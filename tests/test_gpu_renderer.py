"""GPU parity: the fused renderer kernels and the stand-alone stages vs the CPU oracle and the recorded reference
outputs.  Tolerances (fp32 path, stated per tensor): positions / depths 2e-6..1e-5 absolute; gathered features 5e-6;
decoded / composited features 3e-5 absolute on O(1) values (hidden softplus uses MUFU ex2/lg2, |err| < 4e-7 each,
summed over <= 192 hidden units); weights 1e-5."""

import math

import numpy as np
import pytest
import torch

from conftest import T, assert_close, load_golden
from oracle import camera as ocam, renderer as orr

pytestmark = pytest.mark.gpu
DEV = 'cuda'

# Decoder precision modes of the fused kernel: 'fp32' = CUDA-core FFMA (plain fp32), 'tc' = wgmma tensor cores with
# every product evaluated as bf16 hi*hi + hi*lo + lo*hi and fp32 accumulation (operands carry 16 mantissa bits, i.e.
# 2^-17 relative rounding of inputs / weights / hidden activations).  Tolerance on composited features: 3e-5 (fp32),
# 2e-4 (tc) absolute on O(1) values; depth and weights only depend on the decoder through sigma.
PRECISIONS = ['fp32', 'tc']
FEAT_TOL = {'fp32': 3e-5, 'tc': 2e-4}
W_TOL = {'fp32': 1e-5, 'tc': 5e-5}
D_TOL = {'fp32': 1e-5, 'tc': 5e-5}


def three_head_from_dense(w1, b1, w2, b2, H=64):
    """Slice the block-sparse dense decoder of the fixtures into the three heads the kernel takes."""
    w1, b1, w2, b2 = [torch.as_tensor(t) for t in (w1, b1, w2, b2)]
    return [(0, 0, w1[0:H, 0:32], b1[0:H], w2[0:32, 0:H], b2[0:32]),
            (1, 32, w1[H:2 * H, 32:], b1[H:2 * H], w2[32:51, H:2 * H], b2[32:51]),
            (1, 51, w1[2 * H:, 32:], b1[2 * H:], w2[51:52, 2 * H:], b2[51:52])]


@pytest.mark.parametrize('layout,precision', [('nchw', 'fp32'), ('nhwc', 'fp32'), ('nhwc', 'tc')])
def test_raymarch_matches_recorded_reference_chain(layout, precision):
    from ide3d_b200 import render
    g = load_golden('chain')
    tex, seg = T(g['planes_tex'], DEV), T(g['planes_seg'], DEV)
    if layout == 'nhwc':
        tex, seg = tex.contiguous(memory_format=torch.channels_last), seg.contiguous(memory_format=torch.channels_last)
    heads = three_head_from_dense(g['w1'], g['b1'], g['w2'], g['b2'])
    res = tuple(int(v) for v in g['resolution'])
    feat, depth, w = render.raymarch(tex, seg, heads, T(g['camera'], DEV), resolution=res, num_steps=int(g['num_steps']),
                                     box_scale=float(g['box_scale']), jitter_u=T(g['u'], DEV), return_weights=True,
                                     convert_layout=(layout == 'nhwc'), precision=precision)
    assert_close(feat, g['rgb'], FEAT_TOL[precision], what='feat')
    assert_close(depth, g['depth'], D_TOL[precision], what='depth')
    assert_close(w, g['weights'], W_TOL[precision], what='weights')


@pytest.mark.parametrize('precision', PRECISIONS)
def test_raymarch_dense_decoder_relu_lastback(precision):
    from ide3d_b200 import render
    g, d = load_golden('chain'), load_golden('chain_dense')
    res = tuple(int(v) for v in g['resolution'])
    feat, depth, w = render.raymarch(T(g['planes_tex'], DEV), T(g['planes_seg'], DEV),
                                     render.dense_heads(*[T(d[k]) for k in ('w1', 'b1', 'w2', 'b2')]), T(g['camera'], DEV),
                                     resolution=res, num_steps=int(g['num_steps']), box_scale=float(g['box_scale']),
                                     jitter_u=T(g['u'], DEV), clamp_mode='relu', last_back=True, return_weights=True,
                                     precision=precision)
    assert_close(feat, d['rgb'], FEAT_TOL[precision]); assert_close(depth, d['depth'], D_TOL[precision]); assert_close(w, d['weights'], W_TOL[precision])


def _planes(n, plane, g, smooth):
    """White noise is the adversarial input for an fp32 gather: a texel-to-texel slope of O(1) turns the ~3e-7 rounding
    of the world coordinates (cancellation in cam2world: |R p| ~ 3 against t = 2.7) into plane_res * 3e-7 * slope of
    feature error on EITHER implementation.  Generator planes are smooth; `smooth` draws band-limited noise
    (8x8 control points, bicubic) so that the tight tolerance measures the kernel and not that conditioning.
    plane: side of square planes, or (H, W)."""
    size = (plane, plane) if isinstance(plane, int) else tuple(plane)
    if not smooth:
        return torch.randn(n, 96, *size, generator=g)
    lo = torch.randn(n, 96, 8, 8, generator=g)
    return torch.nn.functional.interpolate(lo, size=size, mode='bicubic', align_corners=True).contiguous()


def _random_case(n, plane, seed, hidden=64, three_head=True, smooth=True):
    g = torch.Generator().manual_seed(seed)
    tex = _planes(n, plane, g, smooth)
    seg = _planes(n, plane, g, smooth)
    dec = orr.Decoder.random(hidden=hidden, seed=seed + 1, three_head=three_head)
    yaw = math.pi / 2 + np.linspace(-0.5, 0.5, n).reshape(n, 1).astype(np.float32)
    pitch = np.full((n, 1), math.pi / 2 - 0.1, np.float32)
    cam = torch.from_numpy(ocam.look_at_pose(yaw, pitch, [0, 0, 0.2], radius=2.7, batch_size=n))
    return tex, seg, dec, cam


@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('S,res,opts', [
    (48, (16, 16), dict()),                                              # config-1 shape, small image
    (96, (12, 10), dict(white_back=True, max_depth=3.3)),                # 3 full chunks, non-square, odd tile edge
    (33, (9, 7), dict(last_back=True, clamp_mode='relu')),               # ragged chunk
    (2, (5, 5), dict()),                                                 # two samples: one finite delta + 1e10
    (40, (8, 8), dict(fill_mode='weight')),
])
def test_raymarch_vs_oracle_random(S, res, opts, precision):
    from ide3d_b200 import render
    tex, seg, dec, cam = _random_case(2, 32, seed=S)
    u = torch.rand(2, res[0] * res[1], S, 1, generator=torch.Generator().manual_seed(5))
    ro, do_, wo = orr.render_frames(tex, seg, dec, cam, num_steps=S, resolution=res, jitter_u=u, **opts)
    heads = three_head_from_dense(dec.w1, dec.b1, dec.w2, dec.b2)
    feat, depth, w = render.raymarch(tex.to(DEV), seg.to(DEV), heads, cam.to(DEV), resolution=res, num_steps=S,
                                     jitter_u=u.to(DEV), return_weights=True, precision=precision, **opts)
    assert_close(feat, ro, FEAT_TOL[precision], what='feat'); assert_close(depth, do_, D_TOL[precision], what='depth'); assert_close(w, wo, W_TOL[precision], what='w')


def test_raymarch_white_noise_planes():
    """White-noise planes: tolerance scaled by the conditioning explained in _planes() (32^2 planes -> 3e-4).
    (S = 1 is degenerate in the reference itself: `deltas[:, :, :1]` of an empty tensor is empty, so fancy_integration
    returns all-zero maps, volumetric_rendering.py:40-43; it is not a case the kernels try to mimic.)"""
    from ide3d_b200 import render
    tex, seg, dec, cam = _random_case(2, 32, seed=5, smooth=False)
    heads = three_head_from_dense(dec.w1, dec.b1, dec.w2, dec.b2)
    u = torch.rand(2, 64, 33, 1, generator=torch.Generator().manual_seed(5))
    ro, do_, wo = orr.render_frames(tex, seg, dec, cam, num_steps=33, resolution=(8, 8), jitter_u=u)
    feat, depth, w = render.raymarch(tex.to(DEV), seg.to(DEV), heads, cam.to(DEV), resolution=(8, 8), num_steps=33,
                                     jitter_u=u.to(DEV), return_weights=True)
    assert_close(feat, ro, 3e-4); assert_close(depth, do_, 1e-4); assert_close(w, wo, 1e-4)


@pytest.mark.parametrize('precision', PRECISIONS)
def test_raymarch_hash_jitter_is_bit_compatible_with_oracle_hash(precision):
    from ide3d_b200 import render
    tex, seg, dec, cam = _random_case(2, 24, seed=11, hidden=128, three_head=False)
    S, res, seed = 20, (8, 8), 0x1234_5678_9ABC_DEF1
    ro, do_, wo = orr.render_frames(tex, seg, dec, cam, num_steps=S, resolution=res, jitter_seed=seed)
    feat, depth, w = render.raymarch(tex.to(DEV), seg.to(DEV), render.dense_heads(dec.w1, dec.b1, dec.w2, dec.b2),
                                     cam.to(DEV), resolution=res, num_steps=S, jitter_seed=seed, return_weights=True, precision=precision)
    assert_close(feat, ro, FEAT_TOL[precision]); assert_close(depth, do_, D_TOL[precision]); assert_close(w, wo, W_TOL[precision])


@pytest.mark.parametrize('precision', PRECISIONS)
def test_raymarch_noise_and_no_jitter(precision):
    from ide3d_b200 import render
    tex, seg, dec, cam = _random_case(1, 16, seed=3)
    S, res = 12, (6, 6)
    noise = torch.randn(1, 36, S, 1, generator=torch.Generator().manual_seed(2))
    ro, do_, wo = orr.render_frames(tex, seg, dec, cam, num_steps=S, resolution=res, noise=noise, noise_std=0.7)
    feat, depth, w = render.raymarch(tex.to(DEV), seg.to(DEV), three_head_from_dense(dec.w1, dec.b1, dec.w2, dec.b2),
                                     cam.to(DEV), resolution=res, num_steps=S, noise=noise.to(DEV), noise_std=0.7,
                                     return_weights=True, precision=precision)
    assert_close(feat, ro, FEAT_TOL[precision]); assert_close(depth, do_, D_TOL[precision]); assert_close(w, wo, W_TOL[precision])


@pytest.mark.parametrize('precision', PRECISIONS)
def test_raymarch_full_size_properties(precision):
    """BASELINE config 2 shape (8 frames, 64^2 x 96, 256^2 planes): size-independent properties instead of the slow
    CPU oracle -- weights are a sub-probability along each ray, last_back makes them sum to 1, fill_mode='weight'
    returns exactly the weight sums, linearity of the composited features in the decoder's output bias."""
    from ide3d_b200 import render
    g = torch.Generator(device='cuda').manual_seed(0)
    n = 8
    up = lambda t: torch.nn.functional.interpolate(t, size=(256, 256), mode='bicubic', align_corners=True).contiguous(memory_format=torch.channels_last)
    tex = up(torch.randn(n, 96, 8, 8, device=DEV, generator=g))           # band-limited planes, see _planes()
    seg = up(torch.randn(n, 96, 8, 8, device=DEV, generator=g))
    dec = orr.Decoder.random(hidden=64, seed=1)
    heads = three_head_from_dense(dec.w1, dec.b1, dec.w2, dec.b2)
    yaw = math.pi / 2 + np.linspace(-0.5, 0.5, n).reshape(n, 1).astype(np.float32)
    cam = torch.from_numpy(ocam.look_at_pose(yaw, np.full((n, 1), math.pi / 2, np.float32), [0, 0, 0.2], radius=2.7, batch_size=n)).to(DEV)
    kw = dict(resolution=(64, 64), num_steps=96, jitter_seed=7, return_weights=True, precision=precision)
    feat, depth, w = render.raymarch(tex, seg, heads, cam, **kw)
    wsum = w.sum(2)
    assert torch.isfinite(feat).all() and torch.isfinite(depth).all()
    assert (w >= 0).all() and (wsum <= 1 + 1e-4).all()
    assert (depth >= 2.25 * wsum - 1e-3).all() and (depth <= 3.3 * wsum + 1e-3).all()
    _, _, w_lb = render.raymarch(tex, seg, heads, cam, last_back=True, **kw)
    assert_close(w_lb.sum(2), torch.ones_like(wsum), 2e-5, what='last_back sums to one')
    f_fill, _, _ = render.raymarch(tex, seg, heads, cam, fill_mode='weight', **kw)
    assert_close(f_fill, wsum.expand(-1, -1, 51), 2e-5, what='fill_mode=weight')
    # shifting the colour head's output bias by delta shifts the composited colour by delta * wsum
    heads2 = [(heads[0][0], heads[0][1], heads[0][2], heads[0][3], heads[0][4], heads[0][5] + 0.5)] + heads[1:]
    f2, _, _ = render.raymarch(tex, seg, heads2, cam, **kw)
    assert_close(f2[..., :32] - feat[..., :32], 0.5 * wsum.expand(-1, -1, 32), 5e-5 if precision == 'fp32' else 2e-4, what='bias linearity')
    assert_close(f2[..., 32:], feat[..., 32:], 0.0, what='other heads untouched')
    # a spot-check of 3 rays of frame 5 against the oracle on the same inputs
    sub = slice(5, 6)
    ro, do_, _ = orr.render_frames(tex[sub].cpu().contiguous(), seg[sub].cpu().contiguous(), dec, cam[sub].cpu(),
                                   num_steps=96, resolution=(64, 64), jitter_u=None)
    f_nj, d_nj, _ = render.raymarch(tex[sub], seg[sub], heads, cam[sub], resolution=(64, 64), num_steps=96, precision=precision)
    # 3e-4: where a ray leaves the plane (zeros padding) the bilinear value falls to 0 within one texel, i.e. unit
    # slope per texel; the ~3e-7 fp32 rounding of world coordinates x 128 texels/unit x |feature| ~ 1e-4 on either side.
    assert_close(f_nj, ro, 3e-4, what='full-size frame vs oracle'); assert_close(d_nj, do_, 2e-5)
    assert (f_nj.cpu() - ro).abs().mean().item() < (3e-6 if precision == 'fp32' else 2e-5)


def test_unsupported_decoder_shape_is_reported():
    from ide3d_b200 import render
    tex = torch.randn(1, 96, 8, 8, device=DEV)
    bad = [(2, 0, torch.randn(48, 64), torch.zeros(48), torch.randn(52, 48), torch.zeros(52))]
    with pytest.raises(RuntimeError, match='no fused kernel'):
        render.raymarch(tex, tex, bad, torch.eye(4, device=DEV)[None], resolution=(4, 4), num_steps=4)
    with pytest.raises(ValueError):
        render.raymarch(tex, tex, bad, torch.eye(4, device=DEV)[None], clamp_mode=None)


# ------------------------------------------------------------------------------------------ point queries
def test_sample_voxel_golden_and_edges():
    from ide3d_b200 import render
    g, v = load_golden('chain'), load_golden('voxel')
    heads = three_head_from_dense(g['w1'], g['b1'], g['w2'], g['b2'])
    tex, seg = T(g['planes_tex'], DEV), T(g['planes_seg'], DEV)
    out = render.sample_voxel(tex, seg, heads, T(v['points'], DEV), box_scale=float(g['box_scale']))
    assert_close(out, v['out'], 3e-5)
    sg = render.sample_voxel(tex, seg, heads, T(v['points'], DEV), box_scale=float(g['box_scale']), sigma_only=True)
    assert_close(sg, v['out'][..., -1:], 3e-5)
    # ragged count (not a multiple of 32), far-outside points (all taps masked) and an empty request
    pts = torch.cat([T(v['points'])[:, :37], torch.full((2, 3, 3), 9.0)], 1)
    dec = orr.Decoder(g['w1'], g['b1'], g['w2'], g['b2'])
    ref = orr.sample_voxel(T(g['planes_tex']), T(g['planes_seg']), dec, pts, float(g['box_scale']))
    assert_close(render.sample_voxel(tex, seg, heads, pts.to(DEV), box_scale=float(g['box_scale'])), ref, 3e-5)
    assert render.sample_voxel(tex, seg, heads, torch.zeros(2, 0, 3, device=DEV)).shape == (2, 0, 52)


def test_sigma_grid_matches_create_samples_path():
    from ide3d_b200 import render
    tex, seg, dec, _ = _random_case(1, 32, seed=21)
    heads = three_head_from_dense(dec.w1, dec.b1, dec.w2, dec.b2)
    N = 24
    samples, _, _ = orr.create_samples(N, [0, 0, 0], 1.0)
    ref = orr.sample_voxel(tex, seg, dec, 0.9 * samples, 2.0)[..., -1]
    full = render.sigma_grid(tex.to(DEV), seg.to(DEV), heads, grid_n=N, cube_length=1.0)
    assert_close(full, ref, 3e-5)
    # slab interface = what a rank computes in the z-slab shard; concatenation must equal the whole grid (bit-exact)
    cut = 5000
    a = render.sigma_grid(tex.to(DEV), seg.to(DEV), heads, grid_n=N, cube_length=1.0, first=0, count=cut)
    b = render.sigma_grid(tex.to(DEV), seg.to(DEV), heads, grid_n=N, cube_length=1.0, first=cut)
    assert torch.equal(torch.cat([a, b], 1), full)
    # and the explicit-points kernel agrees with the in-kernel point generator
    exp = render.sample_voxel(tex.to(DEV), seg.to(DEV), heads, (0.9 * samples).to(DEV), sigma_only=True)[..., 0]
    assert_close(full, exp, 1e-6)


# ------------------------------------------------------------------------------------------ stand-alone stages
def test_free_functions_match_recorded_reference():
    from ide3d_b200.training import volumetric_rendering as vr
    for tag in 'ab':
        g = load_golden('rays_' + tag)
        p, z, d = vr.get_initial_rays_trig(int(g['n']), int(g['num_steps']), DEV, float(g['fov']),
                                           tuple(int(v) for v in g['resolution']), float(g['ray_start']), float(g['ray_end']))
        assert_close(p, g['points'], 2e-6); assert_close(z, g['z_vals'], 2e-6); assert_close(d, g['rays_d_cam'], 2e-6)
    g = load_golden('transform')
    torch.manual_seed(123)
    u = torch.rand(g['z_vals'].shape, device=DEV)          # the draw transform_sampled_points makes first
    torch.manual_seed(123)
    pw, zj, dw, ow, _, _ = vr.transform_sampled_points(T(g['points'], DEV), T(g['z_vals'], DEV), T(g['rays_d_cam'], DEV),
                                                       DEV, camera=T(g['camera'], DEV))
    pj, zo = orr.perturb(T(g['points']), T(g['z_vals']), T(g['rays_d_cam']), u.cpu())
    pwo, dwo, owo = orr.to_world(pj, T(g['rays_d_cam']), T(g['camera']))
    assert_close(zj, zo, 2e-6); assert_close(pw, pwo, 3e-6); assert_close(dw, dwo, 2e-6); assert_close(ow, owo, 2e-6)


def test_sample_from_triplane_golden():
    from ide3d_b200.dnnlib.util import sample_from_triplane
    g = load_golden('triplane')
    for fmt in (torch.contiguous_format, torch.channels_last):
        out = sample_from_triplane(T(g['coords'], DEV), T(g['grid'], DEV).contiguous(memory_format=fmt))
        assert_close(out, g['feat'], 5e-6)


@pytest.mark.parametrize('case,kw', [
    ('softplus', dict(clamp_mode='softplus')), ('relu', dict(clamp_mode='relu')),
    ('lastback', dict(clamp_mode='softplus', last_back=True)),
    ('white', dict(clamp_mode='softplus', white_back=True, max_depth=3.5)),
    ('fillw', dict(clamp_mode='relu', fill_mode='weight'))])
def test_fancy_integration_golden(case, kw):
    from ide3d_b200.training import volumetric_rendering as vr
    g = load_golden('integration')
    rgb, dep, w = vr.fancy_integration(T(g['rgb_sigma'], DEV), T(g['rays_d_cam'], DEV), T(g['z_vals'], DEV), DEV,
                                       noise_std=0, **kw)
    assert_close(rgb, g[case + '_rgb'], 1e-5); assert_close(dep, g[case + '_depth'], 1e-5); assert_close(w, g[case + '_weights'], 5e-6)


def test_fancy_integration_needs_clamp_mode():
    from ide3d_b200.training import volumetric_rendering as vr
    g = load_golden('integration')
    with pytest.raises(ValueError):
        vr.fancy_integration(T(g['rgb_sigma'], DEV), T(g['rays_d_cam'], DEV), T(g['z_vals'], DEV), DEV, noise_std=0)


def test_sample_pdf_golden():
    from ide3d_b200.training import volumetric_rendering as vr
    g = load_golden('sample_pdf')
    assert_close(vr.sample_pdf(T(g['bins'], DEV), T(g['weights'], DEV), 8, det=True), g['det'], 5e-6)
    torch.manual_seed(9)
    u = torch.rand(g['bins'].shape[0], 8, device=DEV)
    torch.manual_seed(9)
    out = vr.sample_pdf(T(g['bins'], DEV), T(g['weights'], DEV), 8, det=False)
    assert_close(out, orr.sample_pdf(T(g['bins']), T(g['weights']), 8, det=False, u=u.cpu()), 5e-6)


def test_camera_helpers_golden():
    from ide3d_b200.training import volumetric_rendering as vr
    g = load_golden('camera')
    for i, (h, v) in enumerate(zip(g['h'], g['v'])):
        o, _, _ = vr.sample_camera_positions(DEV, n=1, r=2.7, horizontal_mean=float(h), vertical_mean=float(v), mode=None)
        assert_close(o, g[f'origin{i}'], 2e-6)
        assert_close(vr.create_cam2world_matrix(-o, o, device=DEV), g[f'c2w{i}'], 2e-6)
        la = vr.LookAtPoseSampler.sample(float(h), float(v), torch.tensor([0, 0, 0.2], device=DEV), radius=2.7, device=DEV)
        assert_close(la, g[f'lookat{i}'], 2e-6)


def test_mask2color_matches_reference_loop():
    """dnnlib/seg_tools.py:75-82 (argmax + 19 masked assignments) vs the one-pass kernel; ties -> first maximum; strided input."""
    from ide3d_b200.dnnlib import seg_tools
    from oracle import ops as oops
    g = torch.Generator().manual_seed(2)
    m = torch.randn(3, 19, 21, 17, generator=g)
    m[0, 4, 3, 3] = m[0, 9, 3, 3] = 50.0                                  # tie: argmax returns the first
    want = oops.mask2color(m, seg_tools.COLOR_MAP)
    got = seg_tools.mask2color(m.to(DEV))
    assert got.dtype == torch.float32 and torch.equal(got.cpu(), want)
    got8 = seg_tools.mask2color(m.to(DEV).contiguous(memory_format=torch.channels_last), to_uint8=True)
    assert got8.dtype == torch.uint8 and torch.equal(got8.cpu(), want.to(torch.uint8))
    wide = torch.randn(2, 51, 8, 8, generator=g).to(DEV)                   # the renderer's feat layout: logits are channels 32..50
    sl = wide[:, 32:51]
    assert torch.equal(seg_tools.mask2color(sl).cpu(), oops.mask2color(sl.cpu(), seg_tools.COLOR_MAP))


@pytest.mark.parametrize('precision', PRECISIONS)
def test_hierarchical_two_pass_matches_oracle_composition(precision):
    """a8 wired: coarse fused pass -> ide3d_sample_pdf -> merged, sorted depths -> second fused pass (depths read from a tensor,
    IDE3D_JITTER_ZVALS) vs the oracle's composition of the reference's own stages around sample_pdf
    (volumetric_rendering.py:224-265), same injected uniforms for the stratified jitter and the importance draw."""
    from ide3d_b200 import render
    N, S, NI, res = 2, 24, 16, (8, 8)
    tex, seg, dec, cam = _random_case(N, 32, seed=17)
    g = torch.Generator().manual_seed(17)
    u = torch.rand(N, 64, S, 1, generator=g)
    ui = torch.rand(N * 64, NI, generator=g)
    ro, do_, wo, zo = orr.render_frames_hierarchical(tex, seg, dec, cam, num_steps=S, n_importance=NI, resolution=res, jitter_u=u, importance_u=ui)
    heads = three_head_from_dense(dec.w1, dec.b1, dec.w2, dec.b2)
    feat, depth, w, z = render.raymarch_hierarchical(tex.to(DEV), seg.to(DEV), heads, cam.to(DEV), resolution=res, num_steps=S, n_importance=NI,
                                                     jitter_u=u.to(DEV), importance_u=ui.to(DEV), return_weights=True, return_depths=True,
                                                     precision=precision)
    assert z.shape == (N, 64, S + NI) and bool((z[..., 1:] >= z[..., :-1]).all())
    # the importance depths are a continuous function of the coarse weights: 1e-6-level weight differences move them by <= 1e-5
    assert_close(z, zo.reshape(N, 64, S + NI), 2e-5, what='merged depths')
    assert_close(feat, ro, 3 * FEAT_TOL[precision], what='feat'); assert_close(depth, do_, 3 * D_TOL[precision], what='depth')
    assert_close(w, wo, 3 * W_TOL[precision], what='w')
    # the importance samples concentrate where the coarse weights are: the merged set is not the stratified one
    zc = render.coarse_depths(N, res, S, jitter_u=u.to(DEV), device=DEV)
    assert_close(zc, orr.render_frames(tex, seg, dec, cam, num_steps=S, resolution=res, jitter_u=u, return_stages=True)['z_vals'].reshape(N, 64, S), 1e-6)
    # det=True (no jitter anywhere) is reproducible
    a = render.raymarch_hierarchical(tex.to(DEV), seg.to(DEV), heads, cam.to(DEV), resolution=res, num_steps=S, det=True, precision=precision)
    b = render.raymarch_hierarchical(tex.to(DEV), seg.to(DEV), heads, cam.to(DEV), resolution=res, num_steps=S, det=True, precision=precision)
    assert torch.equal(a[0], b[0]) and a[0].shape == (N, 64, 51)


@pytest.mark.parametrize('precision', PRECISIONS)
def test_hierarchical_matches_recorded_reference_stage_composition(precision):
    """chain_hier.npz: the two passes composed from the reference's own stage functions (tests/golden/make_golden.py
    g_chain_hier) vs the fused kernels + ide3d_sample_pdf, same injected uniforms."""
    from ide3d_b200 import render
    g = load_golden('chain_hier')
    res = tuple(int(v) for v in g['resolution'])
    S, NI = int(g['num_steps']), int(g['n_importance'])
    heads = three_head_from_dense(g['w1'], g['b1'], g['w2'], g['b2'])
    feat, depth, w, z = render.raymarch_hierarchical(T(g['planes_tex'], DEV), T(g['planes_seg'], DEV), heads, T(g['camera'], DEV),
                                                     resolution=res, num_steps=S, n_importance=NI, box_scale=float(g['box_scale']),
                                                     jitter_u=T(g['u'], DEV), importance_u=T(g['importance_u'], DEV),
                                                     return_weights=True, return_depths=True, precision=precision)
    R = res[0] * res[1]
    assert_close(z, T(g['z_all']).reshape(-1, R, S + NI), 2e-5, what='merged depths')
    assert_close(feat, g['rgb'], 3 * FEAT_TOL[precision], what='feat'); assert_close(depth, g['depth'], 3 * D_TOL[precision], what='depth')
    assert_close(w, g['weights'], 3 * W_TOL[precision], what='w')


def test_hierarchical_flag_through_the_generator():
    """rendering_kwargs / render_params 'hierarchical' reaches the renderer (forward only)."""
    from ide3d_b200.compat import random_init_generator
    G = random_init_generator(device=DEV, seed=0, img_resolution=128, plane_resolution=64, render_size=16, channel_max=32)
    with torch.no_grad():
        ws = G.mapping(torch.randn(1, G.z_dim, device=DEV), torch.zeros(1, 25, device=DEV))
        c = torch.eye(4, device=DEV).reshape(1, 16); c[0, 11] = 2.7
        c = torch.cat([c, torch.zeros(1, 9, device=DEV)], 1)
        a = G.synthesis(ws, c=c, render_params=dict(num_steps=12), perturb=None)
        b = G.synthesis(ws, c=c, render_params=dict(num_steps=12, hierarchical=True, n_importance=12), perturb=None)
    assert a.shape == b.shape and torch.isfinite(b).all() and not torch.equal(a, b)
