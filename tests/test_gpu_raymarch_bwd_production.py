"""The backward kernel (ide3d_raymarch_bwd_cam, csrc/raymarch_bwd.cu) and both forward kernels at the shapes production runs: rays
longer than one 32-sample chunk, CTAs that walk several tiles across frames, non-square planes.  The reference is autograd through
the oracle's chain in float64 on the device (oracle.renderer follows its inputs' dtype and device), one frame at a time so that its
footprint stays bounded; the gather goes through F.grid_sample, whose autograd keeps the grid rather than the tap gathers.

Planes are band-limited and tapered to exactly 0 on their outer texels: zero padding then adds no slope at the plane's edge, where
untapered planes turn the fp32 rounding of world coordinates into errors of up to 3e-4 on either implementation (DESIGN §3).

Every tensor is compared against its own magnitude, with no floor: max|err| <= rtol * max|ref| and ||err|| <= ftol * ||ref||
(Frobenius), the second catching a small error spread over many elements; the camera gradient's Frobenius error is taken against the
magnitude of the per-sample terms it sums (compare_gradients)."""

import math

import numpy as np
import pytest
import torch

from oracle import camera as ocam
from oracle import renderer as orr
from test_gpu_pose_grad import spy
from test_gpu_renderer import D_TOL, FEAT_TOL, W_TOL, _planes, three_head_from_dense
from test_pose_grad import oracle_explicit

DEV = 'cuda'

# Launch geometry of the backward kernel (raymarch_bwd.cu:29-32, :509-516): a CTA of 8 warps covers a tile of 4 x 2 rays, one warp
# per ray, marching it in chunks of 32 samples; at most kMaxSteps = 256 samples per ray.  grid = min(SM count, tiles) and CTA b
# takes tiles b, b + grid, b + 2 grid, ... in frame-major order.
TILE_X, TILE_Y, CHUNK, MAX_STEPS = 4, 2, 32, 256

# Tolerances set from one run on an H100 80GB HBM3 (700 W), at most 4x the largest error measured over the cases (in the comment).
# Gradients (rtol, ftol): max|err| <= rtol * max|ref|, ||err|| <= ftol * ||ref|| (camera: ftol * ||sum_s |terms|||, compare_gradients).
GRAD_TOL = {
    'tex': (2.5e-4, 1e-4),      # 6.5e-5, 5.3e-5 (production)
    'seg': (2.5e-4, 1e-4),      # 7.1e-5, 5.3e-5 (production)
    'cam': (5e-4, 8e-6),        # 3.8e-4 (default_steps), 2.2e-6
    'w1': (8e-6, 9e-6),         # 2.1e-6, 2.4e-6 (ragged)
    'b1': (3e-5, 4e-5),         # 8.7e-6, 1.0e-5 (sample_limit)
    'w2': (2e-5, 2e-5),         # 5.9e-6, 6.0e-6 (ragged)
    'b2': (2.4e-4, 1e-4),       # 6.1e-5, 6.1e-5 (ragged: the sigma head's bias, one sum over all samples)
}
# Forward (max abs error) of the two decoder precisions on the tapered planes; within FEAT_TOL / D_TOL / W_TOL of test_gpu_renderer.
FWD_TOL = {
    'fp32': dict(feat=2.5e-5, depth=1e-5, weights=1e-5),      # 6.5e-6 (ragged), 3.8e-6, 3.5e-6 (sample_limit)
    'tc': dict(feat=8e-5, depth=3e-5, weights=1.4e-5),        # 2.0e-5, 8.7e-6 (ragged), 3.7e-6 (sample_limit)
}
assert all(FWD_TOL[p][k] <= lim[p] for p in FWD_TOL for k, lim in (('feat', FEAT_TOL), ('depth', D_TOL), ('weights', W_TOL)))
PEAK_BYTES = 8 << 30          # the float64 reference's footprint on a shared card

# name: (plane sets, views, resolution (W, H), samples S, planes (H, W), jitter, options, what the case reaches)
#   reach: chunks = 32-sample chunks per ray; tail = S % 32 where a partial chunk is claimed; walks = CTAs walk >= 2 tiles and a
#   CTA's tile sequence crosses a frame.
CASES = {
    'production': (2, 1, (64, 64), 96, (256, 256), 'hash', dict(clamp_mode='softplus'), dict(chunks=3, tail=0, walks=True)),
    'default_steps': (2, 1, (64, 64), 48, (128, 128), 'tensor', dict(clamp_mode='relu', white_back=True, max_depth=3.3, last_back=True),
                      dict(chunks=2, tail=16, walks=True)),
    'ragged': (2, 1, (37, 29), 33, (160, 96), 'hash', dict(clamp_mode='relu', noise_std=0.5), dict(chunks=2, tail=1, walks=True)),
    'sample_limit': (1, 1, (16, 12), 256, (64, 64), 'tensor', dict(fill_mode='weight'), dict(chunks=8, tail=0, walks=False)),
    'views': (1, 3, (64, 64), 96, (128, 128), 'frames', dict(), dict(chunks=3, tail=0, walks=True)),
    'hierarchical': (2, 1, (64, 64), 48 + 48, (128, 128), 'zvals', dict(), dict(chunks=3, tail=0, walks=True)),
    'over_limit': (1, 1, (8, 8), 257, (64, 64), 'tensor', dict(), dict(chunks=9, tail=1, walks=False)),
}
HIER_COARSE = 48
BOX_SCALE = 2.0
# default_steps: relu, and a decoder whose sigma off the planes is < 0 (seed 32: -0.012), so rays that leave the box end with alpha = 0,
# the weights sum to < 1 and last_back moves weight onto the last sample (with softplus the 1e10 last delta makes alpha_last = 1)


def taper(n, ramp=16):
    """Separable window along one axis: exactly 0 on the outer texels, sin^2 rise over `ramp` texels, 1 inside."""
    i = torch.arange(n, dtype=torch.float64)
    r = (torch.minimum(i, n - 1 - i) / ramp).clamp(max=1.0)
    return torch.sin(0.5 * math.pi * r).square()


def tapered_planes(n, size, g):
    """Band-limited planes [n, 96, H, W] (test_gpu_renderer._planes) times the separable window."""
    H, W = size
    window = (taper(H)[:, None] * taper(W)[None, :]).float()
    return (_planes(n, (H, W), g, smooth=True) * window).contiguous()


def launch_geometry(frames, res):
    W, H = res
    per_frame = math.ceil(W / TILE_X) * math.ceil(H / TILE_Y)
    tiles = per_frame * frames
    grid = min(torch.cuda.get_device_properties(0).multi_processor_count, tiles)
    crosses = any(len({t // per_frame for t in range(b, tiles, grid)}) > 1 for b in range(grid))
    return tiles, grid, crosses


def check_reach(name):
    sets, views, res, S, plane, jitter, opts, reach = CASES[name]
    assert math.ceil(S / CHUNK) == reach['chunks'] and S > CHUNK and S % CHUNK == reach['tail'], name
    tiles, grid, crosses = launch_geometry(sets * views, res)
    if reach['walks']:
        assert tiles >= 2 * grid and crosses, f'{name}: {tiles} tiles on {grid} CTAs'
    if name == 'ragged':
        assert res[0] % TILE_X and res[1] % TILE_Y and plane[0] != plane[1]
    if name == 'sample_limit':
        assert S == MAX_STEPS
    if name == 'over_limit':
        assert S == MAX_STEPS + 1
    if name == 'views':
        assert views > 1


def make_case(name, seed):
    """Fixtures of one case: planes, heads, cameras, output gradients and the jitter / noise both sides use."""
    sets, views, res, S, plane, jitter, opts, _ = CASES[name]
    n = sets * views
    R = res[0] * res[1]
    g = torch.Generator().manual_seed(seed)
    tex, seg = tapered_planes(sets, plane, g), tapered_planes(sets, plane, g)
    dec = orr.Decoder.random(hidden=64, seed=seed + 1)
    yaw = math.pi / 2 + np.linspace(-0.4, 0.4, n).reshape(n, 1).astype(np.float32)
    cam = torch.from_numpy(ocam.look_at_pose(yaw, np.full((n, 1), math.pi / 2 - 0.1, np.float32), [0, 0, 0.2], radius=2.7, batch_size=n))
    gf, gd = torch.randn(n, R, 51, generator=g), torch.randn(n, R, 1, generator=g)
    fx = dict(name=name, n=n, R=R, tex=tex, seg=seg, dec=dec, cam=cam, gf=gf, gd=gd, kw={}, u=None, noise=None)
    opts = dict(opts)
    if opts.get('noise_std'):
        fx['noise'] = torch.randn(n, R, S, 1, generator=g)
        fx['kw']['noise'] = fx['noise']
    if jitter == 'tensor':
        fx['u'] = torch.rand(n, R, S, 1, generator=g)
        fx['kw']['jitter_u'] = fx['u']
    elif jitter == 'hash':
        seed64 = 0x1234_5678_9ABC_DEF1 + seed
        fx['u'] = torch.from_numpy(orr.hash_uniform(np.arange(n * R * S, dtype=np.uint64), seed64)).reshape(n, R, S, 1)
        fx['kw']['jitter_seed'] = seed64
    elif jitter == 'frames':
        seeds = [5 + seed, 2 ** 40 + 3, 77]
        fx['u'] = torch.stack([torch.from_numpy(orr.hash_uniform(np.arange(R * S, dtype=np.uint64), s)) for s in seeds]).reshape(n, R, S, 1)
        fx['kw']['jitter_seed'] = seeds
    elif jitter == 'zvals':
        fx['u'] = torch.rand(n, R, HIER_COARSE, generator=g)
        fx['ui'] = torch.rand(n * R, S - HIER_COARSE, generator=g)
    fx['opts'] = opts
    return fx


def _device_kw(kw):
    return {k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in kw.items()}


def product(fx):
    """One differentiable render through render.raymarch (or raymarch_hierarchical) and its backward.
    -> dict of gradients (tex, seg, cam and the 12 head tensors), the merged depths of a hierarchical case, and the calls seen."""
    from ide3d_b200 import render, render_grad
    sets, views, res, S, _, jitter, _, _ = CASES[fx['name']]
    heads = [tuple(h[:2]) + tuple(t.to(DEV).requires_grad_(True) for t in h[2:]) for h in three_head_from_dense(fx['dec'].w1, fx['dec'].b1, fx['dec'].w2, fx['dec'].b2)]
    t, s, c = [x.to(DEV).requires_grad_(True) for x in (fx['tex'], fx['seg'], fx['cam'])]
    kernel_calls, chain_calls = [], []
    z = None
    with spy(render, 'raymarch_backward', kernel_calls), spy(render_grad, 'composed_chain', chain_calls):
        if jitter == 'zvals':
            feat, d, _, z = render.raymarch_hierarchical(t, s, heads, c, resolution=res, num_steps=HIER_COARSE, n_importance=S - HIER_COARSE,
                                                         jitter_u=fx['u'].to(DEV), importance_u=fx['ui'].to(DEV), return_depths=True, **fx['opts'])
        else:
            feat, d, _ = render.raymarch(t, s, heads, c, resolution=res, num_steps=S, views=views, **_device_kw(fx['kw']), **fx['opts'])
        (feat * fx['gf'].to(DEV)).sum().add((d * fx['gd'].to(DEV)).sum()).backward()
    names = ('w1', 'b1', 'w2', 'b2')
    grads = dict(tex=t.grad, seg=s.grad, cam=c.grad)
    for i, h in enumerate(heads):
        grads.update({f'{k}[{i}]': x.grad for k, x in zip(names, h[2:])})
    return grads, z, kernel_calls, chain_calls


def forward(fx, precision, z=None):
    """feat, depth, weights of the fused forward kernel at one decoder precision (z: the depths of a hierarchical case's second pass)."""
    from ide3d_b200 import render
    sets, views, res, S, _, _, _, _ = CASES[fx['name']]
    heads = three_head_from_dense(fx['dec'].w1, fx['dec'].b1, fx['dec'].w2, fx['dec'].b2)
    kw = dict(z_vals=z) if z is not None else dict(views=views, **_device_kw(fx['kw']))
    with torch.no_grad():
        return render.raymarch(fx['tex'].to(DEV), fx['seg'].to(DEV), [tuple(h[:2]) + tuple(x.to(DEV) for x in h[2:]) for h in heads],
                               fx['cam'].to(DEV), resolution=res, num_steps=S, return_weights=True, precision=precision, **kw, **fx['opts'])


def reference(fx, z=None):
    """Values and gradients of the same loss by autograd through the float64 oracle on the device, frame by frame (the gradients
    accumulate in the leaves; the views of one plane set add into its gradient).
    -> (values, gradients, peak bytes allocated, sum over samples of |terms| of the camera gradient [N,4,4])."""
    sets, views, res, S, _, _, opts, _ = CASES[fx['name']]
    f64 = dict(device=DEV, dtype=torch.float64)
    seen = []

    def gather(coords, planes):                                           # keeps the grid points: the camera gradient's per-sample terms
        if coords.requires_grad and not any(coords is x for x in seen):
            coords.retain_grad()
            seen.append(coords)
        return orr.sample_triplane_torch(coords, planes)

    t, s, c = [x.to(**f64).requires_grad_(True) for x in (fx['tex'], fx['seg'], fx['cam'])]
    params = [p.to(**f64).requires_grad_(True) for p in (fx['dec'].w1, fx['dec'].b1, fx['dec'].w2, fx['dec'].b2)]
    dec = orr.Decoder(*params)
    gf, gd = fx['gf'].to(**f64), fx['gd'].to(**f64)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    vals = dict(feat=[], depth=[], weights=[])
    cam_abs = torch.zeros(fx['n'], 4, 4, **f64)
    for f in range(fx['n']):
        seen.clear()
        k = f // views
        sel = slice(f, f + 1)
        if z is not None:
            out = oracle_explicit(t[k:k + 1], s[k:k + 1], dec, c[sel], z[sel].to(**f64), res=res, box_scale=BOX_SCALE, gather=gather, **opts)
        else:
            noise = None if fx['noise'] is None else fx['noise'][sel]
            out = orr.render_frames(t[k:k + 1], s[k:k + 1], dec, c[sel], num_steps=S, resolution=res, jitter_u=fx['u'][sel], noise=noise,
                                    box_scale=BOX_SCALE, gather=gather, **opts)
        (out[0] * gf[sel]).sum().add((out[1] * gd[sel]).sum()).backward()
        for key, v in zip(('feat', 'depth', 'weights'), out):
            vals[key].append(v.detach())
        # dL/dM[i][j] = sum_s dL/dpw[s][i] (p_cam[s], 1)[j]: keep sum_s |.| of the terms, the scale of the sum's rounding error
        coords, = seen
        g_pw = coords.grad.reshape(-1, 3) * BOX_SCALE
        M = c[f].detach()
        p_cam = (coords.detach().reshape(-1, 3) / BOX_SCALE - M[:3, 3]) @ M[:3, :3]
        hom = torch.cat([p_cam, torch.ones_like(p_cam[:, :1])], 1)
        cam_abs[f, :3] = g_pw.abs().t() @ hom.abs()
        terms_sum = g_pw.t() @ hom
        del out, coords
    # the terms add up to autograd's camera gradient (the same sums, in another order)
    assert float((terms_sum - c.grad[fx['n'] - 1, :3]).abs().max()) <= 1e-9 * float(cam_abs[fx['n'] - 1].max())
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    vals = {k: torch.cat(v) for k, v in vals.items()}
    w1g, b1g, w2g, b2g = [p.grad for p in params]
    H = 64
    blocks = [(slice(0, H), slice(0, 32), slice(0, 32)), (slice(H, 2 * H), slice(32, 64), slice(32, 51)), (slice(2 * H, 3 * H), slice(32, 64), slice(51, 52))]
    grads = dict(tex=t.grad, seg=s.grad, cam=c.grad)
    for i, (hs, ks, os_) in enumerate(blocks):
        grads.update({f'w1[{i}]': w1g[hs, ks], f'b1[{i}]': b1g[hs], f'w2[{i}]': w2g[os_, hs], f'b2[{i}]': b2g[os_]})
    return vals, grads, peak, cam_abs


def rel_errors(mine, ref, fro_scale=None):
    """(max|err| / max|ref|, ||err|| / ||fro_scale or ref||); an exact match of an all-zero reference is (0, 0)."""
    err = mine.detach().to(device=ref.device, dtype=torch.float64) - ref
    e_max, r_max = float(err.abs().max()), float(ref.abs().max())
    e_fro, r_fro = float(err.norm()), float((ref if fro_scale is None else fro_scale).norm())
    if r_max == 0.0:
        return (0.0, 0.0) if e_max == 0.0 else (math.inf, math.inf)
    return e_max / r_max, e_fro / r_fro


def compare_gradients(mine, ref, cam_abs):
    """-> {name: (rtol, ftol) measured}, and the list of those over GRAD_TOL.
    The camera gradient's Frobenius error is taken relative to ||sum_s |terms|||, not to ||sum_s terms||: it is a sum of ~4e5 per-sample
    terms that cancel (random-signed output gradients), and an fp32 sum's error scales with the sum of the terms' magnitudes.  At
    64^2 rays the cancellation is ~200x: relative to the sum itself, the fp32 composed chain's camera gradient is off by 1e-4..6e-4 and
    rounding only the world coordinates to fp32 moves the float64 reference by 2.3e-5.  The max-error check stays relative to max|ref|."""
    errs, bad = {}, []
    for key, r in ref.items():
        assert mine[key] is not None and mine[key].shape == r.shape, key
        errs[key] = rel_errors(mine[key], r, cam_abs if key == 'cam' else None)
        rtol, ftol = GRAD_TOL[key.split('[')[0]]
        if errs[key][0] > rtol or errs[key][1] > ftol:
            bad.append(f'{key}: max {errs[key][0]:.2e} (rtol {rtol:.0e}), frobenius {errs[key][1]:.2e} (ftol {ftol:.0e})')
    return errs, bad


def compare_forward(fx, vals, z=None):
    """Both decoder precisions against the float64 values: -> {precision/tensor: max abs error}, and those over FWD_TOL."""
    errs, bad = {}, []
    for precision in ('fp32', 'tc'):
        for key, v in zip(('feat', 'depth', 'weights'), forward(fx, precision, z)):
            e = float((v.to(torch.float64) - vals[key]).abs().max())
            errs[f'{precision}/{key}'] = e
            if e > FWD_TOL[precision][key]:
                bad.append(f'{precision} {key}: max abs {e:.2e} (tol {FWD_TOL[precision][key]:.0e})')
    return errs, bad


def report(name, errs, peak):
    print(f'\n[{name}] reference peak {peak / 2 ** 30:.2f} GiB')
    for key, e in errs.items():
        print(f'[{name}] {key:>14s} ' + (f'max {e[0]:.3e} fro {e[1]:.3e}' if isinstance(e, tuple) else f'abs {e:.3e}'))


# ------------------------------------------------------------------------------------------------------------------- CPU

def test_taper_is_zero_on_the_border_texels_and_one_inside():
    g = torch.Generator().manual_seed(0)
    p = tapered_planes(2, (40, 72), g)
    assert p.shape == (2, 96, 40, 72)
    for edge in (p[:, :, 0], p[:, :, -1], p[:, :, :, 0], p[:, :, :, -1]):
        assert bool((edge == 0).all())
    assert bool((p[:, :, 1:-1, 1:-1] != 0).all())
    w = taper(72)
    assert float(w[0]) == 0.0 and float(w[-1]) == 0.0 and bool((w[16:-16] == 1).all()) and bool((w[1:-1] > 0).all())
    assert bool((w[1:17] >= w[:16]).all())                                      # rises monotonically over the ramp


@pytest.mark.parametrize('gather', ['explicit', 'grid_sample'])
def test_float64_oracle_agrees_with_fp32_oracle_over_two_chunks(gather):
    """The float64 chain (same functions, float64 inputs) against the fp32 oracle at S = 40: values and gradients agree to fp32
    rounding, so the float64 reference differs from the fp32 one by rounding alone."""
    S, res, n = 40, (6, 5), 2
    R = res[0] * res[1]
    g = torch.Generator().manual_seed(3)
    tex, seg = tapered_planes(n, (48, 40), g), tapered_planes(n, (48, 40), g)
    dec = orr.Decoder.random(hidden=64, seed=4)
    yaw = math.pi / 2 + np.array([[-0.3], [0.3]], np.float32)
    cam = torch.from_numpy(ocam.look_at_pose(yaw, np.full((n, 1), math.pi / 2 - 0.1, np.float32), [0, 0, 0.2], radius=2.7, batch_size=n))
    u = torch.rand(n, R, S, 1, generator=g)
    gf, gd = torch.randn(n, R, 51, generator=g), torch.randn(n, R, 1, generator=g)
    fn = orr.sample_triplane if gather == 'explicit' else orr.sample_triplane_torch

    def run(dtype):
        leaves = [x.detach().to(dtype, copy=True).requires_grad_(True) for x in (tex, seg, cam, dec.w1, dec.b1, dec.w2, dec.b2)]
        rgb, depth, w = orr.render_frames(leaves[0], leaves[1], orr.Decoder(*leaves[3:]), leaves[2], num_steps=S, resolution=res,
                                          jitter_u=u, last_back=True, white_back=True, max_depth=3.3, gather=fn)
        (rgb * gf.to(dtype)).sum().add((depth * gd.to(dtype)).sum()).backward()
        return [rgb, depth, w], [x.grad for x in leaves]

    v32, g32 = run(torch.float32)
    v64, g64 = run(torch.float64)
    assert all(v.dtype == torch.float64 for v in v64 + g64)
    # measured: feat 8.3e-7, depth 1.1e-6, weights 4.4e-7; gradients 1.1e-5 of their max (tex, seg), <= 1.4e-6 (camera, decoder)
    for a, b, tol in zip(v32, v64, (4e-6, 4e-6, 2e-6)):
        assert float((a.detach().double() - b.detach()).abs().max()) <= tol
    for a, b in zip(g32, g64):
        assert float((a.double() - b).abs().max()) <= 5e-5 * float(b.abs().max())
    # the fp32 path of the same function is the oracle's fp32 chain, bit for bit
    r32 = orr.render_frames(tex, seg, dec, cam, num_steps=S, resolution=res, jitter_u=u, last_back=True, white_back=True, max_depth=3.3, gather=fn)
    assert all(torch.equal(a.detach(), b) for a, b in zip(v32, r32))


# ------------------------------------------------------------------------------------------------------------------- GPU

@pytest.mark.gpu
@pytest.mark.parametrize('name', [k for k in CASES if k != 'over_limit'])
def test_backward_kernel_matches_float64_reference_at_production_shapes(name):
    check_reach(name)
    fx = make_case(name, seed=list(CASES).index(name) + 30)
    grads, z, kernel_calls, chain_calls = product(fx)
    assert kernel_calls and kernel_calls[0]['want_camera'] and not chain_calls, 'the backward kernel path was not taken'
    assert float(grads['cam'][:, 3].abs().max()) == 0.0 and float(grads['cam'][:, :3].abs().max()) > 0
    vals, ref, peak, cam_abs = reference(fx, z)
    errs, bad = compare_gradients(grads, ref, cam_abs)
    del grads, ref
    f_errs, f_bad = compare_forward(fx, vals, z)
    report(name, dict(errs, **f_errs), peak)
    assert peak < PEAK_BYTES, f'reference peak {peak / 2 ** 30:.2f} GiB'
    assert not bad and not f_bad, '\n'.join(bad + f_bad)


@pytest.mark.gpu
def test_just_over_the_sample_limit_the_composed_chain_matches_float64_reference():
    """S = kMaxSteps + 1: the kernel declines (render.raymarch_backward returns None) and the composed chain, in fp32 with TF32 off,
    gives the gradients."""
    name = 'over_limit'
    check_reach(name)
    fx = make_case(name, seed=40)
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        grads, _, kernel_calls, chain_calls = product(fx)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    assert kernel_calls and chain_calls, 'the composed chain was not taken'
    vals, ref, peak, cam_abs = reference(fx)
    errs, bad = compare_gradients(grads, ref, cam_abs)
    f_errs, f_bad = compare_forward(fx, vals)
    report(name, dict(errs, **f_errs), peak)
    assert not bad and not f_bad, '\n'.join(bad + f_bad)

