"""GPU: the multi-view path of gen_images.py batched (ide3d_b200.images).

  * ray-march kernels with `views` (frames sharing a plane set) against the same launch on materialised planes, bit for bit, and
    against the oracle; per-frame jitter seeds against one-frame launches; the backward's plane gradients against the summed copies
  * SynthesisNetwork(views=...) against repeated ws, one backbone pass, and the hierarchical path
  * ide3d_image_strips against torchvision's bytes (tests/golden/image_strips.npz) and oracle/images.py on the device
  * render_multiview against the gen_images.py loop run through this package at batch 1"""

import math

import numpy as np
import pytest
import torch

from conftest import T, assert_close, load_golden
from oracle import camera as ocam, renderer as orr

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')
FEAT_TOL = {'fp32': 3e-5, 'tc': 2e-4}
D_TOL = {'fp32': 1e-5, 'tc': 5e-5}


def _heads(dec, H=64):
    return [(0, 0, dec.w1[0:H, 0:32], dec.b1[0:H], dec.w2[0:32, 0:H], dec.b2[0:32]),
            (1, 32, dec.w1[H:2 * H, 32:], dec.b1[H:2 * H], dec.w2[32:51, H:2 * H], dec.b2[32:51]),
            (1, 51, dec.w1[2 * H:, 32:], dec.b1[2 * H:], dec.w2[51:52, 2 * H:], dec.b2[51:52])]


def _case(sets, views, plane=32, seed=0):
    """Smooth planes for `sets` latents, a decoder, and sets * views cameras (latent-major)."""
    g = torch.Generator().manual_seed(seed)
    smooth = lambda: torch.nn.functional.interpolate(torch.randn(sets, 96, 8, 8, generator=g), size=(plane, plane), mode='bicubic',
                                                     align_corners=True).contiguous()
    tex, seg = smooth(), smooth()
    dec = orr.Decoder.random(hidden=64, seed=seed + 1)
    n = sets * views
    yaw = math.pi / 2 + np.tile(np.linspace(-0.5, 0.5, views), sets).reshape(n, 1).astype(np.float32)
    cam = torch.from_numpy(ocam.look_at_pose(yaw, np.full((n, 1), math.pi / 2 - 0.1, np.float32), [0, 0, 0.2], radius=2.7, batch_size=n))
    return tex, seg, dec, cam


def _jitter_kwargs(jitter, n, res, S, device):
    from ide3d_b200 import render
    if jitter == 'none':
        return {}
    if jitter == 'tensor':
        return dict(jitter_u=torch.rand(n, res[0] * res[1], S, generator=torch.Generator().manual_seed(7)).to(device))
    if jitter == 'hash':
        return dict(jitter_seed=[1000 + 77 * f + (f << 40) for f in range(n)])
    return dict(z_vals=render.coarse_depths(n, res, S, jitter_seed=[5 + f for f in range(n)], device=device))


@pytest.mark.parametrize('precision,layout', [('fp32', 'nchw'), ('fp32', 'nhwc'), ('tc', 'nhwc')])
@pytest.mark.parametrize('jitter', ['none', 'tensor', 'hash', 'zvals'])
def test_views_forward_equals_materialised_planes(precision, layout, jitter):
    """views=3 reads plane set f // 3: bit-identical to the launch on planes repeated per view, and within the renderer tolerances of
    the oracle."""
    from ide3d_b200 import render
    sets, views, S, res = 2, 3, 40, (12, 10)
    tex, seg, dec, cam = _case(sets, views)
    n = sets * views
    heads = _heads(dec)
    kw = dict(resolution=res, num_steps=S, precision=precision, return_weights=True, **_jitter_kwargs(jitter, n, res, S, DEV))
    cl = layout == 'nhwc'
    prep = (lambda t: t.to(DEV).contiguous(memory_format=torch.channels_last)) if cl else (lambda t: t.to(DEV))
    got = render.raymarch(prep(tex), prep(seg), heads, cam.to(DEV), views=views, convert_layout=cl, **kw)
    want = render.raymarch(prep(tex.repeat_interleave(views, 0)), prep(seg.repeat_interleave(views, 0)), heads, cam.to(DEV),
                           convert_layout=cl, **kw)
    for a, b, name in zip(got, want, ('feat', 'depth', 'weights')):
        assert torch.equal(a, b), (name, (a - b).abs().max().item())
    if jitter == 'zvals':
        return
    u = None
    if jitter == 'tensor':
        u = kw['jitter_u'].cpu().reshape(n, -1, S, 1)
    elif jitter == 'hash':
        idx = np.arange(res[0] * res[1] * S, dtype=np.uint64)
        u = torch.from_numpy(np.stack([orr.hash_uniform(idx, s) for s in kw['jitter_seed']])).reshape(n, -1, S, 1)
    ro, do_, _ = orr.render_frames(tex.repeat_interleave(views, 0), seg.repeat_interleave(views, 0), dec, cam, num_steps=S, resolution=res,
                                   jitter_u=u)
    assert_close(got[0], ro, FEAT_TOL[precision], what='feat vs oracle')
    assert_close(got[1], do_, D_TOL[precision], what='depth vs oracle')


@pytest.mark.parametrize('precision', ['fp32', 'tc'])
def test_per_frame_seeds_equal_one_frame_launches(precision):
    """A 6-frame launch (2 plane sets x 3 views) with per-frame seeds is bit-identical to six one-frame launches with those seeds."""
    from ide3d_b200 import render
    sets, views, S, res = 2, 3, 48, (16, 16)
    tex, seg, dec, cam = _case(sets, views, seed=3)
    tex, seg = tex.to(DEV), seg.to(DEV)
    heads = render.PackedDecoder(_heads(dec), DEV)
    seeds = [(2 ** 62 - 1) // (f + 1) for f in range(sets * views)]
    feat, depth, _ = render.raymarch(tex, seg, heads, cam.to(DEV), resolution=res, num_steps=S, jitter_seed=torch.tensor(seeds), views=views,
                                     precision=precision)
    for f, s in enumerate(seeds):
        i = f // views
        f1, d1, _ = render.raymarch(tex[i:i + 1], seg[i:i + 1], heads, cam[f:f + 1].to(DEV), resolution=res, num_steps=S, jitter_seed=s,
                                    precision=precision)
        assert torch.equal(feat[f:f + 1], f1) and torch.equal(depth[f:f + 1], d1), f


def test_backward_views_sum_into_shared_planes():
    """ide3d_raymarch_bwd with views=3: the plane gradients of the three views land in their shared set -- the sum of the gradients of
    the three materialised copies -- and the decoder gradients match."""
    from ide3d_b200 import render
    sets, views, S, res = 2, 3, 32, (8, 8)
    tex, seg, dec, cam = _case(sets, views, seed=9)
    n = sets * views
    g = torch.Generator().manual_seed(2)
    gf, gd = torch.randn(n, res[0] * res[1], 51, generator=g).to(DEV), torch.randn(n, res[0] * res[1], 1, generator=g).to(DEV)
    seeds = [31 * f + 1 for f in range(n)]

    def run(shared):
        t = tex.to(DEV).contiguous(memory_format=torch.channels_last).requires_grad_(True)
        s = seg.to(DEV).contiguous(memory_format=torch.channels_last).requires_grad_(True)
        heads = [(h[0], h[1]) + tuple(p.to(DEV).clone().requires_grad_(True) for p in h[2:]) for h in _heads(dec)]
        if shared:
            feat, depth, _ = render.raymarch(t, s, heads, cam.to(DEV), resolution=res, num_steps=S, jitter_seed=seeds, views=views)
        else:
            feat, depth, _ = render.raymarch(t.repeat_interleave(views, 0), s.repeat_interleave(views, 0), heads, cam.to(DEV), resolution=res,
                                             num_steps=S, jitter_seed=seeds)
        ((feat * gf).sum() + (depth * gd).sum()).backward()
        return [t.grad, s.grad] + [p.grad for h in heads for p in h[2:]]

    got, want = run(True), run(False)
    for k, (a, b) in enumerate(zip(got, want)):
        tol = 5e-4 * max(1.0, b.abs().max().item())
        assert (a - b).abs().max().item() <= tol, (k, (a - b).abs().max().item(), tol)


@pytest.fixture(scope='module')
def small_G():
    from ide3d_b200.training.triplane import TriPlaneGenerator
    torch.manual_seed(0)
    return TriPlaneGenerator(z_dim=32, w_dim=32, img_resolution=128, plane_resolution=64, render_size=32, channel_base=2048, channel_max=64,
                             sr_channels=(32, 32), mapping_kwargs=dict(num_layers=2)).eval().requires_grad_(False).to(DEV)


@pytest.fixture()
def fp32_convs():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def test_synthesis_views_against_repeated_ws(small_G, fp32_convs):
    """views=3 against ws.repeat_interleave(3): image <= 1e-4, depth <= 2e-5, every backbone block ran once on the N latents; the
    hierarchical path with per-frame seeds against its repeated-planes run."""
    from ide3d_b200 import images
    G = small_G
    cams = images.view_cameras(images.YAWS, DEV)
    ws = G.mapping(torch.randn(4, G.z_dim, generator=torch.Generator().manual_seed(3)).to(DEV), cams[:1].repeat(4, 1))
    c = cams.repeat(4, 1)
    seeds = torch.arange(12) * 1000003 + 17
    rows = {}
    hooks = [getattr(G.synthesis, f'vb{r}').register_forward_hook(lambda m, a, o, r=r: rows.setdefault(r, []).append(a[2].shape[0]))
             for r in G.synthesis.voxel_block_resolutions]
    try:
        with torch.no_grad():
            got = G.synthesis(ws, c=c, views=3, seed=seeds, noise_mode='const', return_dict=True)
    finally:
        for h in hooks:
            h.remove()
    assert rows and all(v == [4] for v in rows.values()), rows
    with torch.no_grad():
        want = G.synthesis(ws.repeat_interleave(3, 0), c=c, seed=seeds, noise_mode='const', return_dict=True)
    err = {k: (got[k] - want[k]).abs().max().item() for k in want}
    print('views=3 vs repeated ws, max abs difference:', err)
    assert err['image'] <= 1e-4 and err['image_depth'] <= 2e-5 and err['image_raw'] <= 1e-4, err
    with torch.no_grad():
        kw = dict(render_params=dict(num_steps=24, hierarchical=True, n_importance=16), noise_mode='const', return_dict=True,
                  importance_u=torch.rand(12 * 32 * 32, 16, generator=torch.Generator().manual_seed(4)).to(DEV))
        hier = G.synthesis(ws, c=c, views=3, seed=seeds, **kw)
        hier_rep = G.synthesis(ws.repeat_interleave(3, 0), c=c, seed=seeds, **kw)
    assert (hier['image_depth'] - hier_rep['image_depth']).abs().max().item() <= 2e-5
    assert (hier['image'] - hier_rep['image']).abs().max().item() <= 1e-4


def _decided(seg):
    """Pixels whose class two bilinear evaluations cannot disagree on (the rule of test_gpu_video_frames.py)."""
    finite = torch.nan_to_num(seg, nan=0.0)
    top2 = finite.topk(2, dim=1).values
    return ((top2[:, 0] - top2[:, 1]) > 1e-5 * (1 + finite.abs().max())) | seg.isnan().any(1)


def _strip_mask(mask, views):
    """Per-view pixel mask [S*views, H, W] -> strip layout [S, Hs, Ws] (padding counts as decided: it is always 0)."""
    n, h, w = mask.shape
    if views == 1:
        return mask
    out = torch.ones(n // views, h + 4, views * (w + 2) + 2, dtype=torch.bool, device=mask.device)
    for j in range(views):
        out[:, 2:2 + h, 2 + j * (w + 2):2 + j * (w + 2) + w] = mask[j::views]
    return out


@pytest.mark.parametrize('views', [1, 3])
@pytest.mark.parametrize('strided', [False, True])
def test_strip_kernel_matches_golden_and_oracle(views, strided):
    from ide3d_b200 import images
    from ide3d_b200.training.triplane import upsample_seg
    from oracle.images import compose_strips as oracle_strips
    z = load_golden('image_strips')
    img, seg = T(z[f'v{views}_img'], DEV), T(z[f'v{views}_seg'], DEV)
    if strided:                      # the channel view of a ray-march output [n, r*r, 51], and a channels-last image
        n, c, r, _ = seg.shape
        feat = torch.randn(n, r * r, 51, device=DEV)
        view = feat.permute(0, 2, 1).reshape(n, 51, r, r)[:, 32:]
        view.copy_(seg)
        seg, img = view, img.contiguous(memory_format=torch.channels_last)
    s_img, s_seg = images.compose_strips(img, seg, views)
    assert s_img.dtype == torch.uint8 and s_img.shape == z[f'v{views}_out_img'].shape and s_img.is_contiguous()
    assert torch.equal(s_img.cpu(), torch.from_numpy(z[f'v{views}_out_img']))
    o_img, o_seg = oracle_strips(img, seg, views)
    assert torch.equal(s_img, o_img)
    decided = _strip_mask(_decided(upsample_seg(seg, tuple(img.shape[-2:]))), views)
    ties = int((~decided).sum())
    gold = T(z[f'v{views}_out_seg'], DEV)
    assert torch.equal(s_seg[decided], gold[decided]) and torch.equal(s_seg[decided], o_seg[decided])
    differ = int(((s_seg != gold).any(-1) & ~decided).sum())
    print(f'views={views} strided={strided}: {ties} near-tie seg pixels, {differ} of them differ from torchvision')


def _loop_strips(G, seeds, psi):
    """gen_images.py:88-116 run through this package at batch 1, with the save_image bytes computed on the device."""
    from ide3d_b200 import images
    from ide3d_b200.dnnlib.seg_tools import mask2color
    from oracle.images import grid_bytes
    cs = torch.tensor(images.FRONTAL).float().to(DEV).reshape(1, -1)
    out_img, out_seg, logits = [], [], []
    for seed in seeds:
        torch.manual_seed(seed)
        z = torch.from_numpy(np.random.RandomState(seed).randn(1, G.z_dim)).to(DEV)
        ws = G.mapping(z=z, c=cs, truncation_psi=psi)
        imgs, segs = [], []
        for k, yaw in enumerate(images.YAWS):
            c = images.view_cameras([yaw], DEV)
            img, seg = G.synthesis(ws, c=c, render_params=images.render_params(yaw), noise_mode='const', return_seg=True)
            logits.append(seg)
            imgs.append(img)
            segs.append((mask2color(seg) / 255. - 0.5) / 0.5)
        out_img.append(grid_bytes(torch.cat(imgs)))
        out_seg.append(grid_bytes(torch.cat(segs)))
    return torch.stack(out_img), torch.stack(out_seg), torch.cat(logits)


@pytest.mark.parametrize('config', ['small', 'bench'])
def test_render_multiview_matches_gen_images_loop(small_G, config):
    """render_multiview for seeds [0, 1, 2, 3, 5], psi 0.7, default jitter, against the reference loop at batch 1: image strips within
    one uint8 level (other batch sizes may pick other convolution algorithms), seg strips equal wherever the class is decided despite
    that difference."""
    from ide3d_b200 import images
    if config == 'small':
        G = small_G
    else:
        from ide3d_b200.compat import random_init_generator
        G = random_init_generator(device=DEV, seed=0)
    seeds = [0, 1, 2, 3, 5]
    with torch.no_grad():
        want_img, want_seg, logits = _loop_strips(G, seeds, 0.7)
        got_img, got_seg = images.render_multiview(G, seeds, psi=0.7, batch_seeds=4)
        # the logits of the driver's own batches (4 seeds, the last one padded with repeats of seed 5): the backbone ran at another batch
        # size than the loop's, so they differ from the loop's by delta; a class is decided where the loop's top-two margin exceeds
        # twice that pixel's delta plus the bilinear-evaluation margin
        padded = seeds + [seeds[-1]] * 3
        z = torch.from_numpy(np.concatenate([np.random.RandomState(s).randn(1, G.z_dim) for s in padded])).to(DEV)
        ws = G.mapping(z=z, c=torch.tensor(images.FRONTAL).float().to(DEV).reshape(1, -1).repeat(8, 1), truncation_psi=0.7)
        jit = torch.tensor([images.view_seeds(s, 3) for s in padded])
        cams = images.view_cameras(images.YAWS, DEV)
        batch_logits = torch.cat([G.synthesis(ws[b:b + 4], c=cams.repeat(4, 1), render_params=images.render_params(0), noise_mode='const',
                                              return_seg=True, views=3, seed=jit[b:b + 4].reshape(-1))[1] for b in (0, 4)])[:15]
    got_img, got_seg = torch.from_numpy(got_img).to(DEV), torch.from_numpy(got_seg).to(DEV)
    assert got_img.shape == want_img.shape and got_seg.shape == want_seg.shape
    worst = int((got_img.int() - want_img.int()).abs().max())
    finite = torch.nan_to_num(logits, nan=0.0)
    top2 = finite.topk(2, dim=1).values
    delta = (batch_logits - logits).abs().amax(1)
    decided = _strip_mask((top2[:, 0] - top2[:, 1]) > 2 * delta + 1e-5 * (1 + finite.abs().max()), 3)
    print(f'{config}: max logit difference driver batches vs loop {delta.max().item():.2e}')
    differ = int(((got_seg != want_seg).any(-1) & ~decided).sum())
    print(f'{config}: driver vs loop, max image difference {worst} uint8 levels; {int((~decided).sum())} near-tie seg pixels, '
          f'{differ} of them differ')
    assert worst <= 1
    assert torch.equal(got_seg[decided], want_seg[decided])
