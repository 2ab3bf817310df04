"""GPU: the visualizer's frames (ide3d_b200.viz.renderer) and the display tail kernels (ide3d_viz_image, ide3d_viz_fft).

  * ide3d_viz_image equals the reference's torch tail on the device byte for byte (NCHW, channels-last and strided maps, depth maps,
    512^2 RGB, a 64^2 x 512 layer, float16), its stats are within 1e-6 of float64, and reruns are bit-identical
  * ide3d_viz_fft against float64 numpy: colormap indices within 1 everywhere and equal at >= 99.9 % of the pixels; refused shapes
    take the torch fallback; a constant map gives index 0
  * Renderer.render: a cached frame equals the uncached one bit for bit for every noise mode, after a pose change and a render-type
    change; a weight update that bumps _version invalidates the cache; image_depth / image_raw are the return_dict maps through the
    tail; a captured layer is the module's output on the unlinked path; planes + render_planes is forward for 1 and 3 views"""

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')


def torch_tail(out, render_type='image', sel_channels=3, base_channel=0, img_normalize=False, img_scale_db=0):
    """viz/renderer.py:362-393 in torch on the device: -> (uint8 [H, W, S], float64 stats of the raw map)."""
    out = out.to(torch.float32).clone()
    if sel_channels > out.shape[0]:
        sel_channels = 1
    base_channel = max(min(base_channel, out.shape[0] - sel_channels), 0)
    sel = out[base_channel:base_channel + sel_channels]
    o64, s64 = out.double(), sel.double()
    stats = torch.stack([o64.mean(), s64.mean(), o64.std(), s64.std(), o64.abs().max(), s64.abs().max()])
    if render_type == 'image_depth':
        out -= out.min()
        out /= out.max()
        out -= .5
        out *= -2
    img = sel
    if img_normalize:
        img = img / img.norm(float('inf'), dim=[1, 2], keepdim=True).clip(1e-8, 1e8)
    img = img * (10 ** (img_scale_db / 20))
    return (img * 127.5 + 128).clamp(0, 255).to(torch.uint8).permute(1, 2, 0), stats


def _map(c, h, w, layout='nchw', dtype=torch.float32, seed=0, scale=1.0, offset=0.0):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(1, c, h, w, generator=g) * scale + offset).to(DEV)
    if layout == 'channels_last':
        x = x.contiguous(memory_format=torch.channels_last)
    elif layout == 'strided':
        big = torch.randn(1, c + 2, h, w + 5, device=DEV)
        big[:, 1:c + 1, :, 3:3 + w] = x
        x = big[:, 1:c + 1, :, 3:3 + w]
    return x[0].to(dtype)


IMAGE_CASES = [
    # (C, H, W, layout, dtype, render_type, sel_channels, base_channel, img_normalize, img_scale_db, scale, offset)
    (3, 64, 64, 'nchw', torch.float32, 'image', 3, 0, False, 0, 1.0, 0.0),
    (3, 64, 64, 'channels_last', torch.float32, 'image', 3, 0, True, 6, 1.0, 0.0),
    (3, 64, 48, 'strided', torch.float32, 'image_raw', 1, 2, True, -3.5, 0.7, 0.1),
    (1, 64, 64, 'nchw', torch.float32, 'image_depth', 3, 0, False, 0, 0.05, 2.6),
    (1, 64, 64, 'strided', torch.float32, 'image_depth', 3, 0, True, 2, 0.05, 2.6),
    (3, 512, 512, 'nchw', torch.float32, 'image', 3, 0, False, 0, 1.0, 0.0),
    (3, 512, 512, 'channels_last', torch.float32, 'image', 3, 0, True, 0, 1.0, 0.0),
    (512, 64, 64, 'channels_last', torch.float32, 'image', 3, 100, True, 0, 3.0, 0.0),
    (512, 64, 64, 'nchw', torch.float32, 'image', 600, 7, False, 10, 3.0, 0.0),
    (512, 64, 64, 'nchw', torch.float32, 'image', 5, 510, False, 0, 3.0, 0.0),
    (64, 128, 128, 'channels_last', torch.float16, 'image', 3, 10, True, 0, 2.0, 0.0),
    (3, 256, 256, 'nchw', torch.float16, 'image_depth', 1, 1, False, 0, 0.5, 0.0),
]


@pytest.mark.parametrize('case', IMAGE_CASES, ids=lambda c: f'{c[0]}x{c[1]}x{c[2]}-{c[3]}-{str(c[4])[6:]}-{c[5]}-s{c[6]}b{c[7]}n{int(c[8])}')
def test_viz_image_equals_torch_tail(case):
    from ide3d_b200.torch_utils.ops import viz
    C, H, W, layout, dtype, rt, sel, base, norm, db, scale, offset = case
    x = _map(C, H, W, layout, dtype, seed=C + H, scale=scale, offset=offset)
    ref, ref_stats = torch_tail(x, rt, sel, base, norm, db)
    img, stats = viz.display(x, render_type=rt, sel_channels=sel, base_channel=base, img_normalize=norm, img_scale_db=db)
    assert img.shape == ref.shape
    assert torch.equal(img, ref), f'{(img != ref).sum().item()} bytes differ'
    scale_ref = ref_stats[4:].repeat(3)                      # the inf-norm sets the scale of a mean near zero
    err = (stats.double() - ref_stats).abs()
    assert (err <= 1e-6 * torch.maximum(ref_stats.abs(), scale_ref) + 1e-30).all(), (stats, ref_stats)
    img2, stats2 = viz.display(x, render_type=rt, sel_channels=sel, base_channel=base, img_normalize=norm, img_scale_db=db)
    assert torch.equal(img, img2) and torch.equal(stats, stats2)


def _index_lut(K):
    k = torch.arange(K)
    return torch.stack([k & 255, k >> 8, torch.zeros_like(k)], 1).to(torch.uint8).to(DEV)


def _decode(panel):
    p = panel.to(torch.int64).cpu().numpy()
    return p[..., 0] + 256 * p[..., 1]


def numpy_fft_index(x, beta, range_db, K):
    """The FFT panel's colormap indices in float64 numpy (viz/renderer.py:397-405)."""
    x = x.double().cpu().numpy()
    x = x - x.mean(axis=(1, 2), keepdims=True)
    w0 = torch.kaiser_window(x.shape[1], periodic=False, beta=beta).double().numpy()
    w1 = torch.kaiser_window(x.shape[2], periodic=False, beta=beta).double().numpy()
    x = x * w0[None, :, None] * w1[None, None, :]
    p = (np.abs(np.fft.fft2(x, axes=(1, 2))) ** 2).sum(0)
    p = np.roll(p, (p.shape[0] // 2, p.shape[1] // 2), axis=(0, 1))
    with np.errstate(divide='ignore'):
        db = 10 * np.log10(p / p.mean())
    t = ((db / range_db + 1) / 2) * (K - 1) + 0.5
    return np.clip(np.floor(np.nan_to_num(t, nan=-np.inf)), 0, K - 1).astype(np.int64)


@pytest.mark.parametrize('C', [1, 3, 512])
@pytest.mark.parametrize('N', [4, 8, 64, 256, 512])
def test_viz_fft_against_float64(N, C):
    from ide3d_b200.torch_utils.ops import viz
    K = 1024
    x = _map(C, N, N, 'channels_last' if C == 512 else 'nchw', seed=N + C, scale=2.0, offset=0.3)
    g = torch.Generator().manual_seed(N)
    x = x + torch.nn.functional.interpolate(torch.randn(1, C, 4, 4, generator=g), size=(N, N), mode='bilinear')[0].to(DEV) * 5
    for beta, rng in ((8, 50), (2, 30)):
        panel = torch.empty(N, N, 3, dtype=torch.uint8, device=DEV)
        viz.fft_panel(x, beta, rng, _index_lut(K), panel)
        got, ref = _decode(panel), numpy_fft_index(x, beta, rng, K)
        d = np.abs(got - ref)
        assert d.max() <= 1 and (d == 0).mean() >= 0.999, (d.max(), (d == 0).mean())
        again = torch.empty_like(panel)
        viz.fft_panel(x, beta, rng, _index_lut(K), again)
        assert torch.equal(panel, again)


def test_viz_fft_fallback_and_constant_map():
    from ide3d_b200.torch_utils.ops import viz
    from ide3d_b200 import _lib as L
    K = 256
    assert L.get_lib().ide3d_viz_fft_scratch_bytes(3, 48, 64) == L.UNSUPPORTED
    assert L.get_lib().ide3d_viz_fft_scratch_bytes(3, 2048, 2048) == L.UNSUPPORTED
    x = _map(3, 48, 64, seed=5)
    panel = torch.empty(48, 64, 3, dtype=torch.uint8, device=DEV)
    viz.fft_panel(x, 8, 50, _index_lut(K), panel)
    d = np.abs(_decode(panel) - numpy_fft_index(x, 8, 50, K))
    assert d.max() <= 1 and (d == 0).mean() >= 0.999
    const = torch.full((3, 32, 32), 0.25, device=DEV)
    panel = torch.full((32, 32, 3), 77, dtype=torch.uint8, device=DEV)
    viz.fft_panel(const, 8, 50, _index_lut(K), panel)
    assert (_decode(panel) == 0).all()


def test_display_fft_canvas():
    """The FFT view: the image on the left (one selected channel expanded to three), the panel on the right of the same canvas."""
    from ide3d_b200.torch_utils.ops import viz
    lut = _index_lut(1024)
    x = _map(8, 64, 64, seed=3)
    for sel, fft_all in ((1, True), (3, False)):
        img, _ = viz.display(x, sel_channels=sel, base_channel=2, fft_show=True, fft_all=fft_all, cmap=lut)
        ref, _ = torch_tail(x, sel_channels=sel, base_channel=2)
        assert img.shape == (64, 128, 3) and torch.equal(img[:, :64], ref.expand(64, 64, 3))
        panel = torch.empty(64, 64, 3, dtype=torch.uint8, device=DEV)
        viz.fft_panel(x if fft_all else x[2:2 + sel], 8, 50, lut, panel)
        assert torch.equal(img[:, 64:], panel)


# ------------------------------------------------------------------------------------------------------------------------- Renderer

@pytest.fixture(scope='module')
def G():
    from ide3d_b200.compat import random_init_generator
    G = random_init_generator(device='cuda', seed=0)
    with torch.no_grad():
        for name, p in G.synthesis.named_parameters():   # noise that shows, so the noise modes differ
            if name.endswith('noise_strength'):
                p.fill_(0.05)
    return G


ARGS = dict(w0_seeds=[[3, 0.6], [11, 0.4]], stylemix_idx=[0, 1, 30], stylemix_seed=5, trunc_psi=0.7, random_seed=2)


def _frame(r, G, **kw):
    res = r.render(pkl=G, **dict(ARGS, **kw))
    assert 'error' not in res, res.error
    return res


@pytest.mark.parametrize('noise_mode', ['const', 'random', 'none'])
def test_cached_frame_equals_uncached(G, noise_mode):
    from ide3d_b200.viz.renderer import Renderer
    cached, plain = Renderer(cmap=_index_lut(1024)), Renderer(cmap=_index_lut(1024))
    steps = [dict(yaw=0.2), dict(yaw=-0.35, pitch=0.1), dict(yaw=-0.35, pitch=0.1, render_type='image_depth'),
             dict(yaw=0.1, render_type='image_raw', fft_show=True, sel_channels=3)]
    entry = None
    for kw in steps:
        a = _frame(cached, G, noise_mode=noise_mode, do_backbone_caching=True, **kw)
        entry = entry or cached._backbone
        assert cached._backbone is entry                    # one backbone pass: every later frame is a cache hit
        b = _frame(plain, G, noise_mode=noise_mode, **kw)
        assert np.array_equal(a.image, b.image) and np.array_equal(a.stats, b.stats), kw


def test_weight_update_invalidates_cache(G):
    from ide3d_b200.viz.renderer import Renderer
    r = Renderer()
    a = _frame(r, G, do_backbone_caching=True, yaw=0.3)
    w = G.synthesis.vb16.conv1.weight
    saved = w.detach().clone()
    try:
        with torch.no_grad():
            w.mul_(1.7)
        b = _frame(r, G, do_backbone_caching=True, yaw=0.3)
        c = _frame(Renderer(), G, yaw=0.3)
    finally:
        with torch.no_grad():
            w.copy_(saved)
    assert not np.array_equal(a.image, b.image) and np.array_equal(b.image, c.image)


@pytest.mark.parametrize('render_type', ['image', 'image_depth', 'image_raw'])
def test_render_types_are_the_return_dict_maps(G, render_type):
    from ide3d_b200.viz import renderer as R
    res = _frame(R.Renderer(), G, render_type=render_type, yaw=0.25, img_normalize=render_type == 'image_raw')
    with torch.no_grad():
        w, _, _ = R.latents(G, ARGS['w0_seeds'], ARGS['stylemix_idx'], ARGS['stylemix_seed'], ARGS['trunc_psi'], 0)
        torch.manual_seed(ARGS['random_seed'])
        c = R.camera(0.25, 0, 4.2647, DEV)
        out = G.synthesis(w, c, noise_mode='const', return_dict=True)
    ref, _ = torch_tail(out[render_type][0], render_type, img_normalize=render_type == 'image_raw')
    assert np.array_equal(res.image, ref.cpu().numpy())
    assert res.image.shape[0] == (G.img_resolution if render_type == 'image' else G.synthesis.render_size)


def test_layer_capture_is_the_unlinked_output(G):
    from ide3d_b200.viz import renderer as R
    name = 'synthesis.vb64.conv1'
    res = _frame(R.Renderer(), G, layer_name=name, sel_channels=3, base_channel=5, img_normalize=True, yaw=0.1)
    assert name in [l.name for l in res.layers]
    with torch.no_grad():
        w, _, _ = R.latents(G, ARGS['w0_seeds'], ARGS['stylemix_idx'], ARGS['stylemix_seed'], ARGS['trunc_psi'], 0)
        torch.manual_seed(ARGS['random_seed'])
        c = R.camera(0.1, 0, 4.2647, DEV)
        seen = []
        h = G.synthesis.vb64.conv1.register_forward_hook(lambda m, i, o: seen.append(o))
        try:
            G.synthesis(w, c, noise_mode='const', unlinked=True)
        finally:
            h.remove()
        _, layers = R.run_synthesis_net(G, w, c, unlinked=True, noise_mode='const', force_fp32=False)
    ref, _ = torch_tail(seen[0][0], sel_channels=3, base_channel=5, img_normalize=True)
    assert np.array_equal(res.image, ref.cpu().numpy())
    assert [(l.name, l.shape, l.dtype) for l in res.layers] == [(l.name, l.shape, l.dtype) for l in layers]
    assert res.layers[-1].name == 'synthesis' and res.num_ws == 18 and res.has_noise and not res.has_input_transform


@pytest.mark.parametrize('views', [1, 3])
def test_render_planes_is_forward(G, views):
    from ide3d_b200 import images
    g = torch.Generator().manual_seed(views)
    ws = G.mapping(torch.randn(2, G.z_dim, generator=g).to(DEV), torch.tensor(images.FRONTAL, device=DEV).reshape(1, -1).repeat(2, 1))
    cams = images.view_cameras((-0.3, 0.0, 0.3)[:views], DEV).repeat(2, 1)
    with torch.no_grad():
        torch.manual_seed(0)
        a = G.synthesis(ws, cams, noise_mode='random', views=views)
        torch.manual_seed(0)
        img_v, seg_v, plan = G.synthesis.planes(ws, noise_mode='random')
        b = G.synthesis.render_planes(img_v, seg_v, ws, cams, noise_mode='random', views=views, style_plan=plan)
    assert torch.equal(a, b)
