"""GPU: ide3d_seg_stem / ide3d_seg_labels (csrc/seg_stem.cu) and ide3d_b200.edit on the device.

  * ide3d_seg_stem against the composition in float64 (F.one_hot -> *2-1 -> the module's stem, conv1 and skip) at C0 = 32 and 64,
    N = 1 and 3, over random, blocky, single-class, out-of-range and border-run masks; bit-identical reruns; two launches
  * shapes the kernel refuses fall back to the composition
  * E.geometry(uint8) against E.geometry(float one-hot) at 512^2 with fp32 convolutions
  * edit against encode(pivot render) + one synthesis, its launch count, and K masks against K single calls
  * reenact against the reference's per-frame loop
  * render_mask against the strip kernel's colours and against argmax(interpolate(logits))"""

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


@pytest.fixture
def fp32_convolutions():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _layers(c0, seed):
    from ide3d_b200.encoder import Conv2dLayer, EncoderResBlock
    torch.manual_seed(seed)
    stem, block = Conv2dLayer(19, c0, 1), EncoderResBlock(c0, 2 * c0)
    for m in (stem, block):
        for p in m.parameters():
            if p.ndim == 1:
                p.data.normal_(0, 0.3)
    return stem.to(DEV).requires_grad_(False), block.to(DEV).requires_grad_(False)


def _masks(kind, n, size, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    if kind == 'random':
        return torch.randint(0, 19, (n, size, size), device=DEV, generator=g, dtype=torch.uint8)
    if kind == 'blocky':
        b = torch.randint(0, 19, (n, size // 16, size // 16), device=DEV, generator=g, dtype=torch.uint8)
        return b.repeat_interleave(16, 1).repeat_interleave(16, 2).contiguous()
    if kind == 'one_class':
        return torch.full((n, size, size), 13, device=DEV, dtype=torch.uint8)
    if kind == 'out_of_range':
        return torch.randint(0, 256, (n, size, size), device=DEV, generator=g, dtype=torch.uint8)
    m = torch.randint(0, 19, (n, size, size), device=DEV, generator=g, dtype=torch.uint8)   # 'borders': a class run along every border
    m[:, :2, :], m[:, -2:, :], m[:, :, :2], m[:, :, -2:] = 18, 4, 200, 1
    return m


def _composition64(mask, stem, block):
    from ide3d_b200.encoder import one_hot_input
    import copy
    s64, b64 = copy.deepcopy(stem).double(), copy.deepcopy(block).double()
    for m in (s64, b64.conv1, b64.conv2, b64.skip):
        m.resample_filter = m.resample_filter.float()                                   # FIR taps stay fp32, as conv2d_resample wants
    x = s64(one_hot_input(mask, 19, torch.float64))
    return b64.conv1(x), b64.skip(x)


@pytest.mark.parametrize('c0, size', [(32, 512), (64, 256)])
@pytest.mark.parametrize('n', [1, 3])
@pytest.mark.parametrize('kind', ['random', 'blocky', 'one_class', 'out_of_range', 'borders'])
def test_seg_stem_matches_float64_composition(c0, size, n, kind):
    from ide3d_b200 import _lib
    from ide3d_b200.torch_utils.ops import seg_stem
    stem, block = _layers(c0, c0 + n)
    mask = _masks(kind, n, size, seed=n)
    if kind == 'random' and n == 3:
        mask = mask.transpose(1, 2)                                                      # any strides
    with torch.no_grad():
        n0 = _lib.launch_count()
        y1, skip = seg_stem.seg_stem(mask, stem, block.conv1, block.skip)
        launches = _lib.launch_count() - n0
        y1_ref, skip_ref = _composition64(mask, stem, block)
        y1b, skipb = seg_stem.seg_stem(mask, stem, block.conv1, block.skip)
    torch.cuda.synchronize()
    e1, e2 = rel(y1, y1_ref), rel(skip, skip_ref)
    print(f'C0 {c0} n {n} {kind}: y1 {e1:.2e} skip {e2:.2e} of max|ref|')
    assert y1.shape == (n, c0, size, size) and skip.shape == (n, 2 * c0, size // 2, size // 2)
    assert y1.is_contiguous(memory_format=torch.channels_last) and skip.is_contiguous(memory_format=torch.channels_last)
    assert e1 <= 1e-5 and e2 <= 1e-5
    assert torch.equal(y1, y1b) and torch.equal(skip, skipb)
    assert launches == 2


def test_unsupported_shapes_fall_back_to_composition():
    from ide3d_b200.encoder import HybridEncoder, one_hot_input
    from ide3d_b200.torch_utils.ops import seg_stem
    stem, block = _layers(48, 1)
    assert seg_stem.seg_stem(_masks('random', 1, 64, 0), stem, block.conv1, block.skip) is None               # C0 = 48
    stem, block = _layers(32, 1)
    assert seg_stem.seg_stem(_masks('random', 1, 6, 0), stem, block.conv1, block.skip) is None                # < 8
    torch.manual_seed(0)
    E = HybridEncoder(64, 2, 2, w_dim=16).to(DEV).requires_grad_(False)                                       # C0 = 256: unsupported
    mask = _masks('borders', 2, 64, 3)
    with torch.no_grad():
        assert torch.equal(E.geometry(mask), E.geometry(one_hot_input(mask, 19)))


def test_grad_mode_runs_the_composition():
    from ide3d_b200.encoder import HybridEncoder, one_hot_input
    torch.manual_seed(0)
    E = HybridEncoder(64, 2, 2, w_dim=16).to(DEV)
    mask = _masks('blocky', 1, 64, 2)
    ws = E.geometry(mask)
    ws.square().sum().backward()
    assert E.convs_seg[0].weight.grad is not None and E.convs_seg[1].conv1.weight.grad is not None


@pytest.fixture(scope='module')
def G():
    from ide3d_b200.compat import random_init_generator
    G = random_init_generator(device=DEV, seed=0)
    G.rendering_kwargs['perturb'] = None
    return G


@pytest.fixture(scope='module')
def E(G):
    from ide3d_b200.encoder import HybridEncoder
    torch.manual_seed(1)
    E = HybridEncoder(512, G.num_ws - 8, 8, w_dim=G.w_dim)
    for p in E.parameters():
        if p.ndim == 1:
            p.data.normal_(0, 0.2)
    return E.eval().requires_grad_(False).to(DEV)


def _pivot(G, seed=0, n=1):
    from ide3d_b200 import edit
    z = torch.from_numpy(__import__('numpy').random.RandomState(seed).randn(n, G.z_dim)).float().to(DEV)
    c = torch.tensor(edit.FRONTAL, device=DEV).reshape(1, -1).repeat(n, 1)
    with torch.no_grad():
        return G.mapping(z, c), c


def test_geometry_mask_matches_float_one_hot(E, fp32_convolutions):
    from ide3d_b200.encoder import one_hot_input
    mask = torch.cat([_masks('blocky', 2, 512, 5), _masks('borders', 1, 512, 6), _masks('out_of_range', 1, 512, 7)])
    with torch.no_grad():
        a, b = E.geometry(mask), E.geometry(one_hot_input(mask, 19))
    print(f'geometry: uint8 path vs float one-hot {rel(a, b):.2e} of max|ws|')
    assert rel(a, b) <= 1e-5


def test_edit_is_encode_then_one_synthesis(G, E):
    from ide3d_b200 import _lib, edit
    ws, label = _pivot(G)
    masks = torch.cat([_masks('blocky', 2, 512, 8), _masks('borders', 1, 512, 9)])
    with torch.no_grad():
        n0 = _lib.launch_count()
        ws_edit, img = edit.edit(G, E, ws, label, masks)
        n_edit = _lib.launch_count() - n0
        n0 = _lib.launch_count()
        E.geometry(masks)
        n_geo = _lib.launch_count() - n0
        n0 = _lib.launch_count()
        G.synthesis(ws_edit, label.expand(3, -1), noise_mode='const')
        n_syn = _lib.launch_count() - n0
        n0 = _lib.launch_count()
        E.appearance(torch.zeros(3, 3, 512, 512, device=DEV))
        n_app = _lib.launch_count() - n0
        render = G.synthesis(ws, label, noise_mode='const')
        ws_ref = edit.encode(E, G, render.expand(3, -1, -1, -1).clamp(-1, 1), masks, pivot=ws)
        img_ref = G.synthesis(ws_ref, label.expand(3, -1), noise_mode='const')
        singles = [edit.edit(G, E, ws, label, masks[k]) for k in range(3)]
    print(f'edit launches {n_edit} = geometry {n_geo} + synthesis {n_syn} (image branch alone: {n_app})')
    assert n_edit == n_geo + n_syn and n_app > 0
    assert torch.equal(ws_edit, ws_ref) and torch.equal(img, img_ref)
    e_ws = max(rel(ws_edit[k:k + 1], s[0]) for k, s in enumerate(singles))
    e_img = max(rel(img[k:k + 1], s[1]) for k, s in enumerate(singles))
    print(f'edit: 3 masks in one call vs 3 single calls: ws {e_ws:.2e}, images {e_img:.2e} of max|ref|')
    assert e_ws <= 1e-3 and e_img <= 1e-2


def test_reenact_matches_reference_loop(G, E, fp32_convolutions):
    from ide3d_b200 import edit
    from ide3d_b200.encoder import one_hot_input
    from ide3d_b200.images import view_cameras
    ws, _ = _pivot(G, seed=3, n=2)
    labels = view_cameras((-0.3, 0.0, 0.25), device=DEV)
    masks = torch.cat([_masks('blocky', 2, 512, 10), _masks('borders', 1, 512, 11)])
    rp = dict(edit.REENACT_RENDER_PARAMS, num_steps=24)
    geo = []
    with torch.no_grad():
        out = edit.reenact(G, E, ws, labels, masks, render_params=rp, frames_per_call=2)
        w_avg = G.mapping.w_avg[None, None, :]
        worst = 0.0
        for f in range(3):
            c = labels[f:f + 1].repeat(2, 1)
            cond = G.synthesis(ws, c, noise_mode='const', render_params=rp)
            rec = E(cond, one_hot_input(masks[f:f + 1], 19).repeat(2, 1, 1, 1)) + w_avg
            geo.append(rec[:, :8])
            worst = max(worst, rel(out[f], G.synthesis(rec, c, noise_mode='const', render_params=rp)))
    print(f'reenact vs per-frame loop: images {worst:.2e} of max|ref|')
    assert out.shape == (3, 2, 3, 512, 512)
    assert all(torch.equal(g[0], g[1]) for g in geo)
    assert worst <= 1e-3


def test_render_mask_matches_strip_colours_and_argmax(G):
    from ide3d_b200 import edit, images
    from ide3d_b200.dnnlib.seg_tools import _lut_for
    ws, _ = _pivot(G, seed=4, n=2)
    label = images.view_cameras((-0.4, 0.3), device=DEV)
    with torch.no_grad():
        ids = edit.render_mask(G, ws, label)
        img, seg_raw = G.synthesis(ws, label, noise_mode='const', return_seg='raw')
        _, strip = images.compose_strips(img, seg_raw, 1)
        lut = _lut_for(DEV, 19).to(torch.uint8)
        up = F.interpolate(seg_raw, size=(512, 512), mode='bilinear', align_corners=False)
    assert ids.shape == (2, 512, 512) and ids.dtype == torch.uint8
    assert torch.equal(lut[ids.long()], strip)
    top2 = up.topk(2, dim=1).values
    decided = (top2[:, 0] - top2[:, 1]) > 1e-5
    differ = int((ids != up.argmax(1).to(torch.uint8)).sum())
    print(f'render_mask vs argmax(interpolate): {differ} pixels differ, {int((~decided).sum())} within the 1e-5 top-two margin, '
          f'{len(ids.unique())} classes present')
    assert torch.equal(ids[decided], up.argmax(1).to(torch.uint8)[decided])
