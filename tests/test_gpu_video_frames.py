"""GPU: ide3d_video_frames (csrc/frames.cu) against the reference's composition written with torch ops on the device
(oracle.frames: interpolate + mask2color + the float passes + cat + layout_grid's uint8 conversion), and the batched video driver's
image_seg / image_depth modes against the reference's batch-1 frame loop (gen_videos.py:129-139)."""

import pytest
import torch

from oracle import frames as ofr

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')


def _decided(seg):
    """Pixels where two bilinear evaluations cannot disagree on the class: top-two margin above 1e-5 * (1 + max|logit|), or a NaN
    logit (NaN counts as maximal on both sides, and only one class holds it)."""
    finite = torch.nan_to_num(seg, nan=0.0)
    top2 = finite.topk(2, dim=1).values
    return ((top2[:, 0] - top2[:, 1]) > 1e-5 * (1 + finite.abs().max())) | seg.isnan().any(1)


def _logits(n, r, strided, g):
    """Render-resolution logits, either the channel view of a ray-march output feat [n, r*r, 51] that SynthesisNetwork.forward hands
    out (maps[:, 32:]) or a dense tensor."""
    feat = torch.randn(n, r * r, 51, generator=g).to(DEV) * 3
    seg = feat.permute(0, 2, 1).reshape(n, 51, r, r)[:, 32:]
    return seg if strided else seg.contiguous()


def _check_seg(got, img, seg, what):
    """Image half bit-equal; seg colours equal wherever the class is decided.  Returns (near-tie pixels, those of them whose colour
    differs)."""
    from ide3d_b200.training.triplane import upsample_seg
    want = ofr.compose_frames(img, seg, 'image_seg')
    w = img.shape[-1]
    assert got.shape == want.shape and got.dtype == torch.uint8 and got.is_contiguous(), what
    assert torch.equal(got[..., :w], want[..., :w]), what
    decided = _decided(upsample_seg(seg, tuple(img.shape[-2:])))
    mask = decided[:, None].expand(-1, 3, -1, -1)
    assert torch.equal(got[..., w:][mask], want[..., w:][mask]), (what, int((got[..., w:] != want[..., w:])[mask].sum()))
    return int((~decided).sum()), int(((got[..., w:] != want[..., w:]).any(1) & ~decided).sum())


@pytest.mark.parametrize('r', [16, 48, 64, 128])
@pytest.mark.parametrize('size', [64, 512])
@pytest.mark.parametrize('channels_last', [False, True])
def test_kernel_matches_torch_composition(r, size, channels_last):
    from ide3d_b200 import video
    g = torch.Generator().manual_seed(r * 1000 + size)
    n = 3
    img = (torch.randn(n, 3, size, size, generator=g) * 1.2).to(DEV)         # some values beyond [-1, 1]: the clamp
    if channels_last:
        img = img.contiguous(memory_format=torch.channels_last)
    ties = {}
    for strided in (True, False):
        seg = _logits(n, r, strided, g)
        ties[strided] = _check_seg(video.compose_frames(img, seg, 'image_seg'), img, seg, (r, size, channels_last, strided))
    print(f'render {r} -> {size}, channels_last={channels_last}: of {n * size * size} pixels, near-tie / differing among them: '
          f'strided view {ties[True]}, dense {ties[False]}')
    got = video.compose_frames(img, None, 'image_depth')
    assert got.shape == (n, 3, size, size) and torch.equal(got, ofr.compose_frames(img, None, 'image_depth'))


def test_nan_logit_and_constant_frame():
    """A NaN logit wins its class wherever it reaches an interpolated pixel (torch.argmax counts NaN as maximal); a constant frame
    in image_depth divides 0 by 0, and the kernel writes what torch writes for it."""
    from ide3d_b200 import video
    g = torch.Generator().manual_seed(3)
    img = torch.randn(2, 3, 64, 64, generator=g).to(DEV)
    seg = _logits(2, 16, True, g)
    seg[1, 5, 7, 9] = float('nan')
    got = video.compose_frames(img, seg, 'image_seg')
    _check_seg(got, img, seg, 'nan logit')
    from ide3d_b200.training.triplane import upsample_seg
    hit = upsample_seg(seg, (64, 64))[1, 5].isnan()
    assert hit.sum() > 0
    assert (got[1, :, :, 64:][:, hit] == torch.tensor([204, 0, 204], dtype=torch.uint8, device=DEV)[:, None]).all()   # COLOR_MAP[5]
    img[1] = 0.25
    got = video.compose_frames(img, None, 'image_depth')
    want = ofr.compose_frames(img, None, 'image_depth')
    print('constant frame: torch writes', want[1].unique().tolist())
    assert torch.equal(got, want)


def test_empty_batch_and_bad_arguments():
    from ide3d_b200 import video
    assert video.compose_frames(torch.empty(0, 3, 8, 8, device=DEV), torch.empty(0, 19, 4, 4, device=DEV), 'image_seg').shape == (0, 3, 8, 16)
    assert video.compose_frames(torch.empty(0, 3, 8, 8, device=DEV), None, 'image_depth').shape == (0, 3, 8, 8)
    with pytest.raises(RuntimeError):
        video.compose_frames(torch.zeros(1, 3, 8, 8, device=DEV, dtype=torch.float16), None, 'image_depth')
    with pytest.raises(RuntimeError):
        video.compose_frames(torch.zeros(2, 3, 8, 8, device=DEV), torch.zeros(1, 19, 4, 4, device=DEV), 'image_seg')


# ------------------------------------------------------------------------------------------------ the driver
@pytest.fixture(scope='module')
def G():
    from ide3d_b200.training.triplane import TriPlaneGenerator
    torch.manual_seed(0)
    return TriPlaneGenerator(z_dim=32, w_dim=32, img_resolution=128, plane_resolution=64, render_size=32, channel_base=2048, channel_max=64,
                             sr_channels=(32, 32), mapping_kwargs=dict(num_layers=2)).eval().requires_grad_(False).to(DEV)


def _reference_cell(G, w, c, image_mode):
    """One cell as gen_videos.py:129-135 builds it (batch 1), then layout_grid's uint8 conversion (:29-30)."""
    from oracle.frames import mask2color, to_uint8
    from ide3d_b200.dnnlib.seg_tools import COLOR_MAP
    img, seg = G.synthesis(ws=w, c=c, noise_mode='const', return_seg=True, perturb=None)
    if image_mode == 'image_depth':
        img = -img
        img = (img - img.min()) / (img.max() - img.min()) * 2 - 1
    else:
        col = (mask2color(seg, COLOR_MAP) / 255. - 0.5) / 0.5
        img = torch.cat((img, col), -1)
    return to_uint8(img[0]), seg


@pytest.mark.parametrize('image_mode', ['image_seg', 'image_depth'])
def test_render_interp_video_matches_batch1_loop(G, image_mode, monkeypatch):
    """render_interp_video(image_mode=...) against the reference's per-cell loop; the full-resolution logits tensor is never built on
    the way (the upsample helper raises if it is called)."""
    from ide3d_b200 import video
    from ide3d_b200.training import triplane
    kw = dict(seeds=[0, 1, 2, 3], w_frames=2, grid_dims=(2, 1), truncation_cutoff=4)
    with torch.no_grad():
        ws, c, (F, gh, gw) = video.interp_video_inputs(G, **kw)
        cells = [_reference_cell(G, ws[i:i + 1].float().to(DEV), c[i:i + 1].to(DEV), image_mode) for i in range(ws.shape[0])]

        def no_upsample(*a, **k):
            raise AssertionError('the driver built the full-resolution logits')

        monkeypatch.setattr(triplane, 'upsample_seg', no_upsample)
        grids = video.render_interp_video(G, batch=4, synthesis_kwargs=dict(perturb=None), image_mode=image_mode, **kw)
    k = 2 if image_mode == 'image_seg' else 1
    assert tuple(grids.shape) == (F, gh * 128, gw * k * 128, 3) and grids.dtype == torch.uint8
    worst, ties, differ = 0, 0, 0
    for i, (want, seg) in enumerate(cells):
        f, xi = divmod(i, gw)
        got = grids[f, :, xi * k * 128:(xi + 1) * k * 128].permute(2, 0, 1).to(DEV)
        worst = max(worst, int((got[:, :, :128].int() - want[:, :, :128].int()).abs().max()))
        if image_mode == 'image_seg':
            decided = _decided(seg)[0][None].expand(3, -1, -1)
            ties += int((~decided[0]).sum())
            differ += int(((got[:, :, 128:] != want[:, :, 128:]).any(0) & ~decided[0]).sum())
            assert torch.equal(got[:, :, 128:][decided], want[:, :, 128:][decided]), i
    print(f'{image_mode}: driver vs batch-1 loop, max image difference {worst} uint8 levels, {ties} near-tie seg pixels '
          f'({differ} of them differ)')
    assert worst <= 1
