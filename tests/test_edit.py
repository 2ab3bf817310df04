"""CPU: ide3d_b200.encoder and ide3d_b200.edit against the reference's HybridEncoder, infer_hybrid_encoder.test, the Painter's edit step
and the face animation (tests/golden/edit_trace.npz, recorded by make_edit_golden.py with the weights and stand-in generator of
oracle/edit.py), the table formulation of ide3d_seg_stem, argument validation, and the ABI of the two new entry points."""

import ctypes
import math

import numpy as np
import pytest
import torch

from conftest import load_golden


@pytest.fixture(scope='module')
def trace():
    return load_golden('edit_trace')


@pytest.fixture(scope='module')
def models():
    from ide3d_b200.encoder import HybridEncoder
    from oracle import edit as oe
    torch.manual_seed(0)
    E = HybridEncoder(**oe.ENCODER_ARGS).eval()
    E.load_state_dict(oe.encoder_state(E))
    return E.requires_grad_(False), oe.standin_generator()


def _err(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return ((a - b).abs().max() / b.abs().max()).item()


def _pool(img):
    return torch.nn.functional.avg_pool2d(img.float(), 16)


def test_state_dict_matches_reference_names_and_shapes(trace, models):
    E, _ = models
    sd = E.state_dict()
    assert list(sd) == [str(n) for n in trace['state_names']]
    assert [','.join(map(str, v.shape)) for v in sd.values()] == [str(s) for s in trace['state_shapes']]


def test_encoder_float_and_mask_inputs_match_reference(trace, models):
    """E(img, one_hot * 2 - 1) through the composition, and E(img, uint8 mask) through the table formulation, against the reference's
    E(img, mask2label_np(mask) * 2 - 1).  Mask 0 has ids >= 19 and classes on every border.  Measured: 2.4e-6 and 2.9e-6 of max|ws|."""
    from ide3d_b200.encoder import one_hot_input
    from oracle import edit as oe
    E, _ = models
    masks, images = torch.from_numpy(trace['masks']), oe.golden_images(3)
    ref = trace['encoder_ws']
    with oe.cpu_edit_ops(), torch.no_grad():
        ws_float = E(images, one_hot_input(masks, 19))
        ws_mask = E(images, masks)
    assert _err(ws_float, ref) <= 1e-5 and _err(ws_mask, ref) <= 1e-5, (_err(ws_float, ref), _err(ws_mask, ref))


def test_one_hot_input_is_mask2label(trace):
    from ide3d_b200.encoder import one_hot_input
    m = torch.tensor([[[0, 18], [19, 255]]], dtype=torch.uint8)
    x = one_hot_input(m, 19)
    assert x.shape == (1, 19, 2, 2)
    assert x[0, :, 0, 0].tolist() == [1.0] + [-1.0] * 18 and x[0, 18, 0, 1] == 1 and (x[0, :, 1] == -1).all()


def test_seg_stem_tables_match_composition():
    """oracle.edit.seg_stem (the kernel's formulation) against one_hot * 2 - 1 -> stem -> conv1 / skip at C0 = 16 and 48 (sizes the
    kernel does not take: the formulation holds for any C0), with a class touching every border and ids >= classes."""
    from ide3d_b200.encoder import EncoderResBlock, Conv2dLayer, one_hot_input
    from oracle import edit as oe
    from oracle.backend import cpu_reference_ops
    g = torch.Generator().manual_seed(3)
    for c0, classes in ((16, 19), (48, 7)):
        torch.manual_seed(c0)
        stem, block = Conv2dLayer(classes, c0, 1), EncoderResBlock(c0, 2 * c0)
        for m in (stem, block):
            for p in m.parameters():
                if p.ndim == 1:
                    p.data.normal_(0, 0.3, generator=g)
        mask = torch.randint(0, classes + 3, (2, 12, 10), generator=g, dtype=torch.uint8)
        mask[:, 0, :] = 2
        mask[:, :, -1] = classes + 1
        with cpu_reference_ops(), torch.no_grad():
            x = stem(one_hot_input(mask, classes))
            y1_ref, skip_ref = block.conv1(x), block.skip(x)
            y1, skip = oe.seg_stem(mask, stem, block.conv1, block.skip)
        assert _err(y1, y1_ref) < 1e-6 and _err(skip, skip_ref) < 1e-6


def test_encode_replays_infer_hybrid_encoder(trace, models):
    """infer_hybrid_encoder.test with --target_code: E + w_avg, the pivot's rows from n_latents_geo = 8 on, then the render."""
    from ide3d_b200 import edit
    from oracle import edit as oe
    E, G = models
    image = oe.to_uint8(oe.golden_images(3)[:1]).float() / 127.5 - 1
    with oe.cpu_edit_ops():
        ws = edit.encode(E, G, image, torch.from_numpy(trace['masks'][1]), pivot=torch.from_numpy(trace['pivot']))
        img = G.synthesis(ws, torch.from_numpy(trace['labels'][:1]), noise_mode='const')
    assert _err(ws, trace['encode_ws']) <= 1e-5
    assert torch.equal(ws[:, 8:], torch.from_numpy(trace['pivot'])[:, 8:])
    assert _err(_pool(img), trace['encode_img']) <= 1e-5


def test_edit_replays_painter(trace, models):
    """Painter run_deep_model (inversion=True), one call per mask, against one edit() call with both masks."""
    from ide3d_b200 import edit
    from oracle import edit as oe
    E, G = models
    with oe.cpu_edit_ops():
        ws_edit, img = edit.edit(G, E, torch.from_numpy(trace['pivot']), torch.from_numpy(trace['labels'][:1]),
                                 torch.from_numpy(trace['masks'][1:3]))
    assert ws_edit.shape == (2, 10, 16) and img.shape == (2, 3, 512, 512)
    assert _err(ws_edit, trace['painter_ws']) <= 1e-5
    assert torch.equal(ws_edit[:, 8:], torch.from_numpy(trace['pivot'])[:, 8:].expand(2, -1, -1))
    assert _err(_pool(img), trace['painter_img']) <= 1e-5


def test_reenact_replays_face_animation(trace, models):
    """run_video_animation: seeds 0 and 1 driven by three (mask, camera) frames; two frames per call so the chunking is exercised."""
    from ide3d_b200 import edit
    from oracle import edit as oe
    E, G = models
    c_front = torch.tensor(edit.FRONTAL).reshape(1, -1)
    ws = torch.cat([G.mapping(torch.from_numpy(np.random.RandomState(int(s)).randn(1, G.z_dim)), c_front) for s in trace['anim_seeds']])
    geo = {}
    with oe.cpu_edit_ops():
        from ide3d_b200.encoder import HybridEncoder
        geometry = HybridEncoder.geometry
        HybridEncoder.geometry = lambda self, seg: geo.setdefault(len(geo), geometry(self, seg))
        try:
            img = edit.reenact(G, E, ws, torch.from_numpy(trace['labels']), torch.from_numpy(trace['masks']), frames_per_call=2)
        finally:
            HybridEncoder.geometry = geometry
    assert img.shape == (3, 2, 3, 512, 512)
    assert [g.shape[0] for g in geo.values()] == [2, 1]                 # each mask encoded once, not once per latent
    geo_ws = torch.cat(list(geo.values())) + G.mapping.w_avg
    ref_ws = torch.from_numpy(trace['anim_ws']) + G.mapping.w_avg
    assert _err(geo_ws, ref_ws[:, 0, :8]) <= 1e-5 and _err(geo_ws, ref_ws[:, 1, :8]) <= 1e-5
    assert _err(_pool(img.flatten(0, 1)), trace['anim_img'].reshape(6, 3, 32, 32)) <= 1e-5


def test_render_mask_is_argmax_of_upsampled_logits(models, trace):
    from ide3d_b200 import edit
    from oracle import edit as oe
    _, G = models
    ws = torch.from_numpy(trace['pivot']).repeat(2, 1, 1)
    with oe.cpu_edit_ops():
        m = edit.render_mask(G, ws, torch.from_numpy(trace['labels'][:2]))
        _, seg_raw = G.synthesis(ws, torch.from_numpy(trace['labels'][:2]), return_seg='raw')
    seg = torch.nn.functional.interpolate(seg_raw, size=(512, 512), mode='bilinear', align_corners=False)
    assert m.dtype == torch.uint8 and m.shape == (2, 512, 512) and len(m.unique()) > 3
    assert torch.equal(m, seg.argmax(1).to(torch.uint8))


def test_argument_validation(models, trace):
    from ide3d_b200 import edit
    from ide3d_b200.encoder import HybridEncoder
    E, G = models
    pivot, label = torch.from_numpy(trace['pivot']), torch.from_numpy(trace['labels'][:1])
    mask = torch.from_numpy(trace['masks'][1])
    image = torch.zeros(3, 512, 512)
    with pytest.raises(ValueError, match='rows'):
        edit.edit(G, HybridEncoder(64, 3, 8, w_dim=16), pivot, label, mask)
    with pytest.raises(ValueError, match='rows'):
        edit.edit(G, HybridEncoder(64, 2, 8, w_dim=8), pivot, label, mask)
    with pytest.raises(ValueError, match='uint8'):
        edit.edit(G, E, pivot, label, mask.long())
    with pytest.raises(ValueError, match='uint8'):
        edit.edit(G, E, pivot, label, mask[:256])
    with pytest.raises(ValueError, match='label'):
        edit.edit(G, E, pivot, label[:, :16], mask)
    with pytest.raises(ValueError, match='label'):
        edit.edit(G, E, pivot, label.repeat(3, 1), torch.stack([mask, mask]))
    with pytest.raises(ValueError, match='ws'):
        edit.edit(G, E, pivot[0], label, mask)
    with pytest.raises(ValueError, match=r'\[-1, 1\]'):
        edit.encode(E, G, image + 2, mask)
    with pytest.raises(ValueError, match='image'):
        edit.encode(E, G, image[:, :256], mask)
    with pytest.raises(ValueError, match='label'):
        edit.reenact(G, E, pivot, label.repeat(2, 1), torch.stack([mask] * 3))
    with pytest.raises(ValueError, match='uint8'):
        E.geometry(mask)


def test_seg_stem_entry_points_validate_before_the_device(lib):
    """Malformed parameters return a status without touching the device (the pointers below are never dereferenced)."""
    from ide3d_b200 import _lib
    assert lib.ide3d_seg_stem(None, None) == _lib.INVALID and b'null params' in lib.ide3d_last_error()
    assert lib.ide3d_seg_labels(None, None) == _lib.INVALID and b'null params' in lib.ide3d_last_error()
    assert lib.ide3d_seg_stem_scratch_bytes(19, 32) == 4 * 21 * (9 * 32 + 64)
    assert lib.ide3d_seg_stem_scratch_bytes(19, 48) == _lib.UNSUPPORTED and lib.ide3d_seg_stem_scratch_bytes(32, 32) == _lib.UNSUPPORTED
    fake = 0x10000
    p = _lib.SegStemParams()
    p.mask, p.n, p.h, p.w = fake, 2, 16, 16
    p.mask_stride_n, p.mask_stride_h, p.mask_stride_w = 256, 16, 1
    p.classes, p.c0, p.c1 = 19, 32, 64
    p.w0 = p.b0 = p.w1 = p.b1 = p.ws = p.fir = p.tables = p.y1 = p.skip = fake
    p.wg0 = p.wg1 = p.wgs = 1.0
    cases = [('c0', 48, _lib.UNSUPPORTED, b'c0 must be 32 or 64'), ('c1', 32, _lib.UNSUPPORTED, b'c1 must be 2 * c0'),
             ('classes', 32, _lib.UNSUPPORTED, b'at most 31 classes'), ('h', 15, _lib.UNSUPPORTED, b'even and >= 8'),
             ('w', 6, _lib.UNSUPPORTED, b'even and >= 8'), ('classes', 0, _lib.INVALID, b'bad sizes'), ('n', -1, _lib.INVALID, b'bad sizes'),
             ('mask', None, _lib.INVALID, b'null mask or output'), ('y1', None, _lib.INVALID, b'null mask or output'),
             ('w1', None, _lib.INVALID, b'null weight, bias or filter'), ('fir', None, _lib.INVALID, b'null weight, bias or filter'),
             ('tables', None, _lib.INVALID, b'null tables'), ('skip', fake + 4, _lib.INVALID, b'16-byte aligned')]
    for field, value, status, message in cases:
        saved = getattr(p, field)
        setattr(p, field, value)
        assert lib.ide3d_seg_stem(ctypes.byref(p), None) == status, field
        assert message in lib.ide3d_last_error(), (field, lib.ide3d_last_error())
        setattr(p, field, saved)
    p.n = 0
    assert lib.ide3d_seg_stem(ctypes.byref(p), None) == _lib.OK                                           # empty batch: no launch
    q = _lib.SegLabelsParams()
    q.seg, q.n, q.classes, q.in_h, q.in_w, q.out_h, q.out_w, q.out = fake, 1, 19, 8, 8, 32, 32, None
    assert lib.ide3d_seg_labels(ctypes.byref(q), None) == _lib.INVALID and b'null logits or output' in lib.ide3d_last_error()
    q.out, q.classes = fake, 0
    assert lib.ide3d_seg_labels(ctypes.byref(q), None) == _lib.INVALID and b'bad sizes' in lib.ide3d_last_error()


def test_product_stem_is_cuda_only(models):
    from ide3d_b200.torch_utils.ops import seg_stem
    E, _ = models
    with pytest.raises(RuntimeError, match='CUDA'):
        seg_stem.seg_stem(torch.zeros(1, 512, 512, dtype=torch.uint8), E.convs_seg[0], E.convs_seg[1].conv1, E.convs_seg[1].skip)
    assert math.isclose(E.convs_seg[0].weight_gain, 1 / math.sqrt(19))
