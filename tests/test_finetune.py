"""CPU: ide3d_b200.parsing and ide3d_b200.finetune against the reference's BiSeNet and apps/finetune_hybrid_encoder.py
(tests/golden/finetune_trace.npz, recorded by make_finetune_golden.py with the weights of oracle/finetune.py and oracle/edit.py), the
{0, 1} re-parameterisation of the stem, argument validation, and the ABI of the new entry points."""

import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT, load_golden

NAMES = ('loss_ws', 'loss_gen_l2', 'loss_real_entropy', 'loss_real_cycle')


@pytest.fixture(scope='module')
def trace():
    return load_golden('finetune_trace')


@pytest.fixture(scope='module')
def parser():
    from ide3d_b200.parsing import BiSeNet
    from oracle import finetune as of
    torch.manual_seed(0)
    net = BiSeNet(20)
    net.load_state_dict(of.bisenet_state(net), strict=True)
    return net.eval().requires_grad_(False)


def _encoder():
    from ide3d_b200.encoder import HybridEncoder
    from oracle import edit as oe
    torch.manual_seed(0)
    E = HybridEncoder(**oe.ENCODER_ARGS).eval()
    E.load_state_dict(oe.encoder_state(E))
    return E.requires_grad_(False)


def _image():
    from oracle import edit as oe
    return oe.to_uint8(oe.golden_images(1, seed=44)).float() / 127.5 - 1


def _err(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return ((a - b).abs().max() / b.abs().max()).item()


def test_bisenet_loads_reference_state_and_matches_logits(trace, parser):
    """Same state_dict names as the reference (strict loading, BatchNorm statistics included); forward's logits match the reference's
    on the portrait, and forward is logits() upsampled with align_corners=True."""
    from ide3d_b200.parsing import BiSeNet
    assert list(parser.state_dict()) == [str(n) for n in trace['bisenet_names']]
    with torch.no_grad():
        x = _image()
        full, a, b = parser(x)
        small = parser.logits(x)
    assert a is None and b is None and small.shape == (1, 20, 64, 64) and full.shape == (1, 20, 512, 512)
    assert torch.equal(full, F.interpolate(small, (512, 512), mode='bilinear', align_corners=True))
    assert _err(F.avg_pool2d(full, 16), trace['bisenet_logits']) <= 1e-5
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, 'segNet-20Class.pth')
        torch.save(parser.state_dict(), path)
        net = BiSeNet.load(path)
        assert not net.training and not any(p.requires_grad for p in net.parameters())
        with pytest.raises(FileNotFoundError):
            BiSeNet.load(os.path.join(d, 'missing.pth'))


@pytest.mark.parametrize('tag', ['seg', 'parse'])
def test_finetune_replays_reference(trace, parser, tag):
    """Three steps with --target_seg (mask 1 of oracle.edit.golden_masks) and without (the parse of the image): per-step losses, the
    tuned weights (the stem, block 0 and 16 output channels of projector_seg), the sums of their change and the saved mask.
    Measured: losses 4.3e-7 / 3.0e-7 of max|loss|, tuned weights 2.6e-7 / 3.3e-7 of max|w|, the change itself 2.4e-2 / 5.1e-2 of its
    max (Adam's first steps are about lr * sign(grad): a gradient near zero can change its update by a whole step), the sums of the
    change 3.5e-5 / 2.8e-5; the masks are equal."""
    from ide3d_b200 import finetune
    from oracle import edit as oe, finetune as of
    E = _encoder()
    initial = {k: v.clone() for k, v in E.state_dict().items()}
    G = oe.standin_generator()
    mask = oe.golden_masks()[1] if tag == 'seg' else None
    with of.cpu_finetune_ops():
        E_t, out_mask, losses = finetune.run(G, E, _image(), torch.from_numpy(trace['code']), torch.from_numpy(trace['label']),
                                             parser=parser, mask=mask, steps=3)
    ref = trace[f'{tag}_losses']
    got = np.stack([losses[n] for n in NAMES], 1)
    e_loss = float(np.abs(got - ref).max() / np.abs(ref).max())
    state = E_t.state_dict()
    names = [str(n) for n in trace[f'{tag}_names']]
    delta = {n: state[n].double() - initial[n].double() for n in names}
    whole = [n for n in names if n.startswith(('convs_seg.0.', 'convs_seg.1.')) and not n.endswith('resample_filter')]
    ref_w = {n: initial[n].double() + torch.from_numpy(trace[f'{tag}_d_{n}']).double() for n in whole}
    ref_w['rows'] = initial['projector_seg.weight'][:16].double() + torch.from_numpy(trace[f'{tag}_d_projector_rows']).double()
    got_w = {n: state[n] for n in whole}
    got_w['rows'] = state['projector_seg.weight'][:16]
    e_w = max(_err(got_w[n], ref_w[n]) for n in ref_w)
    e_d = max(max(_err(delta[n], trace[f'{tag}_d_{n}']) for n in whole),
              _err(delta['projector_seg.weight'][:16], trace[f'{tag}_d_projector_rows']))
    sums = np.array([delta[n].sum().item() for n in names])
    e_sums = float(np.abs(sums - trace[f'{tag}_d_sums']).max() / np.abs(trace[f'{tag}_d_sums']).max())
    print(f'{tag}: losses {e_loss:.2e}, tuned weights {e_w:.2e}, their change {e_d:.2e}, sums of the change {e_sums:.2e}')
    assert e_loss <= 1e-5 and e_w <= 1e-5
    assert e_d <= 1e-1 and e_sums <= 1e-3
    assert out_mask.dtype == torch.uint8 and out_mask.shape == (512, 512)
    assert np.array_equal(out_mask.numpy(), trace[f'{tag}_mask'])
    assert not E_t.training and not any(p.requires_grad for p in E_t.parameters())
    assert all(torch.equal(v, initial[k]) for k, v in E.state_dict().items())               # the caller's E is untouched


def test_unsigned_mask_matches_float_zero_one_input():
    """The {0, 1} re-parameterisation of the stem (HybridEncoder._mask_stem) through the table formulation against the {0, 1} one-hot
    float map through the composition in float64: block 0's conv1 / skip outputs' gradients w.r.t. all five parameters (measured
    2.6e-7 of max|g|), and the geometry rows against the fp32 composition (measured 3.9e-6 of max|ws|)."""
    import copy
    from ide3d_b200.encoder import _UnsignedStem, one_hot_input
    from oracle import edit as oe, finetune as of
    E = _encoder()
    E.convs_seg.requires_grad_(True)
    stem, block = E.convs_seg[0], E.convs_seg[1]
    masks = oe.golden_masks()[:2]
    g = torch.Generator().manual_seed(0)
    gy, gs = torch.randn(2, 32, 512, 512, generator=g), torch.randn(2, 64, 256, 256, generator=g)
    with of.cpu_finetune_ops():
        y1, sk = of.seg_stem(masks, _UnsignedStem(stem), block.conv1, block.skip)
        params = [stem.weight, stem.bias, block.conv1.weight, block.conv1.bias, block.skip.weight]
        got = torch.autograd.grad((y1 * gy).sum() + (sk * gs).sum(), params)
        s64, b64 = copy.deepcopy(stem).double(), copy.deepcopy(block).double()
        for m in (s64, b64.conv1, b64.conv2, b64.skip):
            m.resample_filter = m.resample_filter.float()
        x = s64((one_hot_input(masks, 19, torch.float64) + 1) / 2)
        ref = torch.autograd.grad((b64.conv1(x) * gy.double()).sum() + (b64.skip(x) * gs.double()).sum(),
                                  [s64.weight, s64.bias, b64.conv1.weight, b64.conv1.bias, b64.skip.weight])
        with torch.no_grad():
            a = E.geometry(masks, signed=False)
            b = E.geometry((one_hot_input(masks, 19) + 1) / 2)
    errs = [_err(p, q) for p, q in zip(got, ref)]
    assert max(errs) <= 3e-6, errs
    assert _err(a, b) <= 1e-5, _err(a, b)


def test_argument_validation(trace, parser):
    from ide3d_b200 import finetune
    from oracle import edit as oe
    E, G = _encoder(), oe.standin_generator()
    code, label, image = torch.from_numpy(trace['code']), torch.from_numpy(trace['label']), _image()
    with pytest.raises(ValueError, match=r'\[-1, 1\]'):
        finetune.run(G, E, image + 2, code, label, parser=parser, steps=0)
    with pytest.raises(ValueError, match='single portrait'):
        finetune.run(G, E, image.repeat(2, 1, 1, 1), code, label, parser=parser, steps=0)
    with pytest.raises(ValueError, match='ws'):
        finetune.run(G, E, image, code[:, :4], label, parser=parser, steps=0)
    with pytest.raises(ValueError, match='label'):
        finetune.run(G, E, image, code, label[:, :16], parser=parser, steps=0)
    with pytest.raises(ValueError, match='uint8'):
        finetune.run(G, E, image, code, label, parser=parser, mask=torch.zeros(512, 512), steps=0)
    with pytest.raises(ValueError, match='steps'):
        finetune.run(G, E, image, code, label, parser=parser, steps=-1)


def _probe_size():
    probe = r'''
    #include <stdio.h>
    #include "ide3d_b200.h"
    int main(void) { printf("%zu\n", sizeof(ide3d_seg_stem_bwd_params)); return 0; }'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, 'p.c')
        open(c, 'w').write(probe)
        exe = os.path.join(d, 'p')
        subprocess.run(['gcc', '-I', os.path.join(ROOT, 'include'), c, '-o', exe], check=True)
        return int(subprocess.run([exe], capture_output=True, text=True, check=True).stdout)


def test_new_symbols_exported_and_struct_layout(lib):
    from ide3d_b200 import _lib
    for name in ('ide3d_seg_stem_bwd', 'ide3d_seg_stem_bwd_scratch_bytes', 'ide3d_seg_xent_fwd_ac', 'ide3d_seg_xent_bwd_ac',
                 'ide3d_seg_labels_ac'):
        assert name in _lib.exported_symbols() and hasattr(lib, name)
    assert ctypes.sizeof(_lib.SegStemBwdParams) == _probe_size()


def test_new_entry_points_validate_before_the_device(lib):
    """Malformed parameters return a status without touching the device (the pointers below are never dereferenced)."""
    from ide3d_b200 import _lib
    for name in ('ide3d_seg_stem_bwd', 'ide3d_seg_xent_fwd_ac', 'ide3d_seg_xent_bwd_ac', 'ide3d_seg_labels_ac'):
        assert getattr(lib, name)(None, None) == _lib.INVALID and b'null params' in lib.ide3d_last_error(), name
    need = lib.ide3d_seg_stem_bwd_scratch_bytes(2, 16, 16, 19, 32)
    assert need > 0 and need % 16 == 0
    assert lib.ide3d_seg_stem_bwd_scratch_bytes(2, 16, 16, 19, 48) == _lib.UNSUPPORTED
    assert lib.ide3d_seg_stem_bwd_scratch_bytes(2, 15, 16, 19, 32) == _lib.UNSUPPORTED
    assert lib.ide3d_seg_stem_bwd_scratch_bytes(-1, 16, 16, 19, 32) == _lib.INVALID
    fake = 0x10000
    b = _lib.SegStemBwdParams()
    p = b.fwd
    p.mask, p.n, p.h, p.w = fake, 2, 16, 16
    p.mask_stride_n, p.mask_stride_h, p.mask_stride_w = 256, 16, 1
    p.classes, p.c0, p.c1 = 19, 32, 64
    p.w0 = p.b0 = p.w1 = p.b1 = p.ws = p.fir = p.tables = p.y1 = p.skip = fake
    p.wg0 = p.wg1 = p.wgs = 1.0
    b.grad_y1 = b.grad_skip = b.grad_w0 = b.grad_b0 = b.grad_w1 = b.grad_b1 = b.grad_ws = b.scratch = fake
    b.scratch_bytes = need
    cases = [('fwd.c0', 48, _lib.UNSUPPORTED, b'c0 must be 32 or 64'), ('fwd.classes', 32, _lib.UNSUPPORTED, b'at most 31 classes'),
             ('fwd.h', 15, _lib.UNSUPPORTED, b'even and >= 8'), ('fwd.n', -1, _lib.INVALID, b'bad sizes'),
             ('fwd.w1', None, _lib.INVALID, b'null weight, bias or filter'), ('grad_ws', None, _lib.INVALID, b'null gradient output'),
             ('fwd.mask', None, _lib.INVALID, b'null mask, tables or incoming gradient'),
             ('grad_skip', None, _lib.INVALID, b'null mask, tables or incoming gradient'),
             ('grad_y1', fake + 4, _lib.INVALID, b'16-byte aligned'), ('scratch', None, _lib.INVALID, b'scratch'),
             ('scratch_bytes', need - 1, _lib.INVALID, b'scratch holds')]
    for field, value, status, message in cases:
        obj, attr = (b.fwd, field[4:]) if field.startswith('fwd.') else (b, field)
        saved = getattr(obj, attr)
        setattr(obj, attr, value)
        if field.startswith('fwd.'):
            b.fwd = obj
        assert lib.ide3d_seg_stem_bwd(ctypes.byref(b), None) == status, field
        assert message in lib.ide3d_last_error(), (field, lib.ide3d_last_error())
        setattr(obj, attr, saved)
        if field.startswith('fwd.'):
            b.fwd = obj
    q = _lib.SegXentParams()
    q.seg, q.n, q.classes, q.in_h, q.in_w, q.out_h, q.out_w = fake, 1, 33, 8, 8, 32, 32
    q.mask = q.lse = fake
    assert lib.ide3d_seg_xent_fwd_ac(ctypes.byref(q), None) == _lib.INVALID and b'at most 32' in lib.ide3d_last_error()
    q.classes = 20
    assert lib.ide3d_seg_xent_bwd_ac(ctypes.byref(q), None) == _lib.INVALID and b'null grad_loss' in lib.ide3d_last_error()
    r = _lib.SegLabelsParams()
    r.seg, r.n, r.classes, r.in_h, r.in_w, r.out_h, r.out_w, r.out = fake, 1, 20, 8, 8, 32, 32, None
    assert lib.ide3d_seg_labels_ac(ctypes.byref(r), None) == _lib.INVALID and b'null logits or output' in lib.ide3d_last_error()
