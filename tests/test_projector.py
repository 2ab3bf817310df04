"""CPU: ide3d_b200.projector against the reference's three projectors (tests/golden/projector_trace.npz, recorded by
make_projector_golden.py with the stand-ins of oracle/projector.py), the oracle's loss restatements against direct autograd, the
mirror / camera helpers, argument validation, and the ABI of the projector kernels."""

import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import load_golden

MODES = {'w': dict(), 'w_plus': dict(w_plus=True), 'join_view': dict(mirror=True)}


def _replay(mode, features=None, **extra):
    from ide3d_b200 import projector
    from oracle import projector as op
    g = load_golden('projector_trace')
    kw = eval(str(g['kwargs']))                    # the projector keyword arguments the trace was recorded with
    label, target = torch.from_numpy(g['label']), torch.from_numpy(g['target'])
    dist, loss = [], []
    torch.manual_seed(int(g['torch_seed']))
    with op.cpu_projector_ops():
        ws, lab = projector.project(op.StandInGenerator(seed=int(g['generator_seed'])), label, target,
                                    features=features or op.standin_features(), seed=int(g['w_avg_seed']),
                                    on_step=lambda s, d, l: (dist.append(d.item()), loss.append(l.item())), **MODES[mode], **kw, **extra)
    return g, ws, lab, np.array(dist), np.array(loss)


@pytest.mark.parametrize('mode', sorted(MODES))
def test_replays_reference_projector(mode):
    """Same torch ops in the same order as the reference loop: W and W+ are bit-exact.  The join view renders both cameras from one
    backbone pass, so the backbone's gradient is J^T (g1 + g2) rather than J^T g1 + J^T g2: fp32 rounding, which Adam's
    normalised steps keep at the 1e-6 level over the 15 recorded steps."""
    g, ws, lab, dist, loss = _replay(mode)
    ref_ws = torch.from_numpy(g[f'{mode}_ws'])
    if mode != 'w_plus':                          # the reference's W projector returns 18 rows; every row is the one w
        assert ws.shape[1] == 6 and torch.equal(ref_ws, ref_ws[:, :1].expand_as(ref_ws))
        ref_ws = ref_ws[:, :ws.shape[1]]
    assert torch.equal(lab, torch.from_numpy(g['label']))
    if mode == 'join_view':
        torch.testing.assert_close(ws, ref_ws, rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(dist, g[f'{mode}_dist'], rtol=1e-5)
        np.testing.assert_allclose(loss, g[f'{mode}_loss'], rtol=1e-5)
    else:
        assert torch.equal(ws, ref_ws)
        np.testing.assert_array_equal(dist, g[f'{mode}_dist'])
        np.testing.assert_array_equal(loss, g[f'{mode}_loss'])


def test_features_from_file_and_missing_file(tmp_path):
    from ide3d_b200 import projector
    from oracle import projector as op
    path = tmp_path / 'vgg16.pt'
    path.write_bytes(op.standin_features_bytes())
    g, ws, _, dist, _ = _replay('w', features=str(path))
    assert torch.equal(ws, torch.from_numpy(g['w_ws'])[:, :6])
    label, target = op.golden_inputs()
    with pytest.raises(FileNotFoundError):
        projector.project(op.StandInGenerator(), label, target, features=str(tmp_path / 'absent.pt'), num_steps=1, w_avg_samples=4)


def test_caller_generator_untouched():
    from ide3d_b200 import projector
    from oracle import projector as op
    G = op.StandInGenerator()
    before = {k: v.clone() for k, v in G.state_dict().items()}
    label, target = op.golden_inputs()
    with op.cpu_projector_ops():
        projector.project(G, label, target, features=op.standin_features(), num_steps=3, w_avg_samples=8, refine_camera=True)
    assert all(torch.equal(before[k], v) for k, v in G.state_dict().items())
    assert all(not p.requires_grad or p.grad is None for p in G.parameters())


def _oracle_reg_autograd(bufs):
    """The regulariser by direct autograd, each level pooled explicitly (independent of the oracle's loop structure)."""
    total = 0.0
    for b in bufs:
        n = b
        while True:
            total = total + (n * n.roll(1, 1)).mean() ** 2 + (n * n.roll(1, 0)).mean() ** 2
            if n.shape[0] <= 8:
                break
            n = 0.25 * (n[0::2, 0::2] + n[0::2, 1::2] + n[1::2, 0::2] + n[1::2, 1::2])
    return total


def test_oracle_noise_reg_matches_autograd():
    from oracle import projector as op
    g = torch.Generator().manual_seed(0)
    bufs = [torch.randn(s, s, generator=g, dtype=torch.float64, requires_grad=True) for s in (4, 8, 16, 64)]
    a = op.noise_reg(bufs)
    ga = torch.autograd.grad(a, bufs)
    b = _oracle_reg_autograd(bufs)
    gb = torch.autograd.grad(b, bufs)
    torch.testing.assert_close(a, b, rtol=1e-12, atol=0)
    for x, y in zip(ga, gb):
        torch.testing.assert_close(x, y, rtol=1e-10, atol=1e-14)
    # the closed form the kernel evaluates: sum_L 4^-L * 2/N_L * (A_L (n(J-1) + n(J+1)) + B_L (n(I-1) + n(I+1))) at the ancestor
    v = bufs[3].detach()
    grad = torch.zeros_like(v)
    n, L = v, 0
    while True:
        s = n.shape[0]
        A, B = (n * n.roll(1, 1)).mean(), (n * n.roll(1, 0)).mean()
        gl = 2 / (s * s) * (A * (n.roll(1, 1) + n.roll(-1, 1)) + B * (n.roll(1, 0) + n.roll(-1, 0)))
        grad += 4.0 ** -L * gl.repeat_interleave(2 ** L, 0).repeat_interleave(2 ** L, 1)
        if s <= 8:
            break
        n = F.avg_pool2d(n[None, None], 2)[0, 0]
        L += 1
    torch.testing.assert_close(grad, ga[3], rtol=1e-10, atol=1e-14)


def test_oracle_normalize_matches_definition():
    from oracle import projector as op
    b = torch.randn(16, 16, dtype=torch.float64) * 3 + 1
    ref = (b - b.mean()) / ((b - b.mean()).square().mean().sqrt())
    op.noise_normalize_([b])
    torch.testing.assert_close(b, ref, rtol=1e-12, atol=1e-12)


def test_oracle_seg_cross_entropy_matches_autograd():
    from oracle import projector as op
    g = torch.Generator().manual_seed(1)
    raw = torch.randn(2, 8, 8, 19, generator=g, dtype=torch.float64).permute(0, 3, 1, 2).requires_grad_(True)    # strided view
    mask = torch.randint(0, 19, (2, 32, 32), generator=g, dtype=torch.uint8)
    a = op.seg_cross_entropy(raw, mask)
    ga, = torch.autograd.grad(a, raw)
    up = F.interpolate(raw, size=(32, 32), mode='bilinear', align_corners=False)
    b = -(up.log_softmax(1).gather(1, mask.long()[:, None])).mean()
    gb, = torch.autograd.grad(b, raw)
    torch.testing.assert_close(a, b, rtol=1e-12, atol=0)
    torch.testing.assert_close(ga, gb, rtol=1e-10, atol=1e-14)


# the 19-class order of dnnlib/seg_tools.py:35-55 (class index -> name)
CLASS_NAMES = ['background', 'skin', 'nose', 'eye_g', 'l_eye', 'r_eye', 'l_brow', 'r_brow', 'l_ear', 'r_ear', 'mouth', 'u_lip',
               'l_lip', 'hair', 'hat', 'ear_r', 'neck_l', 'neck', 'cloth']


def test_mirror_mask_swaps_left_right_classes():
    from ide3d_b200 import projector
    m = torch.arange(19, dtype=torch.uint8).repeat(2, 1)                     # [2, 19]: column j holds class j
    out = projector.mirror_mask(m)
    expect = torch.tensor(projector.MIRROR_CLASSES, dtype=torch.uint8).flip(0).repeat(2, 1)
    assert torch.equal(out, expect)
    for a, b in ((4, 5), (6, 7), (8, 9)):
        assert projector.MIRROR_CLASSES[a] == b and projector.MIRROR_CLASSES[b] == a
        assert CLASS_NAMES[a].startswith('l_') and CLASS_NAMES[b] == 'r_' + CLASS_NAMES[a][2:]
    assert all(projector.MIRROR_CLASSES[k] == k for k in range(19) if k not in {4, 5, 6, 7, 8, 9})
    assert not any(CLASS_NAMES[k].startswith(('l_', 'r_')) for k in range(19) if k not in {4, 5, 6, 7, 8, 9, 12})   # l_lip: lower lip
    assert torch.equal(projector.mirror_mask(projector.mirror_mask(m)), m)


def test_mirror_label_indices():
    from ide3d_b200 import projector
    label = torch.arange(1, 26, dtype=torch.float32)[None]
    out = projector.mirror_label(label)
    flipped = {1, 2, 3, 4, 8}
    assert all(out[0, i] == (-label[0, i] if i in flipped else label[0, i]) for i in range(25))
    # a mirrored look-at camera: the rotation's x column and the camera position's x flip sign
    from oracle import projector as op
    lab, _ = op.golden_inputs()
    m, mm = lab[0, :16].reshape(4, 4), projector.mirror_label(lab)[0, :16].reshape(4, 4)
    flip = torch.diag(torch.tensor([-1., 1., 1., 1.]))
    torch.testing.assert_close(mm, flip @ m @ torch.diag(torch.tensor([-1., 1., 1., 1.])))


def test_zero_camera_delta_is_identity():
    from ide3d_b200 import projector
    from oracle import projector as op
    lab, _ = op.golden_inputs()
    lab = lab.clone()
    lab[0, 1] = -0.0                                                           # a negative zero survives too
    delta = torch.zeros(6, requires_grad=True)
    out = projector.refine_label(lab, delta)
    assert torch.equal(out.view(torch.int32), lab.view(torch.int32))
    out[0, :12].sum().backward()                                               # and the delta still gets a gradient
    assert delta.grad.abs().sum() > 0
    # a small rotation about +y (yaw) moves the camera on the sphere: the radius is kept
    d = torch.tensor([0.0, 0.05, 0.0, 0.0, 0.0, 0.0])
    m2 = projector.refine_label(lab, d)[0, :16].reshape(4, 4)
    assert math.isclose(m2[:3, 3].norm().item(), lab[0, :16].reshape(4, 4)[:3, 3].norm().item(), rel_tol=1e-6)
    R = projector.rodrigues(torch.tensor([0.3, -0.2, 0.1], dtype=torch.float64))
    torch.testing.assert_close(R @ R.T, torch.eye(3, dtype=torch.float64))
    torch.testing.assert_close(torch.linalg.det(R), torch.tensor(1.0, dtype=torch.float64))


def test_arguments_are_validated():
    from ide3d_b200 import projector
    from oracle import projector as op
    label, target = op.golden_inputs()
    G, f = op.StandInGenerator(), op.standin_features()
    run = lambda **kw: projector.project(G, kw.pop('label', label), kw.pop('target', target), features=f, num_steps=1, w_avg_samples=4, **kw)
    with pytest.raises(ValueError, match='target must be'):
        run(target=target[:, :16])
    with pytest.raises(ValueError, match='label must be'):
        run(label=label[:, :16])
    with pytest.raises(ValueError, match='uint8 class map'):
        run(target_seg=torch.zeros(16, 16, dtype=torch.uint8), seg_weight=1.0)
    with pytest.raises(ValueError, match='uint8 class map'):
        run(target_seg=torch.zeros(32, 32, dtype=torch.int64), seg_weight=1.0)
    with pytest.raises(ValueError, match='has class 19'):
        run(target_seg=torch.full((32, 32), 19, dtype=torch.uint8), seg_weight=1.0)
    with pytest.raises(ValueError, match='needs target_seg'):
        run(seg_weight=1.0)
    with pytest.raises(TypeError):
        projector.load_features(3, 'cpu')


def test_seg_and_camera_run_on_cpu():
    """The whole driver with every option on, through the oracle ops: the camera moves, the seg term enters the loss."""
    from ide3d_b200 import projector
    from oracle import projector as op
    label, target = op.golden_inputs()
    G = op.StandInGenerator()
    with torch.no_grad():
        _, seg_raw = G.synthesis(G.mapping(torch.zeros(1, 16), label), c=label, return_seg='raw')
        mask = op.F.interpolate(seg_raw, size=(32, 32), mode='bilinear', align_corners=False).argmax(1)[0].to(torch.uint8)
    losses = {}
    for w in (0.0, 1.0):
        rec = []
        torch.manual_seed(0)
        with op.cpu_projector_ops():
            ws, lab = projector.project(G, label, target, features=op.standin_features(), num_steps=4, w_avg_samples=8, mirror=True,
                                        refine_camera=True, target_seg=mask, seg_weight=w, on_step=lambda s, d, l: rec.append((d.item(), l.item())))
        losses[w] = rec
    assert not torch.equal(lab, label)
    assert all(l1 > l0 for (_, l0), (_, l1) in zip(losses[0.0][1:], losses[1.0][1:]))


# ------------------------------------------------------------------------------------------------ ABI
FAKE = 0x10000


def _fake_table(_lib, sides=(4, 8)):
    t = _lib.NoiseTable()
    t.count = len(sides)
    for i, s in enumerate(sides):
        t.sides[i], t.bufs[i], t.grads[i] = s, FAKE, FAKE
    t.scratch, t.scratch_floats = FAKE, 1 << 20
    return t


def _fake_xent(_lib):
    p = _lib.SegXentParams()
    p.seg, p.n, p.classes, p.in_h, p.in_w = FAKE, 1, 19, 8, 8
    p.seg_stride_n, p.seg_stride_c, p.seg_stride_h, p.seg_stride_w = 19 * 64, 1, 8 * 19, 19
    p.mask, p.out_h, p.out_w, p.lse, p.partials, p.loss, p.grad_loss, p.grad_seg = FAKE, 32, 32, FAKE, FAKE, FAKE, FAKE, FAKE
    return p


def _setattr(field, value):
    def apply(p):
        setattr(p, field, value)
    return apply


def test_noise_entry_points_validate(lib):
    from ide3d_b200 import _lib
    assert lib.ide3d_noise_reg(None, None, None, None) == _lib.INVALID and b'null table' in lib.ide3d_last_error()
    assert lib.ide3d_noise_normalize(None, None) == _lib.INVALID
    empty = _lib.NoiseTable()
    empty.scratch, empty.scratch_floats = FAKE, 128
    assert lib.ide3d_noise_reg(ctypes.byref(empty), ctypes.c_void_p(FAKE), None, None) == _lib.OK          # no buffers: no-op
    assert lib.ide3d_noise_normalize(ctypes.byref(empty), None) == _lib.OK


@pytest.mark.skipif(torch.cuda.is_available(), reason='passes fake device pointers: run only where no GPU can be reached')
@pytest.mark.parametrize('case, status, message', [
    ('negative count', 'INVALID', b'negative buffer count'),
    ('zero side', 'INVALID', b'has side 0'),
    ('null buffer', 'INVALID', b'null buffer 1'),
    ('null scratch', 'INVALID', b'null scratch'),
    ('small scratch', 'INVALID', b'need 192'),
    ('unaligned scratch', 'INVALID', b'not 8-byte aligned'),
    ('null gradient', 'INVALID', b'null gradient 0'),
    ('null loss, no gradient', 'INVALID', b'null loss'),
    ('side 12', 'UNSUPPORTED', b'not a power of two'),
    ('side 1024', 'UNSUPPORTED', b'not a power of two <= 512'),
    ('65 buffers', 'UNSUPPORTED', b'at most 64'),
])
def test_noise_reg_malformed_params(lib, case, status, message):
    from ide3d_b200 import _lib
    t = _fake_table(_lib, (4, 16))
    loss, scale = ctypes.c_void_p(FAKE), ctypes.c_void_p(FAKE)
    if case == 'negative count':
        t.count = -1
    elif case == 'zero side':
        t.sides[1] = 0
    elif case == 'null buffer':
        t.bufs[1] = None
    elif case == 'null scratch':
        t.scratch = None
    elif case == 'small scratch':
        t.scratch_floats = 100                  # 128 + the 16 x 16 buffer's 8 x 8 level
    elif case == 'unaligned scratch':
        t.scratch = FAKE + 4
    elif case == 'null gradient':
        t.grads[0] = None
    elif case == 'null loss, no gradient':
        loss, scale = None, None
    elif case == 'side 12':
        t.sides[1] = 12
    elif case == 'side 1024':
        t.sides[1] = 1024
    elif case == '65 buffers':
        t.count = 65
    assert lib.ide3d_noise_reg(ctypes.byref(t), loss, scale, None) == getattr(_lib, status)
    assert message in lib.ide3d_last_error()


@pytest.mark.skipif(torch.cuda.is_available(), reason='passes fake device pointers: run only where no GPU can be reached')
@pytest.mark.parametrize('case, message', [
    ('null params', b'null params'),
    ('zero frames', b'bad sizes'),
    ('negative width', b'bad sizes'),
    ('33 classes', b'at most 32'),
    ('null logits', b'null logits'),
    ('null mask', b'null logits, mask'),
    ('stride over 32 bits', b'do not fit 32 bits'),
    ('negative stride', b'do not fit 32 bits'),
    ('null partials', b'null partials'),
    ('null grad', b'null grad_loss or grad_seg'),
])
def test_seg_xent_malformed_params(lib, case, message):
    from ide3d_b200 import _lib
    p = _fake_xent(_lib)
    fwd = case != 'null grad'
    if case == 'zero frames':
        p.n = 0
    elif case == 'negative width':
        p.out_w = -2
    elif case == '33 classes':
        p.classes = 33
    elif case == 'null logits':
        p.seg = None
    elif case == 'null mask':
        p.mask = None
    elif case == 'stride over 32 bits':
        p.seg_stride_c = 1 << 28
    elif case == 'negative stride':
        p.seg_stride_w = -19
    elif case == 'null partials':
        p.partials = None
    elif case == 'null grad':
        p.grad_seg = None
    arg = None if case == 'null params' else ctypes.byref(p)
    rc = (lib.ide3d_seg_xent_fwd if fwd else lib.ide3d_seg_xent_bwd)(arg, None)
    assert rc == _lib.INVALID
    assert message in lib.ide3d_last_error()


def test_projection_ops_refuse_cpu_tensors():
    from ide3d_b200.torch_utils.ops import projection
    with pytest.raises(RuntimeError, match='CUDA'):
        projection.noise_regularizer([torch.randn(8, 8)])
    with pytest.raises(RuntimeError, match='CUDA'):
        projection.noise_normalize_([torch.randn(8, 8)])
    with pytest.raises(RuntimeError, match='CUDA'):
        projection.seg_cross_entropy(torch.randn(1, 19, 8, 8), torch.zeros(1, 16, 16, dtype=torch.uint8))
