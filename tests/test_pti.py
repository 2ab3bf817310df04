"""CPU: ide3d_b200.pti against the reference's pivotal-tuning coach (tests/golden/pti_trace.npz, recorded by make_pti_golden.py with
the stand-ins of oracle/projector.py and oracle/pti.py), lpips_head_torch against the reference's vendored LPIPS head, argument
validation, the free-view cameras, and the ABI of the LPIPS kernels."""

import ctypes

import numpy as np
import pytest
import torch

from conftest import load_golden

RUNS = {'w': 'w', 'w_plus': 'w_plus', 'join_view': 'join_view', 'early_stop': 'w'}


@pytest.fixture(scope='module')
def trace():
    return load_golden('pti_trace')


def _replay(g, key, G=None):
    from ide3d_b200 import pti
    from oracle import projector as op
    from oracle import pti as opti
    label, target = torch.from_numpy(g['label']), torch.from_numpy(g['target'])
    G = G or op.StandInGenerator(seed=int(g['generator_seed']))
    rec = []
    torch.manual_seed(int(g['torch_seed']))
    with opti.cpu_pti_ops():
        G_tuned, ws, lab = pti.run(G, label, target, features=op.standin_features(), lpips=opti.standin_lpips(), projector=RUNS[key],
                                   first_inv_steps=int(g['first_inv_steps']), w_avg_samples=int(g['w_avg_samples']),
                                   steps=int(g['max_pti_steps']), lpips_threshold=float(g[f'{key}_threshold']),
                                   on_step=lambda s, l2, lp, loss: rec.append((l2.numpy(), lp.numpy(), loss.item())))
    l2 = np.stack([r[0] for r in rec]).astype(np.float64)
    lp = np.stack([r[1] for r in rec]).astype(np.float64)
    loss = np.array([r[2] for r in rec], np.float64)
    return G_tuned, ws, lab, l2, lp, loss


@pytest.mark.parametrize('key', sorted(RUNS))
def test_replays_reference_coach(trace, key):
    """Projection, then the tuning loop.  W and W+ (and the early stop): pivot, label and the first step's l2 / lpips / loss bit-exact;
    the later steps and the tuned weights within 1e-6, because the vendored trunk normalises each tapped activation as soon as it
    exists while the head here takes all five at once, so autograd adds the three gradient contributions of a tap in another order
    (a few ulp per step).  The join view renders both cameras from one backbone pass (the backward then sums the views before the
    backbone): held to 1e-5."""
    g = trace
    G_tuned, ws, lab, l2, lp, loss = _replay(g, key)
    pivot = torch.from_numpy(g[f'{key}_pivot'])[:, :ws.shape[1]]
    assert torch.equal(lab, torch.from_numpy(g[f'{key}_label'])) and torch.equal(lab, torch.from_numpy(g['label']))
    ref_l2, ref_lp, ref_loss = g[f'{key}_l2'], g[f'{key}_lpips'], g[f'{key}_loss'].sum(1)
    assert l2.shape == ref_l2.shape and len(loss) == len(ref_loss)
    state = {k[len(f'{key}_state.'):]: torch.from_numpy(g[k]) for k in g if k.startswith(f'{key}_state.')}
    ours = G_tuned.state_dict()
    assert sorted(ours) == sorted(state)
    updates = int((lp.sum(1) > float(g[f'{key}_threshold'])).sum())
    assert updates == int(g[f'{key}_updates'])
    if key == 'early_stop':
        assert updates < int(g['max_pti_steps']) and len(loss) == updates + 1
    if key == 'join_view':
        torch.testing.assert_close(ws, pivot, rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(l2, ref_l2, rtol=1e-5)
        np.testing.assert_allclose(lp, ref_lp, rtol=1e-5)
        np.testing.assert_allclose(loss, ref_loss, rtol=1e-5)
        for k, v in state.items():
            torch.testing.assert_close(ours[k], v, rtol=1e-5, atol=1e-6, msg=k)
    else:
        assert torch.equal(ws, pivot)
        assert (l2[0], lp[0], loss[0]) == (ref_l2[0], ref_lp[0], ref_loss[0])
        np.testing.assert_allclose(l2, ref_l2, rtol=1e-6)
        np.testing.assert_allclose(lp, ref_lp, rtol=1e-6)
        np.testing.assert_allclose(loss, ref_loss, rtol=1e-6)
        for k, v in state.items():
            torch.testing.assert_close(ours[k], v, rtol=1e-6, atol=1e-7, msg=k)


def test_caller_generator_untouched(trace):
    from oracle import projector as op
    G = op.StandInGenerator(seed=int(trace['generator_seed']))
    before = {k: v.clone() for k, v in G.state_dict().items()}
    G_tuned, *_ = _replay(trace, 'w', G=G)
    assert all(torch.equal(before[k], v) for k, v in G.state_dict().items())
    assert all(p.grad is None for p in G.parameters())
    assert not any(torch.equal(before[k], v) for k, v in G_tuned.state_dict().items() if k.endswith('affine'))
    assert not G_tuned.training and not any(p.requires_grad for p in G_tuned.parameters())


def test_lpips_head_torch_matches_vendored_head():
    """lpips_head_torch against the vendored head's own ops (normalize_activation, (fx - fy) ** 2, the 1x1 lin conv, spatial mean,
    torch.sum(cat) / N) on the stand-in trunk's features of the golden target and a perturbed copy, restated here from
    inversion/criteria/lpips/{lpips,utils}.py."""
    from ide3d_b200.torch_utils.ops import lpips as LP
    from oracle import pti as opti
    net = opti.standin_lpips()
    _, target = opti.golden_inputs()
    x = (target + 0.2 * torch.sin(torch.arange(target.numel()).reshape(target.shape).float())).clamp(-1, 1)
    fx, fy = net.trunk(x), net.trunk(target)

    def normalize_activation(t, eps=1e-10):
        return t / (torch.sqrt(torch.sum(t ** 2, dim=1, keepdim=True)) + eps)

    lin = [torch.nn.Conv2d(w.numel(), 1, 1, 1, 0, bias=False) for w in net.lin]
    for conv, w in zip(lin, net.lin):
        conv.weight.data = w.reshape(1, -1, 1, 1).clone()
    diff = [(normalize_activation(a) - normalize_activation(b)) ** 2 for a, b in zip(fx, fy)]
    res = [conv(d).mean((2, 3), True) for d, conv in zip(diff, lin)]
    ref = torch.sum(torch.cat(res, 0)) / x.shape[0]
    ours = LP.lpips_head_torch(fx, fy, net.lin)
    assert ours.shape == (1,) and torch.equal(ours[0], ref)
    assert [tuple(f.shape[1:]) for f in fx] == [(64, 7, 7), (192, 3, 3), (384, 1, 1), (256, 1, 1), (256, 1, 1)]
    # two samples against one broadcast target (the second sample is the target itself)
    v = LP.lpips_head_torch([torch.cat([a, b]) for a, b in zip(fx, fy)], net.target(target), net.lin)
    torch.testing.assert_close(v[0], ref.detach(), rtol=1e-6, atol=0)
    assert float(v[1]) == 0.0


def test_lpips_head_is_cuda_only_and_validates():
    from ide3d_b200.torch_utils.ops import lpips as LP
    x = [torch.randn(1, 4, 3, 3)]
    with pytest.raises(RuntimeError):
        LP.lpips_head(x, x, [torch.ones(4)])
    with pytest.raises(ValueError):
        LP.lpips_head(x, [torch.randn(1, 5, 3, 3)], [torch.ones(4)])
    with pytest.raises(ValueError):
        LP.lpips_head(x, x, [torch.ones(3)])
    with pytest.raises(ValueError):
        LP.lpips_head(x, x + x, [torch.ones(4)])


def test_lpips_weights_from_files(tmp_path):
    import torchvision
    from ide3d_b200.torch_utils.ops.lpips import LPIPS
    from oracle import pti as opti
    trunk = tmp_path / 'alexnet.pth'
    lin = tmp_path / 'alex.pth'
    torch.save(opti.standin_alexnet().state_dict(), trunk)
    torch.save(opti.lin_state_dict(), lin)
    net = LPIPS.alexnet(str(trunk), str(lin))
    ref = opti.standin_lpips()
    assert all(torch.equal(a, b) for a, b in zip(net.state_dict().values(), ref.state_dict().values()))
    with pytest.raises(FileNotFoundError, match='absent.pth'):
        LPIPS.alexnet(str(tmp_path / 'absent.pth'), str(lin))
    with pytest.raises(FileNotFoundError, match='absent_lin.pth'):
        LPIPS.alexnet(str(trunk), str(tmp_path / 'absent_lin.pth'))
    with pytest.raises(ValueError):
        LPIPS(torchvision.models.alexnet(weights=None).features, [torch.ones(3)] * 5)


def test_argument_validation(trace):
    from ide3d_b200 import pti
    from oracle import projector as op
    from oracle import pti as opti
    G = op.StandInGenerator()
    label, target = opti.golden_inputs()
    ws = torch.zeros(1, G.num_ws, G.w_dim)
    lp = opti.standin_lpips()
    with pytest.raises(ValueError, match='target'):
        pti.tune(G, ws, label, target[:, :, :16], lpips=lp, steps=1)
    with pytest.raises(ValueError, match='label'):
        pti.tune(G, ws, label[:, :16], target, lpips=lp, steps=1)
    with pytest.raises(ValueError, match='ws'):
        pti.tune(G, ws[0], label, target, lpips=lp, steps=1)
    with pytest.raises(ValueError, match='lambda'):
        pti.tune(G, ws, label, target, lpips=lp, steps=1, l2_lambda=-1)
    with pytest.raises(ValueError, match='projector'):
        pti.run(G, label, target, features=op.standin_features(), lpips=lp, projector='e4e')
    with pytest.raises(TypeError, match='mirror'):
        pti.run(G, label, target, features=op.standin_features(), lpips=lp, mirror=True)
    with pytest.raises(FileNotFoundError):
        pti.run(G, label, target, features='/nonexistent/vgg16.pt', lpips=lp, first_inv_steps=1, w_avg_samples=4)
    with pytest.raises(ValueError, match='ws'):
        pti.free_view_frames(G, ws[0])


def test_free_view_cameras_follow_run_pti():
    """The camera of frame f: yaw pi (0.5 + 0.1 cos(2 pi f / 120)), pitch pi (0.5 - 0.05 sin(2 pi f / 120)), radius 2.7, looking at
    the origin (run_pti.py:155-171); one period every 120 frames."""
    from ide3d_b200 import pti
    c = pti.free_view_cameras(240)
    assert c.shape == (240, 25)
    m = c[:, :16].reshape(-1, 4, 4)
    origin = m[:, :3, 3]
    torch.testing.assert_close(origin.norm(dim=1), torch.full((240,), 2.7), rtol=1e-6, atol=1e-6)
    torch.testing.assert_close(c[:120], c[120:], rtol=0, atol=1e-6)
    for f in (0, 30, 77):
        h = np.pi * (0.5 + 0.1 * np.cos(2 * np.pi * f / 120))
        v = np.pi * (0.5 - 0.05 * np.sin(2 * np.pi * f / 120))
        want = 2.7 * np.array([np.sin(v) * np.cos(h), np.cos(v), np.sin(v) * np.sin(h)])
        np.testing.assert_allclose(origin[f].numpy(), want, rtol=0, atol=1e-5)
        np.testing.assert_allclose((-m[f, :3, 2]).numpy(), -want / 2.7, rtol=0, atol=1e-5)     # the camera looks at the origin
    assert torch.equal(c[:, 16:], torch.tensor(pti.INTRINSICS).expand(240, 9))


def test_invalidate_caches_drops_every_cache():
    from ide3d_b200.training import triplane
    from ide3d_b200.compat import random_init_generator
    G = random_init_generator(device='cpu', seed=0, z_dim=32, w_dim=32, img_resolution=64, plane_resolution=32, render_size=16,
                              channel_base=512, channel_max=16, sr_channels=(8, 8), mapping_kwargs=dict(num_layers=2))
    layers = [m for m in G.modules() if isinstance(m, triplane.networks.SynthesisLayer)]
    for m in layers:
        m.__dict__['_const_cache'] = {'noise': ((0,), torch.zeros(1))}
    G.synthesis.renderer._packed, G.synthesis.renderer._packed_key = object(), (1,)
    triplane._STYLE_PLANS[G.synthesis] = object()
    triplane.invalidate_caches(G)
    assert all('_const_cache' not in m.__dict__ for m in layers)
    assert G.synthesis.renderer._packed is None and G.synthesis.renderer._packed_key is None
    assert G.synthesis not in triplane._STYLE_PLANS


def test_lpips_entry_points_validate_before_the_device(lib):
    """Malformed tables return a status without touching the device (the pointers below are never dereferenced)."""
    from ide3d_b200 import _lib
    assert lib.ide3d_lpips_fwd(None, None) == _lib.INVALID and b'null params' in lib.ide3d_last_error()
    assert lib.ide3d_lpips_bwd(None, None) == _lib.INVALID
    assert lib.ide3d_lpips_scratch_bytes(None) == _lib.INVALID
    fake = 0x10000
    p = _lib.LpipsParams()
    p.n, p.num_layers = 2, 1
    layer = p.layers[0]
    layer.c, layer.h, layer.w = 4, 3, 5
    layer.x, layer.y, layer.lin = fake, fake, fake
    layer.x_stride = (ctypes.c_int64 * 4)(60, 15, 5, 1)
    layer.y_stride = (ctypes.c_int64 * 4)(0, 15, 5, 1)
    assert lib.ide3d_lpips_scratch_bytes(ctypes.byref(p)) == 8 * (2 * 1 + 2 * 1)     # one CTA per sample, one value per (sample, layer)
    assert lib.ide3d_lpips_fwd(ctypes.byref(p), None) == _lib.INVALID and b'null value or scratch' in lib.ide3d_last_error()
    assert lib.ide3d_lpips_bwd(ctypes.byref(p), None) == _lib.INVALID and b'null grad_value' in lib.ide3d_last_error()
    layer.grad_y, p.grad_value = fake, fake
    layer.gy_stride = (ctypes.c_int64 * 4)(0, 15, 5, 1)
    assert lib.ide3d_lpips_bwd(ctypes.byref(p), None) == _lib.INVALID and b'per sample' in lib.ide3d_last_error()
    layer.grad_y = None
    p.num_layers = 9
    assert lib.ide3d_lpips_fwd(ctypes.byref(p), None) == _lib.UNSUPPORTED and b'at most 8' in lib.ide3d_last_error()
    p.num_layers = 1
    layer.lin = None
    assert lib.ide3d_lpips_fwd(ctypes.byref(p), None) == _lib.INVALID and b'null x, y or lin' in lib.ide3d_last_error()
    layer.lin = fake
    layer.h = 0
    assert lib.ide3d_lpips_fwd(ctypes.byref(p), None) == _lib.INVALID and b'bad sizes' in lib.ide3d_last_error()
    layer.h = 3
    layer.x_stride = (ctypes.c_int64 * 4)(1 << 31, 15, 5, 1)
    assert lib.ide3d_lpips_fwd(ctypes.byref(p), None) == _lib.INVALID and b'31 bits' in lib.ide3d_last_error()
