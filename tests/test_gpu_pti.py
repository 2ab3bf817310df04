"""GPU: the LPIPS head kernels (csrc/lpips.cu) and ide3d_b200.pti on the device.

  * ide3d_lpips_fwd / _bwd against lpips_head_torch autograd (in float64) at the layer shapes of AlexNet on 512^2 images: one and two
    samples, NCHW and channels_last, broadcast and per-sample targets; bit-reproducibility; fixed launch counts; refused tables
  * a planted all-zero feature vector: the kernel's gradient is 0 where torch's is NaN, and through a ReLU both agree
  * tune(mirror=True): the first step's per-view losses and parameter gradients against two single-view synthesis calls
  * tuning lowers l2 + lpips towards a target rendered by a perturbed copy of the generator
  * no stale inference caches after tuning with foreach and fused Adam, and after torch.save / torch.load
  * free_view_frames against the batch-1 loop of run_pti.py:154-182"""

import contextlib
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')
ALEX_512 = [(64, 127, 127), (192, 63, 63), (384, 31, 31), (256, 31, 31), (256, 31, 31)]


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


@pytest.fixture
def fp32_convolutions():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _features(n, shapes, channels_last, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    out = []
    for c, h, w in shapes:
        t = torch.relu(torch.randn(n, c, h, w, device=DEV, generator=g)) * scale
        out.append(t.contiguous(memory_format=torch.channels_last) if channels_last else t)
    return out


def _lin(shapes, seed=7):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return [torch.rand(c, device=DEV, generator=g) / c * 8 for c, _, _ in shapes]


@pytest.mark.parametrize('n', [1, 2])
@pytest.mark.parametrize('channels_last', [False, True])
@pytest.mark.parametrize('broadcast', [False, True])
def test_head_matches_torch_autograd(n, channels_last, broadcast):
    from ide3d_b200.torch_utils.ops import lpips as LP
    fx = [t.requires_grad_(True) for t in _features(n, ALEX_512, channels_last, 1)]
    base = _features(n, ALEX_512, channels_last, 2)
    fy = [(x.detach()[:1] if broadcast else x.detach()) * 0.7 + b[:1 if broadcast else n] * 0.3 for x, b in zip(fx, base)]
    fy = [t.contiguous(memory_format=torch.channels_last) if channels_last else t.contiguous() for t in fy]
    fy = [t.requires_grad_(True) for t in fy]
    lin = _lin(ALEX_512)
    gv = torch.tensor([1.0, -0.5][:n], device=DEV)
    v = LP.lpips_head(fx, fy, lin)
    (v * gv).sum().backward()
    rx = [t.detach().double().requires_grad_(True) for t in fx]
    ry = [t.detach().double().requires_grad_(True) for t in fy]
    rv = LP.lpips_head_torch(rx, ry, [w.double() for w in lin])
    (rv * gv.double()).sum().backward()
    assert v.shape == (n,) and rel(v, rv) <= 1e-6, (v.tolist(), rv.tolist())
    for a, b in zip(fx + fy, rx + ry):
        assert a.grad.shape == b.grad.shape
        assert rel(a.grad, b.grad) <= 1e-5, (tuple(a.shape), rel(a.grad, b.grad))
    if channels_last:
        assert fx[0].grad.is_contiguous(memory_format=torch.channels_last)


def test_head_bit_reproducible_and_fixed_launches():
    from ide3d_b200 import _lib
    from ide3d_b200.torch_utils.ops import lpips as LP

    def run(shapes):
        fx = [t.requires_grad_(True) for t in _features(2, shapes, False, 3)]
        fy = _features(1, shapes, False, 4)
        lin = _lin(shapes)
        n0 = _lib.launch_count()
        v = LP.lpips_head(fx, fy, lin)
        n1 = _lib.launch_count()
        v.sum().backward()
        n2 = _lib.launch_count()
        return v.detach(), [t.grad for t in fx], (n1 - n0, n2 - n1)

    v1, g1, c5 = run(ALEX_512)
    v2, g2, _ = run(ALEX_512)
    assert torch.equal(v1, v2) and all(torch.equal(a, b) for a, b in zip(g1, g2))
    _, _, c1 = run(ALEX_512[:1])
    assert c5 == c1 == (2, 1), (c5, c1)


def test_refused_tables():
    """More than 8 layers: the library answers IDE3D_UNSUPPORTED and lpips_head computes the torch formula (no launch); null pointers
    are IDE3D_INVALID."""
    from ide3d_b200 import _lib
    from ide3d_b200.torch_utils.ops import lpips as LP
    shapes = [(8, 5, 5)] * 9
    fx, fy, lin = _features(1, shapes, False, 5), _features(1, shapes, False, 6), _lin(shapes)
    n0 = _lib.launch_count()
    v = LP.lpips_head(fx, fy, lin)
    assert _lib.launch_count() == n0
    assert torch.equal(v, LP.lpips_head_torch(fx, fy, lin))
    p = LP._params(fx[:1], fy[:1], lin[:1], 1)
    value = torch.empty(1, device=DEV)
    scratch = torch.empty(64, dtype=torch.float64, device=DEV)
    p.value, p.scratch, p.scratch_bytes = value.data_ptr(), scratch.data_ptr(), 512
    lib = _lib.get_lib()
    assert lib.ide3d_lpips_fwd(ctypes.byref(p), _lib.stream_ptr(DEV)) == _lib.OK
    p.num_layers = 9
    assert lib.ide3d_lpips_fwd(ctypes.byref(p), _lib.stream_ptr(DEV)) == _lib.UNSUPPORTED
    p.num_layers = 1
    p.layers[0].y = None
    assert lib.ide3d_lpips_fwd(ctypes.byref(p), _lib.stream_ptr(DEV)) == _lib.INVALID
    p.layers[0].y = fy[0].data_ptr()
    p.scratch = None
    assert lib.ide3d_lpips_fwd(ctypes.byref(p), _lib.stream_ptr(DEV)) == _lib.INVALID
    assert lib.ide3d_lpips_bwd(ctypes.byref(p), _lib.stream_ptr(DEV)) == _lib.INVALID      # grad_value null


def test_zero_feature_vector():
    """A pixel whose feature vector is exactly zero: torch's head gives NaN gradients there, the kernel 0; through a ReLU (the trunk's
    last op before every tap) both give the same, finite gradient."""
    from ide3d_b200.torch_utils.ops import lpips as LP
    shapes = [(16, 9, 9), (32, 5, 5)]
    pre = [t - 0.5 for t in _features(1, shapes, False, 8)]
    pre[0].data[:, :, 4, 4] = -1.0                       # relu -> an all-zero vector at pixel (4, 4) of layer 0
    fy = _features(1, shapes, False, 9)
    lin = _lin(shapes)
    x = [t.detach().clone().requires_grad_(True) for t in pre]
    feats = [torch.relu(t) for t in pre]
    assert feats[0][0, :, 4, 4].abs().max() == 0
    head_k = [f.detach().clone().requires_grad_(True) for f in feats]
    LP.lpips_head(head_k, fy, lin).sum().backward()
    head_t = [f.detach().clone().requires_grad_(True) for f in feats]
    LP.lpips_head_torch(head_t, fy, lin).sum().backward()
    assert torch.isnan(head_t[0].grad[0, :, 4, 4]).all() and torch.equal(head_k[0].grad[0, :, 4, 4], torch.zeros(16, device=DEV))
    assert torch.isfinite(head_k[0].grad).all()
    xk = [t.detach().clone().requires_grad_(True) for t in pre]
    LP.lpips_head([torch.relu(t) for t in xk], fy, lin).sum().backward()
    LP.lpips_head_torch([torch.relu(t) for t in x], fy, lin).sum().backward()
    for a, b in zip(xk, x):
        assert torch.isfinite(a.grad).all() and torch.isfinite(b.grad).all()
        assert rel(a.grad, b.grad) <= 1e-5


# ------------------------------------------------------------------------------------------------ the driver
@pytest.fixture(scope='module')
def bench_G():
    from ide3d_b200.compat import random_init_generator
    G = random_init_generator(device=DEV, seed=0)
    G.rendering_kwargs['perturb'] = None
    return G


@pytest.fixture(scope='module')
def alex():
    from oracle import pti as opti
    return opti.standin_lpips().to(DEV)


def _frontal(yaw=0.0, pitch=0.0):
    from ide3d_b200 import pti
    from ide3d_b200.training.volumetric_rendering import create_cam2world_matrix, sample_camera_positions
    p, _, _ = sample_camera_positions(DEV, n=1, r=2.7, horizontal_mean=torch.pi / 2 + yaw, vertical_mean=torch.pi / 2 + pitch, mode=None)
    c = create_cam2world_matrix(-p, p, device=DEV).reshape(1, -1)
    return torch.cat([c, torch.tensor(pti.INTRINSICS, device=DEV)[None]], 1)


def _pivot(G, seed=3):
    torch.manual_seed(seed)
    with torch.no_grad():
        return G.mapping(torch.randn(1, G.z_dim, device=DEV), _frontal(), truncation_psi=0.7)


def _perturbed_target(G, ws, c, scale=0.02):
    import copy
    T = copy.deepcopy(G)
    g = torch.Generator(device=DEV).manual_seed(11)
    with torch.no_grad():
        for name, p in T.named_parameters():
            if name.startswith(('synthesis.b', 'synthesis.renderer')):
                p.add_(torch.randn(p.shape, device=DEV, generator=g) * scale)
        return T.synthesis(ws, c=c, noise_mode='const', force_fp32=True)[0].clamp(-1, 1)


@contextlib.contextmanager
def capture_first_step_grads(store):
    step = torch.optim.Adam.step

    def wrapped(self, *a, **k):
        if not store:
            store.extend(None if p.grad is None else p.grad.detach().clone() for group in self.param_groups for p in group['params'])
        return step(self, *a, **k)
    torch.optim.Adam.step = wrapped
    try:
        yield
    finally:
        torch.optim.Adam.step = step


def test_mirror_first_step_matches_two_calls(bench_G, alex, fp32_convolutions):
    import copy
    from ide3d_b200 import pti, projector
    G = bench_G
    ws = _pivot(G)
    c = _frontal(0.2, 0.05)
    target = _perturbed_target(G, ws, c)
    rec, grads = [], []
    with capture_first_step_grads(grads):
        pti.tune(G, ws, c, target, lpips=alex, steps=1, mirror=True, lpips_threshold=-1.0,
                 on_step=lambda s, l2, lp, loss: rec.append((l2, lp, loss)))
    l2, lp, loss = rec[0]
    # two single-view calls, the reference's structure (single_id_coach.py:62-76)
    R = copy.deepcopy(G).requires_grad_(True)
    total, per = 0.0, []
    for cam, img_t in ((c, target[None]), (projector.mirror_label(c), torch.flip(target[None], (3,)))):
        img = R.synthesis(ws, c=cam, noise_mode='const', force_fp32=True)
        a, b = torch.nn.functional.mse_loss(img, img_t), alex(img, img_t)[0]
        per.append((a.detach(), b.detach()))
        total = total + (a + b)
    total.backward()
    ref_grads = [p.grad for p in R.parameters()]
    assert rel(loss, total) <= 1e-5
    for v in range(2):
        assert rel(l2[v], per[v][0]) <= 1e-5 and rel(lp[v], per[v][1]) <= 1e-5, (v, l2.tolist(), lp.tolist(), per)
    assert [g is None for g in grads] == [g is None for g in ref_grads]          # the mapping network gets none
    flat = torch.cat([g.flatten() for g in grads if g is not None])
    ref_flat = torch.cat([g.flatten() for g in ref_grads if g is not None])
    print('mirror: loss rel', rel(loss, total), 'grad rel', rel(flat, ref_flat))
    assert rel(flat, ref_flat) <= 1e-4


def test_tuning_lowers_the_loss(bench_G, alex):
    """The target is rendered by a copy of G whose super-resolution and decoder weights are perturbed (0.02 N(0, 1)); 40 steps at
    lr 1e-3 bring l2 + lpips under a quarter of its first value (first H100 run: 2.81 -> 0.051)."""
    from ide3d_b200 import pti
    G = bench_G
    ws = _pivot(G)
    c = _frontal(0.1)
    target = _perturbed_target(G, ws, c)
    rec = []
    pti.tune(G, ws, c, target, lpips=alex, steps=40, lr=1e-3, lpips_threshold=-1.0, on_step=lambda s, l2, lp, loss: rec.append(loss.item()))
    print('tune loss', rec[0], '->', rec[-1])
    assert len(rec) == 40 and rec[-1] <= 0.25 * rec[0], (rec[0], rec[-1])


@pytest.mark.parametrize('adam', [dict(foreach=True), dict(fused=True)])
def test_no_stale_caches_after_tuning(bench_G, alex, adam, tmp_path):
    from ide3d_b200 import pti
    from ide3d_b200.compat import random_init_generator
    from ide3d_b200.training import triplane
    G = bench_G
    ws = _pivot(G)
    c = _frontal(0.1)
    target = _perturbed_target(G, ws, c)
    with torch.no_grad():
        G.synthesis(ws, c=c, noise_mode='const')          # the caller's generator has warm caches
    T = pti.tune(G, ws, c, target, lpips=alex, steps=3, lr=1e-3, lpips_threshold=-1.0, adam_kwargs=adam)
    fresh = random_init_generator(device=DEV, seed=1)
    fresh.rendering_kwargs['perturb'] = None
    fresh.load_state_dict(T.state_dict())

    def render(g):
        with torch.no_grad():
            return g.synthesis(ws, c=c, noise_mode='const')

    a = render(T)
    assert torch.equal(a, render(fresh))
    assert not torch.equal(a, render(G))
    torch.save(T, tmp_path / 'tuned.pt')
    assert torch.equal(torch.load(tmp_path / 'tuned.pt', weights_only=False).synthesis(ws, c=c, noise_mode='const'), a)
    # a fused Adam step after the caches are warm, then the explicit invalidation
    p = [q for q in T.parameters()]
    for q in p:
        q.requires_grad_(True)
        q.grad = torch.full_like(q, 1e-3)
    opt = torch.optim.Adam(p, lr=1e-3, fused=True)
    opt.step()
    T.requires_grad_(False)
    triplane.invalidate_caches(T)
    fresh.load_state_dict(T.state_dict())
    assert torch.equal(render(T), render(fresh))


def test_free_view_frames_match_batch1_loop(bench_G):
    from ide3d_b200 import pti
    import copy
    G = copy.deepcopy(bench_G)
    G.rendering_kwargs['perturb'] = 'hash'
    ws = _pivot(G)
    torch.manual_seed(5)
    frames = pti.free_view_frames(G, ws, num_frames=6, chunk=4)
    assert frames.shape == (6, G.img_resolution, G.img_resolution, 3) and frames.dtype.name == 'uint8'
    cams = pti.free_view_cameras(6, DEV)
    torch.manual_seed(5)
    worst = 0
    with torch.no_grad():
        for f in range(6):
            img = G.synthesis(ws, c=cams[f:f + 1], render_params={'h_stddev': 0., 'v_stddev': 0., 'fov': 18, 'num_steps': 96},
                              noise_mode='const')
            ref = (img * 127.5 + 128).clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1)[0].cpu()
            worst = max(worst, int((torch.from_numpy(frames[f]).int() - ref.int()).abs().max()))
    print('free view: worst uint8 difference', worst)
    assert worst <= 1
