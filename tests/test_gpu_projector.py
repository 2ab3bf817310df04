"""GPU: the projector kernels (csrc/projector.cu) and ide3d_b200.projector on the device.

  * ide3d_noise_reg / ide3d_noise_normalize against the reference's torch loop on the bench generator's noise_const buffers: values,
    gradients, bit-reproducibility, a fixed launch count, and the torch loop for tables the kernels do not take
  * seg_cross_entropy against F.cross_entropy(upsample_seg(...)) autograd on the strided ray-march view
  * SynthesisLayer with a frozen generator and noise_const.requires_grad: the buffers receive their gradient
  * the mirrored view as one views=2 synthesis call against two calls; camera refinement on the backward-kernel path
  * the camera delta's gradient against finite differences, the dist landscape's minimum at the true camera, recovery of a known pose
  * projection of a rendered target: dist and the seg cross-entropy decrease by a margin"""

import contextlib
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')


def rel(a, b):
    a, b = a.detach(), b.detach()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


@pytest.fixture
def fp32_convolutions():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


@pytest.fixture(scope='module')
def bench_buffers():
    from ide3d_b200.compat import random_init_generator
    G = random_init_generator(device=DEV, seed=0)
    torch.manual_seed(0)
    bufs = [b.detach().clone().normal_() for n, b in G.synthesis.named_buffers() if 'noise_const' in n]
    del G
    return bufs


def test_noise_reg_matches_torch_loop(bench_buffers):
    from ide3d_b200.torch_utils.ops import projection
    from oracle import projector as op
    assert len(bench_buffers) >= 10 and max(b.shape[0] for b in bench_buffers) == 512
    a = [b.clone().requires_grad_(True) for b in bench_buffers]
    r = [b.clone().requires_grad_(True) for b in bench_buffers]
    loss = projection.noise_regularizer(a)
    ref = op.noise_reg(r)
    assert rel(loss, ref) <= 1e-6, (loss.item(), ref.item())
    (loss * 1e5).backward()
    (ref * 1e5).backward()
    for x, y in zip(a, r):
        assert rel(x.grad, y.grad) <= 1e-5, (x.shape, rel(x.grad, y.grad))


def test_noise_kernels_bit_reproducible_and_fixed_launches(bench_buffers):
    from ide3d_b200 import _lib
    from ide3d_b200.torch_utils.ops import projection

    def run(bufs):
        live = [b.clone().requires_grad_(True) for b in bufs]
        n0 = _lib.launch_count()
        loss = projection.noise_regularizer(live)
        n1 = _lib.launch_count()
        loss.backward()
        n2 = _lib.launch_count()
        with torch.no_grad():
            normed = [b.detach().clone() for b in live]
        projection.noise_normalize_(normed)
        n3 = _lib.launch_count()
        return loss.detach(), [b.grad for b in live], normed, (n1 - n0, n2 - n1, n3 - n2)

    l1, g1, m1, c_all = run(bench_buffers)
    l2, g2, m2, _ = run(bench_buffers)
    assert torch.equal(l1, l2) and all(torch.equal(x, y) for x, y in zip(g1, g2)) and all(torch.equal(x, y) for x, y in zip(m1, m2))
    _, _, _, c_one = run(bench_buffers[:1])
    assert c_all == c_one == (2, 1, 1), (c_all, c_one)


def test_noise_normalize_matches_torch(bench_buffers):
    from ide3d_b200.torch_utils.ops import projection
    from oracle import projector as op
    a = [(b * 3 + 0.5).contiguous() for b in bench_buffers]
    r = [x.clone() for x in a]
    projection.noise_normalize_(a)
    op.noise_normalize_(r)
    for x, y in zip(a, r):
        assert (x - y).abs().max() <= 2e-6 * y.abs().max(), float((x - y).abs().max())


def test_unsupported_sizes_take_the_torch_loop():
    from ide3d_b200 import _lib
    from ide3d_b200.torch_utils.ops import projection
    from oracle import projector as op
    torch.manual_seed(1)
    bufs = [torch.randn(s, s, device=DEV, requires_grad=True) for s in (12, 16)]
    n0 = _lib.launch_count()
    loss = projection.noise_regularizer(bufs)
    assert _lib.launch_count() == n0
    ref = op.noise_reg([b.detach().clone() for b in bufs])
    assert torch.equal(loss.detach(), ref)
    loss.backward()
    assert all(b.grad is not None for b in bufs)


def _xent_case(frames, R, out, seed):
    """A strided [frames, 19, R, R] view of a ray-march-like [frames, R*R, 51] feature tensor, and a mask."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    feat = torch.randn(frames, R * R, 51, generator=g, device=DEV) * 3
    seg_raw = feat.permute(0, 2, 1).reshape(frames, 51, R, R)[:, 32:]
    mask = torch.randint(0, 19, (frames, out, out), generator=g, device=DEV, dtype=torch.uint8)
    return feat, seg_raw, mask


@pytest.mark.parametrize('R, out, frames', [(16, 64, 1), (16, 512, 2), (64, 64, 3), (64, 512, 2), (128, 64, 2), (128, 512, 1)])
def test_seg_cross_entropy_matches_autograd(R, out, frames):
    from ide3d_b200.torch_utils.ops import projection
    from ide3d_b200.training.triplane import upsample_seg
    feat, seg_raw, mask = _xent_case(frames, R, out, seed=R + out + frames)
    assert not seg_raw.is_contiguous()

    def grad_of(fn):
        f = feat.clone().requires_grad_(True)
        s = f.permute(0, 2, 1).reshape(frames, 51, R, R)[:, 32:]
        loss = fn(s)
        loss.backward()
        return loss.detach(), f.grad.reshape(frames, R, R, 51)[..., 32:].permute(0, 3, 1, 2)

    loss, grad = grad_of(lambda s: projection.seg_cross_entropy(s, mask))
    ref, rgrad = grad_of(lambda s: F.cross_entropy(upsample_seg(s, (out, out)), mask.long()))
    assert rel(loss, ref) <= 1e-6, (loss.item(), ref.item())
    assert rel(grad, rgrad) <= 1e-5, rel(grad, rgrad)
    _, grad2 = grad_of(lambda s: projection.seg_cross_entropy(s, mask))
    assert torch.equal(grad, grad2)


def _small_generator():
    from ide3d_b200.training.triplane import TriPlaneGenerator
    torch.manual_seed(0)
    return TriPlaneGenerator(z_dim=32, w_dim=32, img_resolution=64, plane_resolution=32, render_size=16, channel_base=512, channel_max=16,
                             sr_channels=(8, 8), mapping_kwargs=dict(num_layers=2)).to(DEV).eval()


LABEL = [1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 2.7, 0, 0, 0, 1, 4.2647, 0, 0.5, 0, 4.2647, 0.5, 0, 0, 1.]


def _frontal(yaw=0.0, pitch=0.0):
    from ide3d_b200.training.volumetric_rendering import create_cam2world_matrix, sample_camera_positions
    o, _, _ = sample_camera_positions(DEV, n=1, r=2.7, horizontal_mean=math.pi / 2 + yaw, vertical_mean=math.pi / 2 + pitch, mode=None)
    m = create_cam2world_matrix(-o, o, device=DEV)
    return torch.cat([m.reshape(1, 16), torch.tensor(LABEL[16:], device=DEV).reshape(1, 9)], 1)


def test_frozen_generator_noise_buffers_receive_gradient(fp32_convolutions):
    G = _small_generator().requires_grad_(False)
    with torch.no_grad():
        for n, p in G.named_parameters():
            if n.endswith('noise_strength'):
                p.fill_(0.5)
    ws = torch.randn(1, G.num_ws, G.w_dim, device=DEV) * 0.5
    c = _frontal()
    with torch.no_grad():
        img0 = G.synthesis(ws, c=c, noise_mode='const', perturb=None)
    layers = [m for m in G.synthesis.modules() if hasattr(m, 'noise_const')]
    # buffers that do not require grad keep the inference path (the cached noise product, as before); buffers that do leave it
    for m in layers:
        m.__dict__.pop('_const_cache', None)
    G.synthesis(ws, c=c, noise_mode='const', perturb=None)
    assert all('noise' in m.__dict__.get('_const_cache', {}) for m in layers)
    for m in layers:
        m.__dict__.pop('_const_cache', None)
    for m in layers:
        m.noise_const.requires_grad_(True)
    img = G.synthesis(ws, c=c, noise_mode='const', perturb=None)
    assert not any('noise' in m.__dict__.get('_const_cache', {}) for m in layers)
    assert (img - img0).abs().max() <= 1e-4 * img0.abs().max()
    img.double().square().mean().backward()                 # the loss reduced in float64: the finite difference below resolves it
    grads = [m.noise_const.grad for m in layers]
    assert all(g is not None and torch.isfinite(g).all() for g in grads) and max(float(g.abs().max()) for g in grads) > 0
    # against a central finite difference of the loss along the gradient's own direction (no cancellation between buffers)
    scale = max(float(gr.abs().max()) for gr in grads)
    dirs = [gr / scale for gr in grads]
    analytic = sum(float((gr.double() * d.double()).sum()) for gr, d in zip(grads, dirs))
    eps, fd = 1e-2, []
    with torch.no_grad():
        for sign in (1, -1):
            for m, d in zip(layers, dirs):
                m.noise_const.add_(sign * eps * d)
            fd.append(float(G.synthesis(ws, c=c, noise_mode='const', perturb=None).double().square().mean()))
            for m, d in zip(layers, dirs):
                m.noise_const.sub_(sign * eps * d)
    numeric = (fd[0] - fd[1]) / (2 * eps)
    assert abs(analytic - numeric) <= 1e-2 * abs(numeric), (analytic, numeric)


def test_mirror_views2_matches_two_calls(fp32_convolutions):
    from ide3d_b200 import projector
    G = _small_generator().requires_grad_(False)
    c = _frontal(0.2, 0.05)
    cm = projector.mirror_label(c)
    w0 = torch.randn(1, 1, G.w_dim, device=DEV) * 0.5

    def loss_and_grad(two_calls):
        w = w0.clone().requires_grad_(True)
        ws = w.repeat(1, G.num_ws, 1)
        if two_calls:
            a = G.synthesis(ws, c=c, noise_mode='const', force_fp32=True, perturb=None)
            b = G.synthesis(ws, c=cm, noise_mode='const', force_fp32=True, perturb=None)
            img = torch.cat([a, b])
        else:
            img = G.synthesis(ws, c=torch.cat([c, cm]), noise_mode='const', force_fp32=True, views=2, perturb=None)
        loss = (img[0] - 0.1).square().sum() + (img[1] + 0.1).square().sum()
        loss.backward()
        return loss.detach(), w.grad

    l1, g1 = loss_and_grad(False)
    l2, g2 = loss_and_grad(True)
    assert rel(l1, l2) <= 1e-5 and rel(g1, g2) <= 1e-4, (rel(l1, l2), rel(g1, g2))


@contextlib.contextmanager
def spy(module, name, calls):
    orig = getattr(module, name)
    setattr(module, name, lambda *a, **k: (calls.append(k), orig(*a, **k))[1])
    try:
        yield
    finally:
        setattr(module, name, orig)


def _target(G, ws, c):
    with torch.no_grad():
        img, seg_raw = G.synthesis(ws, c=c, noise_mode='const', force_fp32=True, return_seg='raw', perturb=None)
    target = (img[0] + 1) * 127.5          # not clamped: the random-init generator leaves [-1, 1], and a clamped target is not its render
    from ide3d_b200.training.triplane import upsample_seg
    mask = upsample_seg(seg_raw, (G.img_resolution,) * 2).argmax(1)[0].to(torch.uint8)
    return target, mask


def test_camera_refinement_takes_backward_kernel():
    from ide3d_b200 import projector, render, render_grad
    from oracle import projector as op
    G = _small_generator()
    G.rendering_kwargs['perturb'] = None
    c = _frontal()
    target, mask = _target(G, torch.zeros(1, G.num_ws, G.w_dim, device=DEV), c)
    kernel_calls, chain_calls = [], []
    with spy(render, 'raymarch_backward', kernel_calls), spy(render_grad, 'composed_chain', chain_calls):
        projector.project(G, c, target, features=op.standin_features().to(DEV), num_steps=2, w_avg_samples=16, mirror=True,
                          refine_camera=True, target_seg=mask, seg_weight=1.0)
    assert kernel_calls and all(k.get('want_camera') for k in kernel_calls) and not chain_calls


def _known_target():
    """The small generator (jitter off), a target rendered from a known (w*, c*) and the mask of its own argmax."""
    G = _small_generator()
    G.rendering_kwargs['perturb'] = None
    torch.manual_seed(3)
    z = torch.randn(1, G.z_dim, device=DEV)
    c_star = _frontal(0.15, 0.05)
    with torch.no_grad():
        w_star = G.mapping(z, c_star)
    target, mask = _target(G, w_star, c_star)
    return G, w_star, c_star, target, mask


def pixel_features(img, resize_images=False, return_lpips=True):
    """A feature callable with the projectors' contract that returns the pixels: a photometric dist."""
    return img.flatten(1) / 255


def _pose_error(a, b):
    return float((a[0, :12] - b[0, :12]).norm())


def test_camera_delta_gradient_matches_finite_differences(fp32_convolutions):
    """d dist / d (omega, t) through refine_label and the renderer's backward kernel, at a camera 4 / 2 degrees off, against central
    differences of the same dist; and the dist over yaw and pitch is smallest at c*."""
    from ide3d_b200 import projector
    G, w_star, c_star, target, _ = _known_target()
    G.requires_grad_(False)

    def dist(c):
        img = projector._prepare(G.synthesis(w_star, c=c, noise_mode='const', force_fp32=True))
        return (pixel_features(target[None]) - pixel_features(img)).square().sum()

    c0 = _frontal(0.15 + math.radians(4), 0.05 + math.radians(2))
    delta = torch.zeros(6, device=DEV, requires_grad=True)
    dist(projector.refine_label(c0, delta)).backward()
    fd = []
    with torch.no_grad():
        for k in range(6):
            e = torch.zeros(6, device=DEV)
            e[k] = 1e-3
            fd.append(float(dist(projector.refine_label(c0, e)) - dist(projector.refine_label(c0, -e))) / 2e-3)
    fd = torch.tensor(fd, device=DEV)
    assert (delta.grad - fd).abs().max() <= 1e-2 * fd.abs().max(), (delta.grad.tolist(), fd.tolist())
    with torch.no_grad():
        for axis in range(2):
            sweep = [float(dist(_frontal(0.15 + math.radians(d) * (axis == 0), 0.05 + math.radians(d) * (axis == 1)))) for d in range(-6, 7, 2)]
            assert min(range(len(sweep)), key=sweep.__getitem__) == 3 and sweep[3] <= 1e-6 * max(sweep), sweep


def test_camera_refinement_recovers_pose(fp32_convolutions):
    """Projection from w* with the camera 4 degrees off in yaw and 2 in pitch, no w noise, photometric dist: refine_camera brings the
    pose back (first H100 run: 0.237 -> 0.0195, while w is optimised too)."""
    from ide3d_b200 import projector
    G, w_star, c_star, target, _ = _known_target()
    c0 = _frontal(0.15 + math.radians(4), 0.05 + math.radians(2))
    torch.manual_seed(0)
    _, c_fit = projector.project(G, c0, target, features=pixel_features, num_steps=200, w_avg_samples=64, initial_w=w_star[:, :1],
                                 initial_noise_factor=0.0, refine_camera=True)
    before, after = _pose_error(c0, c_star), _pose_error(c_fit, c_star)
    print('pose error', before, '->', after)
    assert after <= 0.25 * before, (before, after)


def test_projection_lowers_dist_and_seg_xent(fp32_convolutions):
    """Projection from w_avg with the scripted stand-in VGG features towards a target rendered from (w*, c*): dist falls to under 0.4 of
    its first value (first H100 run: 0.173 -> 0.052) and, with seg_weight > 0 and the target's own argmax as the mask, the
    cross-entropy to under 0.85 (1.92 -> 1.43)."""
    from ide3d_b200 import projector
    from ide3d_b200.torch_utils.ops import projection
    from oracle import projector as op
    G, _, c_star, target, mask = _known_target()
    feats = op.standin_features().to(DEV)
    rec, seg_losses = [], []
    torch.manual_seed(0)
    projector.project(G, c_star, target, features=feats, num_steps=100, w_avg_samples=256, on_step=lambda s, d, l: rec.append(d.item()))
    orig = projection.seg_cross_entropy
    projection.seg_cross_entropy = lambda s, m: (lambda v: (seg_losses.append(v.item()), v)[1])(orig(s, m))
    try:
        torch.manual_seed(0)
        projector.project(G, c_star, target, features=feats, num_steps=100, w_avg_samples=256, target_seg=mask, seg_weight=1.0)
    finally:
        projection.seg_cross_entropy = orig
    print('dist', rec[0], '->', rec[-1], 'seg xent', seg_losses[0], '->', seg_losses[-1])
    assert rec[-1] <= 0.4 * rec[0], (rec[0], rec[-1])
    assert seg_losses[-1] <= 0.85 * seg_losses[0], (seg_losses[0], seg_losses[-1])
