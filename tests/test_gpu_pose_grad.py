"""GPU: camera gradients from the backward kernel (ide3d_raymarch_bwd_cam) and differentiable hierarchical renders, against autograd
through the oracle's stage functions, and against the composed-chain backward (render_grad.USE_BACKWARD_KERNEL = False)."""

import contextlib
import math

import numpy as np
import pytest
import torch

from oracle import camera as ocam
from oracle import renderer as orr
from test_gpu_renderer import _random_case, three_head_from_dense
from test_pose_grad import RES, R, S, check_head_grads, oracle_explicit_grads

DEV = 'cuda'
tol = lambda ref: 5e-4 * max(1.0, ref.abs().max().item())


def oracle_grads(tex, seg, dec, cam, u, gf, gd, box_scale=2.0, **opts):
    t, s, c = tex.clone().requires_grad_(True), seg.clone().requires_grad_(True), cam.clone().requires_grad_(True)
    params = [p.clone().requires_grad_(True) for p in (dec.w1, dec.b1, dec.w2, dec.b2)]
    rgb, depth, _ = orr.render_frames(t, s, orr.Decoder(*params), c, num_steps=S, resolution=RES, jitter_u=u, box_scale=box_scale, **opts)
    (rgb * gf).sum().add((depth * gd).sum()).backward()
    return t.grad, s.grad, c.grad, [p.grad for p in params]


def live_heads(dec, grad=True):
    return [tuple(h[:2]) + tuple(t.to(DEV).requires_grad_(grad) for t in h[2:]) for h in three_head_from_dense(dec.w1, dec.b1, dec.w2, dec.b2)]


@contextlib.contextmanager
def spy(module, name, calls):
    orig = getattr(module, name)
    setattr(module, name, lambda *a, **k: (calls.append(k), orig(*a, **k))[1])
    try:
        yield
    finally:
        setattr(module, name, orig)


@contextlib.contextmanager
def composed_chain_backward():
    from ide3d_b200 import render_grad
    render_grad.USE_BACKWARD_KERNEL = False
    try:
        yield
    finally:
        render_grad.USE_BACKWARD_KERNEL = True


def jitter_case(jitter, g):
    """(jitter_u for the product, uniforms for the oracle, hash seed) of one jitter mode."""
    if jitter == 'tensor':
        u = torch.rand(2, R, S, 1, generator=g)
        return u, u, None
    if jitter == 'hash':
        seed = 0x1234_5678_9ABC_DEF1
        return None, torch.from_numpy(orr.hash_uniform(torch.arange(2 * R * S).numpy(), seed)).reshape(2, R, S, 1), seed
    return None, None, None


def render_backward(tex, seg, heads, cam, gf, gd, planes=True, **kw):
    from ide3d_b200 import render
    t, s = [x.to(DEV).requires_grad_(planes) for x in (tex, seg)]
    c = cam.to(DEV).requires_grad_(True)
    feat, d, _ = render.raymarch(t, s, heads, c, resolution=RES, num_steps=S, **kw)
    (feat * gf.to(DEV)).sum().add((d * gd.to(DEV)).sum()).backward()
    return t.grad, s.grad, c.grad


@pytest.mark.gpu
@pytest.mark.parametrize('opts', [dict(), dict(white_back=True, max_depth=3.3, last_back=True), dict(clamp_mode='relu'), dict(fill_mode='weight')])
@pytest.mark.parametrize('jitter', ['tensor', 'hash', 'none'])
def test_camera_gradient_kernel_matches_oracle_autograd(opts, jitter):
    """A camera that requires grad takes the backward kernel (no composed-chain fallback) and its gradient, with the planes' and the
    heads', matches autograd through the oracle and the composed-chain backward."""
    from ide3d_b200 import render, render_grad
    tex, seg, dec, cam = _random_case(2, 16, seed=4)
    g = torch.Generator().manual_seed(1)
    u, u_ref, seed = jitter_case(jitter, g)
    gf, gd = torch.randn(2, R, 51, generator=g), torch.randn(2, R, 1, generator=g)
    gt, gs, gc, gp = oracle_grads(tex, seg, dec, cam, u_ref, gf, gd, **opts)
    kw = dict(jitter_u=None if u is None else u.to(DEV), jitter_seed=seed, **opts)

    heads = live_heads(dec)
    kernel_calls, chain_calls = [], []
    with spy(render, 'raymarch_backward', kernel_calls), spy(render_grad, 'composed_chain', chain_calls):
        t_grad, s_grad, c_grad = render_backward(tex, seg, heads, cam, gf, gd, **kw)
    assert kernel_calls and kernel_calls[0]['want_camera'] and not chain_calls, 'the backward kernel path was not taken'
    assert (c_grad.cpu() - gc).abs().max() <= tol(gc), 'cam'
    assert float(c_grad[:, 3].abs().max()) == 0.0 and float(c_grad[:, :3].abs().max()) > 0
    assert (t_grad.cpu() - gt).abs().max() <= tol(gt), 'tex'
    assert (s_grad.cpu() - gs).abs().max() <= tol(gs), 'seg'
    check_head_grads(heads, gp, tol)

    with composed_chain_backward():
        _, _, c2 = render_backward(tex, seg, live_heads(dec), cam, gf, gd, **kw)
    assert (c_grad - c2).abs().max() <= tol(gc)


@pytest.mark.gpu
@pytest.mark.parametrize('box_scale', [3.0, 4.5])
def test_camera_gradient_with_samples_leaving_the_planes(box_scale):
    """A box scale that pushes part of every ray outside [-1, 1]: taps outside the plane count as zero, including samples whose
    footprint is partly or wholly off the plane."""
    tex, seg, dec, cam = _random_case(2, 16, seed=8)
    st = orr.render_frames(tex, seg, dec, cam, num_steps=S, resolution=RES, box_scale=box_scale, return_stages=True)
    coords = (st['points_world'] * box_scale).abs().amax(-1)
    edge = 1 + 1.0 / 16                                                       # beyond this, all four taps of a plane are off it
    assert bool((coords < 1).any()) and bool(((coords > 1) & (coords < edge)).any()) and bool((coords > edge).any())
    g = torch.Generator().manual_seed(2)
    gf, gd = torch.randn(2, R, 51, generator=g), torch.randn(2, R, 1, generator=g)
    gt, _, gc, _ = oracle_grads(tex, seg, dec, cam, None, gf, gd, box_scale=box_scale)
    t_grad, _, c_grad = render_backward(tex, seg, live_heads(dec), cam, gf, gd, box_scale=box_scale)
    assert (c_grad.cpu() - gc).abs().max() <= tol(gc), 'cam'
    assert (t_grad.cpu() - gt).abs().max() <= tol(gt), 'tex'


@pytest.mark.gpu
def test_camera_only_request_equals_camera_part_of_full_request():
    """Pose refinement with frozen planes and decoder: the taps are read but nothing is scattered, and the camera gradient is that of
    the full request (up to the order of the atomic sums)."""
    from ide3d_b200 import render
    tex, seg, dec, cam = _random_case(2, 16, seed=9)
    g = torch.Generator().manual_seed(3)
    gf, gd = torch.randn(2, R, 51, generator=g), torch.randn(2, R, 1, generator=g)
    _, _, full = render_backward(tex, seg, live_heads(dec), cam, gf, gd, jitter_seed=11)
    calls = []
    with spy(render, 'raymarch_backward', calls):
        t_grad, s_grad, only = render_backward(tex, seg, live_heads(dec, grad=False), cam, gf, gd, planes=False, jitter_seed=11)
    assert t_grad is None and s_grad is None
    assert calls and calls[0]['want_planes'] == (False, False) and not calls[0]['want_params'] and calls[0]['want_camera']
    assert (only - full).abs().max() <= 1e-5 * max(1.0, float(full.abs().max()))


@pytest.mark.gpu
def test_camera_gradient_views_with_per_frame_seeds_equals_materialised_planes():
    """views=3: one plane set, three cameras, per-frame jitter seeds.  Each frame's camera gradient equals the run on planes repeated
    per frame, and the plane gradient is the sum over the views."""
    tex, seg, dec, _ = _random_case(1, 16, seed=12)
    yaw = math.pi / 2 + np.array([[-0.4], [0.0], [0.4]], np.float32)
    cam = torch.from_numpy(ocam.look_at_pose(yaw, np.full((3, 1), math.pi / 2 - 0.1, np.float32), [0, 0, 0.2], radius=2.7, batch_size=3))
    g = torch.Generator().manual_seed(4)
    gf, gd = torch.randn(3, R, 51, generator=g), torch.randn(3, R, 1, generator=g)
    seeds = [5, 2 ** 40 + 3, 77]
    t_v, _, c_v = render_backward(tex, seg, live_heads(dec), cam, gf, gd, jitter_seed=seeds, views=3)
    t_m, _, c_m = render_backward(tex.repeat(3, 1, 1, 1), seg.repeat(3, 1, 1, 1), live_heads(dec), cam, gf, gd, jitter_seed=seeds)
    close = lambda a, b: float((a - b).abs().max()) <= 1e-5 * max(1.0, float(b.abs().max()))
    assert close(c_v, c_m) and close(t_v, t_m.sum(0, keepdim=True))


def hier_case(seed, S_, NI):
    tex, seg, dec, cam = _random_case(2, 16, seed=seed)
    g = torch.Generator().manual_seed(seed)
    u = torch.rand(2, R, S_, generator=g)
    ui = torch.rand(2 * R, NI, generator=g)
    gf, gd = torch.randn(2, R, 51, generator=g), torch.randn(2, R, 1, generator=g)
    return tex, seg, dec, cam, u, ui, gf, gd


def hier_backward(tex, seg, heads, cam, u, ui, gf, gd, S_, NI):
    from ide3d_b200 import render
    t, s, c = [x.to(DEV).requires_grad_(True) for x in (tex, seg, cam)]
    feat, d, _, z = render.raymarch_hierarchical(t, s, heads, c, resolution=RES, num_steps=S_, n_importance=NI, jitter_u=u.to(DEV),
                                                 importance_u=ui.to(DEV), return_depths=True)
    (feat * gf.to(DEV)).sum().add((d * gd.to(DEV)).sum()).backward()
    return feat.detach(), d.detach(), z, t.grad, s.grad, c.grad


@pytest.mark.gpu
def test_hierarchical_render_is_differentiable_and_matches_oracle():
    """Under grad the forward is bit-identical to the no-grad call; the gradients (planes, heads, camera) are those of the second pass
    over the merged depths held fixed, from the backward kernel."""
    from ide3d_b200 import render, render_grad
    S_, NI = S, 10
    tex, seg, dec, cam, u, ui, gf, gd = hier_case(21, S_, NI)
    heads = live_heads(dec)
    kernel_calls, chain_calls = [], []
    with spy(render, 'raymarch_backward', kernel_calls), spy(render_grad, 'composed_chain', chain_calls):
        feat, d, z, t_grad, s_grad, c_grad = hier_backward(tex, seg, heads, cam, u, ui, gf, gd, S_, NI)
    assert kernel_calls and not chain_calls
    with torch.no_grad():
        f0, d0, _, z0 = render.raymarch_hierarchical(tex.to(DEV), seg.to(DEV), live_heads(dec, grad=False), cam.to(DEV), resolution=RES,
                                                     num_steps=S_, n_importance=NI, jitter_u=u.to(DEV), importance_u=ui.to(DEV), return_depths=True)
    assert torch.equal(feat, f0) and torch.equal(d, d0) and torch.equal(z, z0)
    _, _, gt, gs, gc, gp = oracle_explicit_grads(tex, seg, dec, cam, z.cpu(), gf, gd)
    for mine, ref, what in ((t_grad, gt, 'tex'), (s_grad, gs, 'seg'), (c_grad, gc, 'cam')):
        assert (mine.cpu() - ref).abs().max() <= tol(ref), what
    check_head_grads(heads, gp, tol)


@pytest.mark.gpu
def test_hierarchical_beyond_kernel_samples_falls_back_to_composed_chain():
    """S + n_importance > 256: the backward kernel declines, the composed chain over the saved depths gives the same gradients."""
    from ide3d_b200 import render_grad
    S_, NI = 130, 130
    tex, seg, dec, cam, u, ui, gf, gd = hier_case(22, S_, NI)
    heads = live_heads(dec)
    chain_calls = []
    with spy(render_grad, 'composed_chain', chain_calls):
        _, _, z, t_grad, s_grad, c_grad = hier_backward(tex, seg, heads, cam, u, ui, gf, gd, S_, NI)
    assert chain_calls and all(k.get('z_vals') is not None for k in chain_calls)
    _, _, gt, gs, gc, gp = oracle_explicit_grads(tex, seg, dec, cam, z.cpu(), gf, gd)
    for mine, ref, what in ((t_grad, gt, 'tex'), (s_grad, gs, 'seg'), (c_grad, gc, 'cam')):
        assert (mine.cpu() - ref).abs().max() <= tol(ref), what
    check_head_grads(heads, gp, tol)


@pytest.mark.gpu
def test_generator_hierarchical_synthesis_backpropagates_to_ws_decoder_and_camera():
    from ide3d_b200.training.triplane import TriPlaneGenerator
    torch.manual_seed(0)
    G = TriPlaneGenerator(z_dim=32, w_dim=32, img_resolution=64, plane_resolution=32, render_size=16, channel_base=512, channel_max=16,
                          sr_channels=(8, 8), mapping_kwargs=dict(num_layers=2)).cuda().train().requires_grad_(True)
    ws = torch.randn(2, G.num_ws, G.w_dim, device='cuda', requires_grad=True)
    label = torch.tensor([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 2.7, 0, 0, 0, 1, 4.2647, 0, 0.5, 0, 4.2647, 0.5, 0, 0, 1.], device='cuda').repeat(2, 1)
    c = label.requires_grad_(True)
    img = G.synthesis(ws, c=c, noise_mode='const', render_params=dict(num_steps=8, hierarchical=True, n_importance=8), perturb=None)
    img.square().mean().backward()
    assert ws.grad is not None and torch.isfinite(ws.grad).all() and ws.grad.abs().max() > 0
    r = G.synthesis.renderer
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in r.parameters())
    assert r.sigma_net.fc2.weight.grad.abs().max() > 0 and r.tex_net.fc1.weight.grad.abs().max() > 0
    assert c.grad is not None and torch.isfinite(c.grad).all() and c.grad[:, :12].abs().max() > 0
