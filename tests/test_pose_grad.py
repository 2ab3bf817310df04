"""CPU: explicit-depth gradients of the composed chain (the fallback of hierarchical renders under grad) and the ABI of
ide3d_raymarch_bwd_cam.  The reference is autograd through the oracle's stage functions, composed here for explicit depths."""

import ctypes

import pytest
import torch

from oracle import renderer as orr
from test_abi import RAYMARCH_BROKEN, _fake_raymarch_params
from test_gpu_renderer import _random_case, three_head_from_dense

S, RES = 12, (6, 5)
R = RES[0] * RES[1]


def cfg_for(S_, **opts):
    return dict(W=RES[0], H=RES[1], S=S_, fov=18.0, ray_start=2.25, ray_end=3.3, box_scale=opts.get('box_scale', 2.0), jitter_seed=None,
                noise_std=0.0, clamp_mode=opts.get('clamp_mode', 'softplus'), last_back=opts.get('last_back', False),
                white_back=opts.get('white_back', False), max_depth=opts.get('max_depth', 0.0), fill_weight=opts.get('fill_mode') == 'weight')


def oracle_explicit(tex, seg, dec, cam, z, box_scale=2.0, res=RES, gather=orr.sample_triplane, **opts):
    """initial_rays (directions) -> points d * z at the given depths [n,R,S] -> to_world -> gather -> decoder -> composite.
    Rays, depths and camera take the planes' dtype and device (a float64 reference on the GPU: gather=orr.sample_triplane_torch)."""
    n, R_, S_ = z.shape
    assert R_ == res[0] * res[1]
    _, _, d = orr.initial_rays(n, S_, 18.0, res, 2.25, 3.3, dtype=tex.dtype, device=tex.device)
    zz = z.to(device=tex.device, dtype=tex.dtype).reshape(n, R_, S_, 1)
    pw, _, _ = orr.to_world(d.unsqueeze(2) * zz, d, cam.to(device=tex.device, dtype=tex.dtype))
    coords = pw.reshape(n, -1, 3) * box_scale
    out = dec(gather(coords, tex), gather(coords, seg)).reshape(n, R_, S_, orr.N_OUT)
    return orr.composite(out, d, zz, **dict(dict(clamp_mode='softplus'), **opts))


def oracle_explicit_grads(tex, seg, dec, cam, z, gf, gd, **opts):
    """Values and gradients (tex, seg, cam, [w1, b1, w2, b2] of the dense decoder) of oracle_explicit; z takes no gradient."""
    t, s, c = tex.clone().requires_grad_(True), seg.clone().requires_grad_(True), cam.clone().requires_grad_(True)
    params = [p.clone().requires_grad_(True) for p in (dec.w1, dec.b1, dec.w2, dec.b2)]
    rgb, depth, _ = oracle_explicit(t, s, orr.Decoder(*params), c, z.detach(), **opts)
    (rgb * gf).sum().add((depth * gd).sum()).backward()
    return rgb.detach(), depth.detach(), t.grad, s.grad, c.grad, [p.grad for p in params]


def sorted_depths(n, S_, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.sort(2.25 + 1.05 * torch.rand(n, R, S_, generator=g), dim=-1).values


def check_head_grads(heads, gp, tol):
    """Head gradients against the matching blocks of the dense oracle decoder's gradients."""
    H = 64
    w1g, b1g, w2g, b2g = gp
    blocks = [(slice(0, H), slice(0, 32), slice(0, 32)), (slice(H, 2 * H), slice(32, 64), slice(32, 51)), (slice(2 * H, 3 * H), slice(32, 64), slice(51, 52))]
    for (_, _, hw1, hb1, hw2, hb2), (hs, ks, os_) in zip(heads, blocks):
        assert (hw1.grad.cpu() - w1g[hs, ks]).abs().max() <= tol(w1g), 'w1'
        assert (hb1.grad.cpu() - b1g[hs]).abs().max() <= tol(b1g), 'b1'
        assert (hw2.grad.cpu() - w2g[os_, hs]).abs().max() <= tol(w2g), 'w2'
        assert (hb2.grad.cpu() - b2g[os_]).abs().max() <= tol(b2g), 'b2'


@pytest.mark.parametrize('opts', [dict(), dict(white_back=True, max_depth=3.3, last_back=True), dict(clamp_mode='relu')])
def test_composed_chain_explicit_depths_matches_oracle(opts):
    from ide3d_b200 import render_grad as rg
    tex, seg, dec, cam = _random_case(2, 16, seed=4)
    z = sorted_depths(2, S, seed=2)
    g = torch.Generator().manual_seed(1)
    gf, gd = torch.randn(2, R, 51, generator=g), torch.randn(2, R, 1, generator=g)
    rgb, depth, gt, gs, gc, gp = oracle_explicit_grads(tex, seg, dec, cam, z, gf, gd, **opts)

    heads = [tuple(h[:2]) + tuple(t.clone().requires_grad_(True) for t in h[2:]) for h in three_head_from_dense(dec.w1, dec.b1, dec.w2, dec.b2)]
    t, s, c = tex.clone().requires_grad_(True), seg.clone().requires_grad_(True), cam.clone().requires_grad_(True)
    f, d, _ = rg.composed_chain(t, s, heads, c, cfg_for(S, **opts), z_vals=z)
    assert (f - rgb).abs().max() < 3e-5 and (d - depth).abs().max() < 1e-5
    slabs = torch.cat([rg.composed_chain(t, s, heads, c, cfg_for(S, **opts), rays=(r0, min(7, R - r0)), z_vals=z)[0] for r0 in range(0, R, 7)], 1)
    assert (slabs - f).abs().max() < 3e-6
    (f * gf).sum().add((d * gd).sum()).backward()
    tol = lambda ref: 2e-4 * max(1.0, ref.abs().max().item())
    for mine, ref, what in ((t.grad, gt, 'tex'), (s.grad, gs, 'seg'), (c.grad, gc, 'cam')):
        assert (mine - ref).abs().max() <= tol(ref), what
    check_head_grads(heads, gp, tol)


def test_hierarchical_gradient_is_the_fine_pass_with_detached_depths():
    """The gradient of a hierarchical render is the gradient of its second pass over the merged depths, held fixed: the oracle's
    two-pass render equals the explicit-depth composition over its own merged depths, and the composed chain over those depths has
    the gradients autograd gives that composition with all_z detached."""
    from ide3d_b200 import render_grad as rg
    tex, seg, dec, cam = _random_case(2, 16, seed=6)
    NI = 8
    g = torch.Generator().manual_seed(3)
    u = torch.rand(2, R, S, 1, generator=g)
    ui = torch.rand(2 * R, NI, generator=g)
    ro, do_, _, all_z = orr.render_frames_hierarchical(tex, seg, dec, cam, num_steps=S, n_importance=NI, resolution=RES, jitter_u=u, importance_u=ui)
    all_z = all_z.reshape(2, R, S + NI)
    gf, gd = torch.randn(2, R, 51, generator=g), torch.randn(2, R, 1, generator=g)
    rgb, depth, gt, gs, gc, gp = oracle_explicit_grads(tex, seg, dec, cam, all_z, gf, gd)
    assert (rgb - ro).abs().max() < 1e-5 and (depth - do_).abs().max() < 1e-5

    heads = [tuple(h[:2]) + tuple(t.clone().requires_grad_(True) for t in h[2:]) for h in three_head_from_dense(dec.w1, dec.b1, dec.w2, dec.b2)]
    t, s, c = tex.clone().requires_grad_(True), seg.clone().requires_grad_(True), cam.clone().requires_grad_(True)
    f, d, _ = rg.composed_chain(t, s, heads, c, cfg_for(S + NI), z_vals=all_z)
    assert (f - ro).abs().max() < 3e-5 and (d - do_).abs().max() < 1e-5
    (f * gf).sum().add((d * gd).sum()).backward()
    tol = lambda ref: 2e-4 * max(1.0, ref.abs().max().item())
    for mine, ref, what in ((t.grad, gt, 'tex'), (s.grad, gs, 'seg'), (c.grad, gc, 'cam')):
        assert (mine - ref).abs().max() <= tol(ref), what
    check_head_grads(heads, gp, tol)


@pytest.mark.skipif(torch.cuda.is_available(), reason='passes fake device pointers: run only where no GPU can be reached')
@pytest.mark.parametrize('case', sorted(RAYMARCH_BROKEN))
def test_camera_backward_shares_raymarch_validation(lib, case):
    """ide3d_raymarch_bwd_cam rejects the malformed parameters of the shared table with the forward's status and message."""
    from ide3d_b200 import _lib
    breaker, message = RAYMARCH_BROKEN[case]
    p = _fake_raymarch_params(_lib)
    breaker(p)
    fake = ctypes.c_void_p(0x10000)
    assert lib.ide3d_raymarch_fwd(ctypes.byref(p), None) == _lib.INVALID
    fwd_error = lib.ide3d_last_error()
    assert message in fwd_error
    assert lib.ide3d_raymarch_bwd_cam(ctypes.byref(p), fake, None, fake, fake, None, fake, None) == _lib.INVALID
    assert lib.ide3d_last_error() == fwd_error
