"""Backward of the fused renderer (SURVEY.md §8f rank 1: PTI / encoder callers differentiate through G.synthesis,
inversion/training/projectors/w_plus_projector_ide3d.py:115).

Round-1 form: the FORWARD is always the fused sm_90a kernel (render.raymarch); the BACKWARD re-evaluates the same chain
-- rays (volumetric_rendering.py:77-97), jitter (:99-105), cam2world (:122-134), tri-plane gather (dnnlib/util.py:580-617,
grid_sample_gradfix.py:26-29), decoder heads, compositing (:34-74) -- with differentiable torch library ops on the GPU and
lets autograd produce the gradients w.r.t. the planes, the decoder parameters and the camera.  That costs the memory the
fused kernel avoids (every per-sample intermediate is materialised, in slabs of `RAYS_PER_SLAB` rays) and is the piece a
hand-written scatter kernel replaces next; values agree with the kernel to its stated forward tolerance.
Nothing here runs unless a gradient is requested.
"""

import math

import torch
import torch.nn.functional as F

N_FEAT, N_OUT = 32, 52
USE_BACKWARD_KERNEL = True    # ide3d_raymarch_bwd(_cam) for the planes / decoder / camera gradients; False = always differentiate the composed chain
RAYS_PER_SLAB = 1024          # rays per recompute slab: bounds the materialised [n, rays, S, 52+64+...] tensors


def hash_uniform(count, seed, device, first=0):
    """The kernel's counter hash (csrc/raymarch_common.cuh: jitter_hash) in torch integer ops: uniforms in [0,1) for the
    flat sample indices first .. first+count-1 (uint32 wrap)."""
    m = 0xFFFFFFFF
    idx = (torch.arange(first, first + count, device=device, dtype=torch.int64)) & m
    lo, hi = int(seed) & m, (int(seed) >> 32) & m
    h = (idx ^ lo) & m
    h = (h * 0x9E3779B1) & m
    h = h ^ hi
    h = h ^ (h >> 16)
    h = (h * 0x21F0AAAD) & m
    h = h ^ (h >> 15)
    h = (h * 0x735A2D97) & m
    h = h ^ (h >> 15)
    return (h >> 8).to(torch.float32) * (1.0 / 16777216.0)


def hash_uniform_frames(count, seeds, device, first=0):
    """Per-frame twin of hash_uniform (the kernel's per-frame seed mode, ide3d_raymarch_params.jitter_seeds): row f holds the uniforms
    of the frame-local sample indices first .. first+count-1 hashed with seeds[f].  -> [len(seeds), count]"""
    return torch.stack([hash_uniform(count, s, device, first) for s in seeds]) if len(seeds) else torch.empty(0, count, device=device)


def _gather(coords, planes):
    """sample_from_triplane: planes [n,96,H,W], coords [n,P,3] in grid units -> [n,P,32] (sum over xy, yz, xz)."""
    n, c3, h, w = planes.shape
    g = planes.reshape(n, 3, c3 // 3, h, w)
    out = 0
    for k, idx in enumerate(([0, 1], [1, 2], [0, 2])):
        s = F.grid_sample(g[:, k], coords[..., idx].reshape(n, -1, 1, 2), mode='bilinear', padding_mode='zeros', align_corners=False)
        out = out + s[..., 0].permute(0, 2, 1)
    return out


def _decode(f_tex, f_seg, heads):
    """heads: [(in_sel, out_offset, w1, b1, w2, b2)] -> [..., 52]; channels no head writes are 0."""
    out = torch.zeros(f_tex.shape[:-1] + (N_OUT,), dtype=f_tex.dtype, device=f_tex.device)
    for in_sel, off, w1, b1, w2, b2 in heads:
        f = f_tex if in_sel == 0 else f_seg if in_sel == 1 else torch.cat([f_tex, f_seg], -1)
        o = F.softplus(f @ w1.t() + b1) @ w2.t() + b2
        out = out + F.pad(o, (int(off), N_OUT - int(off) - o.shape[-1]))
    return out


def composed_chain(tex, seg, heads, cam2world, cfg, jitter_u=None, noise=None, rays=None, z_vals=None):
    """The renderer chain on materialised tensors.  tex/seg [n,96,H,W]; cam2world [n,4,4]; cfg: dict(W, H, S, fov, ray_start,
    ray_end, box_scale, jitter_seed, noise_std, clamp_mode, last_back, white_back, max_depth, fill_weight[, views]).
    views > 1: the planes hold n / views sets, frame f reads set f // views (materialised here by repeat_interleave, so autograd sums
    the views' gradients into their set); jitter_seed may be a list of per-frame seeds.
    z_vals: explicit sample depths [n,R,S] (render.raymarch's z_vals), used in place of linspace + jitter; they take no gradient.
    rays: optional (first, count) slab of the R = W*H rays.  -> feat [n,r,51], depth [n,r,1], weights [n,r,S,1]."""
    views = int(cfg.get('views', 1) or 1)
    if views > 1:
        tex, seg = tex.repeat_interleave(views, 0), seg.repeat_interleave(views, 0)
    dev = tex.device
    n = tex.shape[0]
    W, H, S = cfg['W'], cfg['H'], cfg['S']
    R = W * H
    r0, rc = rays if rays is not None else (0, R)
    xs = torch.linspace(-1, 1, W, device=dev)
    ys = torch.linspace(1, -1, H, device=dev)
    x = xs.reshape(1, W).expand(H, W).reshape(-1)[r0:r0 + rc]
    y = ys.reshape(H, 1).expand(H, W).reshape(-1)[r0:r0 + rc]
    z = torch.full_like(x, -1.0 / math.tan((2 * math.pi * cfg['fov'] / 360) / 2))
    d = torch.stack([x, y, z], -1)
    d = d / d.norm(dim=-1, keepdim=True)                                     # [r,3]
    zv = torch.linspace(cfg['ray_start'], cfg['ray_end'], S, device=dev)
    u = None
    if z_vals is not None:
        z_vals = z_vals.detach().to(device=dev, dtype=torch.float32).reshape(n, R, S)[:, r0:r0 + rc]
    else:
        z_vals = zv.reshape(1, 1, S).expand(n, rc, S)
        if jitter_u is not None:
            u = jitter_u.reshape(n, R, S)[:, r0:r0 + rc]
        elif cfg.get('jitter_seed') is not None:
            from .render import frame_seeds
            seeds = frame_seeds(cfg['jitter_seed'])
            if seeds is None:
                u = torch.stack([hash_uniform(rc * S, cfg['jitter_seed'], dev, first=(i * R + r0) * S).reshape(rc, S) for i in range(n)])
            else:
                u = hash_uniform_frames(rc * S, seeds, dev, first=r0 * S).reshape(n, rc, S)
    if u is not None and S > 1:
        z_vals = z_vals + (u - 0.5) * (zv[1] - zv[0])
    pts = d.reshape(1, rc, 1, 3) * z_vals.unsqueeze(-1)                      # camera space
    cam = cam2world.reshape(n, 4, 4).to(torch.float32)
    pw = torch.einsum('nij,nrsj->nrsi', cam[:, :3, :3], pts) + cam[:, :3, 3].reshape(n, 1, 1, 3)
    coords = pw.reshape(n, rc * S, 3) * cfg['box_scale']
    raw = _decode(_gather(coords, tex), _gather(coords, seg), heads).reshape(n, rc, S, N_OUT)

    rgbs, sigmas = raw[..., :-1], raw[..., -1:]
    zc = z_vals.unsqueeze(-1)
    deltas = (zc[:, :, 1:] - zc[:, :, :-1]) * d.norm(dim=-1).reshape(1, rc, 1, 1)
    deltas = torch.cat([deltas, 1e10 * torch.ones_like(deltas[:, :, :1])], -2)
    if noise is not None and cfg.get('noise_std'):
        sigmas = sigmas + noise.reshape(n, R, S, 1)[:, r0:r0 + rc] * cfg['noise_std']
    dens = F.softplus(sigmas) if cfg['clamp_mode'] == 'softplus' else F.relu(sigmas)
    alphas = 1 - torch.exp(-deltas * dens)
    shifted = torch.cat([torch.ones_like(alphas[:, :, :1]), 1 - alphas + 1e-10], -2)
    weights = alphas * torch.cumprod(shifted, -2)[:, :, :-1]
    wsum = weights.sum(2)
    if cfg.get('last_back'):
        weights = torch.cat([weights[:, :, :-1], weights[:, :, -1:] + (1 - wsum).unsqueeze(2)], 2)
    feat = (weights * rgbs).sum(-2)
    depth = (weights * zc).sum(-2)
    if cfg.get('white_back'):
        feat = feat + 1 - wsum
    if cfg.get('max_depth'):
        depth = depth + (1 - wsum) * cfg['max_depth']
    if cfg.get('fill_weight'):
        feat = wsum.expand_as(feat)
    return feat, depth, weights


class RaymarchFunction(torch.autograd.Function):
    """forward: render._raymarch_fwd (fused kernel).  backward: autograd through `composed_chain`, slab by slab."""

    @staticmethod
    def forward(ctx, fwd, cfg, head_meta, jitter_u, noise, z_vals, want_weights, tex, seg, cam2world, *params):
        heads = [(m[0], m[1]) + tuple(params[4 * i:4 * i + 4]) for i, m in enumerate(head_meta)]
        feat, depth, weights = fwd(tex, seg, heads, cam2world, jitter_u, noise)
        ctx.cfg, ctx.head_meta, ctx.want_weights = cfg, head_meta, want_weights
        ctx.save_for_backward(tex, seg, cam2world, jitter_u, noise, z_vals, *params)
        if weights is None:
            weights = feat.new_zeros(())
        return feat, depth, weights

    @staticmethod
    def backward(ctx, dfeat, ddepth, dweights):
        tex, seg, cam2world, jitter_u, noise, z_vals, *params = ctx.saved_tensors
        cfg = ctx.cfg
        need = ctx.needs_input_grad[7:]
        # fast path: the backward kernel (ide3d_raymarch_bwd_cam) -- planes, three-head decoder and camera; no per-sample-weight gradients
        want_w = ctx.want_weights and dweights is not None and dweights.ndim == 4 and bool((dweights != 0).any())
        if USE_BACKWARD_KERNEL and tex.is_cuda and not want_w:
            from . import render
            heads = [(m[0], m[1]) + tuple(params[4 * i:4 * i + 4]) for i, m in enumerate(ctx.head_meta)]
            kw = dict(resolution=(cfg['W'], cfg['H']), num_steps=cfg['S'], fov=cfg['fov'], ray_start=cfg['ray_start'], ray_end=cfg['ray_end'],
                      box_scale=cfg['box_scale'], jitter_u=jitter_u, jitter_seed=cfg.get('jitter_seed'), noise=noise, noise_std=cfg.get('noise_std', 0.0),
                      clamp_mode=cfg['clamp_mode'], last_back=cfg['last_back'], white_back=cfg['white_back'], max_depth=cfg['max_depth'],
                      fill_mode='weight' if cfg['fill_weight'] else None, views=cfg.get('views', 1), z_vals=z_vals)
            res = render.raymarch_backward(tex, seg, heads, cam2world, dfeat, ddepth, want_planes=(bool(need[0]), bool(need[1])),
                                           want_params=any(need[3:]), want_camera=bool(need[2]), **kw)
            if res is not None:
                d_tex, d_seg, d_par = res[:3]
                d_cam = res[3].to(cam2world.dtype) if need[2] else None
                gp = [None] * len(params) if d_par is None else [g.reshape(p.shape).to(p.dtype) if nd else None for g, p, nd in zip(d_par, params, need[3:])]
                return (None,) * 7 + (d_tex if need[0] else None, d_seg if need[1] else None, d_cam) + tuple(gp)
        leaves = [t.detach().requires_grad_(bool(nd)) for t, nd in zip((tex, seg, cam2world) + tuple(params), need)]
        wanted = [t for t in leaves if t.requires_grad]
        grads = [torch.zeros_like(t) for t in wanted]
        if wanted:
            l_tex, l_seg, l_cam, *l_params = leaves
            heads = [(m[0], m[1]) + tuple(l_params[4 * i:4 * i + 4]) for i, m in enumerate(ctx.head_meta)]
            R = cfg['W'] * cfg['H']
            for r0 in range(0, R, RAYS_PER_SLAB):
                rc = min(RAYS_PER_SLAB, R - r0)
                with torch.enable_grad():
                    feat, depth, weights = composed_chain(l_tex, l_seg, heads, l_cam, cfg, jitter_u, noise, rays=(r0, rc), z_vals=z_vals)
                    outs, gouts = [feat, depth], [dfeat[:, r0:r0 + rc], ddepth[:, r0:r0 + rc]]
                    if ctx.want_weights and dweights is not None and dweights.ndim == 4:
                        outs.append(weights); gouts.append(dweights[:, r0:r0 + rc])
                g = torch.autograd.grad(outs, wanted, gouts, allow_unused=True)
                for acc, gi in zip(grads, g):
                    if gi is not None:
                        acc.add_(gi)
        it = iter(grads)
        out = [next(it) if t.requires_grad else None for t in leaves]
        return (None,) * 7 + tuple(out)
