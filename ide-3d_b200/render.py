"""Functional front-end of the fused renderer kernels (ide3d_raymarch_fwd / ide3d_sample_voxel / ide3d_sigma_grid).

Everything takes CUDA tensors and raises otherwise.  The decoder is passed as a list of heads
``(in_sel, out_offset, w1 [hid,in], b1 [hid], w2 [out,hid], b2 [out])`` with in_sel 0 = texture features,
1 = shape features, 2 = both (64 inputs) -- the ide3d_decoder of include/ide3d_b200.h.
"""

import ctypes as C

import torch

from . import _lib as L

N_FEAT, N_SEG, N_OUT = 32, 19, 52

# When set to a list, every fused ray-march launch appends (start_event, end_event, frames) recorded on the launching
# stream -- how bench.py measures the kernel's own duration live inside the full synthesis step.
kernel_events = None


class PackedDecoder:
    """fp32 device copies of the head parameters plus the C struct that points at them (kept alive together)."""

    def __init__(self, heads, device):
        assert 1 <= len(heads) <= 4
        self.tensors = []
        self.meta = [(int(h[0]), int(h[1])) for h in heads]          # (in_sel, out_offset) per head
        self.struct = L.Decoder()
        self.struct.num_heads = len(heads)
        for i, (in_sel, out_off, w1, b1, w2, b2) in enumerate(heads):
            ts = [t.detach().to(device=device, dtype=torch.float32).contiguous() for t in (w1, b1, w2, b2)]
            n_in = N_FEAT * (2 if in_sel == 2 else 1)
            if ts[0].shape[1] != n_in or ts[2].shape[1] != ts[0].shape[0] or ts[1].numel() != ts[0].shape[0] \
                    or ts[3].numel() != ts[2].shape[0]:
                raise RuntimeError('ide3d_b200: inconsistent decoder head shapes')
            self.tensors += ts
            self.struct.heads[i] = L.MlpHead(int(in_sel), ts[0].shape[0], int(out_off), ts[2].shape[0],
                                             *[t.data_ptr() for t in ts])


def dense_heads(w1, b1, w2, b2):
    """A dense [hid,64] / [52,hid] decoder as a single head."""
    return [(2, 0, w1, b1, w2, b2)]


def as_planes(t):
    """float32 channels-last view of a tri-plane tensor [N,96,H,W] (one ide3d_planes_to_nhwc pass if needed)."""
    L.require_cuda(t)
    if t.dtype != torch.float32:
        t = t.float()
    if t.stride(1) == 1 and t.is_contiguous(memory_format=torch.channels_last):
        return t
    n, c, h, w = t.shape
    out = torch.empty([n, c, h, w], dtype=torch.float32, device=t.device, memory_format=torch.channels_last)
    s = t.stride()
    L.check(L.get_lib().ide3d_planes_to_nhwc(L.ptr(t), n, c, h, w, s[0], s[1], s[2], s[3], L.ptr(out), L.stream_ptr(t.device)))
    return out


def _decoder(dec, device):
    return dec if isinstance(dec, PackedDecoder) else PackedDecoder(dec, device)


def raymarch(planes_tex, planes_seg, decoder, cam2world, resolution=(64, 64), num_steps=48, fov=18.0, ray_start=2.25,
             ray_end=3.3, box_scale=2.0, jitter_u=None, jitter_seed=None, noise=None, noise_std=0.0,
             clamp_mode='softplus', last_back=False, white_back=False, max_depth=None, fill_mode=None,
             return_weights=False, convert_layout=True, precision='auto', z_vals=None):
    """Fused render of N frames.  -> feat [N,R,51], depth [N,R,1], weights [N,R,S,1] | None.
    jitter_u: explicit uniforms [N,R,S]; jitter_seed: in-kernel counter hash; neither: no jitter.
    z_vals: explicit sample depths [N,R,S] ascending along S (replaces linspace + jitter; num_steps is taken from it).
    precision: 'auto' | 'fp32' (CUDA-core FFMA decoder) | 'tc' (wgmma tensor-core decoder, bf16x3 products).
    Differentiable w.r.t. the planes, the camera and the decoder parameters (when `decoder` is a list of heads holding the
    live parameters): the forward is the same fused kernel, the backward is render_grad.RaymarchFunction."""
    kw = dict(resolution=resolution, num_steps=num_steps, fov=fov, ray_start=ray_start, ray_end=ray_end, box_scale=box_scale,
              jitter_seed=jitter_seed, noise_std=noise_std, clamp_mode=clamp_mode, last_back=last_back, white_back=white_back,
              max_depth=max_depth, fill_mode=fill_mode, return_weights=return_weights, convert_layout=convert_layout, precision=precision)
    if z_vals is not None:
        if torch.is_grad_enabled() and z_vals.requires_grad:
            raise RuntimeError('ide3d_b200.render.raymarch: z_vals is not differentiable (the reference detaches the importance samples too)')
        kw.update(z_vals=z_vals, num_steps=int(z_vals.shape[-1]))
        num_steps = int(z_vals.shape[-1])
        if torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in [planes_tex, planes_seg, cam2world]):
            raise NotImplementedError('ide3d_b200.render.raymarch: the backward pass has no explicit-depth (hierarchical) mode yet')
    if isinstance(decoder, PackedDecoder):
        meta, params = decoder.meta, list(decoder.tensors)
    else:
        meta, params = [(int(h[0]), int(h[1])) for h in decoder], [t for h in decoder for t in h[2:6]]
    if torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in [planes_tex, planes_seg, cam2world] + params):
        from . import render_grad
        if clamp_mode not in ('softplus', 'relu'):
            raise ValueError('Need to choose clamp mode')
        W, H = (resolution, resolution) if isinstance(resolution, int) else resolution
        cfg = dict(W=int(W), H=int(H), S=int(num_steps), fov=float(fov), ray_start=float(ray_start), ray_end=float(ray_end),
                   box_scale=float(box_scale), jitter_seed=None if jitter_u is not None else jitter_seed, noise_std=float(noise_std or 0.0),
                   clamp_mode=clamp_mode, last_back=bool(last_back), white_back=bool(white_back), max_depth=float(max_depth or 0.0),
                   fill_weight=(fill_mode == 'weight'))

        def fwd(tex, seg, heads, cam, ju, nz):
            return _raymarch_impl(tex, seg, heads, cam, jitter_u=ju, noise=nz, **kw)

        n = planes_tex.shape[0]
        feat, depth, weights = render_grad.RaymarchFunction.apply(fwd, cfg, meta, jitter_u, noise, bool(return_weights), planes_tex.float(),
                                                                  planes_seg.float(), cam2world.reshape(n, 4, 4).float(), *params)
        return feat, depth, (weights if return_weights else None)
    return _raymarch_impl(planes_tex, planes_seg, decoder, cam2world, jitter_u=jitter_u, noise=noise, **kw)


def coarse_depths(n, resolution, num_steps, ray_start=2.25, ray_end=3.3, jitter_u=None, jitter_seed=None, device='cuda'):
    """z_vals [N, R, S] of the first (stratified) pass exactly as the fused kernel generates them: torch.linspace(ray_start, ray_end, S)
    (volumetric_rendering.py:91) + (u - 0.5) * (z[1] - z[0]) (:99-105), u = jitter_u or the kernel's counter hash."""
    W, H = (resolution, resolution) if isinstance(resolution, int) else resolution
    R, S = W * H, int(num_steps)
    z = torch.linspace(ray_start, ray_end, S, device=device, dtype=torch.float32)
    zv = z.reshape(1, 1, S).expand(n, R, S)
    if jitter_u is None and jitter_seed is not None:
        from .render_grad import hash_uniform
        jitter_u = hash_uniform(n * R * S, jitter_seed, device)
    if jitter_u is None:
        return zv.contiguous()
    spacing = (z[1] - z[0]) if S > 1 else z.new_zeros(())
    return zv + (jitter_u.to(device=device, dtype=torch.float32).reshape(n, R, S) - 0.5) * spacing


@torch.no_grad()
def raymarch_hierarchical(planes_tex, planes_seg, decoder, cam2world, resolution=(64, 64), num_steps=48, n_importance=None,
                          ray_start=2.25, ray_end=3.3, jitter_u=None, jitter_seed=None, importance_u=None, det=False,
                          return_weights=False, return_depths=False, **kw):
    """Two-pass (coarse -> importance) render, the hierarchical sampling that `sample_pdf` exists for
    (volumetric_rendering.py:224-265; used as in pi-GAN / StyleNeRF's renderers, dnnlib/camera.py:638):
        1. coarse fused pass over the stratified depths, returning the compositing weights;
        2. `ide3d_sample_pdf`: n_importance depths per ray drawn from the piecewise-constant pdf weights[1:-1] (+1e-5) over the
           midpoints of the coarse depths (importance_u [N*R, n_importance] injects the uniform draws; det=True uses linspace);
        3. the coarse and fine depths merged and sorted per ray; second fused pass over all S + n_importance samples with the depths
           read from that tensor (IDE3D_JITTER_ZVALS) -- compositing over the merged set, as the reference composition does.
    Forward only.  -> feat [N,R,51], depth [N,R,1], weights [N,R,S+n_importance,1] | None (, z_vals [N,R,S+n_importance])."""
    from .training.volumetric_rendering import sample_pdf_u
    L.require_cuda(planes_tex, planes_seg, cam2world)
    dev = planes_tex.device
    n = planes_tex.shape[0]
    W, H = (resolution, resolution) if isinstance(resolution, int) else resolution
    R, S = W * H, int(num_steps)
    n_imp = S if n_importance is None else int(n_importance)
    assert S >= 3, 'hierarchical sampling needs at least 3 coarse samples (weights[1:-1])'
    tex, seg = as_planes(planes_tex), as_planes(planes_seg)
    dec = _decoder(decoder, dev)
    z = coarse_depths(n, (W, H), S, ray_start, ray_end, jitter_u=jitter_u, jitter_seed=jitter_seed, device=dev)
    kw = dict(kw, convert_layout=False)
    noise_std = float(kw.pop('noise_std', 0.0) or 0.0)
    kw.pop('noise', None)                                  # drawn per pass (the two passes have different sample counts)
    draw = (lambda s_: dict(noise=torch.randn(n, R, s_, device=dev), noise_std=noise_std)) if noise_std else (lambda s_: {})
    _, _, w = _raymarch_impl(tex, seg, dec, cam2world, resolution=(W, H), ray_start=ray_start, ray_end=ray_end, z_vals=z,
                             num_steps=S, return_weights=True, **draw(S), **kw)
    z_mid = 0.5 * (z[..., :-1] + z[..., 1:])
    if det:
        u = torch.linspace(0, 1, n_imp, device=dev).expand(n * R, n_imp)
    elif importance_u is not None:
        u = importance_u.to(device=dev, dtype=torch.float32).reshape(n * R, n_imp)
    else:
        u = torch.rand(n * R, n_imp, device=dev)
    fine = sample_pdf_u(z_mid.reshape(n * R, S - 1), w.reshape(n * R, S)[:, 1:-1] + 1e-5, u)
    all_z = torch.sort(torch.cat([z, fine.reshape(n, R, n_imp)], -1), dim=-1).values
    feat, depth, weights = _raymarch_impl(tex, seg, dec, cam2world, resolution=(W, H), ray_start=ray_start, ray_end=ray_end,
                                          z_vals=all_z, num_steps=S + n_imp, return_weights=return_weights, **draw(S + n_imp), **kw)
    return (feat, depth, weights, all_z) if return_depths else (feat, depth, weights)


def _raymarch_impl(planes_tex, planes_seg, decoder, cam2world, resolution=(64, 64), num_steps=48, fov=18.0, ray_start=2.25,
                   ray_end=3.3, box_scale=2.0, jitter_u=None, jitter_seed=None, noise=None, noise_std=0.0,
                   clamp_mode='softplus', last_back=False, white_back=False, max_depth=None, fill_mode=None,
                   return_weights=False, convert_layout=True, precision='auto', z_vals=None):
    if clamp_mode not in ('softplus', 'relu'):
        raise ValueError('Need to choose clamp mode')
    if fill_mode not in (None, 'weight'):
        raise NotImplementedError(f'fill_mode={fill_mode!r} is not supported by the fused renderer')
    L.require_cuda(planes_tex, planes_seg, cam2world)
    tex = as_planes(planes_tex) if convert_layout else planes_tex
    seg = as_planes(planes_seg) if convert_layout else planes_seg
    dev = tex.device
    n = tex.shape[0]
    W, H = (resolution, resolution) if isinstance(resolution, int) else resolution
    R, S = W * H, int(num_steps)
    cam = cam2world.to(device=dev, dtype=torch.float32).reshape(n, 16).contiguous()
    dec = _decoder(decoder, dev)
    feat = torch.empty([n, R, N_OUT - 1], dtype=torch.float32, device=dev)
    depth = torch.empty([n, R, 1], dtype=torch.float32, device=dev)
    weights = torch.empty([n, R, S, 1], dtype=torch.float32, device=dev) if return_weights else None
    p = L.RaymarchParams()
    p.tex, p.seg, p.dec = L.triplane_view(tex), L.triplane_view(seg), dec.struct
    p.cam2world = L.ptr(cam)
    p.n, p.res_w, p.res_h, p.num_steps = n, W, H, S
    p.fov_deg, p.ray_start, p.ray_end, p.box_scale = float(fov), float(ray_start), float(ray_end), float(box_scale)
    if z_vals is not None:
        z_vals = z_vals.detach().to(device=dev, dtype=torch.float32).reshape(n, R, S).contiguous()
        p.jitter_mode, p.jitter_u = L.JITTER_ZVALS, L.ptr(z_vals)
    elif jitter_u is not None:
        jitter_u = jitter_u.to(device=dev, dtype=torch.float32).reshape(n, R, S).contiguous()
        p.jitter_mode, p.jitter_u = L.JITTER_TENSOR, L.ptr(jitter_u)
    elif jitter_seed is not None:
        p.jitter_mode, p.jitter_seed = L.JITTER_HASH, int(jitter_seed) & 0xFFFFFFFFFFFFFFFF
    else:
        p.jitter_mode = L.JITTER_NONE
    if noise is not None and noise_std:
        noise = noise.to(device=dev, dtype=torch.float32).reshape(n, R, S).contiguous()
        p.noise, p.noise_std = L.ptr(noise), float(noise_std)
    p.clamp_mode = L.CLAMP_SOFTPLUS if clamp_mode == 'softplus' else L.CLAMP_RELU
    p.last_back, p.white_back = int(bool(last_back)), int(bool(white_back))
    p.max_depth, p.fill_weight = float(max_depth or 0.0), int(fill_mode == 'weight')
    p.out_feat, p.out_depth, p.out_weights = L.ptr(feat), L.ptr(depth), L.ptr(weights)
    p.precision = L.PRECISION[precision]
    with torch.cuda.device(dev):
        if kernel_events is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        L.check(L.get_lib().ide3d_raymarch_fwd(C.byref(p), L.stream_ptr(dev)))
        if kernel_events is not None:
            e1.record()
            kernel_events.append((e0, e1, n))
    return feat, depth, weights


def sample_voxel(planes_tex, planes_seg, decoder, points, box_scale=2.0, sigma_only=False):
    """Decode world-space points [N,P,3] -> [N,P,52] (or [N,P,1] sigma)."""
    tex, seg = as_planes(planes_tex), as_planes(planes_seg)
    dev = tex.device
    pts = points.to(device=dev, dtype=torch.float32).contiguous()
    n, P = pts.shape[0], pts.shape[1]
    dec = _decoder(decoder, dev)
    out = torch.empty([n, P, 1 if sigma_only else N_OUT], dtype=torch.float32, device=dev)
    tv, sv = L.triplane_view(tex), L.triplane_view(seg)
    with torch.cuda.device(dev):
        L.check(L.get_lib().ide3d_sample_voxel(C.byref(tv), C.byref(sv), C.byref(dec.struct), L.ptr(pts), P,
                                               float(box_scale), int(sigma_only), L.ptr(out), L.stream_ptr(dev)))
    return out


def sigma_grid(planes_tex, planes_seg, decoder, grid_n=256, voxel_origin=(0, 0, 0), cube_length=2.0, pre_scale=0.9,
               box_scale=2.0, first=0, count=None):
    """Density for flat voxel indices [first, first+count) of the grid 0.9*create_samples(grid_n, origin, cube)
    (extract_shapes.py:74-103), points generated in the kernel.  -> [N, count]."""
    tex, seg = as_planes(planes_tex), as_planes(planes_seg)
    dev = tex.device
    count = grid_n ** 3 - first if count is None else count
    dec = _decoder(decoder, dev)
    out = torch.empty([tex.shape[0], count], dtype=torch.float32, device=dev)
    tv, sv = L.triplane_view(tex), L.triplane_view(seg)
    org = (C.c_float * 3)(*[float(v) for v in voxel_origin])
    with torch.cuda.device(dev):
        L.check(L.get_lib().ide3d_sigma_grid(C.byref(tv), C.byref(sv), C.byref(dec.struct), int(grid_n), C.byref(org),
                                             float(cube_length), float(pre_scale), float(box_scale), int(first),
                                             int(count), L.ptr(out), L.stream_ptr(dev)))
    return out


def raymarch_backward(planes_tex, planes_seg, decoder, cam2world, grad_feat, grad_depth, resolution=(64, 64), num_steps=48, fov=18.0,
                      ray_start=2.25, ray_end=3.3, box_scale=2.0, jitter_u=None, jitter_seed=None, noise=None, noise_std=0.0,
                      clamp_mode='softplus', last_back=False, white_back=False, max_depth=None, fill_mode=None, z_vals=None,
                      want_planes=(True, True), want_params=True):
    """ide3d_raymarch_bwd: gradients of (feat, depth) of `raymarch` w.r.t. the planes and the three decoder heads, one kernel that
    recomputes the per-sample chain (no materialised intermediates).  -> (d_tex | None, d_seg | None, [dW1, db1, dW2, db2] x 3 | None),
    or None when the configuration has no backward kernel (the caller then differentiates the composed chain)."""
    L.require_cuda(planes_tex, planes_seg, cam2world, grad_feat)
    tex, seg = as_planes(planes_tex), as_planes(planes_seg)
    dev = tex.device
    n = tex.shape[0]
    W, H = (resolution, resolution) if isinstance(resolution, int) else resolution
    R, S = W * H, int(num_steps if z_vals is None else z_vals.shape[-1])
    dec = _decoder(decoder, dev)
    if dec.meta != [(0, 0), (1, N_FEAT), (1, N_FEAT + N_SEG)] or S > 256:
        return None
    shapes = [tuple(t.shape) for t in dec.tensors]
    if shapes != [(64, 32), (64,), (32, 64), (32,), (64, 32), (64,), (19, 64), (19,), (64, 32), (64,), (1, 64), (1,)]:
        return None
    cam = cam2world.detach().to(device=dev, dtype=torch.float32).reshape(n, 16).contiguous()
    p = L.RaymarchParams()
    p.tex, p.seg, p.dec = L.triplane_view(tex), L.triplane_view(seg), dec.struct
    p.cam2world = L.ptr(cam)
    p.n, p.res_w, p.res_h, p.num_steps = n, W, H, S
    p.fov_deg, p.ray_start, p.ray_end, p.box_scale = float(fov), float(ray_start), float(ray_end), float(box_scale)
    keep = []
    if z_vals is not None:
        zt = z_vals.detach().to(device=dev, dtype=torch.float32).reshape(n, R, S).contiguous(); keep.append(zt)
        p.jitter_mode, p.jitter_u = L.JITTER_ZVALS, L.ptr(zt)
    elif jitter_u is not None:
        ju = jitter_u.detach().to(device=dev, dtype=torch.float32).reshape(n, R, S).contiguous(); keep.append(ju)
        p.jitter_mode, p.jitter_u = L.JITTER_TENSOR, L.ptr(ju)
    elif jitter_seed is not None:
        p.jitter_mode, p.jitter_seed = L.JITTER_HASH, int(jitter_seed) & 0xFFFFFFFFFFFFFFFF
    else:
        p.jitter_mode = L.JITTER_NONE
    if noise is not None and noise_std:
        nz = noise.detach().to(device=dev, dtype=torch.float32).reshape(n, R, S).contiguous(); keep.append(nz)
        p.noise, p.noise_std = L.ptr(nz), float(noise_std)
    p.clamp_mode = L.CLAMP_SOFTPLUS if clamp_mode == 'softplus' else L.CLAMP_RELU
    p.last_back, p.white_back = int(bool(last_back)), int(bool(white_back))
    p.max_depth, p.fill_weight = float(max_depth or 0.0), int(fill_mode == 'weight')
    gf = grad_feat.detach().to(device=dev, dtype=torch.float32).reshape(n, R, N_OUT - 1).contiguous()
    gd = None if grad_depth is None else grad_depth.detach().to(device=dev, dtype=torch.float32).reshape(n, R).contiguous()
    d_tex = torch.zeros_like(tex) if want_planes[0] else None               # channels-last, like the forward's planes
    d_seg = torch.zeros_like(seg) if want_planes[1] else None
    d_par = [torch.zeros(sh, dtype=torch.float32, device=dev) for sh in shapes] if want_params else None
    ptrs = None
    if d_par is not None:
        ptrs = (C.c_void_p * 12)(*[t.data_ptr() for t in d_par])
    with torch.cuda.device(dev):
        rc = L.get_lib().ide3d_raymarch_bwd(C.byref(p), L.ptr(gf), L.ptr(gd), L.ptr(d_tex), L.ptr(d_seg), ptrs, L.stream_ptr(dev))
    if L.check(rc, allow_unsupported=True) == L.UNSUPPORTED:
        return None
    return d_tex, d_seg, d_par
