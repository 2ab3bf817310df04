"""Plugin-level entry points: the functions the reference's pybind11 modules export, re-implemented on
top of the C-ABI library.  Same argument lists, same validation messages (TORCH_CHECK -> RuntimeError),
same return conventions (including filtered_lrelu's `return_code = -1` = "no specialised kernel").

    bias_act_plugin.bias_act                     torch_utils/ops/bias_act.cpp:32
    upfirdn2d_plugin.upfirdn2d                   torch_utils/ops/upfirdn2d.cpp:16
    filtered_lrelu_plugin.filtered_lrelu         torch_utils/ops/filtered_lrelu.cpp:16
    filtered_lrelu_plugin.filtered_lrelu_act_    torch_utils/ops/filtered_lrelu.cpp:213
"""

import ctypes as C

import torch

from . import _lib as L


def _req(cond, msg):
    if not cond:
        raise RuntimeError(msg)


def _has(t):
    return t is not None and t.numel() > 0


def _suggest_memory_format(x):
    # at::Tensor::suggest_memory_format(): channels_last iff the tensor is laid out that way
    if x.ndim == 4 and x.is_contiguous(memory_format=torch.channels_last) and not x.is_contiguous():
        return torch.channels_last
    return torch.contiguous_format


# ------------------------------------------------------------------------------------------- bias_act
def bias_act(x, b, xref, yref, dy, grad, dim, act, alpha, gain, clamp):
    L.require_cuda(x)
    _req(not _has(b) or (b.dtype == x.dtype and b.device == x.device), 'b must have the same dtype and device as x')
    for name, t in (('xref', xref), ('yref', yref), ('dy', dy)):
        _req(not _has(t) or (t.shape == x.shape and t.dtype == x.dtype and t.device == x.device),
             f'{name} must have the same shape, dtype, and device as x')
    _req(not _has(b) or b.ndim == 1, 'b must have rank 1')
    _req(not _has(b) or (0 <= dim < x.ndim), 'dim is out of bounds')
    _req(not _has(b) or b.shape[0] == x.shape[dim], 'b has wrong number of elements')
    _req(grad >= 0, 'grad must be non-negative')
    dense = x.is_contiguous() or (x.ndim == 4 and x.is_contiguous(memory_format=torch.channels_last))
    _req(dense, 'x must be non-overlapping and dense')
    for t in (xref, yref, dy):
        _req(not _has(t) or t.stride() == x.stride(), 'xref, yref and dy must have the same layout as x')
    if _has(b):
        b = b.contiguous()
    y = torch.empty_like(x)
    if x.numel() == 0:
        return y
    step_b = x.stride(dim) if _has(b) else 1
    rc = L.get_lib().ide3d_bias_act(L.ptr(x), L.ptr(b) if _has(b) else None, L.ptr(xref) if _has(xref) else None,
                                    L.ptr(yref) if _has(yref) else None, L.ptr(dy) if _has(dy) else None, L.ptr(y),
                                    L.dtype_code(x), int(grad), int(act), float(alpha), float(gain), float(clamp),
                                    x.numel(), b.numel() if _has(b) else 0, step_b, L.stream_ptr(x.device))
    L.check(rc)
    return y


def modconv_epilogue(x, scale, noise, b, act, alpha, gain, clamp, next_scale=None, only_next=False, out_dtype=None):
    """bias_act(x * scale[:, :, None, None] + noise, b) in one pass (extension, forward only).  x [N,C,H,W] dense NCHW or
    channels_last; scale [N,C] | None; noise [H,W] / [1,1,H,W] / [N,1,H,W] | None; b [C] | None.  With next_scale [N,C] a
    second tensor y * next_scale[:, :, None, None] is written in the same pass -> (y, y2), or y2 alone if only_next.
    out_dtype torch.float16 (channels_last float32 x, linear / lrelu): y and y2 are written in fp16, each rounded once from the
    float32 result.  Returns None when the kernel does not take the shape (caller composes the reference ops instead)."""
    L.require_cuda(x)
    _req(x.ndim == 4, 'x must be rank 4')
    n, c, h, w = x.shape
    cl = (not x.is_contiguous()) and x.is_contiguous(memory_format=torch.channels_last)
    _req(x.is_contiguous() or cl, 'x must be non-overlapping and dense')
    out_dtype = x.dtype if out_dtype is None else out_dtype
    mixed = out_dtype != x.dtype
    _req(not mixed or (x.dtype == torch.float32 and out_dtype == torch.float16), 'out_dtype must be the dtype of x, or float16 for float32 x')
    vec = 16 // x.element_size()
    if x.numel() == 0 or (cl and c % vec != 0) or (not cl and (h * w) % vec != 0) or (mixed and (not cl or act not in (1, 3))):
        return None
    if _has(scale):
        _req(scale.numel() == n * c, 'scale must have N*C elements')
        scale = scale.to(dtype=x.dtype).reshape(n, c).contiguous()
    noise_batch = 1
    if _has(noise):
        _req(noise.numel() in (h * w, n * h * w), 'noise must be [H,W] or [N,1,H,W]')
        noise_batch = noise.numel() // (h * w)
        noise = noise.to(dtype=x.dtype).contiguous()
    if _has(b):
        _req(b.ndim == 1 and b.shape[0] == c, 'b has wrong number of elements')
        b = b.to(dtype=x.dtype).contiguous()
    y = y2 = None
    if _has(next_scale):
        _req(next_scale.numel() == n * c, 'next_scale must have N*C elements')
        next_scale = next_scale.to(dtype=x.dtype).reshape(n, c).contiguous()
        y2 = torch.empty_like(x, dtype=out_dtype)
    if not (only_next and y2 is not None):
        y = torch.empty_like(x, dtype=out_dtype)
    rc = L.get_lib().ide3d_modconv_epilogue(L.ptr(x), L.ptr(scale) if _has(scale) else None, L.ptr(noise) if _has(noise) else None,
                                            L.ptr(b) if _has(b) else None, L.ptr(y) if y is not None else None,
                                            L.ptr(next_scale) if y2 is not None else None, L.ptr(y2) if y2 is not None else None,
                                            L.dtype2(x.dtype, out_dtype) if mixed else L.dtype_code(x), int(act), float(alpha),
                                            float(gain), float(clamp), n, c, h * w,
                                            noise_batch, int(cl), L.stream_ptr(x.device))
    if L.check(rc, allow_unsupported=True) == L.UNSUPPORTED:
        return None
    if y2 is None:
        return y
    return y2 if y is None else (y, y2)


def modconv_epilogue_rgb(x, scale, noise, b, act, alpha, gain, clamp, emit_y=True, y_scale=None, next_scale=None, rgb=None, fp32_tail=False):
    """`modconv_epilogue` for channels_last x with the consumers of its output folded in (extension, forward only):
    y = t (* y_scale[:, :, None, None]) if emit_y; y2 = t * next_scale[:, :, None, None] if next_scale is given; with
    rgb = (weight [O,C,1,1], styles [N,C], bias [O] | None), O <= 4, the ToRGB output conv1x1(t * styles, weight) + bias as a dense
    NCHW [N,O,H,W] float32 tensor.  x float32, or with fp32_tail float16 (the output of an fp16 convolution; y and y2 are then
    fp16, each rounded once from the float32 result).  Every other operand is used in float32.  Returns the list of the requested outputs in the
    order (y, y2, rgb), or None when the kernel does not take the shape (caller composes the reference ops instead)."""
    L.require_cuda(x)
    _req(x.ndim == 4, 'x must be rank 4')
    n, c, h, w = x.shape
    cl = (not x.is_contiguous()) and x.is_contiguous(memory_format=torch.channels_last)
    if not cl or x.dtype != (torch.float16 if fp32_tail else torch.float32) or c % 4 != 0 or c > 512 or x.numel() == 0:
        return None
    f32 = torch.float32

    def per_sample(t, name):
        if not _has(t):
            return None
        _req(t.numel() == n * c, f'{name} must have N*C elements')
        return t.to(dtype=f32).reshape(n, c).contiguous()

    scale, y_scale, next_scale = per_sample(scale, 'scale'), per_sample(y_scale, 'y_scale'), per_sample(next_scale, 'next_scale')
    noise_batch = 1
    if _has(noise):
        _req(noise.numel() in (h * w, n * h * w), 'noise must be [H,W] or [N,1,H,W]')
        noise_batch = noise.numel() // (h * w)
        noise = noise.to(dtype=f32).contiguous()
    if _has(b):
        _req(b.ndim == 1 and b.shape[0] == c, 'b has wrong number of elements')
        b = b.to(dtype=f32).contiguous()
    _req(y_scale is None or emit_y, 'y_scale needs emit_y')
    wrgb = srgb = brgb = out_rgb = None
    o = 0
    if rgb is not None:
        wrgb, srgb, brgb = rgb
        o = wrgb.shape[0]
        if o > 4:
            return None
        _req(wrgb.numel() == o * c, 'rgb weight must be [O, C, 1, 1]')
        wrgb = wrgb.to(dtype=f32).reshape(o, c).contiguous()
        srgb = per_sample(srgb, 'rgb styles')
        if brgb is not None:
            _req(brgb.numel() == o, 'rgb bias must have O elements')
            brgb = brgb.to(dtype=f32).contiguous()
        out_rgb = torch.empty([n, o, h, w], dtype=f32, device=x.device)
    y = torch.empty_like(x) if emit_y else None
    y2 = torch.empty_like(x) if next_scale is not None else None
    _req(y is not None or y2 is not None or out_rgb is not None, 'no output requested')
    opt = lambda t: L.ptr(t) if t is not None else None
    rc = L.get_lib().ide3d_modconv_epilogue_rgb(L.ptr(x), opt(scale), opt(noise), opt(b), opt(y_scale), opt(y), opt(next_scale), opt(y2),
                                                opt(wrgb), opt(srgb), opt(brgb), opt(out_rgb), o,
                                                L.F32 if x.dtype == f32 else L.dtype2(x.dtype, x.dtype), int(act), float(alpha),
                                                float(gain), float(clamp), n, c, h * w, noise_batch, L.stream_ptr(x.device))
    if L.check(rc, allow_unsupported=True) == L.UNSUPPORTED:
        return None
    return [t for t in (y, y2, out_rgb) if t is not None]


# ------------------------------------------------------------------------------------------- upfirdn2d
def upfirdn2d(x, f, upx, upy, downx, downy, padx0, padx1, pady0, pady1, flip, gain, add=None, bias=None, epilogue=None):
    """Extensions (return None if the kernel cannot fuse them, so the caller composes the reference ops):
    add / bias: y = upfirdn2d(x) + add + bias[c] in one pass;
    epilogue = dict(scale, noise, b, act (1|3), alpha, gain, clamp, next_scale, only_next, fp32_tail): the modulated-convolution tail
    applied to the filter output, -> y | (y, y2) | y2 exactly like `modconv_epilogue`; with fp32_tail and fp16 x the tail operands
    stay float32 (y / y2 fp16, rounded once), else they take the dtype of x.
    add of another dtype than x: float16 add onto float32 x."""
    L.require_cuda(x, f)
    _req(f.device == x.device, 'f must reside on the same device as x')
    _req(f.dtype == torch.float32, 'f must be float32')
    _req(x.numel() > 0, 'x has zero size')
    _req(f.numel() > 0, 'f has zero size')
    _req(x.ndim == 4, 'x must be rank 4')
    _req(f.ndim == 2, 'f must be rank 2')
    _req(f.shape[0] >= 1 and f.shape[1] >= 1, 'f must be at least 1x1')
    _req(upx >= 1 and upy >= 1, 'upsampling factor must be at least 1')
    _req(downx >= 1 and downy >= 1, 'downsampling factor must be at least 1')
    n, c, h, w = x.shape
    fh, fw = f.shape
    out_w = (w * upx + padx0 + padx1 - fw + downx) // downx
    out_h = (h * upy + pady0 + pady1 - fh + downy) // downy
    _req(out_w >= 1 and out_h >= 1, 'output must be at least 1x1')
    y = torch.empty([n, c, out_h, out_w], dtype=x.dtype, device=x.device, memory_format=_suggest_memory_format(x))
    xs, ys, fs = x.stride(), y.stride(), f.stride()
    p = L.UpfirParams(L.ptr(x), L.ptr(f), L.ptr(y), L.dtype_code(x), upx, upy, downx, downy, padx0, pady0,
                      1 if flip else 0, float(gain), w, h, c, n, xs[3], xs[2], xs[1], xs[0],
                      fw, fh, fs[1], fs[0], out_w, out_h, ys[3], ys[2], ys[1], ys[0])
    if epilogue is not None:
        e = epilogue
        if not (y.is_contiguous(memory_format=torch.channels_last) and not y.is_contiguous()) or e['act'] not in (1, 3) or x.dtype == torch.float64:
            return None
        tail = torch.float32 if e.get('fp32_tail') else x.dtype
        if tail != x.dtype:
            _req(x.dtype == torch.float16, 'fp32_tail needs float16 x')
            p.dtype = L.dtype2(x.dtype, x.dtype)

        def prep(t, numel):
            if t is None:
                return None
            _req(t.numel() == numel, 'epilogue operand has the wrong number of elements')
            return t.to(dtype=tail).contiguous()
        scale, b, scale2 = prep(e.get('scale'), n * c), prep(e.get('b'), c), prep(e.get('next_scale'), n * c)
        noise = e.get('noise')
        noise_batch = 1
        if noise is not None:
            _req(noise.numel() in (out_h * out_w, n * out_h * out_w), 'noise must be [H,W] or [N,1,H,W]')
            noise_batch = noise.numel() // (out_h * out_w)
            noise = noise.to(dtype=tail).contiguous()
        y2 = torch.empty_like(y) if scale2 is not None else None
        want_y = not (e.get('only_next') and y2 is not None)
        if not want_y:
            p.y = None
        ep = L.FirEpilogue(L.ptr(scale) if scale is not None else None, L.ptr(noise) if noise is not None else None,
                           L.ptr(b) if b is not None else None, L.ptr(scale2) if scale2 is not None else None,
                           L.ptr(y2) if y2 is not None else None, int(e['act']), float(e['alpha']), float(e['gain']),
                           float(e['clamp']), noise_batch)
        rc = L.get_lib().ide3d_upfirdn2d_epilogue(C.byref(p), C.byref(ep), L.stream_ptr(x.device))
        if L.check(rc, allow_unsupported=True) == L.UNSUPPORTED:
            return None
        if y2 is None:
            return y
        return (y, y2) if want_y else y2
    if add is not None:
        mixed = add.dtype == torch.float16 and x.dtype == torch.float32
        if tuple(add.shape) != (n, c, out_h, out_w) or (add.dtype != x.dtype and not mixed) or add.stride(1) != 1 or not y.is_contiguous(memory_format=torch.channels_last) or y.is_contiguous():
            return None
        if mixed:
            p.dtype = L.dtype2(x.dtype, add.dtype)
        if bias is not None:
            bias = bias.to(dtype=x.dtype).contiguous()
        a = add.stride()
        rc = L.get_lib().ide3d_upfirdn2d_add(C.byref(p), L.ptr(add), a[0], a[2], a[3], L.ptr(bias) if bias is not None else None,
                                             L.stream_ptr(x.device))
        return None if L.check(rc, allow_unsupported=True) == L.UNSUPPORTED else y
    L.check(L.get_lib().ide3d_upfirdn2d(C.byref(p), L.stream_ptr(x.device)))
    return y


# ------------------------------------------------------------------------------------------- filtered_lrelu
def filtered_lrelu(x, fu, fd, b, si, up, down, px0, px1, py0, py1, sx, sy, gain, slope, clamp, flip_filters, writeSigns):
    """-> (y, so, return_code); return_code -1 with (None, None) means "no fused kernel" (filtered_lrelu.cpp:52-56)."""
    L.require_cuda(x, fu, fd, b)
    _req(fu.device == x.device and fd.device == x.device and b.device == x.device, 'all input tensors must reside on the same device')
    _req(fu.dtype == torch.float32 and fd.dtype == torch.float32, 'fu and fd must be float32')
    _req(b.dtype == x.dtype, 'x and b must have the same dtype')
    _req(x.dtype in (torch.float16, torch.float32), 'x and b must be float16 or float32')
    _req(x.ndim == 4, 'x must be rank 4')
    _req(x.numel() > 0, 'x is empty')
    _req(fu.ndim in (1, 2) and fd.ndim in (1, 2), 'fu and fd must be rank 1 or 2')
    _req(fu.numel() > 0, 'fu is empty')
    _req(fd.numel() > 0, 'fd is empty')
    _req(b.ndim == 1 and b.shape[0] == x.shape[1], 'b must be a vector with the same number of channels as x')
    _req(up >= 1 and down >= 1, 'up and down must be at least 1')
    n, c, xh, xw = x.shape
    fut_w, fut_h = fu.shape[-1] - 1, fu.shape[0] - 1
    fdt_w, fdt_h = fd.shape[-1] - 1, fd.shape[0] - 1
    cw = xw * up + (px0 + px1) - fut_w
    ch = xh * up + (py0 + py1) - fut_h
    _req(cw > fdt_w and ch > fdt_h, 'upsampled buffer must be at least the size of downsampling filter')
    yw = (cw - fdt_w + (down - 1)) // down
    yh = (ch - fdt_h + (down - 1)) // down
    _req(yw > 0 and yh > 0, 'output must be at least 1x1')
    read_signs = _has(si)
    s = si if read_signs else None
    so = None
    sw = sh = 0
    y = torch.empty([n, c, yh, yw], dtype=x.dtype, device=x.device, memory_format=_suggest_memory_format(x))
    if writeSigns:
        sw_active = yw * down - (down - 1) + fdt_w
        sh = yh * down - (down - 1) + fdt_h
        sw = (sw_active + 15) & ~15
        s = so = torch.empty([n, c, sh, sw >> 2], dtype=torch.uint8, device=x.device)
    elif read_signs:
        _req(s.is_contiguous(), 'signs must be contiguous')
        _req(s.dtype == torch.uint8, 'signs must be uint8')
        _req(s.ndim == 4 and s.shape[0] == n and s.shape[1] == c, 'signs must have same batch & channels as x')
        sw, sh = s.shape[3] << 2, s.shape[2]
    fu_c, fd_c = fu.contiguous(), fd.contiguous()
    xs, ys = x.stride(), y.stride()
    p = L.FlreluParams(L.ptr(x), L.ptr(b.contiguous()), L.ptr(fu_c), L.ptr(fd_c), L.ptr(y), L.ptr(s) if s is not None else None,
                       L.dtype_code(x), up, down, fu.shape[-1], fu.shape[0] if fu.ndim == 2 else 0,
                       fd.shape[-1], fd.shape[0] if fd.ndim == 2 else 0, px0, py0, 1 if flip_filters else 0,
                       float(gain), float(slope), float(min(clamp, 3.0e38)), xw, xh, c, n, xs[3], xs[2], xs[1], xs[0],
                       yw, yh, ys[3], ys[2], ys[1], ys[0], sw, sh, sx, sy, 1 if writeSigns else 0,
                       1 if (read_signs and not writeSigns) else 0)
    rc = L.check(L.get_lib().ide3d_filtered_lrelu(C.byref(p), L.stream_ptr(x.device)), allow_unsupported=True)
    if rc == L.UNSUPPORTED:
        return None, None, -1
    return y, so, 0


def filtered_lrelu_act_(x, si, sx, sy, gain, slope, clamp, writeSigns):
    """In place on x; returns the freshly written sign tensor (or None)."""
    L.require_cuda(x)
    _req(x.ndim == 4, 'x must be rank 4')
    _req(x.numel() > 0, 'x is empty')
    _req(x.dtype in (torch.float16, torch.float32, torch.float64), 'x must be float16, float32 or float64')
    read_signs = _has(si)
    s, so = (si if read_signs else None), None
    n, c, h, w = x.shape
    if writeSigns:
        sw = (w + 15) & ~15
        s = so = torch.empty([n, c, h, sw >> 2], dtype=torch.uint8, device=x.device)
    if s is not None:
        _req(s.is_contiguous(), 'signs must be contiguous')
        _req(s.dtype == torch.uint8, 'signs must be uint8')
        _req(s.device == x.device, 'signs must reside on the same device as x')
        _req(s.ndim == 4 and s.shape[0] == n and s.shape[1] == c, 'signs must have same batch & channels as x')
    xs = x.stride()
    p = L.FlreluActParams(L.ptr(x), L.ptr(s) if s is not None else None, L.dtype_code(x), w, h, c, n,
                          xs[3], xs[2], xs[1], xs[0], (s.shape[3] << 2) if s is not None else 0,
                          s.shape[2] if s is not None else 0, sx, sy, float(gain), float(slope),
                          float(min(clamp, 3.0e38)), 1 if writeSigns else 0, 1 if (read_signs and not writeSigns) else 0)
    L.check(L.get_lib().ide3d_filtered_lrelu_act(C.byref(p), L.stream_ptr(x.device)))
    return so


class _Plugin:
    """What custom_ops.get_plugin() hands back: an object with the pybind module's attributes."""

    def __init__(self, name, **funcs):
        self.__name__ = name
        self.__dict__.update(funcs)


PLUGINS = {
    'bias_act_plugin': _Plugin('bias_act_plugin', bias_act=bias_act, modconv_epilogue=modconv_epilogue,
                                 modconv_epilogue_rgb=modconv_epilogue_rgb),
    'upfirdn2d_plugin': _Plugin('upfirdn2d_plugin', upfirdn2d=upfirdn2d),
    'filtered_lrelu_plugin': _Plugin('filtered_lrelu_plugin', filtered_lrelu=filtered_lrelu,
                                     filtered_lrelu_act_=filtered_lrelu_act_),
}
