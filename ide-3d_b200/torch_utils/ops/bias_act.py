"""Fused bias + activation (+ gain, clamp) on sm_90a.

Same public surface as the reference's torch_utils/ops/bias_act.py: `activation_funcs` (:21-31) and
`bias_act(x, b=None, dim=1, act='linear', alpha=None, gain=None, clamp=None, impl='cuda')` (:52).
Compute goes through `bias_act_plugin.bias_act` -> ide3d_bias_act (csrc/bias_act.cu).  There is no
PyTorch fallback in this package: CPU tensors and impl='ref' raise (the CPU restatement is oracle/ops.py,
test infrastructure only).
"""

import math

import torch

from .. import custom_ops


class _Spec(dict):
    __getattr__ = dict.__getitem__


def _spec(def_alpha, def_gain, cuda_idx, ref, has_2nd_grad):
    return _Spec(def_alpha=def_alpha, def_gain=def_gain, cuda_idx=cuda_idx, ref=ref, has_2nd_grad=has_2nd_grad)


_SQRT2 = math.sqrt(2)
activation_funcs = {
    'linear':   _spec(0,   1,      1, '',  False),
    'relu':     _spec(0,   _SQRT2, 2, 'y', False),
    'lrelu':    _spec(0.2, _SQRT2, 3, 'y', False),
    'tanh':     _spec(0,   1,      4, 'y', True),
    'sigmoid':  _spec(0,   1,      5, 'y', True),
    'elu':      _spec(0,   1,      6, 'y', True),
    'selu':     _spec(0,   1,      7, 'y', True),
    'softplus': _spec(0,   1,      8, 'y', True),
    'swish':    _spec(0,   _SQRT2, 9, 'x', True),
}

_plugin = None


def _init():
    global _plugin
    if _plugin is None:
        _plugin = custom_ops.get_plugin(module_name='bias_act_plugin', sources=['bias_act.cu'])
    return True


def _layout(x):
    """Tensor in a dense layout the kernel accepts (contiguous or channels_last), like bias_act.py:145-146."""
    if x.ndim == 4 and x.is_contiguous(memory_format=torch.channels_last):
        return x
    return x.contiguous()


class _BiasAct(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, b, dim, spec, alpha, gain, clamp):
        x = _layout(x)
        y = _plugin.bias_act(x, b, None, None, None, 0, dim, spec.cuda_idx, alpha, gain, clamp)
        ctx.cfg = (dim, spec, alpha, gain, clamp)
        ctx.has_bias = b is not None
        ctx.cl = (x.ndim == 4 and not x.is_contiguous())
        ctx.save_for_backward(x if 'x' in spec.ref or spec.has_2nd_grad else None, b if b is not None else None,
                              y if 'y' in spec.ref else None)
        return y

    @staticmethod
    def backward(ctx, dy):
        dim, spec, alpha, gain, clamp = ctx.cfg
        x, b, y = ctx.saved_tensors
        dx = db = None
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
            dy = dy.contiguous(memory_format=torch.channels_last) if ctx.cl else dy.contiguous()
            dx = dy
            if spec.cuda_idx != 1 or gain != 1 or clamp >= 0:
                dx = _BiasActGrad.apply(dy, x, b, y, dim, spec, alpha, gain, clamp)
        if ctx.needs_input_grad[1] and ctx.has_bias:
            db = dx.sum([i for i in range(dx.ndim) if i != dim])
        return dx, db, None, None, None, None, None


class _BiasActGrad(torch.autograd.Function):
    """dx = dy * gain * act'(x + b) (grad=1 kernel); its own backward uses the grad=2 kernel for the second-order term, so
    double backward (R1 / path-length regularisers) is exact -- the reference's BiasActCudaGrad, bias_act.py:178-203."""

    @staticmethod
    def forward(ctx, dy, x, b, y, dim, spec, alpha, gain, clamp):
        ctx.cfg = (dim, spec, alpha, gain, clamp)
        ctx.cl = (dy.ndim == 4 and not dy.is_contiguous())
        dx = _plugin.bias_act(dy, b, x, y, None, 1, dim, spec.cuda_idx, alpha, gain, clamp)
        ctx.save_for_backward(dy if spec.has_2nd_grad else None, x, b, y)
        return dx

    @staticmethod
    def backward(ctx, d_dx):
        dim, spec, alpha, gain, clamp = ctx.cfg
        d_dx = d_dx.contiguous(memory_format=torch.channels_last) if ctx.cl else d_dx.contiguous()
        dy, x, b, y = ctx.saved_tensors
        d_dy = d_x = d_b = None
        if ctx.needs_input_grad[0]:
            d_dy = _BiasActGrad.apply(d_dx, x, b, y, dim, spec, alpha, gain, clamp)
        if spec.has_2nd_grad and (ctx.needs_input_grad[1] or ctx.needs_input_grad[2]):
            d_x = _plugin.bias_act(d_dx, b, x, y, dy, 2, dim, spec.cuda_idx, alpha, gain, clamp)
        if spec.has_2nd_grad and ctx.needs_input_grad[2]:
            d_b = d_x.sum([i for i in range(d_x.ndim) if i != dim])
        return d_dy, d_x, d_b, None, None, None, None, None, None


def bias_act(x, b=None, dim=1, act='linear', alpha=None, gain=None, clamp=None, impl='cuda'):
    """y = clamp(gain * act(x + b)).  Arguments as in the reference (bias_act.py:52-86)."""
    assert isinstance(x, torch.Tensor)
    assert impl in ['ref', 'cuda']
    if impl == 'ref':
        raise NotImplementedError("ide3d_b200 has no PyTorch reference path; impl='ref' lives in oracle/ops.py (tests only)")
    if x.device.type != 'cuda':
        raise RuntimeError('ide3d_b200.bias_act: x must be a CUDA tensor (no CPU path in this package)')
    _init()
    assert clamp is None or clamp >= 0
    spec = activation_funcs[act]
    alpha = float(alpha if alpha is not None else spec.def_alpha)
    gain = float(gain if gain is not None else spec.def_gain)
    clamp = float(clamp if clamp is not None else -1)
    if b is not None:
        assert isinstance(b, torch.Tensor) and b.ndim == 1
        assert 0 <= dim < x.ndim
        assert b.shape[0] == x.shape[dim]
    # identity short-cut of the reference (bias_act.py:149)
    if act == 'linear' and gain == 1 and clamp < 0 and b is None:
        return x
    if torch.is_grad_enabled() and (x.requires_grad or (b is not None and b.requires_grad)):
        return _BiasAct.apply(x, b, dim, spec, alpha, gain, clamp)
    return _plugin.bias_act(_layout(x), b, None, None, None, 0, dim, spec.cuda_idx, alpha, gain, clamp)


def scaled_bias_act(x, scale=None, noise=None, b=None, act='linear', alpha=None, gain=None, clamp=None, next_scale=None,
                    only_next=False, emit_y=True, y_scale=None, rgb=None, out_dtype=None, fp32_tail=False):
    """Extension: ``bias_act(fma(x, scale[:, :, None, None], noise), b, act=...)`` -- the tail of an activation-scaled
    modulated convolution (inversion/networks.py:104-105 then :512) -- as ONE sm_90a pass when nothing needs a gradient;
    otherwise exactly that composition of the two reference ops (so autograd behaves as in the reference).
    x [N,C,H,W]; scale [N,C] (demodulation coefficients) | None; noise broadcastable [.,1,H,W] | None; b [C] | None.
    next_scale [N,C]: additionally return ``y * next_scale[:, :, None, None]`` (the style modulation that opens the next
    modulated convolution, :100) -> (y, y_next); with only_next just y_next.
    Further consumers folded into the same pass: emit_y=False drops y (as only_next), y_scale [N,C] returns ``y * y_scale``
    in place of y (the next block's first modulation), rgb=(weight [O,C,1,1], styles [N,C], bias [O] | None) adds the ToRGB
    output ``conv1x1(y * styles, weight) + bias`` as a dense NCHW tensor (ToRGBLayer, :700-707).  With any of these the
    result is the list of the requested outputs in the order (y, y2, rgb).
    out_dtype=torch.float16 (float32 x, without the folded consumers): y / y2 rounded once to fp16 -- the input of an fp16
    convolution.  fp32_tail (float16 x, the output of such a convolution, with folded consumers): scale, noise, b and the
    styles stay float32 and so does the arithmetic; y / y2 are fp16, each rounded once."""
    from . import fma
    if x.device.type != 'cuda':
        raise RuntimeError('ide3d_b200.scaled_bias_act: x must be a CUDA tensor (no CPU path in this package)')
    _init()
    if rgb is not None or y_scale is not None or not emit_y:
        assert out_dtype is None
        return _scaled_bias_act_fold(x, scale, noise, b, act, alpha, gain, clamp, next_scale, emit_y and not only_next, y_scale, rgb,
                                     fp32_tail)
    assert not fp32_tail, 'fp32_tail needs a folded consumer (y_scale, rgb or emit_y=False)'
    spec = activation_funcs[act]
    needs_grad = torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (x, scale, noise, b, next_scale))
    if not needs_grad and x.ndim == 4:
        out = _plugin.modconv_epilogue(_layout(x), scale, noise, b, spec.cuda_idx, float(alpha if alpha is not None else spec.def_alpha),
                                       float(gain if gain is not None else spec.def_gain), float(clamp if clamp is not None else -1),
                                       next_scale=next_scale, only_next=only_next, out_dtype=out_dtype)
        if out is not None:
            return out
    if out_dtype is not None and out_dtype != x.dtype:
        out = scaled_bias_act(x, scale, noise, b, act=act, alpha=alpha, gain=gain, clamp=clamp, next_scale=next_scale, only_next=only_next)
        return out.to(out_dtype) if isinstance(out, torch.Tensor) else tuple(t.to(out_dtype) for t in out)
    if scale is not None and noise is not None:
        x = fma.fma(x, scale.to(x.dtype).reshape(x.shape[0], -1, 1, 1), noise.to(x.dtype))
    elif scale is not None:
        x = x * scale.to(x.dtype).reshape(x.shape[0], -1, 1, 1)
    elif noise is not None:
        x = x + noise.to(x.dtype)
    y = bias_act(x, None if b is None else b.to(x.dtype), act=act, alpha=alpha, gain=gain, clamp=clamp)
    if next_scale is None:
        return y
    y2 = y * next_scale.to(y.dtype).reshape(y.shape[0], -1, 1, 1)
    return y2 if only_next else (y, y2)


def _scaled_bias_act_fold(x, scale, noise, b, act, alpha, gain, clamp, next_scale, emit_y, y_scale, rgb, fp32_tail=False):
    """`scaled_bias_act` with its consumers folded in: one `ide3d_modconv_epilogue_rgb` pass for channels_last float32 / float16 x;
    for anything else (gradients, other layouts / dtypes / widths) today's composition -- the epilogue, the products with the
    styles and, for rgb, the cuDNN 1x1 convolution followed by the bias."""
    from . import conv2d_resample
    spec = activation_funcs[act]
    alpha = float(alpha if alpha is not None else spec.def_alpha)
    gain = float(gain if gain is not None else spec.def_gain)
    clamp_f = float(clamp if clamp is not None else -1)
    needs_grad = torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (x, scale, noise, b, next_scale, y_scale, *(rgb or ())))
    if not needs_grad and x.ndim == 4:
        out = _plugin.modconv_epilogue_rgb(x, scale, noise, b, spec.cuda_idx, alpha, gain, clamp_f, emit_y=emit_y, y_scale=y_scale,
                                           next_scale=next_scale, rgb=rgb, fp32_tail=fp32_tail)
        if out is not None:
            return out
    if fp32_tail and x.dtype != torch.float32:              # the same tail composed in float32, fp16 outputs rounded once
        out = _scaled_bias_act_fold(x.float(), scale, noise, b, act, alpha, gain, clamp, next_scale, emit_y, y_scale, rgb)
        n_x = int(emit_y) + int(next_scale is not None)
        return [t.to(x.dtype) if i < n_x else t for i, t in enumerate(out)]
    y = scaled_bias_act(x, scale, noise, b, act=act, alpha=alpha, gain=gain, clamp=clamp)
    mod = lambda s: y * s.to(y.dtype).reshape(y.shape[0], -1, 1, 1)
    out = []
    if emit_y:
        out.append(y if y_scale is None else mod(y_scale))
    if next_scale is not None:
        out.append(mod(next_scale))
    if rgb is not None:
        weight, styles, bias = rgb
        r = conv2d_resample.conv2d_resample(x=mod(styles), w=weight.to(y.dtype))
        r = bias_act(r, None if bias is None else bias.to(r.dtype))
        out.append(r.contiguous())
    return out
