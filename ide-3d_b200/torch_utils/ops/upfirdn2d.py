"""upfirdn2d family on sm_90a: pad -> zero-upsample -> FIR -> decimate.

Public surface of the reference's torch_utils/ops/upfirdn2d.py: `setup_filter` (:70), `upfirdn2d` (:118),
`filter2d` (:277), `upsample2d` (:313), `downsample2d` (:352) -- same arguments and semantics.  Compute
goes through `upfirdn2d_plugin.upfirdn2d` -> ide3d_upfirdn2d (csrc/upfirdn2d.cu).  No CPU path here
(oracle/ops.py holds the CPU restatement for the tests).
"""

import numpy as np
import torch

from .. import custom_ops

_plugin = None


def _init():
    global _plugin
    if _plugin is None:
        _plugin = custom_ops.get_plugin(module_name='upfirdn2d_plugin', sources=['upfirdn2d.cu'])
    return True


def _parse_scaling(scaling):
    if isinstance(scaling, int):
        scaling = [scaling, scaling]
    assert isinstance(scaling, (list, tuple)) and all(isinstance(v, int) for v in scaling)
    sx, sy = scaling
    assert sx >= 1 and sy >= 1
    return sx, sy


def _parse_padding(padding):
    if isinstance(padding, int):
        padding = [padding, padding]
    assert isinstance(padding, (list, tuple)) and all(isinstance(v, int) for v in padding)
    if len(padding) == 2:
        px, py = padding
        padding = [px, px, py, py]
    px0, px1, py0, py1 = padding
    return px0, px1, py0, py1


def _get_filter_size(f):
    if f is None:
        return 1, 1
    assert isinstance(f, torch.Tensor) and f.ndim in [1, 2]
    fw, fh = int(f.shape[-1]), int(f.shape[0])
    assert fw >= 1 and fh >= 1
    return fw, fh


def setup_filter(f, device=torch.device('cpu'), normalize=True, flip_filter=False, gain=1, separable=None):
    """Prepare a 2D FIR filter for `upfirdn2d()`: 1-D taps with < 8 entries become an outer product, the
    DC gain is normalised to 1, `gain` is split over the dimensions (reference :70-115)."""
    if f is None:
        f = 1
    f = torch.as_tensor(f, dtype=torch.float32)
    assert f.ndim in [0, 1, 2] and f.numel() > 0
    if f.ndim == 0:
        f = f[np.newaxis]
    if separable is None:
        separable = (f.ndim == 1 and f.numel() >= 8)
    if f.ndim == 1 and not separable:
        f = f.ger(f)
    assert f.ndim == (1 if separable else 2)
    if normalize:
        f = f / f.sum()
    if flip_filter:
        f = f.flip(list(range(f.ndim)))
    f = f * (gain ** (f.ndim / 2))
    return f.to(device=device)


def _run(x, f, upx, upy, downx, downy, px0, px1, py0, py1, flip, gain):
    """One or two plugin calls: a 1-D filter is applied along x, then along y (reference :243-245)."""
    if f is None:
        f = torch.ones([1, 1], dtype=torch.float32, device=x.device)
    if f.ndim == 1 and f.shape[0] == 1:
        f = f.square().unsqueeze(0)                  # 1 tap separable == 1x1 full filter
    assert f.dtype == torch.float32 and f.ndim in [1, 2]
    if f.device != x.device:
        f = f.to(x.device)
    if f.ndim == 2:
        return _plugin.upfirdn2d(x, f, upx, upy, downx, downy, px0, px1, py0, py1, flip, gain)
    y = _plugin.upfirdn2d(x, f.unsqueeze(0), upx, 1, downx, 1, px0, px1, 0, 0, flip, 1.0)
    return _plugin.upfirdn2d(y, f.unsqueeze(1), 1, upy, 1, downy, 0, 0, py0, py1, flip, gain)


class _Upfirdn2d(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, f, cfg):
        upx, upy, downx, downy, px0, px1, py0, py1, flip, gain = cfg
        y = _run(x, f, upx, upy, downx, downy, px0, px1, py0, py1, flip, gain)
        ctx.save_for_backward(f)
        ctx.cfg = cfg
        ctx.x_shape = x.shape
        return y

    @staticmethod
    def backward(ctx, dy):
        (f,) = ctx.saved_tensors
        upx, upy, downx, downy, px0, px1, py0, py1, flip, gain = ctx.cfg
        _, _, ih, iw = ctx.x_shape
        _, _, oh, ow = dy.shape
        fw, fh = _get_filter_size(f)
        # adjoint = same op with up/down swapped, flipped filter and complementary padding (reference :251-266)
        p = (fw - px0 - 1, iw * upx - ow * downx + px0 - upx + 1, fh - py0 - 1, ih * upy - oh * downy + py0 - upy + 1)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = _Upfirdn2d.apply(dy, f, (downx, downy, upx, upy, p[0], p[1], p[2], p[3], (not flip), gain))
        return dx, None, None


def upfirdn2d(x, f, up=1, down=1, padding=0, flip_filter=False, gain=1, impl='cuda'):
    """Pad, upsample, filter and downsample a batch of 2D images (reference :118-162)."""
    assert isinstance(x, torch.Tensor)
    assert impl in ['ref', 'cuda']
    if impl == 'ref':
        raise NotImplementedError("ide3d_b200 has no PyTorch reference path; impl='ref' lives in oracle/ops.py (tests only)")
    if x.device.type != 'cuda':
        raise RuntimeError('ide3d_b200.upfirdn2d: x must be a CUDA tensor (no CPU path in this package)')
    _init()
    upx, upy = _parse_scaling(up)
    downx, downy = _parse_scaling(down)
    px0, px1, py0, py1 = _parse_padding(padding)
    cfg = (upx, upy, downx, downy, px0, px1, py0, py1, bool(flip_filter), float(gain))
    if torch.is_grad_enabled() and x.requires_grad:
        return _Upfirdn2d.apply(x, f, cfg)
    return _run(x, f, *cfg)


def filter2d(x, f, padding=0, flip_filter=False, gain=1, impl='cuda'):
    """Filter with `f`, output the same size as the input (reference :277-309)."""
    px0, px1, py0, py1 = _parse_padding(padding)
    fw, fh = _get_filter_size(f)
    p = [px0 + fw // 2, px1 + (fw - 1) // 2, py0 + fh // 2, py1 + (fh - 1) // 2]
    return upfirdn2d(x, f, padding=p, flip_filter=flip_filter, gain=gain, impl=impl)


def upsample2d(x, f, up=2, padding=0, flip_filter=False, gain=1, impl='cuda'):
    """Upsample by an integer factor; output is `up` times the input size (reference :313-348)."""
    upx, upy = _parse_scaling(up)
    px0, px1, py0, py1 = _parse_padding(padding)
    fw, fh = _get_filter_size(f)
    p = [px0 + (fw + upx - 1) // 2, px1 + (fw - upx) // 2, py0 + (fh + upy - 1) // 2, py1 + (fh - upy) // 2]
    return upfirdn2d(x, f, up=up, padding=p, flip_filter=flip_filter, gain=gain * upx * upy, impl=impl)


def upfirdn2d_epilogue(x, f, padding=0, gain=1, flip_filter=False, scale=None, noise=None, b=None, act='linear', alpha=None,
                       act_gain=None, clamp=None, next_scale=None, only_next=False, fp32_tail=False):
    """Extension: ``bias_act.scaled_bias_act(upfirdn2d(x, f, padding=padding, gain=gain), scale, noise, b, ...)`` -- what
    follows the transposed convolution of an up=2 SynthesisLayer (conv2d_resample.py:125; inversion/networks.py:104-105, :512)
    -- as one pass when x is channels_last (C % 4 == 0), f is the 4x4 filter and nothing needs a gradient; otherwise that
    composition.  Returns y, (y, y_next) or y_next like `scaled_bias_act`.
    fp32_tail (float16 x, the output of an fp16 convolution): the FIR and the tail run in float32 with float32 scale / noise / b /
    next_scale; the outputs are fp16, each rounded once."""
    from . import bias_act
    if x.device.type != 'cuda':
        raise RuntimeError('ide3d_b200.upfirdn2d_epilogue: x must be a CUDA tensor (no CPU path in this package)')
    _init()
    spec = bias_act.activation_funcs[act]
    needs_grad = torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (x, scale, noise, b, next_scale))
    if not needs_grad and f is not None and f.ndim == 2 and spec.cuda_idx in (1, 3):
        px0, px1, py0, py1 = _parse_padding(padding)
        e = dict(scale=scale, noise=noise, b=b, act=spec.cuda_idx, alpha=float(alpha if alpha is not None else spec.def_alpha),
                 gain=float(act_gain if act_gain is not None else spec.def_gain), clamp=float(clamp if clamp is not None else -1),
                 next_scale=next_scale, only_next=only_next, fp32_tail=fp32_tail)
        out = _plugin.upfirdn2d(x, f.to(x.device), 1, 1, 1, 1, px0, px1, py0, py1, bool(flip_filter), float(gain), epilogue=e)
        if out is not None:
            return out
    y = upfirdn2d(x.float() if fp32_tail else x, f, padding=padding, gain=gain, flip_filter=flip_filter)
    return bias_act.scaled_bias_act(y, scale=scale, noise=noise, b=b, act=act, alpha=alpha, gain=act_gain, clamp=clamp,
                                    next_scale=next_scale, only_next=only_next, out_dtype=x.dtype if fp32_tail else None)


def upsample2d_add(x, f, y, b=None, up=2):
    """Extension: ``upsample2d(x, f, up) + y + b[None, :, None, None]`` -- the skip-connection step of a 'skip' synthesis
    block (inversion/networks.py:841-844, with the ToRGB bias of :707 folded in).  One pass when x is channels_last with
    C % 4 == 0, f is the 2-D 4x4 filter, y has stride_c == 1 and nothing needs a gradient; otherwise the composition of the
    reference ops (``y`` is then not modified).  y may be float16 on float32 x (the output of an fp16 1x1 convolution)."""
    if x.device.type != 'cuda':
        raise RuntimeError('ide3d_b200.upsample2d_add: x must be a CUDA tensor (no CPU path in this package)')
    _init()
    needs_grad = torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (x, y, b))
    if not needs_grad and f is not None and f.ndim == 2 and (y.dtype == x.dtype or (y.dtype == torch.float16 and x.dtype == torch.float32)):
        upx, upy = _parse_scaling(up)
        fw, fh = _get_filter_size(f)
        p = [(fw + upx - 1) // 2, (fw - upx) // 2, (fh + upy - 1) // 2, (fh - upy) // 2]
        out = _plugin.upfirdn2d(x, f.to(x.device), upx, upy, 1, 1, p[0], p[1], p[2], p[3], False, float(upx * upy), add=y, bias=b)
        if out is not None:
            return out
    out = upsample2d(x, f, up=up) + y
    return out if b is None else out + b.to(out.dtype).reshape(1, -1, 1, 1)


def downsample2d(x, f, down=2, padding=0, flip_filter=False, gain=1, impl='cuda'):
    """Downsample by an integer factor; output is 1/`down` of the input size (reference :352-387)."""
    downx, downy = _parse_scaling(down)
    px0, px1, py0, py1 = _parse_padding(padding)
    fw, fh = _get_filter_size(f)
    p = [px0 + (fw - downx + 1) // 2, px1 + (fw - downx) // 2, py0 + (fh - downy + 1) // 2, py1 + (fh - downy) // 2]
    return upfirdn2d(x, f, down=down, padding=p, flip_filter=flip_filter, gain=gain, impl=impl)
