"""Filtered leaky ReLU on sm_90a: bias -> up-FIR -> gain*lrelu*clamp -> down-FIR.

Public surface of the reference's torch_utils/ops/filtered_lrelu.py:56 `filtered_lrelu(x, fu, fd, b, up, down,
padding, gain, slope, clamp, flip_filter, impl)`.  The fused plugin call returns `return_code = -1` when it has
no kernel for the configuration; the op then runs the same generic composition the reference uses
(filtered_lrelu.py:223-229): bias add, `upfirdn2d` (gain up^2), `filtered_lrelu_act_` (in place, optional
2-bit sign tensor), `upfirdn2d`.  Gradients re-use the forward with up/down swapped and the stored signs
(reference :239-268).  No CPU path (oracle/ops.py is the CPU restatement for the tests).
"""

import warnings

import numpy as np
import torch

from .. import custom_ops
from . import upfirdn2d

_plugin = None


def _init():
    global _plugin
    if _plugin is None:
        _plugin = custom_ops.get_plugin(module_name='filtered_lrelu_plugin', sources=['filtered_lrelu.cu'])
    return True


def _get_filter_size(f):
    if f is None:
        return 1, 1
    assert isinstance(f, torch.Tensor) and 1 <= f.ndim <= 2
    return f.shape[-1], f.shape[0]   # width, height


def _parse_padding(padding):
    if isinstance(padding, int):
        padding = [padding, padding]
    assert isinstance(padding, (list, tuple)) and all(isinstance(v, (int, np.integer)) for v in padding)
    padding = [int(v) for v in padding]
    if len(padding) == 2:
        px, py = padding
        padding = [px, px, py, py]
    px0, px1, py0, py1 = padding
    return px0, px1, py0, py1


def _forward(x, fu, fd, b, si, sx, sy, up, down, px0, px1, py0, py1, gain, slope, clamp, flip_filter, write_signs):
    """-> (y, signs_out).  Fused kernel when the library has one, generic composition otherwise."""
    dev = x.device
    if fu is None:
        fu = torch.ones([1, 1], dtype=torch.float32, device=dev)
    if fd is None:
        fd = torch.ones([1, 1], dtype=torch.float32, device=dev)
    fu, fd = fu.to(dev), fd.to(dev)
    if up == 1 and fu.ndim == 1 and fu.shape[0] == 1:
        fu = fu.square()[None]
    if down == 1 and fd.ndim == 1 and fd.shape[0] == 1:
        fd = fd.square()[None]
    if b is None:
        b = torch.zeros([x.shape[1]], dtype=x.dtype, device=dev)
    return_code = -1
    if x.dtype in (torch.float16, torch.float32):
        y, so, return_code = _plugin.filtered_lrelu(x, fu, fd, b, si, up, down, px0, px1, py0, py1, sx, sy, gain,
                                                    slope, clamp, flip_filter, write_signs)
    if return_code < 0:
        y = x.add(b.unsqueeze(-1).unsqueeze(-1))
        y = upfirdn2d.upfirdn2d(x=y, f=fu, up=up, padding=[px0, px1, py0, py1], gain=up ** 2, flip_filter=flip_filter)
        so = _plugin.filtered_lrelu_act_(y, si, sx, sy, gain, slope, clamp, write_signs)
        y = upfirdn2d.upfirdn2d(x=y, f=fd, down=down, flip_filter=flip_filter)
    return y, so, fu, fd


class _FilteredLRelu(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, fu, fd, b, si, sx, sy, cfg):
        up, down, px0, px1, py0, py1, gain, slope, clamp, flip_filter = cfg
        write_signs = (si is None) and (x.requires_grad or (b is not None and b.requires_grad))
        strides = [x.stride(i) for i in range(x.ndim) if x.size(i) > 1]
        if any(a < c for a, c in zip(strides[:-1], strides[1:])):
            warnings.warn('low-performance memory layout detected in filtered_lrelu input', RuntimeWarning)
        y, so, fu_used, fd_used = _forward(x, fu, fd, b, si, sx, sy, up, down, px0, px1, py0, py1, gain, slope, clamp,
                                           flip_filter, write_signs)
        ctx.save_for_backward(fu_used, fd_used, si if si is not None else so)
        ctx.cfg, ctx.x_shape, ctx.y_shape, ctx.s_ofs = cfg, x.shape, y.shape, (sx, sy)
        return y

    @staticmethod
    def backward(ctx, dy):
        fu, fd, si = ctx.saved_tensors
        up, down, px0, px1, py0, py1, gain, slope, clamp, flip_filter = ctx.cfg
        _, _, xh, xw = ctx.x_shape
        _, _, yh, yw = ctx.y_shape
        sx, sy = ctx.s_ofs
        dx = db = None
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[3]:
            pp = [(fu.shape[-1] - 1) + (fd.shape[-1] - 1) - px0, xw * up - yw * down + px0 - (up - 1),
                  (fu.shape[0] - 1) + (fd.shape[0] - 1) - py0, xh * up - yh * down + py0 - (up - 1)]
            gg = gain * (up ** 2) / (down ** 2)
            sx = sx - (fu.shape[-1] - 1) + px0
            sy = sy - (fu.shape[0] - 1) + py0
            dx = _FilteredLRelu.apply(dy, fd, fu, None, si, sx, sy,
                                      (down, up, pp[0], pp[1], pp[2], pp[3], gg, slope, float('inf'), not flip_filter))
        if ctx.needs_input_grad[3]:
            db = dx.sum([0, 2, 3])
        return dx, None, None, db, None, None, None, None


def filtered_lrelu(x, fu=None, fd=None, b=None, up=1, down=1, padding=0, gain=np.sqrt(2), slope=0.2, clamp=None,
                   flip_filter=False, impl='cuda'):
    """Filtered leaky ReLU for a batch of 2D images; steps and arguments as in the reference (:56-116)."""
    assert isinstance(x, torch.Tensor)
    assert impl in ['ref', 'cuda']
    if impl == 'ref':
        raise NotImplementedError("ide3d_b200 has no PyTorch reference path; impl='ref' lives in oracle/ops.py (tests only)")
    if x.device.type != 'cuda':
        raise RuntimeError('ide3d_b200.filtered_lrelu: x must be a CUDA tensor (no CPU path in this package)')
    _init()
    assert x.ndim == 4
    assert isinstance(up, int) and up >= 1
    assert isinstance(down, int) and down >= 1
    px0, px1, py0, py1 = _parse_padding(padding)
    assert gain == float(gain) and gain > 0
    assert slope == float(slope) and slope >= 0
    assert clamp is None or (clamp == float(clamp) and clamp >= 0)
    cfg = (up, down, px0, px1, py0, py1, float(gain), float(slope), float(clamp if clamp is not None else 'inf'),
           bool(flip_filter))
    if torch.is_grad_enabled() and (x.requires_grad or (b is not None and b.requires_grad)):
        return _FilteredLRelu.apply(x, fu, fd, b, None, 0, 0, cfg)
    y, _, _, _ = _forward(x, fu, fd, b, None, 0, 0, up, down, px0, px1, py0, py1, cfg[6], cfg[7], cfg[8], cfg[9], False)
    return y
