"""The HybridEncoder's geometry stem from a class-id mask (ide3d_seg_stem, ide3d_seg_stem_bwd) and class ids at image resolution
(ide3d_seg_labels, ide3d_seg_labels_ac), all csrc/seg_stem.cu.

    seg_stem(mask, stem, conv1, skip)   uint8 [N, H, W] -> (y1 [N, C0, H, W], skip [N, C1, H/2, W/2]), fp32 channels_last: block 0's
                                        conv1 output (what conv2 reads) and its skip branch, for the input one_hot(mask) * 2 - 1.
                                        Differentiable w.r.t. the three layers' weights and biases (the mask is not): the backward is
                                        ide3d_seg_stem_bwd.  `stem` is anything with weight, bias and weight_gain (the encoder passes a
                                        re-parameterised stem for a {0, 1} one-hot).  None when the kernel does not take the shape
                                        (IDE3D_UNSUPPORTED): the caller then runs the composition.
    seg_labels(seg_raw, size, align_corners=False)   [N, C, h, w] logits, any strides -> uint8 [N, H, W] class ids of the bilinear
                                        upsampling (align_corners=True: BiSeNet's rule)

CUDA tensors only; oracle/edit.py::cpu_edit_ops swaps in torch restatements for the CPU tests.
"""

import ctypes as C

import torch

from ... import _lib as L


def _stem_params(mask, w0, b0, w1, b1, ws, fir, gains, tables):
    p = L.SegStemParams()
    p.mask, (p.n, p.h, p.w) = mask.data_ptr(), mask.shape
    p.mask_stride_n, p.mask_stride_h, p.mask_stride_w = mask.stride()
    p.classes, p.c0, p.c1 = w0.shape[1], w0.shape[0], ws.shape[0]
    p.w0, p.b0, p.wg0 = w0.data_ptr(), b0.data_ptr(), gains[0]
    p.w1, p.b1, p.wg1 = w1.data_ptr(), b1.data_ptr(), gains[1]
    p.ws, p.wgs, p.fir = ws.data_ptr(), gains[2], fir.data_ptr()
    p.tables = tables.data_ptr()
    return p


class _SegStem(torch.autograd.Function):
    """(mask, w0 [C0, K], b0, w1 [C0, C0, 3, 3], b1, ws [C1, C0], fir, gains) -> (y1, skip) channels_last [N, H, W, C]."""

    @staticmethod
    def forward(ctx, mask, w0, b0, w1, b1, ws, fir, gains):
        n, h, w = mask.shape
        c0, c1, dev = w0.shape[0], ws.shape[0], mask.device
        lib = L.get_lib()
        tables = torch.empty(int(lib.ide3d_seg_stem_scratch_bytes(w0.shape[1], c0)) // 4, dtype=torch.float32, device=dev)
        y1 = torch.empty([n, h, w, c0], dtype=torch.float32, device=dev)
        sk = torch.empty([n, h // 2, w // 2, c1], dtype=torch.float32, device=dev)
        p = _stem_params(mask, w0, b0, w1, b1, ws, fir, gains, tables)
        p.y1, p.skip = y1.data_ptr(), sk.data_ptr()
        L.check(lib.ide3d_seg_stem(C.byref(p), L.stream_ptr(dev)))
        ctx.save_for_backward(mask, w0, b0, w1, b1, ws, fir, tables)
        ctx.gains = gains
        return y1, sk

    @staticmethod
    def backward(ctx, g_y1, g_skip):
        mask, w0, b0, w1, b1, ws, fir, tables = ctx.saved_tensors
        n, h, w = mask.shape
        lib = L.get_lib()
        grads = [torch.empty_like(t) for t in (w0, b0, w1, b1, ws)]
        scratch = torch.empty(int(lib.ide3d_seg_stem_bwd_scratch_bytes(n, h, w, w0.shape[1], w0.shape[0])), dtype=torch.uint8,
                              device=mask.device)
        g_y1, g_skip = g_y1.float().contiguous(), g_skip.float().contiguous()
        p = L.SegStemBwdParams()
        p.fwd = _stem_params(mask, w0, b0, w1, b1, ws, fir, ctx.gains, tables)
        p.grad_y1, p.grad_skip = g_y1.data_ptr(), g_skip.data_ptr()
        p.grad_w0, p.grad_b0, p.grad_w1, p.grad_b1, p.grad_ws = (g.data_ptr() for g in grads)
        p.scratch, p.scratch_bytes = scratch.data_ptr(), scratch.numel()
        L.check(lib.ide3d_seg_stem_bwd(C.byref(p), L.stream_ptr(mask.device)))
        return (None, *(g if need else None for g, need in zip(grads, ctx.needs_input_grad[1:6])), None, None)


def seg_stem(mask, stem, conv1, skip):
    """stem, conv1, skip: the three Conv2dLayer modules (1x1 with bias, 3x3 lrelu with bias, 1x1 down-2 without bias)."""
    L.require_cuda(mask)
    if mask.dtype != torch.uint8 or mask.ndim != 3:
        raise RuntimeError(f'ide3d_b200.seg_stem: mask must be uint8 [N, H, W], got {mask.dtype} {tuple(mask.shape)}')
    n, h, w = mask.shape
    c0, classes = int(stem.weight.shape[0]), int(stem.weight.shape[1])
    c1 = int(skip.weight.shape[0])
    if int(L.get_lib().ide3d_seg_stem_scratch_bytes(classes, c0)) < 0 or c1 != 2 * c0 or h % 2 or w % 2 or h < 8 or w < 8:
        return None
    if tuple(skip.resample_filter.shape) != (4, 4):
        return None
    dev = mask.device
    f32 = lambda t: t.to(device=dev, dtype=torch.float32).contiguous()
    gains = (float(stem.weight_gain), float(conv1.weight_gain), float(skip.weight_gain))
    y1, sk = _SegStem.apply(mask, f32(stem.weight).reshape(c0, classes), f32(stem.bias), f32(conv1.weight), f32(conv1.bias),
                            f32(skip.weight).reshape(c1, c0), f32(skip.resample_filter).detach(), gains)
    return y1.permute(0, 3, 1, 2), sk.permute(0, 3, 1, 2)


def seg_labels(seg_raw, size, align_corners=False):
    L.require_cuda(seg_raw)
    if seg_raw.dtype != torch.float32 or seg_raw.ndim != 4:
        raise RuntimeError(f'ide3d_b200.seg_labels: logits must be float32 [N, C, h, w], got {seg_raw.dtype} {tuple(seg_raw.shape)}')
    out_h, out_w = size
    n, c, ih, iw = seg_raw.shape
    out = torch.empty([n, out_h, out_w], dtype=torch.uint8, device=seg_raw.device)
    p = L.SegLabelsParams()
    p.seg, p.n, p.classes, p.in_h, p.in_w = seg_raw.data_ptr(), n, c, ih, iw
    p.seg_stride_n, p.seg_stride_c, p.seg_stride_h, p.seg_stride_w = seg_raw.stride()
    p.out_h, p.out_w, p.out = out_h, out_w, out.data_ptr()
    lib = L.get_lib()
    L.check((lib.ide3d_seg_labels_ac if align_corners else lib.ide3d_seg_labels)(C.byref(p), L.stream_ptr(seg_raw.device)))
    return out
