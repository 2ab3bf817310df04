"""The HybridEncoder's geometry stem from a class-id mask (ide3d_seg_stem) and the generator's class ids at image resolution
(ide3d_seg_labels), both csrc/seg_stem.cu.

    seg_stem(mask, stem, conv1, skip)   uint8 [N, H, W] -> (y1 [N, C0, H, W], skip [N, C1, H/2, W/2]), fp32 channels_last: block 0's
                                        conv1 output (what conv2 reads) and its skip branch, for the input one_hot(mask) * 2 - 1.
                                        None when the kernel does not take the shape (IDE3D_UNSUPPORTED): the caller then runs the
                                        composition.
    seg_labels(seg_raw, size)           [N, C, h, w] logits, any strides -> uint8 [N, H, W] class ids of the bilinear upsampling

CUDA tensors only; oracle/edit.py::cpu_edit_ops swaps in torch restatements for the CPU tests.
"""

import ctypes as C

import torch

from ... import _lib as L


def seg_stem(mask, stem, conv1, skip):
    """stem, conv1, skip: the three Conv2dLayer modules (1x1 with bias, 3x3 lrelu with bias, 1x1 down-2 without bias)."""
    L.require_cuda(mask)
    if mask.dtype != torch.uint8 or mask.ndim != 3:
        raise RuntimeError(f'ide3d_b200.seg_stem: mask must be uint8 [N, H, W], got {mask.dtype} {tuple(mask.shape)}')
    n, h, w = mask.shape
    c0, classes = int(stem.weight.shape[0]), int(stem.weight.shape[1])
    c1 = int(skip.weight.shape[0])
    lib = L.get_lib()
    scratch = int(lib.ide3d_seg_stem_scratch_bytes(classes, c0))
    if scratch < 0 or c1 != 2 * c0 or h % 2 or w % 2 or h < 8 or w < 8:
        return None
    dev = mask.device
    f32 = lambda t: t.detach().to(device=dev, dtype=torch.float32).contiguous()
    w0, b0 = f32(stem.weight).reshape(c0, classes), f32(stem.bias)
    w1, b1 = f32(conv1.weight), f32(conv1.bias)
    ws, fir = f32(skip.weight).reshape(c1, c0), f32(skip.resample_filter)
    if fir.shape != (4, 4):
        return None
    tables = torch.empty(scratch // 4, dtype=torch.float32, device=dev)
    y1 = torch.empty([n, h, w, c0], dtype=torch.float32, device=dev)
    sk = torch.empty([n, h // 2, w // 2, c1], dtype=torch.float32, device=dev)
    p = L.SegStemParams()
    p.mask, p.n, p.h, p.w = mask.data_ptr(), n, h, w
    p.mask_stride_n, p.mask_stride_h, p.mask_stride_w = mask.stride()
    p.classes, p.c0, p.c1 = classes, c0, c1
    p.w0, p.b0, p.wg0 = w0.data_ptr(), b0.data_ptr(), float(stem.weight_gain)
    p.w1, p.b1, p.wg1 = w1.data_ptr(), b1.data_ptr(), float(conv1.weight_gain)
    p.ws, p.wgs, p.fir = ws.data_ptr(), float(skip.weight_gain), fir.data_ptr()
    p.tables, p.y1, p.skip = tables.data_ptr(), y1.data_ptr(), sk.data_ptr()
    if L.check(lib.ide3d_seg_stem(C.byref(p), L.stream_ptr(dev)), allow_unsupported=True) == L.UNSUPPORTED:
        return None
    return y1.permute(0, 3, 1, 2), sk.permute(0, 3, 1, 2)


def seg_labels(seg_raw, size):
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
    L.check(L.get_lib().ide3d_seg_labels(C.byref(p), L.stream_ptr(seg_raw.device)))
    return out
