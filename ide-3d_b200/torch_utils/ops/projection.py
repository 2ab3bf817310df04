"""The projector's own losses on sm_90a (csrc/projector.cu), as autograd functions.

    noise_regularizer(buffers)      the noise regulariser of inversion/training/projectors/w_projector_ide3d.py:113-122, one scalar
                                    over all buffers; ide3d_noise_reg computes it and, in the backward, every buffer's gradient
    noise_normalize_(buffers)       the renormalisation after each optimiser step (:138-142), in place (ide3d_noise_normalize)
    seg_cross_entropy(seg_raw, mask, align_corners=False)   F.cross_entropy(upsample_seg(seg_raw, mask.shape[-2:]), mask) without
                                    the upsampled logits (ide3d_seg_xent_fwd / _bwd); align_corners=True upsamples as BiSeNet does
                                    (ide3d_seg_xent_fwd_ac / _bwd_ac), for encoder fine-tuning

A buffer table the kernels have no specialisation for (a side that is not a power of two up to 512, more than 64 buffers -- the
library answers IDE3D_UNSUPPORTED -- or a buffer that is not a dense fp32 square) runs the reference's torch loop instead.  CUDA
tensors only.
"""

import ctypes as C

import torch

from ... import _lib as L


class _Unsupported(Exception):
    pass


def _dense_square(b):
    return b.dtype == torch.float32 and b.ndim == 2 and b.shape[0] == b.shape[1] and b.is_contiguous()


def _levels(side):
    n = 1
    while side > 8:
        side >>= 1
        n += 1
    return n


def _scratch_floats(sides):
    """include/ide3d_b200.h: 128 floats (one double per buffer) and the pyramid levels above every buffer."""
    return 2 * L.NOISE_MAX_BUFFERS + sum((s >> l) ** 2 for s in sides for l in range(1, _levels(s)))


def _table(buffers, grads=None, scratch=None):
    t = L.NoiseTable()
    t.count = len(buffers)
    for i, b in enumerate(buffers[:L.NOISE_MAX_BUFFERS]):
        t.sides[i], t.bufs[i] = b.shape[0], b.data_ptr()
        if grads is not None:
            t.grads[i] = grads[i].data_ptr()
    if scratch is not None:
        t.scratch, t.scratch_floats = scratch.data_ptr(), scratch.numel()
    return t


def noise_reg_torch(buffers):
    """The reference's loop (w_projector_ide3d.py:113-122): what the kernel computes, for tables it does not take."""
    reg = 0.0
    for v in buffers:
        noise = v[None, None, :, :]
        while True:
            reg += (noise * torch.roll(noise, shifts=1, dims=3)).mean() ** 2
            reg += (noise * torch.roll(noise, shifts=1, dims=2)).mean() ** 2
            if noise.shape[2] <= 8:
                break
            noise = torch.nn.functional.avg_pool2d(noise, kernel_size=2)
    return reg


class _NoiseReg(torch.autograd.Function):
    @staticmethod
    def forward(ctx, *buffers):
        scratch = torch.empty(_scratch_floats([b.shape[0] for b in buffers]), dtype=torch.float32, device=buffers[0].device)
        loss = torch.empty(1, dtype=torch.float32, device=buffers[0].device)
        t = _table(buffers, scratch=scratch)
        rc = L.get_lib().ide3d_noise_reg(C.byref(t), loss.data_ptr(), None, L.stream_ptr(loss.device))
        if rc == L.UNSUPPORTED:
            raise _Unsupported()
        L.check(rc)
        ctx.save_for_backward(*buffers)
        return loss.reshape(())

    @staticmethod
    def backward(ctx, grad_output):
        buffers = ctx.saved_tensors
        grads = [torch.empty_like(b) for b in buffers]
        scratch = torch.empty(_scratch_floats([b.shape[0] for b in buffers]), dtype=torch.float32, device=buffers[0].device)
        scale = grad_output.detach().reshape(1).to(torch.float32).contiguous()
        t = _table(buffers, grads=grads, scratch=scratch)
        L.check(L.get_lib().ide3d_noise_reg(C.byref(t), None, scale.data_ptr(), L.stream_ptr(scale.device)))
        return tuple(g if need else None for g, need in zip(grads, ctx.needs_input_grad))


def noise_regularizer(buffers):
    """Sum over `buffers` (each [side, side]) and their avg-pool pyramids of mean(n * roll(n, 1, W))^2 + mean(n * roll(n, 1, H))^2,
    as a 0-d tensor that back-propagates to every buffer requiring grad.  Two launches forward, one backward."""
    buffers = list(buffers)
    if not buffers:
        raise ValueError('noise_regularizer: no buffers')
    L.require_cuda(*buffers)
    if all(_dense_square(b) for b in buffers):
        try:
            return _NoiseReg.apply(*buffers)
        except _Unsupported:
            pass
    return noise_reg_torch(buffers)


@torch.no_grad()
def noise_normalize_(buffers):
    """buf -= buf.mean(); buf *= buf.square().mean().rsqrt() for every buffer, in place, in one launch."""
    buffers = list(buffers)
    L.require_cuda(*buffers)
    if buffers and all(_dense_square(b) for b in buffers):
        t = _table(buffers)
        rc = L.get_lib().ide3d_noise_normalize(C.byref(t), L.stream_ptr(buffers[0].device))
        if rc != L.UNSUPPORTED:
            L.check(rc)
            return
    for buf in buffers:
        buf -= buf.mean()
        buf *= buf.square().mean().rsqrt()


def _xent_params(seg_raw, mask, lse):
    p = L.SegXentParams()
    p.seg = seg_raw.data_ptr()
    p.n, p.classes, p.in_h, p.in_w = seg_raw.shape
    p.seg_stride_n, p.seg_stride_c, p.seg_stride_h, p.seg_stride_w = seg_raw.stride()
    p.mask, (p.out_h, p.out_w) = mask.data_ptr(), mask.shape[1:]
    p.lse = lse.data_ptr()
    return p


class _SegXent(torch.autograd.Function):
    @staticmethod
    def forward(ctx, seg_raw, mask, align_corners):
        n, h, w = mask.shape
        lse = torch.empty([n, h, w], dtype=torch.float32, device=seg_raw.device)
        partials = torch.empty(n * h, dtype=torch.float64, device=seg_raw.device)
        loss = torch.empty(1, dtype=torch.float32, device=seg_raw.device)
        p = _xent_params(seg_raw, mask, lse)
        p.partials, p.loss = partials.data_ptr(), loss.data_ptr()
        lib = L.get_lib()
        L.check((lib.ide3d_seg_xent_fwd_ac if align_corners else lib.ide3d_seg_xent_fwd)(C.byref(p), L.stream_ptr(seg_raw.device)))
        ctx.save_for_backward(seg_raw, mask, lse)
        ctx.align_corners = align_corners
        return loss.reshape(())

    @staticmethod
    def backward(ctx, grad_output):
        seg_raw, mask, lse = ctx.saved_tensors
        grad = torch.empty(seg_raw.shape, dtype=torch.float32, device=seg_raw.device)
        g = grad_output.detach().reshape(1).to(torch.float32).contiguous()
        p = _xent_params(seg_raw, mask, lse)
        p.grad_loss, p.grad_seg = g.data_ptr(), grad.data_ptr()
        lib = L.get_lib()
        L.check((lib.ide3d_seg_xent_bwd_ac if ctx.align_corners else lib.ide3d_seg_xent_bwd)(C.byref(p), L.stream_ptr(seg_raw.device)))
        return grad, None, None


def seg_cross_entropy(seg_raw, mask, align_corners=False):
    """F.cross_entropy(interpolate(seg_raw, mask.shape[-2:], mode='bilinear', align_corners=align_corners), mask.long()), mean reduction.
    seg_raw float32 [N, C, R, R'] with C <= 32, any strides (the return_seg='raw' view of G.synthesis); mask uint8 [N, H, W] with
    values < C.  The values are not checked here (that would synchronise every call; the projector validates its mask once): the
    kernels read a label >= C as C - 1, where F.cross_entropy would raise."""
    L.require_cuda(seg_raw, mask)
    if seg_raw.dtype != torch.float32 or seg_raw.ndim != 4 or not 1 <= seg_raw.shape[1] <= 32:
        raise RuntimeError(f'seg_cross_entropy: seg_raw must be float32 [N, C <= 32, R, R], got {seg_raw.dtype} {tuple(seg_raw.shape)}')
    if mask.dtype != torch.uint8 or mask.ndim != 3 or mask.shape[0] != seg_raw.shape[0]:
        raise RuntimeError(f'seg_cross_entropy: mask must be uint8 [{seg_raw.shape[0]}, H, W], got {mask.dtype} {tuple(mask.shape)}')
    return _SegXent.apply(seg_raw, mask.contiguous(), bool(align_corners))
