// Per-pixel semantic class of an upsampled logits map, shared by the frame kernels (frames.cu) and the image strips (strips.cu):
// interpolate(mode='bilinear', align_corners=False) of the render-resolution logits evaluated at one output pixel, then the class
// argmax.  Every float operation is explicitly rounded, as the reference's torch ops are, so the upsampled logits never need to exist.
// The template parameter AC selects align_corners=True's source position instead (BiSeNet's upsampling, inversion/BiSeNet.py:249);
// the default keeps every existing caller on align_corners=False.
#pragma once

#include "common.cuh"

namespace ide3d {

// interpolate(mode='bilinear') source position of output index d.  align_corners=False: max(scale * (d + 0.5) - 0.5, 0) with
// scale = in / out; align_corners=True: scale * d with scale = (in - 1) / (out - 1) (0 for out = 1).  i0 = floor, i1 = i0 + 1 clamped
// to the last row / column, l1 = fraction.
struct Tap {
    int i0, i1;
    float l0, l1;
};
template <bool AC = false>
__device__ __forceinline__ Tap bilinear_tap(int d, int in, int out) {
    float s;
    if (AC) {
        const float scale = out > 1 ? __fdiv_rn((float)(in - 1), (float)(out - 1)) : 0.f;
        s = __fmul_rn(scale, (float)d);
    } else {
        const float scale = __fdiv_rn((float)in, (float)out);
        s = __fsub_rn(__fmul_rn(scale, __fadd_rn((float)d, 0.5f)), 0.5f);
        s = s < 0.f ? 0.f : s;
    }
    Tap t;
    t.i0 = (int)s;
    t.i1 = t.i0 + (t.i0 < in - 1 ? 1 : 0);
    t.l1 = __fsub_rn(s, (float)t.i0);
    t.l0 = __fsub_rn(1.f, t.l1);
    return t;
}

// Class of output pixel (x, y) of an out_h x out_w image from the logits s [classes, in_h, in_w] (element strides sc, sh, sw):
// v = h0 * (w0 * v00 + w1 * v01) + h1 * (w0 * v10 + w1 * v11) per class, first maximum wins, NaN counts as maximal (torch.argmax).
template <bool AC = false>
__device__ __forceinline__ int seg_class_at(const float* s, int classes, int in_h, int in_w, long long sc, long long sh, long long sw,
                                            int x, int y, int out_h, int out_w) {
    const Tap ty = bilinear_tap<AC>(y, in_h, out_h), tx = bilinear_tap<AC>(x, in_w, out_w);
    const float* r0 = s + ty.i0 * sh;
    const float* r1 = s + ty.i1 * sh;
    const long long c0 = tx.i0 * sw, c1 = tx.i1 * sw;
    float best = 0.f;
    int arg = 0;
    for (int k = 0; k < classes; ++k) {
        const long long kc = k * sc;
        const float top = __fadd_rn(__fmul_rn(tx.l0, __ldg(r0 + kc + c0)), __fmul_rn(tx.l1, __ldg(r0 + kc + c1)));
        const float bot = __fadd_rn(__fmul_rn(tx.l0, __ldg(r1 + kc + c0)), __fmul_rn(tx.l1, __ldg(r1 + kc + c1)));
        const float v = __fadd_rn(__fmul_rn(ty.l0, top), __fmul_rn(ty.l1, bot));
        if (k == 0 || v > best || (v != v && best == best)) { best = v; arg = k; }
    }
    return arg;
}

// The taps of output pixel (x, y) and the logit of one class there, with seg_class_at's arithmetic (projector.cu's cross-entropy
// evaluates one class at a time from these).
struct SegTaps {
    const float *r0, *r1;
    long long c0, c1;
    Tap tx, ty;
};
template <bool AC = false>
__device__ __forceinline__ SegTaps seg_taps_at(const float* s, int in_h, int in_w, long long sh, long long sw, int x, int y, int out_h,
                                               int out_w) {
    SegTaps t;
    t.ty = bilinear_tap<AC>(y, in_h, out_h);
    t.tx = bilinear_tap<AC>(x, in_w, out_w);
    t.r0 = s + t.ty.i0 * sh;
    t.r1 = s + t.ty.i1 * sh;
    t.c0 = t.tx.i0 * sw;
    t.c1 = t.tx.i1 * sw;
    return t;
}
__device__ __forceinline__ float seg_logit_at(const SegTaps& t, long long kc) {
    const float top = __fadd_rn(__fmul_rn(t.tx.l0, __ldg(t.r0 + kc + t.c0)), __fmul_rn(t.tx.l1, __ldg(t.r0 + kc + t.c1)));
    const float bot = __fadd_rn(__fmul_rn(t.tx.l0, __ldg(t.r1 + kc + t.c0)), __fmul_rn(t.tx.l1, __ldg(t.r1 + kc + t.c1)));
    return __fadd_rn(__fmul_rn(t.ty.l0, top), __fmul_rn(t.ty.l1, bot));
}

}  // namespace ide3d
