// The two parts of a projection step (inversion/training/projectors/w_projector_ide3d.py) that are not the generator:
//   ide3d_noise_reg / ide3d_noise_normalize  the noise regulariser (:113-122) with its gradient, and the renormalisation (:138-142),
//                                            over the whole table of noise buffers in a fixed number of launches (the reference walks
//                                            an avg-pool pyramid per buffer: a few hundred small torch kernels per step);
//   ide3d_seg_xent_fwd / _bwd                the semantic-mask loss (extension): cross-entropy of the bilinearly upsampled logits,
//                                            evaluated per output pixel from the render-resolution logits (seg_common.cuh);
//                                            _fwd_ac / _bwd_ac are the same kernels with align_corners=True (BiSeNet's upsampling).
// Every reduction runs in a fixed order (per-thread strides, then a shuffle / shared-memory tree): no float atomics, bit-reproducible.
#include "seg_common.cuh"

namespace ide3d {

constexpr int kNoiseThreads = 1024;
constexpr int kNoiseMaxSide = 512;
constexpr int kNoiseMaxLevels = 8;          // 512 -> 8: seven levels
constexpr int kXentThreads = 256;

// Sum of one double per thread over the block, in a fixed order.  Every thread of the block calls it; every thread gets the sum.
template <int kThreads>
__device__ __forceinline__ double block_sum(double v, double* red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) red[warp] = v;
    __syncthreads();
    if (warp == 0) {
        v = lane < kThreads / 32 ? red[lane] : 0.0;
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
        if (lane == 0) red[32] = v;
    }
    __syncthreads();
    const double s = red[32];
    __syncthreads();                          // red is reused by the next call
    return s;
}

// ------------------------------------------------------------------------------------------------ noise regulariser
struct NoiseArgs {
    int count;
    int sides[IDE3D_NOISE_MAX_BUFFERS];
    const float* bufs[IDE3D_NOISE_MAX_BUFFERS];
    float* grads[IDE3D_NOISE_MAX_BUFFERS];
    long long pyramid[IDE3D_NOISE_MAX_BUFFERS];   // float offset of the buffer's levels >= 1 in scratch
    float* scratch;                               // [0, 2 * IDE3D_NOISE_MAX_BUFFERS): one double per buffer (its loss)
    const float* grad_scale;
};

__host__ __device__ inline int noise_levels(int side) {
    int n = 1;
    while (side > 8) { side >>= 1; ++n; }
    return n;
}

__host__ __device__ inline int ilog2(int v) {
    int l = 0;
    while ((1 << l) < v) ++l;
    return l;
}

// One CTA per buffer.  Level L + 1 is avg_pool2d(level L, 2) with the reference's rounding (the four taps summed in row order, then
// divided by 4), written to scratch; the CTA's barriers order the levels, so no level exists outside this kernel's scratch.
// loss_b = sum_L A_L^2 + B_L^2 with A_L = mean(n * roll(n, 1, W)), B_L = mean(n * roll(n, 1, H)).  The gradient of pixel (i, j) is
// sum_L 4^-L * 2 / side_L^2 * (A_L * (n(I, J-1) + n(I, J+1)) + B_L * (n(I-1, J) + n(I+1, J))) at its level-L ancestor (I, J).
__global__ void __launch_bounds__(kNoiseThreads) noise_reg_kernel(NoiseArgs a) {
    __shared__ double red[33];
    __shared__ float sa[kNoiseMaxLevels], sb[kNoiseMaxLevels];
    const int b = blockIdx.x, side = a.sides[b], tid = threadIdx.x;
    const float* base = a.bufs[b];
    float* pyr = a.scratch + a.pyramid[b];
    const int nl = noise_levels(side);
    const float* cur = base;
    long long off = 0;
    double loss = 0.0;
    for (int l = 0, s = side; l < nl; ++l, s >>= 1) {
        if (l > 0) {
            float* dst = pyr + off;
            const int ps = s * 2, sh = ilog2(s);
            for (int k = tid; k < s * s; k += kNoiseThreads) {
                const float* p = cur + (long long)(2 * (k >> sh)) * ps + 2 * (k & (s - 1));
                dst[k] = __fdiv_rn(__fadd_rn(__fadd_rn(__fadd_rn(p[0], p[1]), p[ps]), p[ps + 1]), 4.f);
            }
            __syncthreads();
            cur = dst;
            off += (long long)s * s;
        }
        const int m = s - 1, sh = ilog2(s);
        double pa = 0.0, pb = 0.0;
        for (int k = tid; k < s * s; k += kNoiseThreads) {
            const int i = k >> sh, j = k & m;
            const float v = cur[k];
            pa += (double)__fmul_rn(v, cur[i * s + ((j - 1) & m)]);
            pb += (double)__fmul_rn(v, cur[((i - 1) & m) * s + j]);
        }
        const double A = block_sum<kNoiseThreads>(pa, red) / ((double)s * s);
        const double B = block_sum<kNoiseThreads>(pb, red) / ((double)s * s);
        loss += A * A + B * B;
        if (tid == 0) { sa[l] = (float)A; sb[l] = (float)B; }
    }
    if (tid == 0) reinterpret_cast<double*>(a.scratch)[b] = loss;
    if (a.grad_scale == nullptr) return;
    __syncthreads();
    const float gs = __ldg(a.grad_scale);
    float* g = a.grads[b];
    const int sh0 = ilog2(side);
    for (int k = tid; k < side * side; k += kNoiseThreads) {
        const int i = k >> sh0, j = k & (side - 1);
        float acc = 0.f;
        const float* c = base;
        long long loff = 0;
        for (int l = 0, s = side; l < nl; ++l, s >>= 1) {
            if (l > 0) {
                c = pyr + loff;
                loff += (long long)s * s;
            }
            const int I = i >> l, J = j >> l, m = s - 1;
            const float w = c[I * s + ((J - 1) & m)] + c[I * s + ((J + 1) & m)];
            const float h = c[((I - 1) & m) * s + J] + c[((I + 1) & m) * s + J];
            const float coef = 2.f / ((float)s * (float)s) / (float)(1 << (2 * l));
            acc += coef * (sa[l] * w + sb[l] * h);
        }
        g[k] = acc * gs;
    }
}

__global__ void noise_loss_kernel(const double* per_buffer, int count, float* loss) {
    double s = 0.0;
    for (int b = 0; b < count; ++b) s += per_buffer[b];
    *loss = (float)s;
}

// One CTA per buffer: buf -= mean(buf); buf *= rsqrt(mean(buf^2)), each mean accumulated in double and rounded once.
__global__ void __launch_bounds__(kNoiseThreads) noise_normalize_kernel(NoiseArgs a) {
    __shared__ double red[33];
    const int b = blockIdx.x, tid = threadIdx.x;
    const int n = a.sides[b] * a.sides[b];
    float* x = const_cast<float*>(a.bufs[b]);
    double s = 0.0;
    for (int k = tid; k < n; k += kNoiseThreads) s += x[k];
    const float mean = (float)(block_sum<kNoiseThreads>(s, red) / n);
    double q = 0.0;
    for (int k = tid; k < n; k += kNoiseThreads) {
        const float d = __fsub_rn(x[k], mean);
        q += (double)__fmul_rn(d, d);
    }
    const float r = rsqrtf((float)(block_sum<kNoiseThreads>(q, red) / n));
    for (int k = tid; k < n; k += kNoiseThreads) x[k] = __fmul_rn(__fsub_rn(x[k], mean), r);
}

static int noise_args(const ide3d_noise_table* t, bool need_scratch, NoiseArgs& a) {
    IDE3D_REQUIRE(t, "noise: null table");
    IDE3D_REQUIRE(t->count >= 0, "noise: negative buffer count %d", t->count);
    if (t->count > IDE3D_NOISE_MAX_BUFFERS) {
        snprintf(error_buffer(), 512, "noise: %d buffers, at most %d per table", t->count, IDE3D_NOISE_MAX_BUFFERS);
        return IDE3D_UNSUPPORTED;
    }
    a.count = t->count;
    long long need = 2 * IDE3D_NOISE_MAX_BUFFERS;
    for (int b = 0; b < t->count; ++b) {
        const int s = t->sides[b];
        IDE3D_REQUIRE(s > 0, "noise: buffer %d has side %d", b, s);
        IDE3D_REQUIRE(t->bufs[b], "noise: null buffer %d", b);
        if ((s & (s - 1)) != 0 || s > kNoiseMaxSide) {
            snprintf(error_buffer(), 512, "noise: buffer %d side %d is not a power of two <= %d", b, s, kNoiseMaxSide);
            return IDE3D_UNSUPPORTED;
        }
        a.sides[b] = s;
        a.bufs[b] = t->bufs[b];
        a.grads[b] = t->grads[b];
        a.pyramid[b] = need;
        for (int l = 1, q = s >> 1; l < noise_levels(s); ++l, q >>= 1) need += (long long)q * q;
    }
    if (need_scratch) {
        IDE3D_REQUIRE(t->scratch, "noise: null scratch");
        IDE3D_REQUIRE((reinterpret_cast<uintptr_t>(t->scratch) & 7) == 0, "noise: scratch not 8-byte aligned");
        IDE3D_REQUIRE(t->scratch_floats >= need, "noise: scratch holds %lld floats, need %lld", (long long)t->scratch_floats, need);
    }
    a.scratch = t->scratch;
    a.grad_scale = nullptr;
    return IDE3D_OK;
}

// ------------------------------------------------------------------------------------------------ semantic cross-entropy
// Forward: one CTA per (output row, frame).  Per pixel: the bilinear logits (seg_logit_at), max, log-sum-exp, NLL of the mask class;
// the row's NLL sum (double) goes to partials[frame * out_h + row] and one more CTA folds the partials in order.  AC: the source
// position rule (seg_common.cuh), align_corners=True for the _ac entry points.
template <bool AC>
__global__ void __launch_bounds__(kXentThreads) seg_xent_fwd_kernel(ide3d_seg_xent_params p) {
    __shared__ double red[33];
    const int y = blockIdx.x, n = blockIdx.y;
    const float* s = p.seg + n * p.seg_stride_n;
    const uint8_t* mrow = p.mask + ((long long)n * p.out_h + y) * p.out_w;
    float* lrow = p.lse + ((long long)n * p.out_h + y) * p.out_w;
    double acc = 0.0;
    for (int x = threadIdx.x; x < p.out_w; x += kXentThreads) {
        const SegTaps t = seg_taps_at<AC>(s, p.in_h, p.in_w, p.seg_stride_h, p.seg_stride_w, x, y, p.out_h, p.out_w);
        const int label = min((int)mrow[x], p.classes - 1);
        float mx = -INFINITY, vl = 0.f;
        for (int k = 0; k < p.classes; ++k) {
            const float v = seg_logit_at(t, k * p.seg_stride_c);
            mx = fmaxf(mx, v);
            if (k == label) vl = v;
        }
        float se = 0.f;
        for (int k = 0; k < p.classes; ++k) se += expf(seg_logit_at(t, k * p.seg_stride_c) - mx);
        const float lse = mx + logf(se);
        lrow[x] = lse;
        acc += (double)(lse - vl);
    }
    const double row = block_sum<kXentThreads>(acc, red);
    if (threadIdx.x == 0) p.partials[(long long)n * p.out_h + y] = row;
}

__global__ void __launch_bounds__(kNoiseThreads) seg_xent_loss_kernel(const double* partials, int rows, double count, float* loss) {
    __shared__ double red[33];
    double s = 0.0;
    for (int k = threadIdx.x; k < rows; k += kNoiseThreads) s += partials[k];
    s = block_sum<kNoiseThreads>(s, red);
    if (threadIdx.x == 0) *loss = (float)(s / count);
}

// First output index whose taps can reach source index i (lo) and one past the last (hi): a tap of output d reaches i0 = floor(src(d))
// and i0 + 1, so i0 in {i - 1, i}; one extra index each side absorbs the rounding of src.  align_corners=False: src(d) = (d + 0.5) *
// in / out - 0.5; align_corners=True: src(d) = d * (in - 1) / (out - 1), and every output reads texel 0 when in = 1.
template <bool AC>
__device__ __forceinline__ void tap_window(int i, int in, int out, int& lo, int& hi) {
    if (AC) {
        if (in == 1) { lo = 0; hi = out; return; }
        const double r = (double)(out - 1) / (in - 1);
        lo = max(0, (int)floor((i - 1) * r) - 1);
        hi = min(out, (int)ceil((i + 1) * r) + 2);
        return;
    }
    const double r = (double)out / in;
    lo = max(0, (int)floor((i - 0.5) * r - 0.5) - 1);
    hi = min(out, (int)ceil((i + 1.5) * r - 0.5) + 2);
}

// Backward: one thread per (frame, class, source texel), ix fastest.  It visits the output pixels of its tap window and sums
// w_y * w_x * (softmax_k - [mask == k]) in row order; softmax_k = exp(logit_k - lse) from the saved log-sum-exp.
template <bool AC>
__global__ void __launch_bounds__(kXentThreads) seg_xent_bwd_kernel(ide3d_seg_xent_params p, float scale) {
    const long long idx = (long long)blockIdx.x * kXentThreads + threadIdx.x;
    const long long total = (long long)p.n * p.classes * p.in_h * p.in_w;
    if (idx >= total) return;
    const int ix = (int)(idx % p.in_w), iy = (int)((idx / p.in_w) % p.in_h);
    const int k = (int)((idx / ((long long)p.in_w * p.in_h)) % p.classes), n = (int)(idx / ((long long)p.in_w * p.in_h * p.classes));
    const float* s = p.seg + n * p.seg_stride_n;
    const long long kc = k * p.seg_stride_c;
    int y0, y1, x0, x1;
    tap_window<AC>(iy, p.in_h, p.out_h, y0, y1);
    tap_window<AC>(ix, p.in_w, p.out_w, x0, x1);
    const float g = scale * __ldg(p.grad_loss);
    float acc = 0.f;
    for (int y = y0; y < y1; ++y) {
        const Tap ty = bilinear_tap<AC>(y, p.in_h, p.out_h);
        const float wy = (ty.i0 == iy ? ty.l0 : 0.f) + (ty.i1 == iy ? ty.l1 : 0.f);
        if (!(ty.i0 == iy || ty.i1 == iy)) continue;
        const long long row = ((long long)n * p.out_h + y) * p.out_w;
        float racc = 0.f;
        for (int x = x0; x < x1; ++x) {
            const Tap tx = bilinear_tap<AC>(x, p.in_w, p.out_w);
            if (!(tx.i0 == ix || tx.i1 == ix)) continue;
            const float wx = (tx.i0 == ix ? tx.l0 : 0.f) + (tx.i1 == ix ? tx.l1 : 0.f);
            const SegTaps t = seg_taps_at<AC>(s, p.in_h, p.in_w, p.seg_stride_h, p.seg_stride_w, x, y, p.out_h, p.out_w);
            const float prob = expf(seg_logit_at(t, kc) - __ldg(p.lse + row + x));
            const float d = min((int)__ldg(p.mask + row + x), p.classes - 1) == k ? prob - 1.f : prob;
            racc += wx * d;
        }
        acc += wy * racc;
    }
    p.grad_seg[idx] = acc * g;
}

static bool fits31(long long n, long long c, long long h, long long w, long long sn, long long sc, long long sh, long long sw) {
    if (sn < 0 || sc < 0 || sh < 0 || sw < 0) return false;
    const long long last = (n - 1) * sn + (c - 1) * sc + (h - 1) * sh + (w - 1) * sw;
    return last < (1LL << 31) && n * c * h * w < (1LL << 31);
}

static int check_xent(const ide3d_seg_xent_params* p) {
    IDE3D_REQUIRE(p, "seg_xent: null params");
    IDE3D_REQUIRE(p->n > 0 && p->classes > 0 && p->in_h > 0 && p->in_w > 0 && p->out_h > 0 && p->out_w > 0,
                  "seg_xent: bad sizes (n %d, classes %d, in %dx%d, out %dx%d)", p->n, p->classes, p->in_h, p->in_w, p->out_h, p->out_w);
    IDE3D_REQUIRE(p->classes <= 32, "seg_xent: %d classes, at most 32", p->classes);
    IDE3D_REQUIRE(p->seg && p->mask && p->lse, "seg_xent: null logits, mask or lse");
    IDE3D_REQUIRE(fits31(p->n, p->classes, p->in_h, p->in_w, p->seg_stride_n, p->seg_stride_c, p->seg_stride_h, p->seg_stride_w),
                  "seg_xent: logit strides do not fit 32 bits");
    IDE3D_REQUIRE(fits31(p->n, 1, p->out_h, p->out_w, (long long)p->out_h * p->out_w, 0, p->out_w, 1), "seg_xent: output does not fit 32 bits");
    IDE3D_REQUIRE(p->out_h <= 65535, "seg_xent: output height %d > 65535", p->out_h);
    IDE3D_REQUIRE(p->n <= 65535, "seg_xent: %d frames > 65535", p->n);
    return IDE3D_OK;
}

}  // namespace ide3d

extern "C" int ide3d_noise_reg(const ide3d_noise_table* t, float* loss, const float* grad_scale, ide3d_stream_t stream) {
    ide3d::NoiseArgs a;
    const int rc = ide3d::noise_args(t, true, a);
    if (rc != IDE3D_OK) return rc;
    IDE3D_REQUIRE(loss || grad_scale, "noise_reg: null loss and no gradient requested");
    if (grad_scale)
        for (int b = 0; b < t->count; ++b) IDE3D_REQUIRE(t->grads[b], "noise_reg: null gradient %d", b);
    a.grad_scale = grad_scale;
    if (t->count == 0) return IDE3D_OK;
    ide3d::noise_reg_kernel<<<t->count, ide3d::kNoiseThreads, 0, (cudaStream_t)stream>>>(a);
    IDE3D_CHECK_LAUNCH("noise_reg_kernel");
    if (loss) {
        ide3d::noise_loss_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(reinterpret_cast<const double*>(t->scratch), t->count, loss);
        IDE3D_CHECK_LAUNCH("noise_loss_kernel");
    }
    return IDE3D_OK;
}

extern "C" int ide3d_noise_normalize(const ide3d_noise_table* t, ide3d_stream_t stream) {
    ide3d::NoiseArgs a;
    const int rc = ide3d::noise_args(t, false, a);
    if (rc != IDE3D_OK) return rc;
    if (t->count == 0) return IDE3D_OK;
    ide3d::noise_normalize_kernel<<<t->count, ide3d::kNoiseThreads, 0, (cudaStream_t)stream>>>(a);
    IDE3D_CHECK_LAUNCH("noise_normalize_kernel");
    return IDE3D_OK;
}

template <bool AC>
static int seg_xent_fwd(const ide3d_seg_xent_params* p, ide3d_stream_t stream) {
    const int rc = ide3d::check_xent(p);
    if (rc != IDE3D_OK) return rc;
    IDE3D_REQUIRE(p->partials && p->loss, "seg_xent_fwd: null partials or loss");
    ide3d::seg_xent_fwd_kernel<AC><<<dim3((unsigned)p->out_h, (unsigned)p->n), ide3d::kXentThreads, 0, (cudaStream_t)stream>>>(*p);
    IDE3D_CHECK_LAUNCH("seg_xent_fwd_kernel");
    ide3d::seg_xent_loss_kernel<<<1, ide3d::kNoiseThreads, 0, (cudaStream_t)stream>>>(p->partials, p->n * p->out_h,
                                                                                      (double)p->n * p->out_h * p->out_w, p->loss);
    IDE3D_CHECK_LAUNCH("seg_xent_loss_kernel");
    return IDE3D_OK;
}

template <bool AC>
static int seg_xent_bwd(const ide3d_seg_xent_params* p, ide3d_stream_t stream) {
    const int rc = ide3d::check_xent(p);
    if (rc != IDE3D_OK) return rc;
    IDE3D_REQUIRE(p->grad_loss && p->grad_seg, "seg_xent_bwd: null grad_loss or grad_seg");
    const long long total = (long long)p->n * p->classes * p->in_h * p->in_w;
    const float scale = (float)(1.0 / ((double)p->n * p->out_h * p->out_w));
    ide3d::seg_xent_bwd_kernel<AC><<<(unsigned)ide3d::ceil_div(total, (long long)ide3d::kXentThreads), ide3d::kXentThreads, 0,
                                     (cudaStream_t)stream>>>(*p, scale);
    IDE3D_CHECK_LAUNCH("seg_xent_bwd_kernel");
    return IDE3D_OK;
}

extern "C" int ide3d_seg_xent_fwd(const ide3d_seg_xent_params* p, ide3d_stream_t stream) { return seg_xent_fwd<false>(p, stream); }
extern "C" int ide3d_seg_xent_bwd(const ide3d_seg_xent_params* p, ide3d_stream_t stream) { return seg_xent_bwd<false>(p, stream); }
extern "C" int ide3d_seg_xent_fwd_ac(const ide3d_seg_xent_params* p, ide3d_stream_t stream) { return seg_xent_fwd<true>(p, stream); }
extern "C" int ide3d_seg_xent_bwd_ac(const ide3d_seg_xent_params* p, ide3d_stream_t stream) { return seg_xent_bwd<true>(p, stream); }
