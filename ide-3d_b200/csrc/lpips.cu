// The LPIPS v0.1 head of pivotal tuning (inversion/criteria/lpips/lpips.py:29-35, normalize_activation in utils.py:6-8), fused over
// every tapped layer of one call:
//   ide3d_lpips_fwd   value[n] = sum_l mean_p sum_c lin_l[c] (u_c - v_c)^2, u / v the channel-normalised features; two launches
//   ide3d_lpips_bwd   the gradient to the features of the render (and of the target when asked); one launch
// The reference runs normalise / subtract / square / 1x1 conv / mean per layer, forward and backward: a few dozen small kernels.
// Work unit: one CTA per (layer, sample, 256 consecutive pixels), one thread per pixel walking the channels; for NCHW the lanes of
// a warp read consecutive pixels of a channel (coalesced), for channels_last each lane reads its own contiguous channel vector.
// Every reduction runs in a fixed order (per-thread channel loop, a shuffle / shared-memory tree, a serial fold): no float atomics.
#include "common.cuh"

namespace ide3d {

constexpr int kLpipsThreads = 256;
constexpr float kLpipsEps = 1e-10f;            // normalize_activation's eps

struct LpipsArgs {
    ide3d_lpips_params p;
    int blocks_per_sample[IDE3D_LPIPS_MAX_LAYERS];   // ceil(h * w / 256)
    int first_block[IDE3D_LPIPS_MAX_LAYERS + 1];     // first CTA of layer l; first_block[num_layers] = grid size
    double* partials;                                // [grid]: the CTAs' sums
    double* layer_values;                            // [n * num_layers]
};

__device__ __forceinline__ double lpips_block_sum(double v, double* red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) red[warp] = v;
    __syncthreads();
    if (warp == 0) {
        v = lane < kLpipsThreads / 32 ? red[lane] : 0.0;
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    }
    return v;                                        // valid in thread 0
}

// The CTA's layer, sample and pixel.  Returns false for the threads past the layer's last pixel.
struct Pixel {
    int layer, n, hw;
    long long x, y;                                  // element offsets of channel 0
    long long gx, gy;
};

__device__ __forceinline__ bool locate(const LpipsArgs& a, Pixel& px) {
    const int b = blockIdx.x;
    int l = 0;
    while (l + 1 < a.p.num_layers && b >= a.first_block[l + 1]) ++l;
    const ide3d_lpips_layer& L = a.p.layers[l];
    const int local = b - a.first_block[l];
    const int n = local / a.blocks_per_sample[l];
    const int pix = (local - n * a.blocks_per_sample[l]) * kLpipsThreads + threadIdx.x;
    px.layer = l;
    px.n = n;
    px.hw = L.h * L.w;
    px.x = px.y = px.gx = px.gy = 0;
    if (pix >= px.hw) return false;
    const int hh = pix / L.w, ww = pix - hh * L.w;
    px.x = n * L.x_stride[0] + hh * L.x_stride[2] + ww * L.x_stride[3];
    px.y = n * L.y_stride[0] + hh * L.y_stride[2] + ww * L.y_stride[3];
    px.gx = n * L.gx_stride[0] + hh * L.gx_stride[2] + ww * L.gx_stride[3];
    px.gy = n * L.gy_stride[0] + hh * L.gy_stride[2] + ww * L.gy_stride[3];
    return true;
}

// sum_c x_c^2 and sum_c y_c^2 at one pixel
__device__ __forceinline__ void squared_norms(const ide3d_lpips_layer& L, const Pixel& px, float& sx, float& sy) {
    const float* x = L.x + px.x;
    const float* y = L.y + px.y;
    sx = 0.f;
    sy = 0.f;
    for (int c = 0; c < L.c; ++c) {
        const float xv = __ldg(x + c * L.x_stride[1]), yv = __ldg(y + c * L.y_stride[1]);
        sx = __fmaf_rn(xv, xv, sx);
        sy = __fmaf_rn(yv, yv, sy);
    }
}

__global__ void __launch_bounds__(kLpipsThreads) lpips_fwd_kernel(const __grid_constant__ LpipsArgs a) {
    __shared__ double red[kLpipsThreads / 32];
    Pixel px;
    float acc = 0.f;
    if (locate(a, px)) {
        const ide3d_lpips_layer& L = a.p.layers[px.layer];
        float sx, sy;
        squared_norms(L, px, sx, sy);
        const float isx = __frcp_rn(sqrtf(sx) + kLpipsEps), isy = __frcp_rn(sqrtf(sy) + kLpipsEps);
        const float* x = L.x + px.x;
        const float* y = L.y + px.y;
        for (int c = 0; c < L.c; ++c) {
            const float d = __ldg(x + c * L.x_stride[1]) * isx - __ldg(y + c * L.y_stride[1]) * isy;
            acc = __fmaf_rn(__ldg(L.lin + c), d * d, acc);
        }
    }
    const double s = lpips_block_sum((double)acc, red);
    if (threadIdx.x == 0) a.partials[blockIdx.x] = s;
}

// One CTA per sample: lane l folds layer l's partials in block order and divides by h * w; lane 0 adds the layers in order.
__global__ void __launch_bounds__(32) lpips_fold_kernel(const __grid_constant__ LpipsArgs a) {
    __shared__ double lv[IDE3D_LPIPS_MAX_LAYERS];
    const int n = blockIdx.x, l = threadIdx.x;
    if (l < a.p.num_layers) {
        const double* part = a.partials + a.first_block[l] + (long long)n * a.blocks_per_sample[l];
        double s = 0.0;
        for (int k = 0; k < a.blocks_per_sample[l]; ++k) s += part[k];
        s /= (double)a.p.layers[l].h * a.p.layers[l].w;
        lv[l] = s;
        a.layer_values[(long long)n * a.p.num_layers + l] = s;
    }
    __syncwarp();
    if (l == 0) {
        double v = 0.0;
        for (int k = 0; k < a.p.num_layers; ++k) v += lv[k];
        a.p.value[n] = (float)v;
    }
}

// One thread per (layer, sample, pixel): norms, then sum_c g_c x_c and sum_c g_c y_c, then the gradient of every channel.
__global__ void __launch_bounds__(kLpipsThreads) lpips_bwd_kernel(const __grid_constant__ LpipsArgs a) {
    Pixel px;
    if (!locate(a, px)) return;
    const ide3d_lpips_layer& L = a.p.layers[px.layer];
    float sx, sy;
    squared_norms(L, px, sx, sy);
    const float nx = sqrtf(sx), ny = sqrtf(sy);
    const float isx = __frcp_rn(nx + kLpipsEps), isy = __frcp_rn(ny + kLpipsEps);
    const float gs = __ldg(a.p.grad_value + px.n) * (2.f / (float)px.hw);
    const float* x = L.x + px.x;
    const float* y = L.y + px.y;
    float tx = 0.f, ty = 0.f;
    for (int c = 0; c < L.c; ++c) {
        const float xv = __ldg(x + c * L.x_stride[1]), yv = __ldg(y + c * L.y_stride[1]);
        const float g = gs * __ldg(L.lin + c) * (xv * isx - yv * isy);
        tx = __fmaf_rn(g, xv, tx);
        ty = __fmaf_rn(g, yv, ty);
    }
    // d u_k / d x_j = s (delta_kj - s x_k x_j / ||x||), s = 1 / (||x|| + eps); a zero vector gets 0 (torch: NaN)
    const float kx = nx > 0.f ? isx * isx / nx * tx : 0.f, ky = ny > 0.f ? isy * isy / ny * ty : 0.f;
    const float mx = nx > 0.f ? isx : 0.f, my = ny > 0.f ? isy : 0.f;
    float* gx = L.grad_x ? L.grad_x + px.gx : nullptr;
    float* gy = L.grad_y ? L.grad_y + px.gy : nullptr;
    for (int c = 0; c < L.c; ++c) {
        const float xv = __ldg(x + c * L.x_stride[1]), yv = __ldg(y + c * L.y_stride[1]);
        const float g = gs * __ldg(L.lin + c) * (xv * isx - yv * isy);
        if (gx) gx[c * L.gx_stride[1]] = mx * g - kx * xv;
        if (gy) gy[c * L.gy_stride[1]] = ky * yv - my * g;
    }
}

static bool lpips_fits31(long long n, long long c, long long h, long long w, const int64_t* s) {
    if (s[0] < 0 || s[1] < 0 || s[2] < 0 || s[3] < 0) return false;
    return (n - 1) * s[0] + (c - 1) * s[1] + (h - 1) * s[2] + (w - 1) * s[3] < (1LL << 31);
}

// Validates the table and fills the launch geometry.  Scratch: the CTAs' partials, then the per-(sample, layer) values.
static int lpips_args(const ide3d_lpips_params* p, bool backward, LpipsArgs& a, long long& scratch_doubles) {
    IDE3D_REQUIRE(p, "lpips: null params");
    IDE3D_REQUIRE(p->n > 0 && p->num_layers > 0, "lpips: %d samples, %d layers", p->n, p->num_layers);
    if (p->num_layers > IDE3D_LPIPS_MAX_LAYERS) {
        snprintf(error_buffer(), 512, "lpips: %d layers, at most %d per call", p->num_layers, IDE3D_LPIPS_MAX_LAYERS);
        return IDE3D_UNSUPPORTED;
    }
    a.p = *p;
    long long blocks = 0;
    for (int l = 0; l < p->num_layers; ++l) {
        const ide3d_lpips_layer& L = p->layers[l];
        IDE3D_REQUIRE(L.c > 0 && L.h > 0 && L.w > 0, "lpips: layer %d has bad sizes (c %d, h %d, w %d)", l, L.c, L.h, L.w);
        IDE3D_REQUIRE(L.x && L.y && L.lin, "lpips: layer %d has a null x, y or lin", l);
        IDE3D_REQUIRE(lpips_fits31(p->n, L.c, L.h, L.w, L.x_stride), "lpips: layer %d x strides do not fit 31 bits", l);
        IDE3D_REQUIRE(lpips_fits31(p->n, L.c, L.h, L.w, L.y_stride), "lpips: layer %d y strides do not fit 31 bits", l);
        IDE3D_REQUIRE((long long)L.h * L.w < (1LL << 31), "lpips: layer %d has more than 2^31 pixels", l);
        if (backward) {
            IDE3D_REQUIRE(!L.grad_x || lpips_fits31(p->n, L.c, L.h, L.w, L.gx_stride), "lpips: layer %d grad_x strides do not fit 31 bits", l);
            IDE3D_REQUIRE(!L.grad_y || lpips_fits31(p->n, L.c, L.h, L.w, L.gy_stride), "lpips: layer %d grad_y strides do not fit 31 bits", l);
            IDE3D_REQUIRE(!L.grad_y || p->n == 1 || L.gy_stride[0] != 0, "lpips: layer %d grad_y must be per sample", l);
        }
        a.blocks_per_sample[l] = (int)ceil_div((long long)L.h * L.w, (long long)kLpipsThreads);
        a.first_block[l] = (int)blocks;
        blocks += (long long)p->n * a.blocks_per_sample[l];
        IDE3D_REQUIRE(blocks < (1LL << 31), "lpips: more than 2^31 blocks");
    }
    a.first_block[p->num_layers] = (int)blocks;
    scratch_doubles = blocks + (long long)p->n * p->num_layers;
    a.partials = nullptr;
    a.layer_values = nullptr;
    return IDE3D_OK;
}

// ---------------------------------------------------------------------------------------------------------------------------------
// The multi-tap L1 head of the encoder's VGG loss (apps/train_hybrid_encoder.py:143-152): total = sum_l w_l mean|x_l - y_l|.  The
// same structure as the LPIPS head: one grid over every layer (a CTA finds its layer from its block index), partials in double, a
// second launch that folds them in block order; the backward is one launch.  Work unit: one CTA per kFeatTile consecutive elements of
// one layer.  A layer whose x, y (and grad_x) share one dense layout (NCHW or channels_last) is walked as a flat array, with float4
// accesses when aligned; any other layer is walked in logical NCHW order through its strides.

constexpr int kFeatVec = 4;
constexpr int kFeatIters = 4;
constexpr long long kFeatTile = (long long)kLpipsThreads * kFeatVec * kFeatIters;   // elements per CTA
enum FeatMode { kFeatStrided = 0, kFeatFlat = 1, kFeatFlat4 = 2 };

struct FeatL1Args {
    ide3d_feat_l1_params p;
    long long numel[IDE3D_FEAT_L1_MAX_LAYERS];
    int mode[IDE3D_FEAT_L1_MAX_LAYERS];
    int first_block[IDE3D_FEAT_L1_MAX_LAYERS + 1];
    double* partials;                                // [grid]
};

__device__ __forceinline__ int feat_layer(const FeatL1Args& a) {
    int l = 0;
    while (l + 1 < a.p.num_layers && (int)blockIdx.x >= a.first_block[l + 1]) ++l;
    return l;
}

// element offset of logical NCHW index e under strides s
__device__ __forceinline__ long long feat_offset(const ide3d_feat_l1_layer& L, long long e, const int64_t* s) {
    const long long w = e % L.w;
    e /= L.w;
    const long long h = e % L.h;
    e /= L.h;
    const long long c = e % L.c;
    return (e / L.c) * s[0] + c * s[1] + h * s[2] + w * s[3];
}

__global__ void __launch_bounds__(kLpipsThreads) feat_l1_fwd_kernel(const __grid_constant__ FeatL1Args a) {
    __shared__ double red[kLpipsThreads / 32];
    const int l = feat_layer(a);
    const ide3d_feat_l1_layer& L = a.p.layers[l];
    const long long n = a.numel[l];
    const long long base = (long long)(blockIdx.x - a.first_block[l]) * kFeatTile;
    float acc = 0.f;
    if (a.mode[l] == kFeatFlat4) {
        const float4* x = reinterpret_cast<const float4*>(L.x);
        const float4* y = reinterpret_cast<const float4*>(L.y);
#pragma unroll
        for (int it = 0; it < kFeatIters; ++it) {
            const long long e = base + ((long long)it * kLpipsThreads + threadIdx.x) * kFeatVec;
            if (e < n) {
                const float4 u = __ldg(x + e / kFeatVec), v = __ldg(y + e / kFeatVec);
                acc += fabsf(u.x - v.x) + fabsf(u.y - v.y) + fabsf(u.z - v.z) + fabsf(u.w - v.w);
            }
        }
    } else {
        for (int it = 0; it < kFeatIters * kFeatVec; ++it) {
            const long long e = base + (long long)it * kLpipsThreads + threadIdx.x;
            if (e < n) {
                const long long ox = a.mode[l] == kFeatFlat ? e : feat_offset(L, e, L.x_stride);
                const long long oy = a.mode[l] == kFeatFlat ? e : feat_offset(L, e, L.y_stride);
                acc += fabsf(__ldg(L.x + ox) - __ldg(L.y + oy));
            }
        }
    }
    const double s = lpips_block_sum((double)acc, red);
    if (threadIdx.x == 0) a.partials[blockIdx.x] = s;
}

// One CTA: per layer, thread t sums partials t, t + 256, ... in order, a fixed tree adds the threads; thread 0 adds the layers in order.
__global__ void __launch_bounds__(kLpipsThreads) feat_l1_fold_kernel(const __grid_constant__ FeatL1Args a) {
    __shared__ double red[kLpipsThreads / 32];
    double total = 0.0;
    for (int l = 0; l < a.p.num_layers; ++l) {
        double s = 0.0;
        for (int b = a.first_block[l] + threadIdx.x; b < a.first_block[l + 1]; b += kLpipsThreads) s += a.partials[b];
        s = lpips_block_sum(s, red);
        if (threadIdx.x == 0) {
            const double mean = s / (double)a.numel[l];
            a.p.value[l] = (float)mean;
            total += (double)a.p.layers[l].weight * mean;
        }
        __syncthreads();                             // red is reused by the next layer
    }
    if (threadIdx.x == 0) a.p.value[a.p.num_layers] = (float)total;
}

__device__ __forceinline__ float feat_sgn(float d) { return (float)((d > 0.f) - (d < 0.f)); }

// grad_x = g w_l / numel_l sgn(x - y), torch's sgn (0 where x == y); g read from device memory.
__global__ void __launch_bounds__(kLpipsThreads) feat_l1_bwd_kernel(const __grid_constant__ FeatL1Args a) {
    const int l = feat_layer(a);
    const ide3d_feat_l1_layer& L = a.p.layers[l];
    const long long n = a.numel[l];
    const long long base = (long long)(blockIdx.x - a.first_block[l]) * kFeatTile;
    const float gs = __ldg(a.p.grad_value) * (float)((double)L.weight / (double)n);
    if (a.mode[l] == kFeatFlat4) {
        const float4* x = reinterpret_cast<const float4*>(L.x);
        const float4* y = reinterpret_cast<const float4*>(L.y);
        float4* gx = reinterpret_cast<float4*>(L.grad_x);
#pragma unroll
        for (int it = 0; it < kFeatIters; ++it) {
            const long long e = base + ((long long)it * kLpipsThreads + threadIdx.x) * kFeatVec;
            if (e < n) {
                const float4 u = __ldg(x + e / kFeatVec), v = __ldg(y + e / kFeatVec);
                gx[e / kFeatVec] = make_float4(gs * feat_sgn(u.x - v.x), gs * feat_sgn(u.y - v.y), gs * feat_sgn(u.z - v.z),
                                               gs * feat_sgn(u.w - v.w));
            }
        }
    } else {
        for (int it = 0; it < kFeatIters * kFeatVec; ++it) {
            const long long e = base + (long long)it * kLpipsThreads + threadIdx.x;
            if (e < n) {
                const bool flat = a.mode[l] == kFeatFlat;
                const long long ox = flat ? e : feat_offset(L, e, L.x_stride);
                const long long oy = flat ? e : feat_offset(L, e, L.y_stride);
                const long long og = flat ? e : feat_offset(L, e, L.gx_stride);
                L.grad_x[og] = gs * feat_sgn(__ldg(L.x + ox) - __ldg(L.y + oy));
            }
        }
    }
}

// True when strides s describe a dense, non-overlapping layout of [n, c, h, w] (size-1 dimensions ignored).
static bool feat_dense(const int* size, const int64_t* s) {
    int order[4] = {0, 1, 2, 3};
    for (int i = 0; i < 4; ++i)                      // fastest dimension first
        for (int j = i + 1; j < 4; ++j)
            if (s[order[j]] < s[order[i]]) { const int t = order[i]; order[i] = order[j]; order[j] = t; }
    long long expect = 1;
    for (int i = 0; i < 4; ++i) {
        const int d = order[i];
        if (size[d] == 1) continue;
        if (s[d] != expect) return false;
        expect *= size[d];
    }
    return true;
}

static int feat_l1_args(const ide3d_feat_l1_params* p, bool backward, FeatL1Args& a) {
    IDE3D_REQUIRE(p, "feat_l1: null params");
    IDE3D_REQUIRE(p->n > 0 && p->num_layers > 0, "feat_l1: %d samples, %d layers", p->n, p->num_layers);
    if (p->num_layers > IDE3D_FEAT_L1_MAX_LAYERS || p->dtype != IDE3D_F32) {
        snprintf(error_buffer(), 512, "feat_l1: %d layers of dtype %d; the kernel takes at most %d fp32 layers", p->num_layers, p->dtype,
                 IDE3D_FEAT_L1_MAX_LAYERS);
        return IDE3D_UNSUPPORTED;
    }
    a.p = *p;
    long long blocks = 0;
    for (int l = 0; l < p->num_layers; ++l) {
        const ide3d_feat_l1_layer& L = p->layers[l];
        IDE3D_REQUIRE(L.c > 0 && L.h > 0 && L.w > 0, "feat_l1: layer %d has bad sizes (c %d, h %d, w %d)", l, L.c, L.h, L.w);
        IDE3D_REQUIRE(L.x && L.y, "feat_l1: layer %d has a null x or y", l);
        IDE3D_REQUIRE(!backward || L.grad_x, "feat_l1: layer %d has a null grad_x", l);
        for (int k = 0; k < 4; ++k)
            IDE3D_REQUIRE(L.x_stride[k] >= 0 && L.y_stride[k] >= 0 && (!backward || L.gx_stride[k] >= 0),
                          "feat_l1: layer %d has a negative stride", l);
        const int size[4] = {p->n, L.c, L.h, L.w};
        a.numel[l] = (long long)p->n * L.c * L.h * L.w;
        bool flat = feat_dense(size, L.x_stride);
        for (int k = 0; k < 4; ++k) {
            if (size[k] == 1) continue;
            flat = flat && L.y_stride[k] == L.x_stride[k] && (!backward || L.gx_stride[k] == L.x_stride[k]);
        }
        const bool aligned = ((reinterpret_cast<uintptr_t>(L.x) | reinterpret_cast<uintptr_t>(L.y) |
                               (backward ? reinterpret_cast<uintptr_t>(L.grad_x) : 0)) & 15) == 0;
        a.mode[l] = !flat ? kFeatStrided : (aligned && a.numel[l] % kFeatVec == 0) ? kFeatFlat4 : kFeatFlat;
        a.first_block[l] = (int)blocks;
        blocks += ceil_div(a.numel[l], kFeatTile);
        IDE3D_REQUIRE(blocks < (1LL << 31), "feat_l1: more than 2^31 blocks");
    }
    a.first_block[p->num_layers] = (int)blocks;
    a.partials = nullptr;
    return IDE3D_OK;
}

}  // namespace ide3d

extern "C" int64_t ide3d_feat_l1_scratch_bytes(const ide3d_feat_l1_params* p) {
    ide3d::FeatL1Args a;
    const int rc = ide3d::feat_l1_args(p, false, a);
    return rc != IDE3D_OK ? (int64_t)rc : (int64_t)8 * a.first_block[p->num_layers];
}

extern "C" int ide3d_feat_l1_fwd(const ide3d_feat_l1_params* p, ide3d_stream_t stream) {
    ide3d::FeatL1Args a;
    const int rc = ide3d::feat_l1_args(p, false, a);
    if (rc != IDE3D_OK) return rc;
    const long long grid = a.first_block[p->num_layers];
    IDE3D_REQUIRE(p->value && p->scratch, "feat_l1_fwd: null value or scratch");
    IDE3D_REQUIRE((reinterpret_cast<uintptr_t>(p->scratch) & 7) == 0, "feat_l1_fwd: scratch not 8-byte aligned");
    IDE3D_REQUIRE(p->scratch_bytes >= 8 * grid, "feat_l1_fwd: scratch holds %lld bytes, need %lld", (long long)p->scratch_bytes, 8 * grid);
    a.partials = static_cast<double*>(p->scratch);
    ide3d::feat_l1_fwd_kernel<<<(unsigned)grid, ide3d::kLpipsThreads, 0, (cudaStream_t)stream>>>(a);
    IDE3D_CHECK_LAUNCH("feat_l1_fwd_kernel");
    ide3d::feat_l1_fold_kernel<<<1, ide3d::kLpipsThreads, 0, (cudaStream_t)stream>>>(a);
    IDE3D_CHECK_LAUNCH("feat_l1_fold_kernel");
    return IDE3D_OK;
}

extern "C" int ide3d_feat_l1_bwd(const ide3d_feat_l1_params* p, ide3d_stream_t stream) {
    ide3d::FeatL1Args a;
    const int rc = ide3d::feat_l1_args(p, true, a);
    if (rc != IDE3D_OK) return rc;
    IDE3D_REQUIRE(p->grad_value, "feat_l1_bwd: null grad_value");
    ide3d::feat_l1_bwd_kernel<<<(unsigned)a.first_block[p->num_layers], ide3d::kLpipsThreads, 0, (cudaStream_t)stream>>>(a);
    IDE3D_CHECK_LAUNCH("feat_l1_bwd_kernel");
    return IDE3D_OK;
}

extern "C" int64_t ide3d_lpips_scratch_bytes(const ide3d_lpips_params* p) {
    ide3d::LpipsArgs a;
    long long doubles = 0;
    const int rc = ide3d::lpips_args(p, false, a, doubles);
    return rc != IDE3D_OK ? (int64_t)rc : (int64_t)(8 * doubles);
}

extern "C" int ide3d_lpips_fwd(const ide3d_lpips_params* p, ide3d_stream_t stream) {
    ide3d::LpipsArgs a;
    long long doubles = 0;
    const int rc = ide3d::lpips_args(p, false, a, doubles);
    if (rc != IDE3D_OK) return rc;
    IDE3D_REQUIRE(p->value && p->scratch, "lpips_fwd: null value or scratch");
    IDE3D_REQUIRE((reinterpret_cast<uintptr_t>(p->scratch) & 7) == 0, "lpips_fwd: scratch not 8-byte aligned");
    IDE3D_REQUIRE(p->scratch_bytes >= 8 * doubles, "lpips_fwd: scratch holds %lld bytes, need %lld", (long long)p->scratch_bytes,
                  8 * doubles);
    a.partials = static_cast<double*>(p->scratch);
    a.layer_values = a.partials + a.first_block[p->num_layers];
    ide3d::lpips_fwd_kernel<<<(unsigned)a.first_block[p->num_layers], ide3d::kLpipsThreads, 0, (cudaStream_t)stream>>>(a);
    IDE3D_CHECK_LAUNCH("lpips_fwd_kernel");
    ide3d::lpips_fold_kernel<<<(unsigned)p->n, 32, 0, (cudaStream_t)stream>>>(a);
    IDE3D_CHECK_LAUNCH("lpips_fold_kernel");
    return IDE3D_OK;
}

extern "C" int ide3d_lpips_bwd(const ide3d_lpips_params* p, ide3d_stream_t stream) {
    ide3d::LpipsArgs a;
    long long doubles = 0;
    const int rc = ide3d::lpips_args(p, true, a, doubles);
    if (rc != IDE3D_OK) return rc;
    IDE3D_REQUIRE(p->grad_value, "lpips_bwd: null grad_value");
    ide3d::lpips_bwd_kernel<<<(unsigned)a.first_block[p->num_layers], ide3d::kLpipsThreads, 0, (cudaStream_t)stream>>>(a);
    IDE3D_CHECK_LAUNCH("lpips_bwd_kernel");
    return IDE3D_OK;
}
