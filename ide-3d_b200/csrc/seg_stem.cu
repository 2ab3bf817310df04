// The opening of the HybridEncoder's geometry branch (inversion/networks.py:1638-1646) from a uint8 class-id mask, and the generator's
// own class ids at image resolution.
//
// ide3d_seg_stem.  The branch's input is one_hot(mask) * 2 - 1: 19 distinct values per pixel.  The 1x1 stem, block 0's 3x3 conv1 and
// its FIR-down + 1x1 skip are linear in that input (up to conv1's bias and lrelu), so all three are exact functions of the class ids:
//   T[k]      = wg0 * (2 W0[:, k] - sum_j W0[:, j]) + b0            stem output of class k (row K: "no class", -wg0 sum_j W0[:, j] + b0)
//   L1[t][k]  = wg1 * W1[:, :, t] @ T[k]                            conv1's contribution of tap t from a pixel of class k
//   S[k]      = wgs * Ws @ T[k]                                     the skip's 1x1 convolution of a pixel of class k
//   y1[p]     = lrelu(sum_{t inside} L1[t][m(p + t)] + b1) * sqrt(2)
//   skip[q]   = sum_{a inside} f~[a] * S[m(2q + a - 1)]              f~ = f flipped (upfirdn2d's convolution)
// Taps outside the image read the stem's zero padding, not a class: a zero table row (index K + 1) stands for them.
// Launch 1: one CTA builds T, L1 and S in double (each entry one dot product in index order) into the caller's scratch as fp32.
// Launch 2: one CTA per 16 x 16 tile of y1 (and the 8 x 8 tile of skip it covers) stages the 18 x 18 halo of table rows and the tables
// in shared memory; C0 / 4 threads per pixel each write one float4, so a pixel's channels_last row is one coalesced store.  Sums run
// in a fixed order and nothing is atomic: reruns are bit-identical.
//
// ide3d_seg_stem_bwd.  The gradients of w0, b0, w1, b1 and ws from grad_y1 and grad_skip, through the same tables:
//   gz[p]      = sqrt 2 * grad_y1[p] * (z[p] > 0 ? 1 : 0.2)          z recomputed from the forward's tables, in the forward's order
//   gL1[t][k]  = sum_{p: tap t of p inside, m(p + t) = k} gz[p]       gS[k] = sum_q sum_{a inside, m(2q + a - 1) = k} f~[a] grad_skip[q]
//   gW1[o, i, t] = wg1 sum_k gL1[t][k][o] T[k][i]                    gWs[o, i] = wgs sum_k gS[k][o] T[k][i]
//   gT[k][i]   = wg1 sum_{t, o} W1[o, i, t] gL1[t][k][o] + wgs sum_o Ws[o, i] gS[k][o]
//   gb0[i]     = sum_k gT[k][i]      gW0[i, j] = wg0 (2 gT[j][i] - sum_k gT[k][i])      gb1 = sum_k gL1[centre tap][k]
// Launch 1: a fixed grid of CTAs, each over the 16 x 16 tiles blockIdx.x, blockIdx.x + gridDim.x, ...  Per tile the CTA stages gz in
// shared memory, then every bin column -- (tap, channel) of gL1, (FIR row, channel) of gS -- has one owner thread that walks the
// tile's pixels in order and adds each run of equal class ids to its bin.  The CTA's bins go to its slice of the scratch.
// Launch 2 folds the slices in block order in double; launch 3 (one CTA) runs the chain above in double in a fixed order.  Three
// launches whatever n, no atomics: reruns are bit-identical.
//
// ide3d_seg_labels.  Per output pixel seg_class_at (seg_common.cuh): the class the frame and strip kernels colour; _ac with
// align_corners=True.
#include <algorithm>

#include "seg_common.cuh"

namespace ide3d {

constexpr int kStemTile = 16;                  // y1 tile side; the skip tile is kStemTile / 2
constexpr int kStemHalo = kStemTile + 2;       // rows / columns -1 .. 16 of the tile
constexpr int kStemThreads = 256;
constexpr int kTableThreads = 256;

// rows of the tables in scratch and shared memory: K classes, "no class", "outside the image" (zeros)
__host__ __device__ inline int stem_rows(int classes) { return classes + 2; }

__global__ void __launch_bounds__(kTableThreads) seg_stem_tables_kernel(ide3d_seg_stem_params p) {
    extern __shared__ double tsm[];                                    // T [(K + 1), C0]
    const int K = p.classes, C0 = p.c0, C1 = p.c1, R = stem_rows(K);
    for (int c = threadIdx.x; c < C0; c += blockDim.x) {
        double sum = 0.0;
        for (int j = 0; j < K; ++j) sum += (double)p.w0[(long long)c * K + j];
        const double wg0 = (double)p.wg0, b0 = (double)p.b0[c];
        for (int k = 0; k < K; ++k) tsm[k * C0 + c] = wg0 * (2.0 * (double)p.w0[(long long)c * K + k] - sum) + b0;
        tsm[K * C0 + c] = -wg0 * sum + b0;
    }
    __syncthreads();
    float* L1 = p.tables;                                              // [9][R][C0]
    float* S = p.tables + 9LL * R * C0;                                // [R][C1]
    const int n1 = 9 * R * C0, ns = R * C1;
    for (int e = threadIdx.x; e < n1 + ns; e += blockDim.x) {
        if (e < n1) {
            const int o = e % C0, k = (e / C0) % R, t = e / (C0 * R);
            double acc = 0.0;
            if (k <= K) {
                const float* w = p.w1 + (long long)o * C0 * 9 + t;     // W1[o, i, t]
                for (int i = 0; i < C0; ++i) acc += (double)w[i * 9] * tsm[k * C0 + i];
                acc *= (double)p.wg1;
            }
            L1[e] = (float)acc;
        } else {
            const int f = e - n1, o = f % C1, k = f / C1;
            double acc = 0.0;
            if (k <= K) {
                const float* w = p.ws + (long long)o * C0;
                for (int i = 0; i < C0; ++i) acc += (double)w[i] * tsm[k * C0 + i];
                acc *= (double)p.wgs;
            }
            S[f] = (float)acc;
        }
    }
}

__device__ __forceinline__ void add4(float4& a, const float4 b) { a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w; }
__device__ __forceinline__ void fma4(float4& a, float s, const float4 b) {
    a.x = fmaf(s, b.x, a.x); a.y = fmaf(s, b.y, a.y); a.z = fmaf(s, b.z, a.z); a.w = fmaf(s, b.w, a.w);
}
__device__ __forceinline__ float lrelu_gain(float v) { return (v > 0.f ? v : v * 0.2f) * 1.41421356237309515f; }

template <int C0>
__global__ void __launch_bounds__(kStemThreads) seg_stem_kernel(ide3d_seg_stem_params p) {
    constexpr int C1 = 2 * C0;
    constexpr int TP = C0 / 4, TS = C1 / 4;                            // threads per y1 pixel / per skip pixel
    const int K = p.classes, R = stem_rows(K);
    extern __shared__ float4 sm4[];
    float4* L1 = sm4;                                                  // [9][R][C0 / 4]
    float4* S = L1 + 9 * R * TP;                                       // [R][C1 / 4]
    unsigned char* ids = (unsigned char*)(S + R * TS);                 // [18][18]
    const int x0 = blockIdx.x * kStemTile, y0 = blockIdx.y * kStemTile, n = blockIdx.z;
    const float4* tables = (const float4*)p.tables;
    for (int i = threadIdx.x; i < 9 * R * TP + R * TS; i += kStemThreads) sm4[i] = tables[i];
    const unsigned char* m = p.mask + (long long)n * p.mask_stride_n;
    for (int i = threadIdx.x; i < kStemHalo * kStemHalo; i += kStemThreads) {
        const int hy = i / kStemHalo, hx = i % kStemHalo, y = y0 - 1 + hy, x = x0 - 1 + hx;
        int k = K + 1;
        if (y >= 0 && y < p.h && x >= 0 && x < p.w) {
            k = m[(long long)y * p.mask_stride_h + (long long)x * p.mask_stride_w];
            k = k < K ? k : K;
        }
        ids[i] = (unsigned char)k;
    }
    float fk[16];
#pragma unroll
    for (int a = 0; a < 16; ++a) fk[a] = p.fir[15 - a];                 // flipped: upfirdn2d convolves
    __syncthreads();

    // y1: TP threads per pixel, one float4 of channels each
    const int c4 = threadIdx.x % TP;
    const float4 b1 = ((const float4*)p.b1)[c4];
    for (int px = threadIdx.x / TP; px < kStemTile * kStemTile; px += kStemThreads / TP) {
        const int ty = px / kStemTile, tx = px % kStemTile, y = y0 + ty, x = x0 + tx;
        if (y >= p.h || x >= p.w) continue;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int t = 0; t < 9; ++t) {
            const int k = ids[(ty + t / 3) * kStemHalo + tx + t % 3];
            add4(acc, L1[(t * R + k) * TP + c4]);
        }
        add4(acc, b1);
        const float4 out = make_float4(lrelu_gain(acc.x), lrelu_gain(acc.y), lrelu_gain(acc.z), lrelu_gain(acc.w));
        ((float4*)p.y1)[(((long long)n * p.h + y) * p.w + x) * TP + c4] = out;
    }

    // skip: TS threads per output pixel; taps 2q - 1 .. 2q + 2 fall inside the halo
    const int s4 = threadIdx.x % TS, hh = p.h / 2, hw = p.w / 2;
    for (int px = threadIdx.x / TS; px < (kStemTile / 2) * (kStemTile / 2); px += kStemThreads / TS) {
        const int qy = px / (kStemTile / 2), qx = px % (kStemTile / 2), y = y0 / 2 + qy, x = x0 / 2 + qx;
        if (y >= hh || x >= hw) continue;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int a = 0; a < 16; ++a) {
            const int k = ids[(2 * qy + a / 4) * kStemHalo + 2 * qx + a % 4];
            fma4(acc, fk[a], S[k * TS + s4]);
        }
        ((float4*)p.skip)[(((long long)n * hh + y) * hw + x) * TS + s4] = acc;
    }
}

template <bool AC>
__global__ void __launch_bounds__(256) seg_labels_kernel(ide3d_seg_labels_params p) {
    const int x = blockIdx.x * 64 + threadIdx.x, y = blockIdx.y * 4 + threadIdx.y, n = blockIdx.z;
    if (x >= p.out_w || y >= p.out_h) return;
    const int k = seg_class_at<AC>(p.seg + (long long)n * p.seg_stride_n, p.classes, p.in_h, p.in_w, p.seg_stride_c, p.seg_stride_h,
                               p.seg_stride_w, x, y, p.out_h, p.out_w);
    p.out[((long long)n * p.out_h + y) * p.out_w + x] = (unsigned char)k;
}

// ------------------------------------------------------------------------------------------------ backward
constexpr int kBwdThreads = 544;               // 17 warps: the 9 C0 + 4 C1 = 17 C0 bin columns, C0 / 32 per thread
constexpr int kBwdCtas = 264;                  // CTAs of the accumulation launch at most (two per SM of an H100 at C0 = 32)
constexpr int kFoldThreads = 256;
constexpr int kChainThreads = 1024;

// bins of one CTA: gL1 [9][R][C0], then gS [4 FIR rows][R][C1] (rows K + 1, "outside the image", collect what no gradient needs)
__host__ __device__ inline long long bwd_bins(int classes, int c0) { return (long long)stem_rows(classes) * (9LL * c0 + 8LL * c0); }
__host__ __device__ inline long long bwd_totals(int classes, int c0) { return (long long)(classes + 1) * (9LL * c0 + 2LL * c0); }
inline int bwd_ctas(int n, int h, int w) {
    const long long tiles = (long long)n * ceil_div(h, kStemTile) * ceil_div(w, kStemTile);
    return (int)std::max(1LL, std::min(tiles, (long long)kBwdCtas));
}
inline long long bwd_totals_bytes(int classes, int c0) { return (8 * bwd_totals(classes, c0) + 15) / 16 * 16; }

template <int C0>
__global__ void __launch_bounds__(kBwdThreads) seg_stem_bwd_accum_kernel(ide3d_seg_stem_bwd_params b, int tiles_x, int tiles_y,
                                                                         float* partials) {
    constexpr int C1 = 2 * C0, TP = C0 / 4, COLS = 17 * C0;
    const ide3d_seg_stem_params& p = b.fwd;
    const int K = p.classes, R = stem_rows(K), nb = R * COLS;
    extern __shared__ float4 bsm4[];
    float* bins = (float*)bsm4;                                        // [nb]
    float* gz = bins + nb;                                             // [256][C0]
    unsigned char* ids = (unsigned char*)(gz + kStemTile * kStemTile * C0);   // [18][18]
    for (int i = threadIdx.x; i < nb; i += kBwdThreads) bins[i] = 0.f;
    const float4* L1 = (const float4*)p.tables;
    const int c4 = threadIdx.x % TP;
    const float4 b1 = __ldg((const float4*)p.b1 + c4);
    const int hh = p.h / 2, hw = p.w / 2, per_image = tiles_x * tiles_y, total = per_image * p.n;
    for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
        const int n = tile / per_image, r = tile % per_image;
        const int y0 = (r / tiles_x) * kStemTile, x0 = (r % tiles_x) * kStemTile;
        __syncthreads();                                               // the previous tile's owners are done with ids and gz
        const unsigned char* m = p.mask + (long long)n * p.mask_stride_n;
        for (int i = threadIdx.x; i < kStemHalo * kStemHalo; i += kBwdThreads) {
            const int hy = i / kStemHalo, hx = i % kStemHalo, y = y0 - 1 + hy, x = x0 - 1 + hx;
            int k = K + 1;
            if (y >= 0 && y < p.h && x >= 0 && x < p.w) {
                k = m[(long long)y * p.mask_stride_h + (long long)x * p.mask_stride_w];
                k = k < K ? k : K;
            }
            ids[i] = (unsigned char)k;
        }
        __syncthreads();
        // gz: the forward's pre-activation sum (same tables, same order), then lrelu's derivative
        for (int px = threadIdx.x / TP; px < kStemTile * kStemTile; px += kBwdThreads / TP) {
            const int ty = px / kStemTile, tx = px % kStemTile, y = y0 + ty, x = x0 + tx;
            float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
            if (y < p.h && x < p.w) {
                float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                for (int t = 0; t < 9; ++t) add4(z, __ldg(L1 + (t * R + ids[(ty + t / 3) * kStemHalo + tx + t % 3]) * TP + c4));
                add4(z, b1);
                const float4 gy = __ldg((const float4*)b.grad_y1 + (((long long)n * p.h + y) * p.w + x) * TP + c4);
                const float s2 = 1.41421356237309515f;
                g.x = z.x > 0.f ? gy.x * s2 : gy.x * s2 * 0.2f;
                g.y = z.y > 0.f ? gy.y * s2 : gy.y * s2 * 0.2f;
                g.z = z.z > 0.f ? gy.z * s2 : gy.z * s2 * 0.2f;
                g.w = z.w > 0.f ? gy.w * s2 : gy.w * s2 * 0.2f;
            }
            ((float4*)gz)[px * TP + c4] = g;
        }
        __syncthreads();
        // owners: one thread per bin column walks the tile in order, flushing each run of one class id into the bin
        for (int col = threadIdx.x; col < COLS; col += kBwdThreads) {
            if (col < 9 * C0) {
                const int t = col / C0, o = col % C0, dy = t / 3, dx = t % 3;
                float* bin = bins + t * R * C0 + o;
                int kp = ids[dy * kStemHalo + dx];
                float run = 0.f;
                for (int px = 0; px < kStemTile * kStemTile; ++px) {
                    const int k = ids[(px / kStemTile + dy) * kStemHalo + px % kStemTile + dx];
                    if (k != kp) {
                        bin[kp * C0] += run;
                        run = 0.f;
                        kp = k;
                    }
                    run += gz[px * C0 + o];
                }
                bin[kp * C0] += run;
            } else {
                const int c = col - 9 * C0, ay = c / C1, o = c % C1;
                float f[4];
#pragma unroll
                for (int ax = 0; ax < 4; ++ax) f[ax] = __ldg(p.fir + 15 - (ay * 4 + ax));     // flipped: upfirdn2d convolves
                float* bin = bins + 9 * R * C0 + ay * R * C1 + o;
                const float* gs = b.grad_skip + (long long)n * hh * hw * C1 + o;
                for (int q = 0; q < (kStemTile / 2) * (kStemTile / 2); ++q) {
                    const int qy = q / (kStemTile / 2), qx = q % (kStemTile / 2), y = y0 / 2 + qy, x = x0 / 2 + qx;
                    if (y >= hh || x >= hw) continue;
                    const float g = __ldg(gs + ((long long)y * hw + x) * C1);
                    const unsigned char* row = ids + (2 * qy + ay) * kStemHalo + 2 * qx;
#pragma unroll
                    for (int ax = 0; ax < 4; ++ax) bin[row[ax] * C1] += f[ax] * g;
                }
            }
        }
    }
    __syncthreads();
    float* out = partials + (long long)blockIdx.x * nb;
    for (int i = threadIdx.x; i < nb; i += kBwdThreads) out[i] = bins[i];
}

// totals (double): gL1 [9][K + 1][C0] then gS [K + 1][C1], each the sum over the CTAs' slices in block order (gS: then FIR rows)
__global__ void __launch_bounds__(kFoldThreads) seg_stem_bwd_fold_kernel(int classes, int c0, int ctas, const float* partials,
                                                                        double* totals) {
    const int K = classes, R = stem_rows(K), c1 = 2 * c0;
    const long long nb = bwd_bins(K, c0);
    const int n1 = 9 * (K + 1) * c0, ns = (K + 1) * c1;
    const int e = blockIdx.x * kFoldThreads + threadIdx.x;
    if (e >= n1 + ns) return;
    double acc = 0.0;
    if (e < n1) {
        const int o = e % c0, k = (e / c0) % (K + 1), t = e / (c0 * (K + 1));
        const float* src = partials + (t * R + k) * c0 + o;
        for (int b = 0; b < ctas; ++b) acc += (double)src[b * nb];
    } else {
        const int f = e - n1, o = f % c1, k = f / c1;
        const float* src = partials + 9LL * R * c0 + (long long)k * c1 + o;
        for (int b = 0; b < ctas; ++b)
            for (int ay = 0; ay < 4; ++ay) acc += (double)src[b * nb + (long long)ay * R * c1];
    }
    totals[e] = acc;
}

__global__ void __launch_bounds__(kChainThreads) seg_stem_bwd_chain_kernel(ide3d_seg_stem_bwd_params b, const double* totals) {
    extern __shared__ double csm[];
    const ide3d_seg_stem_params& p = b.fwd;
    const int K = p.classes, C0 = p.c0, C1 = p.c1;
    double* T = csm;                                                   // [K + 1][C0], as the table launch builds it
    double* gT = csm + (K + 1) * C0;                                   // [K + 1][C0]
    const double* gL1 = totals;                                        // [9][K + 1][C0]
    const double* gS = totals + 9 * (K + 1) * C0;                      // [K + 1][C1]
    const double wg0 = (double)p.wg0, wg1 = (double)p.wg1, wgs = (double)p.wgs;
    for (int c = threadIdx.x; c < C0; c += blockDim.x) {
        double sum = 0.0;
        for (int j = 0; j < K; ++j) sum += (double)p.w0[(long long)c * K + j];
        const double b0 = (double)p.b0[c];
        for (int k = 0; k < K; ++k) T[k * C0 + c] = wg0 * (2.0 * (double)p.w0[(long long)c * K + k] - sum) + b0;
        T[K * C0 + c] = -wg0 * sum + b0;
    }
    __syncthreads();
    const int nt = (K + 1) * C0, n1 = C0 * C0 * 9, ns = C1 * C0;
    for (int e = threadIdx.x; e < nt + n1 + ns; e += blockDim.x) {
        if (e < nt) {                                                  // gT first: the longest sums
            const int i = e % C0, k = e / C0;
            double a1 = 0.0, as = 0.0;
            for (int t = 0; t < 9; ++t)
                for (int o = 0; o < C0; ++o) a1 += (double)p.w1[((long long)o * C0 + i) * 9 + t] * gL1[(t * (K + 1) + k) * C0 + o];
            for (int o = 0; o < C1; ++o) as += (double)p.ws[(long long)o * C0 + i] * gS[k * C1 + o];
            gT[e] = wg1 * a1 + wgs * as;
        } else if (e < nt + n1) {
            const int f = e - nt, t = f % 9, i = (f / 9) % C0, o = f / (9 * C0);
            double acc = 0.0;
            for (int k = 0; k <= K; ++k) acc += gL1[(t * (K + 1) + k) * C0 + o] * T[k * C0 + i];
            b.grad_w1[f] = (float)(wg1 * acc);
        } else {
            const int f = e - nt - n1, i = f % C0, o = f / C0;
            double acc = 0.0;
            for (int k = 0; k <= K; ++k) acc += gS[k * C1 + o] * T[k * C0 + i];
            b.grad_ws[f] = (float)(wgs * acc);
        }
    }
    __syncthreads();
    for (int e = threadIdx.x; e < C0 * (K + 2); e += blockDim.x) {
        if (e < C0 * (K + 1)) {                                        // gW0 [C0][K], then gb0 [C0]
            const int i = e / (K + 1), j = e % (K + 1);
            double sum = 0.0;
            for (int k = 0; k <= K; ++k) sum += gT[k * C0 + i];
            if (j < K) b.grad_w0[(long long)i * K + j] = (float)(wg0 * (2.0 * gT[j * C0 + i] - sum));
            else b.grad_b0[i] = (float)sum;
        } else {                                                       // gb1: every pixel's centre tap is inside the image
            const int o = e - C0 * (K + 1);
            double acc = 0.0;
            for (int k = 0; k <= K; ++k) acc += gL1[(4 * (K + 1) + k) * C0 + o];
            b.grad_b1[o] = (float)acc;
        }
    }
}

}  // namespace ide3d

// The forward's validation, shared with the backward: IDE3D_UNSUPPORTED for a shape the tables do not take.
static int check_stem_shape(const ide3d_seg_stem_params* p) {
    IDE3D_REQUIRE(p->n >= 0 && p->n <= 65535 && p->h >= 1 && p->w >= 1 && p->classes >= 1 && p->c0 >= 1 && p->c1 >= 1,
                  "seg_stem: bad sizes (n %d, h %d, w %d, classes %d, c0 %d, c1 %d)", p->n, p->h, p->w, p->classes, p->c0, p->c1);
    if (p->c0 != 32 && p->c0 != 64)
        IDE3D_FAIL(IDE3D_UNSUPPORTED, "seg_stem: c0 must be 32 or 64, got %d", p->c0);
    if (p->c1 != 2 * p->c0) IDE3D_FAIL(IDE3D_UNSUPPORTED, "seg_stem: c1 must be 2 * c0, got %d for c0 %d", p->c1, p->c0);
    if (p->classes > IDE3D_SEG_STEM_MAX_CLASSES)
        IDE3D_FAIL(IDE3D_UNSUPPORTED, "seg_stem: at most %d classes, got %d", IDE3D_SEG_STEM_MAX_CLASSES, p->classes);
    if (p->h % 2 || p->w % 2 || p->h < 8 || p->w < 8)
        IDE3D_FAIL(IDE3D_UNSUPPORTED, "seg_stem: height and width must be even and >= 8, got %d x %d", p->h, p->w);
    IDE3D_REQUIRE((long long)p->h * p->w * p->c0 < (1LL << 40), "seg_stem: image too large (%d x %d)", p->h, p->w);
    return IDE3D_OK;
}

extern "C" int64_t ide3d_seg_stem_scratch_bytes(int classes, int c0) {
    if (classes < 1 || classes > IDE3D_SEG_STEM_MAX_CLASSES || (c0 != 32 && c0 != 64)) return IDE3D_UNSUPPORTED;
    return 4LL * ide3d::stem_rows(classes) * (9LL * c0 + 2LL * c0);
}

extern "C" int ide3d_seg_stem(const ide3d_seg_stem_params* p, ide3d_stream_t stream) {
    IDE3D_REQUIRE(p, "seg_stem: null params");
    const int rc = check_stem_shape(p);
    if (rc != IDE3D_OK) return rc;
    if (p->n == 0) return IDE3D_OK;
    IDE3D_REQUIRE(p->mask && p->y1 && p->skip, "seg_stem: null mask or output");
    IDE3D_REQUIRE(p->w0 && p->b0 && p->w1 && p->b1 && p->ws && p->fir, "seg_stem: null weight, bias or filter");
    IDE3D_REQUIRE(p->tables, "seg_stem: null tables scratch");
    IDE3D_REQUIRE(((uintptr_t)p->y1 | (uintptr_t)p->skip | (uintptr_t)p->b1 | (uintptr_t)p->tables) % 16 == 0,
                  "seg_stem: y1, skip, b1 and tables must be 16-byte aligned");
    const int R = ide3d::stem_rows(p->classes);
    const cudaStream_t s = (cudaStream_t)stream;
    const size_t tsmem = sizeof(double) * (size_t)(p->classes + 1) * p->c0;
    ide3d::seg_stem_tables_kernel<<<1, ide3d::kTableThreads, tsmem, s>>>(*p);
    IDE3D_CHECK_LAUNCH("seg_stem_tables_kernel");
    const size_t smem = 4 * (size_t)R * (9 * p->c0 + p->c1) + ide3d::kStemHalo * ide3d::kStemHalo;
    const dim3 grid((unsigned)ide3d::ceil_div(p->w, ide3d::kStemTile), (unsigned)ide3d::ceil_div(p->h, ide3d::kStemTile), (unsigned)p->n);
    if (p->c0 == 32) {
        IDE3D_CUDA(cudaFuncSetAttribute(ide3d::seg_stem_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        ide3d::seg_stem_kernel<32><<<grid, ide3d::kStemThreads, smem, s>>>(*p);
    } else {
        IDE3D_CUDA(cudaFuncSetAttribute(ide3d::seg_stem_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        ide3d::seg_stem_kernel<64><<<grid, ide3d::kStemThreads, smem, s>>>(*p);
    }
    IDE3D_CHECK_LAUNCH("seg_stem_kernel");
    return IDE3D_OK;
}

extern "C" int64_t ide3d_seg_stem_bwd_scratch_bytes(int n, int h, int w, int classes, int c0) {
    if (n < 0 || n > 65535 || h < 1 || w < 1) return IDE3D_INVALID;
    if (ide3d_seg_stem_scratch_bytes(classes, c0) < 0 || h % 2 || w % 2 || h < 8 || w < 8) return IDE3D_UNSUPPORTED;
    return ide3d::bwd_totals_bytes(classes, c0) + 4LL * ide3d::bwd_ctas(n, h, w) * ide3d::bwd_bins(classes, c0);
}

extern "C" int ide3d_seg_stem_bwd(const ide3d_seg_stem_bwd_params* b, ide3d_stream_t stream) {
    IDE3D_REQUIRE(b, "seg_stem_bwd: null params");
    const ide3d_seg_stem_params* p = &b->fwd;
    const int rc = check_stem_shape(p);
    if (rc != IDE3D_OK) return rc;
    IDE3D_REQUIRE(p->w0 && p->b0 && p->w1 && p->b1 && p->ws && p->fir, "seg_stem_bwd: null weight, bias or filter");
    IDE3D_REQUIRE(b->grad_w0 && b->grad_b0 && b->grad_w1 && b->grad_b1 && b->grad_ws, "seg_stem_bwd: null gradient output");
    if (p->n > 0) {
        IDE3D_REQUIRE(p->mask && p->tables && b->grad_y1 && b->grad_skip, "seg_stem_bwd: null mask, tables or incoming gradient");
        IDE3D_REQUIRE(((uintptr_t)p->tables | (uintptr_t)p->b1 | (uintptr_t)b->grad_y1) % 16 == 0,
                      "seg_stem_bwd: tables, b1 and grad_y1 must be 16-byte aligned");
    }
    const int64_t need = ide3d_seg_stem_bwd_scratch_bytes(p->n, p->h, p->w, p->classes, p->c0);
    IDE3D_REQUIRE(b->scratch && (uintptr_t)b->scratch % 16 == 0, "seg_stem_bwd: null or unaligned scratch");
    IDE3D_REQUIRE(b->scratch_bytes >= need, "seg_stem_bwd: scratch holds %lld bytes, need %lld", (long long)b->scratch_bytes,
                  (long long)need);
    const cudaStream_t s = (cudaStream_t)stream;
    double* totals = (double*)b->scratch;
    float* partials = (float*)((char*)b->scratch + ide3d::bwd_totals_bytes(p->classes, p->c0));
    const int ctas = ide3d::bwd_ctas(p->n, p->h, p->w);
    const int tx = ide3d::ceil_div(p->w, ide3d::kStemTile), ty = ide3d::ceil_div(p->h, ide3d::kStemTile);
    const size_t smem = 4 * (size_t)ide3d::bwd_bins(p->classes, p->c0) + 4 * (size_t)ide3d::kStemTile * ide3d::kStemTile * p->c0 +
                        ide3d::kStemHalo * ide3d::kStemHalo;
    if (p->c0 == 32) {
        IDE3D_CUDA(cudaFuncSetAttribute(ide3d::seg_stem_bwd_accum_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        ide3d::seg_stem_bwd_accum_kernel<32><<<ctas, ide3d::kBwdThreads, smem, s>>>(*b, tx, ty, partials);
    } else {
        IDE3D_CUDA(cudaFuncSetAttribute(ide3d::seg_stem_bwd_accum_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        ide3d::seg_stem_bwd_accum_kernel<64><<<ctas, ide3d::kBwdThreads, smem, s>>>(*b, tx, ty, partials);
    }
    IDE3D_CHECK_LAUNCH("seg_stem_bwd_accum_kernel");
    const long long nt = ide3d::bwd_totals(p->classes, p->c0);
    ide3d::seg_stem_bwd_fold_kernel<<<(unsigned)ide3d::ceil_div(nt, (long long)ide3d::kFoldThreads), ide3d::kFoldThreads, 0, s>>>(
        p->classes, p->c0, ctas, partials, totals);
    IDE3D_CHECK_LAUNCH("seg_stem_bwd_fold_kernel");
    const size_t csmem = 2 * sizeof(double) * (size_t)(p->classes + 1) * p->c0;
    ide3d::seg_stem_bwd_chain_kernel<<<1, ide3d::kChainThreads, csmem, s>>>(*b, totals);
    IDE3D_CHECK_LAUNCH("seg_stem_bwd_chain_kernel");
    return IDE3D_OK;
}

template <bool AC>
static int seg_labels(const ide3d_seg_labels_params* p, ide3d_stream_t stream) {
    IDE3D_REQUIRE(p, "seg_labels: null params");
    IDE3D_REQUIRE(p->n >= 0 && p->n <= 65535 && p->classes >= 1 && p->classes <= 256 && p->in_h >= 1 && p->in_w >= 1 && p->out_h >= 1 &&
                  p->out_w >= 1 && p->out_h <= 65535 * 4,
                  "seg_labels: bad sizes (n %d, classes %d, in %d x %d, out %d x %d)", p->n, p->classes, p->in_h, p->in_w, p->out_h, p->out_w);
    if (p->n == 0) return IDE3D_OK;
    IDE3D_REQUIRE(p->seg && p->out, "seg_labels: null logits or output");
    const dim3 block(64, 4), grid((unsigned)ide3d::ceil_div(p->out_w, 64), (unsigned)ide3d::ceil_div(p->out_h, 4), (unsigned)p->n);
    ide3d::seg_labels_kernel<AC><<<grid, block, 0, (cudaStream_t)stream>>>(*p);
    IDE3D_CHECK_LAUNCH("seg_labels_kernel");
    return IDE3D_OK;
}

extern "C" int ide3d_seg_labels(const ide3d_seg_labels_params* p, ide3d_stream_t stream) { return seg_labels<false>(p, stream); }
extern "C" int ide3d_seg_labels_ac(const ide3d_seg_labels_params* p, ide3d_stream_t stream) { return seg_labels<true>(p, stream); }
