// The display tail of viz/renderer.py:369-406: statistics, uint8 image and FFT panel of one [C, H, W] map.
//
// ide3d_viz_image, two launches:
//   reduce:  CTA (chunk g, channel c) -> float64 sum and sum of squares, float32 min and max of its pixels, in a fixed order (one
//            partial per CTA, no atomics).
//   image:   every CTA first folds the partials of the channels it needs in index order, then converts its pixels with torch's float32
//            operations in torch's order (depth normalisation, inf-norm normalisation, dB gain, (x * 127.5 + 128).clamp(0, 255) -> uint8).
//            CTA 0 also writes the six statistics.
// ide3d_viz_fft, five launches: per-channel means; the rows of the windowed maps through fft.cuh's float64 FFT (half plane, as
// spectra.cu); the columns, one |X|^2 plane per channel; the channel sum with per-CTA partials of the plane's sum; the panel (dB against
// the mean power, colormap index, half-size roll) written into the canvas.
#include "fft.cuh"

namespace ide3d {
namespace {

constexpr int kRedThreads = 256;
constexpr int kMaxChunks = 64;                  // reduction CTAs per channel
constexpr int kPixPerChunk = 4096;

struct Partial {
    double sum, sumsq;
    float mn, mx;
};

template <typename T>
__device__ __forceinline__ float load_f(const T* p) {
    if constexpr (sizeof(T) == 2) return __half2float(*reinterpret_cast<const __half*>(p));
    else return *p;
}

// fixed-order block reduction of one double (every thread gets the result)
template <int kThreads>
__device__ __forceinline__ double block_sum(double v, double* sh) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    double s = 0.0;
    for (int w = 0; w < kThreads / 32; ++w) s += sh[w];
    __syncthreads();
    return s;
}

template <typename T>
__global__ void __launch_bounds__(kRedThreads) viz_reduce_kernel(const T* __restrict__ x, int H, int W, long long sc, long long sh,
                                                                  long long sw, int chunks, Partial* __restrict__ part) {
    const int g = blockIdx.x, c = blockIdx.y;
    const long long n = (long long)H * W, per = ceil_div<long long>(n, chunks);
    const long long p0 = g * per, p1 = p0 + per < n ? p0 + per : n;
    double s = 0.0, ss = 0.0;
    float mn = INFINITY, mx = -INFINITY;
    for (long long p = p0 + threadIdx.x; p < p1; p += kRedThreads) {
        const int y = (int)(p / W), xx = (int)(p - (long long)y * W);
        const float v = load_f(x + c * sc + y * sh + xx * sw);
        s += (double)v;
        ss += (double)v * (double)v;
        mn = fminf(mn, v);
        mx = fmaxf(mx, v);
    }
    __shared__ double shd[kRedThreads / 32];
    __shared__ float shf[2][kRedThreads / 32];
    s = block_sum<kRedThreads>(s, shd);
    ss = block_sum<kRedThreads>(ss, shd);
    for (int o = 16; o > 0; o >>= 1) {
        mn = fminf(mn, __shfl_down_sync(0xffffffffu, mn, o));
        mx = fmaxf(mx, __shfl_down_sync(0xffffffffu, mx, o));
    }
    if ((threadIdx.x & 31) == 0) {
        shf[0][threadIdx.x >> 5] = mn;
        shf[1][threadIdx.x >> 5] = mx;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 0; w < kRedThreads / 32; ++w) {
            mn = fminf(mn, shf[0][w]);
            mx = fmaxf(mx, shf[1][w]);
        }
        part[(long long)c * chunks + g] = Partial{s, ss, mn, mx};
    }
}

// The partials of channels [c0, c1), folded in index order.
__device__ __forceinline__ Partial fold(const Partial* part, int chunks, int c0, int c1) {
    Partial r{0.0, 0.0, INFINITY, -INFINITY};
    for (long long i = (long long)c0 * chunks; i < (long long)c1 * chunks; ++i) {
        const Partial p = part[i];
        r.sum += p.sum;
        r.sumsq += p.sumsq;
        r.mn = fminf(r.mn, p.mn);
        r.mx = fmaxf(r.mx, p.mx);
    }
    return r;
}

// viz/renderer.py:380-385 on one value: out -= out.min(); out /= out.max(); out -= .5; out *= -2 (range = fl(max - min), which is
// torch's max of fl(x - min) because rounding is monotonic)
__device__ __forceinline__ float depth_norm(float v, float mn, float range) {
    return __fmul_rn(__fsub_rn(__fdiv_rn(__fsub_rn(v, mn), range), 0.5f), -2.f);
}

struct ImageArgs {
    int C, H, W, base, sel, depth, normalize, out_channels, chunks;
    long long sc, sh, sw;
    float gain;
    unsigned char* out;
    long long osh, osw, osc;
    float* stats;
    const Partial* part;
};

constexpr int kImgThreads = 256;
constexpr int kMaxSel = 1024;                   // channels whose norm a CTA keeps in shared memory

template <typename T>
__global__ void __launch_bounds__(kImgThreads) viz_image_kernel(const T* __restrict__ x, ImageArgs a) {
    __shared__ float norm[kMaxSel];
    __shared__ float glob[2];
    const int tid = threadIdx.x;
    if (a.depth && tid == 0) {
        const Partial all = fold(a.part, a.chunks, 0, a.C);
        glob[0] = all.mn;
        glob[1] = __fsub_rn(all.mx, all.mn);
    }
    __syncthreads();
    const float dmn = glob[0], drange = glob[1];
    if (a.normalize) {
        for (int j = tid; j < a.sel; j += kImgThreads) {
            const Partial p = fold(a.part, a.chunks, a.base + j, a.base + j + 1);
            float lo = p.mn, hi = p.mx;
            if (a.depth) {
                lo = depth_norm(lo, dmn, drange);
                hi = depth_norm(hi, dmn, drange);
            }
            // img.norm(inf, dim=[1, 2]).clip(1e-8, 1e8)
            norm[j] = fminf(fmaxf(fmaxf(fabsf(lo), fabsf(hi)), 1e-8f), 1e8f);
        }
    }
    if (blockIdx.x == 0 && a.stats != nullptr && tid < 2) {
        // stats: mean, std (unbiased), inf-norm of the whole map (tid 0) and of the channel window (tid 1), before any normalisation
        const Partial p = tid == 0 ? fold(a.part, a.chunks, 0, a.C) : fold(a.part, a.chunks, a.base, a.base + a.sel);
        const double n = (double)(tid == 0 ? a.C : a.sel) * a.H * a.W;
        const double mean = p.sum / n;
        const double var = (p.sumsq - p.sum * mean) / (n - 1.0);
        a.stats[0 + tid] = (float)mean;
        a.stats[2 + tid] = (float)sqrt(var > 0.0 ? var : 0.0);
        a.stats[4 + tid] = fmaxf(fabsf(p.mn), fabsf(p.mx));
    }
    __syncthreads();
    const long long npix = (long long)a.H * a.W;
    for (long long p = (long long)blockIdx.x * kImgThreads + tid; p < npix; p += (long long)gridDim.x * kImgThreads) {
        const int y = (int)(p / a.W), xx = (int)(p - (long long)y * a.W);
        unsigned char* o = a.out + y * a.osh + xx * a.osw;
        for (int j = 0; j < a.out_channels; ++j) {
            const int s = j < a.sel ? j : a.sel - 1;             // one selected channel fills every output channel (expand_as)
            float v = load_f(x + (a.base + s) * a.sc + y * a.sh + xx * a.sw);
            if (a.depth) v = depth_norm(v, dmn, drange);
            if (a.normalize) v = __fdiv_rn(v, norm[s]);
            v = __fmul_rn(v, a.gain);
            o[j * a.osc] = torch_u8(v);
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------------------- FFT

constexpr int kFftThreads = 256;
constexpr int kFftTile = 2048;
constexpr int kFftPer = kFftTile / kFftThreads;
constexpr int kFftMinN = 4, kFftMaxN = 1024;

struct FftArgs {
    int C, N, logN, H, F, logF;                 // H = N / 2 + 1 half-plane columns, F = kFftTile / N sequences per tile
    long long sc, sh, sw;
    const double* window;                       // [N]
    double* mean;                               // [C]
    double2* Y;                                 // [C, H, N]: row spectra, k2-major
    double* pc;                                 // [C, H, N]: |X|^2 per channel, k2-major
    double* P;                                  // [H, N]: sum over channels
    double* part;                               // [bins CTAs]: partial sums of the full plane
    int parts;
    float range_db;
    const unsigned char* lut;
    int K;
    unsigned char* out;
    long long osh, osw, osc;
};

template <typename T>
__global__ void __launch_bounds__(kFftThreads) viz_mean_kernel(const T* __restrict__ x, FftArgs a) {
    __shared__ double sh[kFftThreads / 32];
    const int c = blockIdx.x, N = a.N;
    double s = 0.0;
    for (int p = threadIdx.x; p < N * N; p += kFftThreads) s += (double)load_f(x + c * a.sc + (p >> a.logN) * a.sh + (p & (N - 1)) * a.sw);
    s = block_sum<kFftThreads>(s, sh);
    if (threadIdx.x == 0) a.mean[c] = s / ((double)N * N);
}

// rows: (x - mean_c) * w[n1] w[n2] -> Y[c, k2, n1] for k2 <= N / 2
template <typename T>
__global__ void __launch_bounds__(kFftThreads) viz_fft_rows_kernel(const T* __restrict__ x, FftArgs a) {
    extern __shared__ double2 viz_smem[];
    const int N = a.N;
    double2* tw = viz_smem;                                          // [N]
    double2* buf = tw + N;                                           // [F, N + 1]
    double* win = reinterpret_cast<double*>(buf + a.F * (N + 1));    // [N]
    twiddle_table<kFftThreads>(tw, N);
    for (int j = threadIdx.x; j < N; j += kFftThreads) win[j] = a.window[j];
    __syncthreads();
    const int tasks = a.C * N;                                       // task = c * N + n1
    const int tiles = ceil_div(tasks, a.F);
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int task0 = tile * a.F;
#pragma unroll 2
        for (int k = 0; k < kFftPer; ++k) {
            const int e = threadIdx.x + k * kFftThreads;
            const int f = e >> a.logN, n2 = e & (N - 1);
            const int task = task0 + f;
            double u = 0.0;
            if (task < tasks) {
                const int c = task >> a.logN, n1 = task & (N - 1);
                u = ((double)load_f(x + c * a.sc + n1 * a.sh + n2 * a.sw) - a.mean[c]) * (win[n1] * win[n2]);
            }
            buf[f * (N + 1) + n2] = make_double2(u, 0.0);
        }
        __syncthreads();
        dif_fft<kFftThreads, kFftTile>(buf, tw, N, a.logN, N);
        for (int e = threadIdx.x; e < a.F * a.H; e += kFftThreads) {
            const int f = e & (a.F - 1), m = e >> a.logF;
            const int task = task0 + f;
            if (task >= tasks) continue;
            const int c = task >> a.logN, n1 = task & (N - 1);
            a.Y[((long long)c * a.H + m) * N + n1] = buf[f * (N + 1) + bitrev(m, a.logN)];
        }
        __syncthreads();
    }
}

// columns: Y[c, k2, :] -> |X[c, k1, k2]|^2 into pc[c, k2, k1]
__global__ void __launch_bounds__(kFftThreads) viz_fft_cols_kernel(FftArgs a) {
    extern __shared__ double2 viz_smem[];
    const int N = a.N;
    double2* tw = viz_smem;
    double2* buf = tw + N;
    twiddle_table<kFftThreads>(tw, N);
    __syncthreads();
    const int tasks = a.C * a.H;                                     // task = c * H + k2
    const int tiles = ceil_div(tasks, a.F);
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int task0 = tile * a.F;
#pragma unroll 2
        for (int k = 0; k < kFftPer; ++k) {
            const int e = threadIdx.x + k * kFftThreads;
            const int f = e >> a.logN, n1 = e & (N - 1);
            const int task = task0 + f;
            buf[f * (N + 1) + n1] = task < tasks ? a.Y[(long long)task * N + n1] : make_double2(0.0, 0.0);
        }
        __syncthreads();
        dif_fft<kFftThreads, kFftTile>(buf, tw, N, a.logN, N);
        for (int e = threadIdx.x; e < kFftTile; e += kFftThreads) {
            const int f = e >> a.logN, m = e & (N - 1);
            const int task = task0 + f;
            if (task >= tasks) continue;
            const double2 z = buf[f * (N + 1) + bitrev(m, a.logN)];
            a.pc[(long long)task * N + m] = z.x * z.x + z.y * z.y;
        }
        __syncthreads();
    }
}

// P[k2, k1] = sum_c pc[c, k2, k1] in channel order; part[CTA] = this CTA's share of the full plane's sum (the columns 0 < k2 < N / 2
// stand for themselves and their mirror)
__global__ void __launch_bounds__(kFftThreads) viz_fft_sum_kernel(FftArgs a) {
    __shared__ double sh[kFftThreads / 32];
    const long long bins = (long long)a.H * a.N;
    const long long i = (long long)blockIdx.x * kFftThreads + threadIdx.x;
    double w = 0.0;
    if (i < bins) {
        double s = 0.0;
        for (int c = 0; c < a.C; ++c) s += a.pc[(long long)c * bins + i];
        a.P[i] = s;
        const int k2 = (int)(i >> a.logN);
        w = (k2 == 0 || k2 == a.N / 2) ? s : 2.0 * s;
    }
    w = block_sum<kFftThreads>(w, sh);
    if (threadIdx.x == 0) a.part[blockIdx.x] = w;
}

// panel pixel (y, x) = colormap[index of 10 log10(P[(y + N/2) % N, (x + N/2) % N] / mean P)]
__global__ void __launch_bounds__(kFftThreads) viz_fft_panel_kernel(FftArgs a) {
    __shared__ double sh[kFftThreads / 32];
    double s = 0.0;
    for (int j = threadIdx.x; j < a.parts; j += kFftThreads) s += a.part[j];
    const double mean = block_sum<kFftThreads>(s, sh) / ((double)a.N * a.N);
    const int N = a.N, hi = a.K - 1;
    const long long npix = (long long)N * N;
    for (long long p = (long long)blockIdx.x * kFftThreads + threadIdx.x; p < npix; p += (long long)gridDim.x * kFftThreads) {
        const int y = (int)(p >> a.logN), xx = (int)(p & (N - 1));
        const int k1 = (y + N / 2) & (N - 1), k2 = (xx + N / 2) & (N - 1);
        const double v = k2 <= N / 2 ? a.P[(long long)k2 * N + k1] : a.P[(long long)(N - k2) * N + ((N - k1) & (N - 1))];
        int idx = 0;                                                 // a zero bin (-inf dB) and a constant map (mean 0) give index 0
        if (mean > 0.0 && v > 0.0) {
            const double db = 10.0 * log10(v / mean);
            const double t = (db / a.range_db + 1.0) * 0.5 * hi + 0.5;
            idx = t <= 0.0 ? 0 : t >= hi ? hi : (int)t;
        }
        const unsigned char* col = a.lut + idx * 3;
        unsigned char* o = a.out + y * a.osh + xx * a.osw;
        o[0] = col[0];
        o[a.osc] = col[1];
        o[2 * a.osc] = col[2];
    }
}

int viz_chunks(int H, int W) {
    const long long c = ceil_div<long long>((long long)H * W, kPixPerChunk);
    return (int)(c < kMaxChunks ? c : kMaxChunks);
}

int fft_shape(int C, int H, int W) {
    if (H != W || H < kFftMinN || H > kFftMaxN || log2_exact(H) < 0)
        IDE3D_FAIL(IDE3D_UNSUPPORTED, "viz_fft: map %d x %d is not square with a power-of-two side in [%d, %d]", H, W, kFftMinN, kFftMaxN);
    if (C < 1) IDE3D_FAIL(IDE3D_INVALID, "viz_fft: %d channels", C);
    return IDE3D_OK;
}

// scratch layout of ide3d_viz_fft, in bytes from the start
struct FftScratch {
    long long mean, Y, pc, P, part, total;
};

FftScratch fft_scratch(int C, int N) {
    const long long H = N / 2 + 1, bins = H * N, parts = ceil_div<long long>(bins, kFftThreads);
    auto up = [](long long b) { return (b + 255) & ~255LL; };
    FftScratch s{};
    s.mean = 0;
    s.Y = up(s.mean + (long long)C * 8);
    s.pc = up(s.Y + (long long)C * bins * 16);
    s.P = up(s.pc + (long long)C * bins * 8);
    s.part = up(s.P + bins * 8);
    s.total = up(s.part + parts * 8);
    return s;
}

size_t fft_smem(int N, bool window) {
    return (size_t)(N + (kFftTile / N) * (N + 1)) * sizeof(double2) + (window ? (size_t)N * sizeof(double) : 0);
}

}  // namespace
}  // namespace ide3d

using namespace ide3d;

extern "C" int64_t ide3d_viz_image_scratch_bytes(int c, int h, int w) {
    if (c < 1 || h < 1 || w < 1) return IDE3D_INVALID;
    return (int64_t)c * viz_chunks(h, w) * (int64_t)sizeof(Partial);
}

extern "C" int ide3d_viz_image(const void* x, int dtype, int c, int h, int w, int64_t stride_c, int64_t stride_h, int64_t stride_w,
                               int base_channel, int sel_channels, int depth, int normalize, float gain, uint8_t* out, int out_channels,
                               int64_t out_stride_h, int64_t out_stride_w, int64_t out_stride_c, float* stats, void* scratch,
                               int64_t scratch_bytes, ide3d_stream_t stream) {
    IDE3D_REQUIRE(c >= 1 && h >= 1 && w >= 1, "viz_image: bad map shape [%d, %d, %d]", c, h, w);
    IDE3D_REQUIRE(dtype == IDE3D_F32 || dtype == IDE3D_F16, "viz_image: dtype %d is not float32 or float16", dtype);
    IDE3D_REQUIRE(sel_channels >= 1 && base_channel >= 0 && base_channel + sel_channels <= c,
                  "viz_image: channel window [%d, %d) outside [0, %d)", base_channel, base_channel + sel_channels, c);
    IDE3D_REQUIRE(sel_channels <= kMaxSel || !normalize, "viz_image: normalisation of more than %d channels", kMaxSel);
    IDE3D_REQUIRE(out_channels >= 1, "viz_image: %d output channels", out_channels);
    IDE3D_REQUIRE(x != nullptr && out != nullptr && scratch != nullptr, "viz_image: null map, output or scratch pointer");
    IDE3D_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 15) == 0, "viz_image: scratch must be 16-byte aligned");
    const int64_t need = ide3d_viz_image_scratch_bytes(c, h, w);
    IDE3D_REQUIRE(scratch_bytes >= need, "viz_image: scratch of %lld bytes, %lld needed", (long long)scratch_bytes, (long long)need);
    const int chunks = viz_chunks(h, w);
    cudaStream_t st = (cudaStream_t)stream;
    Partial* part = static_cast<Partial*>(scratch);
    const dim3 rgrid((unsigned)chunks, (unsigned)c);
    ImageArgs a{c, h, w, base_channel, sel_channels, depth != 0, normalize != 0, out_channels, chunks, stride_c, stride_h, stride_w, gain,
                out, out_stride_h, out_stride_w, out_stride_c, stats, part};
    const long long npix = (long long)h * w;
    const unsigned igrid = (unsigned)(ceil_div<long long>(npix, kImgThreads) < 8LL * sm_count() ? ceil_div<long long>(npix, kImgThreads)
                                                                                                 : 8LL * sm_count());
    if (dtype == IDE3D_F32) {
        viz_reduce_kernel<float><<<rgrid, kRedThreads, 0, st>>>(static_cast<const float*>(x), h, w, stride_c, stride_h, stride_w, chunks, part);
        IDE3D_CHECK_LAUNCH("viz_reduce_kernel");
        viz_image_kernel<float><<<igrid, kImgThreads, 0, st>>>(static_cast<const float*>(x), a);
    } else {
        viz_reduce_kernel<__half><<<rgrid, kRedThreads, 0, st>>>(static_cast<const __half*>(x), h, w, stride_c, stride_h, stride_w, chunks,
                                                                 part);
        IDE3D_CHECK_LAUNCH("viz_reduce_kernel");
        viz_image_kernel<__half><<<igrid, kImgThreads, 0, st>>>(static_cast<const __half*>(x), a);
    }
    IDE3D_CHECK_LAUNCH("viz_image_kernel");
    return IDE3D_OK;
}

extern "C" int64_t ide3d_viz_fft_scratch_bytes(int c, int h, int w) {
    const int rc = fft_shape(c, h, w);
    if (rc != IDE3D_OK) return rc;
    return fft_scratch(c, h).total;
}

extern "C" int ide3d_viz_fft(const void* x, int dtype, int c, int h, int w, int64_t stride_c, int64_t stride_h, int64_t stride_w,
                             const double* window, float range_db, const uint8_t* lut, int lut_size, uint8_t* out, int64_t out_stride_h,
                             int64_t out_stride_w, int64_t out_stride_c, void* scratch, int64_t scratch_bytes, ide3d_stream_t stream) {
    int rc = fft_shape(c, h, w);
    if (rc != IDE3D_OK) return rc;
    IDE3D_REQUIRE(dtype == IDE3D_F32 || dtype == IDE3D_F16, "viz_fft: dtype %d is not float32 or float16", dtype);
    IDE3D_REQUIRE(lut_size >= 1, "viz_fft: colormap of %d entries", lut_size);
    IDE3D_REQUIRE(x != nullptr && window != nullptr && lut != nullptr && out != nullptr && scratch != nullptr,
                  "viz_fft: null map, window, colormap, output or scratch pointer");
    IDE3D_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 255) == 0, "viz_fft: scratch must be 256-byte aligned");
    const FftScratch s = fft_scratch(c, h);
    IDE3D_REQUIRE(scratch_bytes >= s.total, "viz_fft: scratch of %lld bytes, %lld needed", (long long)scratch_bytes, s.total);
    const int N = h;
    char* base = static_cast<char*>(scratch);
    FftArgs a{};
    a.C = c;
    a.N = N;
    a.logN = log2_exact(N);
    a.H = N / 2 + 1;
    a.F = kFftTile / N;
    a.logF = log2_exact(a.F);
    a.sc = stride_c;
    a.sh = stride_h;
    a.sw = stride_w;
    a.window = window;
    a.mean = reinterpret_cast<double*>(base + s.mean);
    a.Y = reinterpret_cast<double2*>(base + s.Y);
    a.pc = reinterpret_cast<double*>(base + s.pc);
    a.P = reinterpret_cast<double*>(base + s.P);
    a.part = reinterpret_cast<double*>(base + s.part);
    a.parts = (int)ceil_div<long long>((long long)a.H * N, kFftThreads);
    a.range_db = range_db;
    a.lut = lut;
    a.K = lut_size;
    a.out = out;
    a.osh = out_stride_h;
    a.osw = out_stride_w;
    a.osc = out_stride_c;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t rs = fft_smem(N, true), cs = fft_smem(N, false);
    int rgrid = 0, cgrid = 0;
    if (dtype == IDE3D_F32) {
        if ((rc = persistent_grid(viz_fft_rows_kernel<float>, kFftThreads, rs, ceil_div(c * N, a.F), rgrid)) != IDE3D_OK) return rc;
    } else {
        if ((rc = persistent_grid(viz_fft_rows_kernel<__half>, kFftThreads, rs, ceil_div(c * N, a.F), rgrid)) != IDE3D_OK) return rc;
    }
    if ((rc = persistent_grid(viz_fft_cols_kernel, kFftThreads, cs, ceil_div(c * a.H, a.F), cgrid)) != IDE3D_OK) return rc;
    if (dtype == IDE3D_F32) {
        viz_mean_kernel<float><<<c, kFftThreads, 0, st>>>(static_cast<const float*>(x), a);
        IDE3D_CHECK_LAUNCH("viz_mean_kernel");
        viz_fft_rows_kernel<float><<<rgrid, kFftThreads, rs, st>>>(static_cast<const float*>(x), a);
    } else {
        viz_mean_kernel<__half><<<c, kFftThreads, 0, st>>>(static_cast<const __half*>(x), a);
        IDE3D_CHECK_LAUNCH("viz_mean_kernel");
        viz_fft_rows_kernel<__half><<<rgrid, kFftThreads, rs, st>>>(static_cast<const __half*>(x), a);
    }
    IDE3D_CHECK_LAUNCH("viz_fft_rows_kernel");
    viz_fft_cols_kernel<<<cgrid, kFftThreads, cs, st>>>(a);
    IDE3D_CHECK_LAUNCH("viz_fft_cols_kernel");
    viz_fft_sum_kernel<<<a.parts, kFftThreads, 0, st>>>(a);
    IDE3D_CHECK_LAUNCH("viz_fft_sum_kernel");
    const long long npix = (long long)N * N;
    const unsigned pgrid = (unsigned)(ceil_div<long long>(npix, kFftThreads) < 4LL * sm_count() ? ceil_div<long long>(npix, kFftThreads)
                                                                                                : 4LL * sm_count());
    viz_fft_panel_kernel<<<pgrid, kFftThreads, 0, st>>>(a);
    IDE3D_CHECK_LAUNCH("viz_fft_panel_kernel");
    return IDE3D_OK;
}
