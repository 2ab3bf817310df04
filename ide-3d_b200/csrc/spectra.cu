// Average power spectrum of avg_spectra.py `calc` (ide3d_spectrum_accum / _finalize) and the exact image moments of `stats`
// (ide3d_image_moments).
//
// The reference zero-pads each whitened, windowed N x N channel to P x P (P = N * interp) and runs a complex128 fftn over the
// whole plane.  Only the N x N block is non-zero, and with k = interp * m + r every length-P zero-padded DFT of a length-N
// sequence u is interp twiddled length-N DFTs:
//
//     U[interp * m + r] = sum_{n < N} (u[n] w_P^{n r}) w_N^{n m}.
//
// So the plane is never built.  Two passes, both float64, both radix-2 decimation-in-frequency FFTs in shared memory on tiles of
// kTile complex values (kTile / N sequences side by side, rows padded by one element against bank conflicts):
//
//   rows:    each of the N non-zero rows of every image and channel -> Y[b, c, k2, n1] for the half plane k2 <= P / 2 only (the
//            input is real, so the other half is its conjugate mirror).  Y is the caller's scratch, k2-major so that the column
//            pass reads contiguous n1.
//   columns: each (k2, r) pair owns the P / interp bins k1 = interp * m + r of column k2.  For every image in index order it
//            transforms the C channels' columns, forms mean_c |Z|^2 and adds it to a register accumulator, which starts from and
//            ends in the half-plane spectrum [P / 2 + 1, P] (k2-major).  One owner per bin, images in order: no atomics, reruns
//            are bit-identical, and the result does not depend on how the images are split into calls.
//
// Twiddles come from one table of w_P^j, j < P, built per CTA with sincospi (w_N^k = w_P^{interp k}); the CTAs are persistent.  The FFT
// itself is fft.cuh's, shared with the visualizer's FFT panel (viz.cu).
#include "fft.cuh"

namespace ide3d {
namespace {

constexpr int kThreads = 256;
constexpr int kTile = 2048;                     // complex values per FFT tile
constexpr int kPer = kTile / kThreads;          // tile elements per thread
constexpr int kMinN = 16, kMaxN = 1024, kMaxP = 4096, kMaxC = 4;

struct SpecArgs {
    const uint8_t* img;
    int64_t sn, sc, sh, sw;
    const double* lut;          // [256] (v - mean) / std
    const double* window;       // [N]
    double2* Y;                 // [B, C, H, N]
    double* S;                  // [H, P]
    int B, C, N, logN, I, logI, P, H, F, logF;
};

__global__ void __launch_bounds__(kThreads) spectrum_rows_kernel(SpecArgs a) {
    extern __shared__ double2 spec_smem[];
    double2* tw = spec_smem;                               // [P]
    double2* buf = tw + a.P;                               // [F, N + 1]
    double* lut = reinterpret_cast<double*>(buf + a.F * (a.N + 1));    // [256]
    double* win = lut + 256;                               // [N]
    twiddle_table<kThreads>(tw, a.P);
    for (int j = threadIdx.x; j < 256; j += kThreads) lut[j] = a.lut[j];
    for (int j = threadIdx.x; j < a.N; j += kThreads) win[j] = a.window[j];
    __syncthreads();

    const int N = a.N;
    const int64_t tasks = (int64_t)a.B * a.C * a.I * N;     // task = ((b * C + c) * I + r) * N + n1
    const int64_t tiles = ceil_div<int64_t>(tasks, a.F);
    for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int64_t task0 = tile * a.F;
#pragma unroll 2
        for (int k = 0; k < kPer; ++k) {
            const int e = threadIdx.x + k * kThreads;
            const int f = e >> a.logN, n2 = e & (N - 1);
            const int64_t task = task0 + f;
            double2 v = make_double2(0.0, 0.0);
            if (task < tasks) {
                const int n1 = (int)(task & (N - 1));
                const int64_t rest = task >> a.logN;
                const int r = (int)(rest & (a.I - 1));
                const int64_t bc = rest >> a.logI;
                const int b = (int)(bc / a.C), c = (int)(bc % a.C);
                const uint8_t x = a.img[b * a.sn + c * a.sc + n1 * a.sh + n2 * a.sw];
                const double u = lut[x] * (win[n1] * win[n2]);
                const double2 w = tw[(n2 * r) & (a.P - 1)];
                v = make_double2(u * w.x, u * w.y);
            }
            buf[f * (N + 1) + n2] = v;
        }
        __syncthreads();
        dif_fft<kThreads, kTile>(buf, tw, a.N, a.logN, a.P);
        // m <= N / 2 is all the half plane k2 = I m + r <= P / 2 needs
        const int outs = a.F * (N / 2 + 1);
        for (int e = threadIdx.x; e < outs; e += kThreads) {
            const int f = e & (a.F - 1), m = e >> a.logF;
            const int64_t task = task0 + f;
            if (task >= tasks) continue;
            const int n1 = (int)(task & (N - 1));
            const int64_t rest = task >> a.logN;
            const int r = (int)(rest & (a.I - 1));
            const int64_t bc = rest >> a.logI;
            const int k2 = m * a.I + r;
            if (k2 > a.P / 2) continue;
            a.Y[(bc * a.H + k2) * N + n1] = buf[f * (N + 1) + bitrev(m, a.logN)];
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kThreads) spectrum_cols_kernel(SpecArgs a) {
    extern __shared__ double2 spec_smem[];
    double2* tw = spec_smem;
    double2* buf = tw + a.P;
    twiddle_table<kThreads>(tw, a.P);
    __syncthreads();

    const int N = a.N;
    const int tasks = a.H * a.I;                           // task = k2 * I + r, owns bins (k1 = I m + r, k2)
    const int tiles = ceil_div(tasks, a.F);
    const double nc = a.C;
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int task0 = tile * a.F;
        double acc[kPer];
        int64_t bin[kPer];
#pragma unroll
        for (int k = 0; k < kPer; ++k) {                   // output element e -> (f, m): consecutive f are consecutive k1
            const int e = threadIdx.x + k * kThreads;
            const int f = e & (a.F - 1), m = e >> a.logF;
            const int task = task0 + f;
            bin[k] = task < tasks ? (int64_t)(task >> a.logI) * a.P + m * a.I + (task & (a.I - 1)) : -1;
            acc[k] = bin[k] >= 0 ? a.S[bin[k]] : 0.0;
        }
        for (int b = 0; b < a.B; ++b) {
            double pw[kPer];
#pragma unroll
            for (int k = 0; k < kPer; ++k) pw[k] = 0.0;
            for (int c = 0; c < a.C; ++c) {
                const double2* Yc = a.Y + (int64_t)(b * a.C + c) * a.H * N;
#pragma unroll 2
                for (int k = 0; k < kPer; ++k) {
                    const int e = threadIdx.x + k * kThreads;
                    const int f = e >> a.logN, n1 = e & (N - 1);
                    const int task = task0 + f;
                    double2 v = make_double2(0.0, 0.0);
                    if (task < tasks) v = cmul(Yc[(int64_t)(task >> a.logI) * N + n1], tw[(n1 * (task & (a.I - 1))) & (a.P - 1)]);
                    buf[f * (N + 1) + n1] = v;
                }
                __syncthreads();
                dif_fft<kThreads, kTile>(buf, tw, a.N, a.logN, a.P);
#pragma unroll
                for (int k = 0; k < kPer; ++k) {
                    const int e = threadIdx.x + k * kThreads;
                    const int f = e & (a.F - 1), m = e >> a.logF;
                    const double2 z = buf[f * (N + 1) + bitrev(m, a.logN)];
                    pw[k] += z.x * z.x + z.y * z.y;
                }
                __syncthreads();
            }
#pragma unroll
            for (int k = 0; k < kPer; ++k) acc[k] += pw[k] / nc;
        }
#pragma unroll
        for (int k = 0; k < kPer; ++k)
            if (bin[k] >= 0) a.S[bin[k]] = acc[k];
    }
}

// out[k1, k2] = S[k2, k1] / count for k2 <= P / 2, else the conjugate mirror S[P - k2, -k1 mod P] / count
__global__ void __launch_bounds__(256) spectrum_finalize_kernel(const double* __restrict__ S, int P, double count, double* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= (int64_t)P * P) return;
    const int k1 = (int)(i / P), k2 = (int)(i % P);
    const double v = k2 <= P / 2 ? S[(int64_t)k2 * P + k1] : S[(int64_t)(P - k2) * P + ((P - k1) & (P - 1))];
    out[i] = v / count;
}

// moments[0] += number of values, moments[1] += sum x, moments[2] += sum x^2 (exact integers; integer atomics are order-free)
__global__ void __launch_bounds__(256) image_moments_kernel(const uint8_t* __restrict__ img, int C, int H, int W, int64_t rows,
                                                            int64_t sn, int64_t sc, int64_t sh, int64_t sw,
                                                            unsigned long long* __restrict__ moments) {
    unsigned long long s1 = 0, s2 = 0;
    for (int64_t row = blockIdx.x; row < rows; row += gridDim.x) {
        const int y = (int)(row % H);
        const int64_t bc = row / H;
        const uint8_t* p = img + (bc / C) * sn + (bc % C) * sc + y * sh;
        for (int x = threadIdx.x; x < W; x += 256) {
            const unsigned v = p[x * sw];
            s1 += v;
            s2 += v * v;
        }
    }
    for (int o = 16; o > 0; o >>= 1) {
        s1 += __shfl_down_sync(0xffffffffu, s1, o);
        s2 += __shfl_down_sync(0xffffffffu, s2, o);
    }
    __shared__ unsigned long long part[2][8];
    if ((threadIdx.x & 31) == 0) {
        part[0][threadIdx.x >> 5] = s1;
        part[1][threadIdx.x >> 5] = s2;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; ++w) {
            s1 += part[0][w];
            s2 += part[1][w];
        }
        if (blockIdx.x == 0) atomicAdd(moments, (unsigned long long)rows * W);
        atomicAdd(moments + 1, s1);
        atomicAdd(moments + 2, s2);
    }
}

// IDE3D_UNSUPPORTED for a shape the kernels do not cover, IDE3D_OK otherwise
int spectrum_shape(const char* fn, int C, int N, int interp) {
    if (N < kMinN || N > kMaxN || log2_exact(N) < 0)
        IDE3D_FAIL(IDE3D_UNSUPPORTED, "%s: image size %d is not a power of two in [%d, %d]", fn, N, kMinN, kMaxN);
    if (interp != 1 && interp != 2 && interp != 4 && interp != 8) IDE3D_FAIL(IDE3D_UNSUPPORTED, "%s: interp %d not in {1, 2, 4, 8}", fn, interp);
    if (N * interp > kMaxP) IDE3D_FAIL(IDE3D_UNSUPPORTED, "%s: spectrum size %d exceeds %d", fn, N * interp, kMaxP);
    if (C < 1 || C > kMaxC) IDE3D_FAIL(IDE3D_UNSUPPORTED, "%s: %d channels outside [1, %d]", fn, C, kMaxC);
    return IDE3D_OK;
}

size_t rows_smem(int N, int P) { return (size_t)(P + (kTile / N) * (N + 1)) * sizeof(double2) + (size_t)(256 + N) * sizeof(double); }
size_t cols_smem(int N, int P) { return (size_t)(P + (kTile / N) * (N + 1)) * sizeof(double2); }

}  // namespace
}  // namespace ide3d

using namespace ide3d;

extern "C" int64_t ide3d_spectrum_scratch_bytes(int n, int c, int size, int interp) {
    if (n < 0) return IDE3D_INVALID;
    if (spectrum_shape("spectrum_scratch_bytes", c, size, interp) != IDE3D_OK) return IDE3D_UNSUPPORTED;
    const int64_t H = (int64_t)size * interp / 2 + 1;
    return (int64_t)n * c * H * size * (int64_t)sizeof(double2);
}

extern "C" int ide3d_spectrum_accum(const uint8_t* images, int n, int c, int size, int64_t stride_n, int64_t stride_c, int64_t stride_h,
                                    int64_t stride_w, const double* lut, const double* window, int interp, double* spectrum, void* scratch,
                                    int64_t scratch_bytes, ide3d_stream_t stream) {
    IDE3D_REQUIRE(n >= 0, "spectrum_accum: negative image count %d", n);
    int rc = spectrum_shape("spectrum_accum", c, size, interp);
    if (rc != IDE3D_OK) return rc;
    IDE3D_REQUIRE(lut != nullptr && window != nullptr && spectrum != nullptr, "spectrum_accum: null lut, window or spectrum pointer");
    IDE3D_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 15) == 0, "spectrum_accum: scratch must be 16-byte aligned");
    const int64_t need = ide3d_spectrum_scratch_bytes(n, c, size, interp);
    IDE3D_REQUIRE(scratch_bytes >= need, "spectrum_accum: scratch of %lld bytes, %lld needed", (long long)scratch_bytes, (long long)need);
    if (n == 0) return IDE3D_OK;
    IDE3D_REQUIRE(images != nullptr && scratch != nullptr, "spectrum_accum: null images or scratch pointer");
    SpecArgs a{};
    a.img = images;
    a.sn = stride_n;
    a.sc = stride_c;
    a.sh = stride_h;
    a.sw = stride_w;
    a.lut = lut;
    a.window = window;
    a.Y = static_cast<double2*>(scratch);
    a.S = spectrum;
    a.B = n;
    a.C = c;
    a.N = size;
    a.logN = log2_exact(size);
    a.I = interp;
    a.logI = log2_exact(interp);
    a.P = size * interp;
    a.H = a.P / 2 + 1;
    a.F = kTile / size;
    a.logF = log2_exact(a.F);
    cudaStream_t st = (cudaStream_t)stream;
    int grid = 0;
    const size_t rs = rows_smem(size, a.P), cs = cols_smem(size, a.P);
    if ((rc = persistent_grid(spectrum_rows_kernel, kThreads, rs, ceil_div<int64_t>((int64_t)n * c * interp * size, a.F), grid)) != IDE3D_OK)
        return rc;
    spectrum_rows_kernel<<<grid, kThreads, rs, st>>>(a);
    IDE3D_CHECK_LAUNCH("spectrum_rows_kernel");
    if ((rc = persistent_grid(spectrum_cols_kernel, kThreads, cs, ceil_div(a.H * interp, a.F), grid)) != IDE3D_OK) return rc;
    spectrum_cols_kernel<<<grid, kThreads, cs, st>>>(a);
    IDE3D_CHECK_LAUNCH("spectrum_cols_kernel");
    return IDE3D_OK;
}

extern "C" int ide3d_spectrum_finalize(const double* spectrum, int size, int interp, int64_t count, double* out, ide3d_stream_t stream) {
    int rc = spectrum_shape("spectrum_finalize", 1, size, interp);
    if (rc != IDE3D_OK) return rc;
    IDE3D_REQUIRE(spectrum != nullptr && out != nullptr, "spectrum_finalize: null spectrum or output pointer");
    IDE3D_REQUIRE(count >= 1, "spectrum_finalize: image count %lld < 1", (long long)count);
    const int P = size * interp;
    spectrum_finalize_kernel<<<(unsigned)ceil_div<int64_t>((int64_t)P * P, 256), 256, 0, (cudaStream_t)stream>>>(spectrum, P, (double)count, out);
    IDE3D_CHECK_LAUNCH("spectrum_finalize_kernel");
    return IDE3D_OK;
}

extern "C" int ide3d_image_moments(const uint8_t* images, int n, int c, int h, int w, int64_t stride_n, int64_t stride_c, int64_t stride_h,
                                   int64_t stride_w, uint64_t* moments, ide3d_stream_t stream) {
    IDE3D_REQUIRE(n >= 0 && c >= 1 && h >= 1 && w >= 1, "image_moments: bad shape [%d, %d, %d, %d]", n, c, h, w);
    IDE3D_REQUIRE(moments != nullptr, "image_moments: null moments pointer");
    IDE3D_REQUIRE((reinterpret_cast<uintptr_t>(moments) & 7) == 0, "image_moments: moments must be 8-byte aligned");
    if (n == 0) return IDE3D_OK;
    IDE3D_REQUIRE(images != nullptr, "image_moments: null images pointer");
    const int64_t rows = (int64_t)n * c * h;
    const unsigned grid = (unsigned)(rows < 4LL * sm_count() ? rows : 4LL * sm_count());
    image_moments_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(images, c, h, w, rows, stride_n, stride_c, stride_h, stride_w,
                                                                 reinterpret_cast<unsigned long long*>(moments));
    IDE3D_CHECK_LAUNCH("image_moments_kernel");
    return IDE3D_OK;
}
