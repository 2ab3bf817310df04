// PIL.Image.resize(size, LANCZOS) of 8-bit L and RGB images (ide3d_resample_u8): Pillow's ImagingResample (libImaging/Resample.c),
// reproduced bit for bit.  The caller builds each axis's integer tables with Pillow's own double arithmetic (precompute_coeffs,
// normalize_coeffs_8bpc); the kernels run Pillow's two integer passes on them:
//
//   horizontal: for each kept row, out[x] = clip8(2^21 + sum_i in[xmin + i] * kx[x][i]) into a uint8 intermediate of the rows the
//               vertical pass reads (Pillow's ybox_first .. ybox_last), or straight into the output when the vertical pass is skipped;
//   vertical:   out[y] = clip8(2^21 + sum_i tmp[ymin + i] * ky[y][i]), from the intermediate, or from the input when the
//               horizontal pass is skipped.
//
// A pass is skipped exactly when Pillow skips it (its axis keeps its size), because a skipped pass also skips a rounding; with both
// skipped the call is a copy.  int32 accumulation as in Pillow: 22 fractional bits leave room for 255 * sum |k| without overflow.
#include "common.cuh"

namespace ide3d {
namespace {

constexpr int kPrecisionBits = 22;
constexpr int kThreads = 128;

__device__ __forceinline__ uint8_t clip8(int v) {
    if (v >= (1 << kPrecisionBits << 8)) return 255;
    if (v <= 0) return 0;
    return (uint8_t)(v >> kPrecisionBits);
}

struct Plane {                  // uint8 [n, h, w, C] through byte strides, channels contiguous
    const uint8_t* p;
    int64_t sn, sh, sw;
};

struct OutPlane {
    uint8_t* p;
    int64_t sn, sh, sw;
};

// rows r < rows of every image: out row r = horizontal resample of input row row0 + r
template <int C>
__global__ void __launch_bounds__(kThreads) resample_h_kernel(Plane in, int row0, OutPlane out, int out_w, int rows, int n,
                                                              const int32_t* __restrict__ bounds, const int32_t* __restrict__ coeffs,
                                                              int ksize) {
    const int x = blockIdx.x * kThreads + threadIdx.x;
    if (x >= out_w) return;
    const int xmin = bounds[2 * x], xmax = bounds[2 * x + 1];
    const int32_t* k = coeffs + (int64_t)x * ksize;
    for (int64_t rb = blockIdx.y; rb < (int64_t)n * rows; rb += gridDim.y) {
        const int b = (int)(rb / rows), r = (int)(rb % rows);
        const uint8_t* src = in.p + b * in.sn + (int64_t)(row0 + r) * in.sh + (int64_t)xmin * in.sw;
        int ss[C];
#pragma unroll
        for (int c = 0; c < C; ++c) ss[c] = 1 << (kPrecisionBits - 1);
        for (int i = 0; i < xmax; ++i) {
            const int w = __ldg(k + i);
#pragma unroll
            for (int c = 0; c < C; ++c) ss[c] += (int)src[i * in.sw + c] * w;
        }
        uint8_t* dst = out.p + b * out.sn + (int64_t)r * out.sh + (int64_t)x * out.sw;
#pragma unroll
        for (int c = 0; c < C; ++c) dst[c] = clip8(ss[c]);
    }
}

// output row y of every image = vertical resample of source rows bounds[2y] - row0 .. + bounds[2y + 1]
template <int C>
__global__ void __launch_bounds__(kThreads) resample_v_kernel(Plane in, int row0, OutPlane out, int out_w, int out_h, int n,
                                                              const int32_t* __restrict__ bounds, const int32_t* __restrict__ coeffs,
                                                              int ksize) {
    const int x = blockIdx.x * kThreads + threadIdx.x;
    if (x >= out_w) return;
    for (int64_t yb = blockIdx.y; yb < (int64_t)n * out_h; yb += gridDim.y) {
        const int b = (int)(yb / out_h), y = (int)(yb % out_h);
        const int ymin = bounds[2 * y] - row0, ymax = bounds[2 * y + 1];
        const int32_t* k = coeffs + (int64_t)y * ksize;
        const uint8_t* src = in.p + b * in.sn + (int64_t)ymin * in.sh + (int64_t)x * in.sw;
        int ss[C];
#pragma unroll
        for (int c = 0; c < C; ++c) ss[c] = 1 << (kPrecisionBits - 1);
        for (int i = 0; i < ymax; ++i) {
            const int w = __ldg(k + i);
#pragma unroll
            for (int c = 0; c < C; ++c) ss[c] += (int)src[i * in.sh + c] * w;
        }
        uint8_t* dst = out.p + b * out.sn + (int64_t)y * out.sh + (int64_t)x * out.sw;
#pragma unroll
        for (int c = 0; c < C; ++c) dst[c] = clip8(ss[c]);
    }
}

template <int C>
__global__ void __launch_bounds__(kThreads) resample_copy_kernel(Plane in, OutPlane out, int w, int h, int n) {
    const int x = blockIdx.x * kThreads + threadIdx.x;
    if (x >= w) return;
    for (int64_t yb = blockIdx.y; yb < (int64_t)n * h; yb += gridDim.y) {
        const int b = (int)(yb / h), y = (int)(yb % h);
        const uint8_t* src = in.p + b * in.sn + (int64_t)y * in.sh + (int64_t)x * in.sw;
        uint8_t* dst = out.p + b * out.sn + (int64_t)y * out.sh + (int64_t)x * out.sw;
#pragma unroll
        for (int c = 0; c < C; ++c) dst[c] = src[c];
    }
}

int64_t align16(int64_t v) { return (v + 15) & ~(int64_t)15; }

int64_t table_bytes(int out, int ksize) { return align16((int64_t)out * ksize * 4) + align16((int64_t)out * 2 * 4); }

// every output position's taps lie in [0, in) (and in [lo, hi) for the vertical table) and number at most ksize
int check_table(const char* axis, const int32_t* bounds, int out, int in, int ksize, int lo, int hi) {
    for (int i = 0; i < out; ++i) {
        const int first = bounds[2 * i], count = bounds[2 * i + 1];
        if (lo < 0 || first < lo || count < 0 || count > ksize || (int64_t)first + count > hi || hi > in)
            IDE3D_FAIL(IDE3D_INVALID, "resample_u8: %s table entry %d (first %d, %d taps) does not fit input size %d, ksize %d", axis, i,
                       first, count, in, ksize);
    }
    return IDE3D_OK;
}

template <int C>
int launch(Plane in, int n, int in_h, int in_w, OutPlane out, int out_h, int out_w, const int32_t* bx, const int32_t* kx, int ksize_x,
           const int32_t* by, const int32_t* ky, int ksize_y, int ybox_first, int ybox_rows, uint8_t* tmp, cudaStream_t st) {
    const bool need_h = out_w != in_w, need_v = out_h != in_h;
    auto grid = [&](int w, int rows) {
        const int64_t ys = (int64_t)n * rows;
        return dim3((unsigned)ceil_div(w, kThreads), (unsigned)(ys < 65535 ? ys : 65535));
    };
    if (!need_h && !need_v) {
        resample_copy_kernel<C><<<grid(out_w, out_h), kThreads, 0, st>>>(in, out, out_w, out_h, n);
        IDE3D_CHECK_LAUNCH("resample_copy_kernel");
        return IDE3D_OK;
    }
    Plane vsrc = in;
    int row0 = 0;
    if (need_h) {
        OutPlane hdst = out;
        int rows = out_h, first = 0;
        if (need_v) {
            hdst = OutPlane{tmp, (int64_t)ybox_rows * out_w * C, (int64_t)out_w * C, C};
            rows = ybox_rows;
            first = ybox_first;
        }
        resample_h_kernel<C><<<grid(out_w, rows), kThreads, 0, st>>>(in, first, hdst, out_w, rows, n, bx, kx, ksize_x);
        IDE3D_CHECK_LAUNCH("resample_h_kernel");
        if (!need_v) return IDE3D_OK;
        vsrc = Plane{tmp, hdst.sn, hdst.sh, hdst.sw};
        row0 = ybox_first;
    }
    resample_v_kernel<C><<<grid(out_w, out_h), kThreads, 0, st>>>(vsrc, row0, out, out_w, out_h, n, by, ky, ksize_y);
    IDE3D_CHECK_LAUNCH("resample_v_kernel");
    return IDE3D_OK;
}

}  // namespace
}  // namespace ide3d

using namespace ide3d;

extern "C" int64_t ide3d_resample_u8_scratch_bytes(int n, int c, int in_h, int out_h, int out_w, int ksize_x, int ksize_y) {
    if (n < 1 || (c != 1 && c != 3) || in_h < 1 || out_h < 1 || out_w < 1 || ksize_x < 1 || ksize_y < 1) return IDE3D_INVALID;
    return table_bytes(out_w, ksize_x) + table_bytes(out_h, ksize_y) + align16((int64_t)n * in_h * out_w * c);
}

extern "C" int ide3d_resample_u8(const uint8_t* in, int n, int c, int in_h, int in_w, int64_t in_stride_n, int64_t in_stride_h,
                                 int64_t in_stride_w, uint8_t* out, int out_h, int out_w, int64_t out_stride_n, int64_t out_stride_h,
                                 int64_t out_stride_w, int ksize_x, const int32_t* bounds_x, const int32_t* coeffs_x, int ksize_y,
                                 const int32_t* bounds_y, const int32_t* coeffs_y, void* scratch, int64_t scratch_bytes,
                                 ide3d_stream_t stream) {
    IDE3D_REQUIRE(in != nullptr && out != nullptr, "resample_u8: null input or output pointer");
    IDE3D_REQUIRE(bounds_x != nullptr && coeffs_x != nullptr && bounds_y != nullptr && coeffs_y != nullptr,
                  "resample_u8: null table pointer");
    IDE3D_REQUIRE(c == 1 || c == 3, "resample_u8: %d channels, need 1 (L) or 3 (RGB)", c);
    IDE3D_REQUIRE(n >= 1 && in_h >= 1 && in_w >= 1 && out_h >= 1 && out_w >= 1, "resample_u8: bad sizes n %d, in %dx%d, out %dx%d", n,
                  in_w, in_h, out_w, out_h);
    IDE3D_REQUIRE(ksize_x >= 1 && ksize_y >= 1, "resample_u8: bad ksize %d, %d", ksize_x, ksize_y);
    int rc = check_table("horizontal", bounds_x, out_w, in_w, ksize_x, 0, in_w);
    if (rc != IDE3D_OK) return rc;
    const int ybox_first = bounds_y[0], ybox_last = bounds_y[2 * (out_h - 1)] + bounds_y[2 * (out_h - 1) + 1];
    rc = check_table("vertical", bounds_y, out_h, in_h, ksize_y, ybox_first, ybox_last);
    if (rc != IDE3D_OK) return rc;
    IDE3D_REQUIRE(scratch != nullptr, "resample_u8: null scratch pointer");
    IDE3D_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 15) == 0, "resample_u8: scratch must be 16-byte aligned");
    const int64_t need = ide3d_resample_u8_scratch_bytes(n, c, in_h, out_h, out_w, ksize_x, ksize_y);
    IDE3D_REQUIRE(scratch_bytes >= need, "resample_u8: scratch of %lld bytes, %lld needed", (long long)scratch_bytes, (long long)need);

    uint8_t* s = static_cast<uint8_t*>(scratch);
    int32_t* kx = reinterpret_cast<int32_t*>(s);
    int32_t* bx = reinterpret_cast<int32_t*>(s + align16((int64_t)out_w * ksize_x * 4));
    s += table_bytes(out_w, ksize_x);
    int32_t* ky = reinterpret_cast<int32_t*>(s);
    int32_t* by = reinterpret_cast<int32_t*>(s + align16((int64_t)out_h * ksize_y * 4));
    uint8_t* tmp = s + table_bytes(out_h, ksize_y);
    cudaStream_t st = (cudaStream_t)stream;
    // pageable sources: each copy is staged before the call returns, so the caller may free its tables
    IDE3D_CUDA(cudaMemcpyAsync(kx, coeffs_x, (size_t)out_w * ksize_x * 4, cudaMemcpyHostToDevice, st));
    IDE3D_CUDA(cudaMemcpyAsync(bx, bounds_x, (size_t)out_w * 2 * 4, cudaMemcpyHostToDevice, st));
    IDE3D_CUDA(cudaMemcpyAsync(ky, coeffs_y, (size_t)out_h * ksize_y * 4, cudaMemcpyHostToDevice, st));
    IDE3D_CUDA(cudaMemcpyAsync(by, bounds_y, (size_t)out_h * 2 * 4, cudaMemcpyHostToDevice, st));

    const Plane ip{in, in_stride_n, in_stride_h, in_stride_w};
    const OutPlane op{out, out_stride_n, out_stride_h, out_stride_w};
    const int rows = ybox_last - ybox_first;
    return c == 3 ? launch<3>(ip, n, in_h, in_w, op, out_h, out_w, bx, kx, ksize_x, by, ky, ksize_y, ybox_first, rows, tmp, st)
                  : launch<1>(ip, n, in_h, in_w, op, out_h, out_w, bx, kx, ksize_x, by, ky, ksize_y, ybox_first, rows, tmp, st);
}
