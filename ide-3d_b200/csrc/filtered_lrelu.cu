// filtered_lrelu for sm_90a.
//   ide3d_filtered_lrelu_act : in-place gain * lrelu * clamp with 2-bit sign write / read -- the activation
//                              stage of the generic composition (filtered_lrelu.cu:1105-1211,
//                              filtered_lrelu.cpp:213-290).
//   ide3d_filtered_lrelu     : fused bias -> up-FIR -> act -> down-FIR (filtered_lrelu.cu:139-1099).
//                              Returns IDE3D_UNSUPPORTED for configurations without a fused kernel, which the
//                              caller resolves exactly like the reference's return code -1
//                              (filtered_lrelu.cpp:52-56, filtered_lrelu.py:223-229): upfirdn2d + act + upfirdn2d.
//
// Sign tensor (filtered_lrelu.cpp:82-96): uint8 [N, C, s_h, s_w/4], 2 bits per element, 4 elements per byte
// in x order; code 1 = value was negative (backward multiplies by slope), code 2 = value was clamped
// (backward gradient is 0; clamp wins over sign).  Filters are kernel arguments / shared memory here, never
// global __constant__ state, so concurrent streams are safe (the reference is not: filtered_lrelu.cu:77-78).
#include "common.cuh"
#include "elem.cuh"
#include "filtered_lrelu.cuh"

namespace ide3d {

struct ActArgs {
    void* x;
    unsigned char* s;
    int xw, xh, xc, xn;
    long long sxw, sxh, sxc, sxn;
    int sw, sh, sox, soy;
    float gain, slope, clamp;
};

// MODE 0: plain forward, 1: write signs, 2: read signs.  One thread per element in x; a 16-lane group
// owns one 32-bit word of the sign tensor (16 elements * 2 bits).
template <typename T, int MODE>
__global__ void __launch_bounds__(256) lrelu_act_kernel(const ActArgs p) {
    const int lane16 = threadIdx.x & 15;
    const int width = (MODE == 1) ? p.sw : p.xw;              // launch covers the sign row when writing
    const int height = (MODE == 1) ? p.sh : p.xh;
    const long long planes = (long long)p.xc * p.xn;
    const long long words_x = (width + 15) >> 4;              // 16-element groups per row
    const long long total = planes * height * words_x * 16;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long grp = i >> 4;
        const int gx = (int)(grp % words_x);
        long long r = grp / words_x;
        const int y = (int)(r % height);
        const long long q = r / height;                       // n*C + c
        const int x = gx * 16 + lane16;
        const int n = (int)(q / p.xc), c = (int)(q - (long long)n * p.xc);
        T* pv = (T*)p.x + n * p.sxn + c * p.sxc + (long long)y * p.sxh + (long long)x * p.sxw;
        if (MODE == 1) {
            unsigned s = 0;
            if (x < p.xw && y < p.xh) {
                float v = load_f32<T>(pv) * p.gain;
                if (v < 0.f) { v *= p.slope; s = 1; }
                if (fabsf(v) > p.clamp) { v = (v < 0.f) ? -p.clamp : p.clamp; s = 2; }
                store_f32<T>(pv, v);
            }
            s <<= (lane16 << 1);
            const unsigned m = (threadIdx.x & 16) ? 0xffff0000u : 0x0000ffffu;
            s |= __shfl_xor_sync(m, s, 1);
            s |= __shfl_xor_sync(m, s, 2);
            s |= __shfl_xor_sync(m, s, 4);
            s |= __shfl_xor_sync(m, s, 8);
            if (lane16 == 0 && x < p.sw) {
                const long long is = x + (long long)p.sw * (y + (long long)p.sh * q);
                reinterpret_cast<unsigned*>(p.s)[is >> 4] = s;
            }
        } else if (x < p.xw) {
            float v = load_f32<T>(pv) * p.gain;
            if (MODE == 2) {
                const unsigned sx = (unsigned)(x + p.sox), sy = (unsigned)(y + p.soy);
                if (sx < (unsigned)p.sw && sy < (unsigned)p.sh) {
                    const long long is = (sx >> 2) + (long long)(p.sw >> 2) * (sy + (long long)p.sh * q);
                    unsigned s = p.s[is];
                    s >>= (sx & 3) << 1;
                    if (s & 1) v *= p.slope;
                    if (s & 2) v = 0.f;
                }
            } else {
                if (v < 0.f) v *= p.slope;
                if (fabsf(v) > p.clamp) v = (v < 0.f) ? -p.clamp : p.clamp;
            }
            store_f32<T>(pv, v);
        }
    }
}

template <typename T>
static int launch_act(const ActArgs& a, int write_signs, int read_signs, cudaStream_t st) {
    const int width = write_signs ? a.sw : a.xw, height = write_signs ? a.sh : a.xh;
    const long long total = (long long)a.xc * a.xn * height * ((width + 15) >> 4) * 16;
    const unsigned grid = capped_grid(ceil_div<long long>(total, 256), 16);
    if (write_signs) lrelu_act_kernel<T, 1><<<grid, 256, 0, st>>>(a);
    else if (read_signs) lrelu_act_kernel<T, 2><<<grid, 256, 0, st>>>(a);
    else lrelu_act_kernel<T, 0><<<grid, 256, 0, st>>>(a);
    IDE3D_CHECK_LAUNCH("lrelu_act_kernel");
    return IDE3D_OK;
}

}  // namespace ide3d

using namespace ide3d;

extern "C" int ide3d_filtered_lrelu_act(const ide3d_filtered_lrelu_act_params* q, ide3d_stream_t stream) {
    IDE3D_REQUIRE(q && q->x, "filtered_lrelu_act: null tensor");
    IDE3D_REQUIRE(q->x_w > 0 && q->x_h > 0 && q->x_c > 0 && q->x_n > 0, "x is empty");
    IDE3D_REQUIRE(!(q->write_signs && q->read_signs), "filtered_lrelu_act: cannot read and write signs at once");
    if (q->write_signs || q->read_signs) {
        IDE3D_REQUIRE(q->s != nullptr, "signs tensor missing");
        IDE3D_REQUIRE(q->s_w > 0 && q->s_h > 0 && (q->s_w & 3) == 0, "signs width must be a positive multiple of 4 elements");
        if (q->write_signs) {
            IDE3D_REQUIRE((q->s_w & 15) == 0, "written signs width must be a multiple of 16 elements");
            IDE3D_REQUIRE(q->s_w >= q->x_w && q->s_h >= q->x_h, "signs tensor smaller than x");
            IDE3D_REQUIRE((reinterpret_cast<uintptr_t>(q->s) & 3) == 0, "signs tensor must be 4-byte aligned");
        }
    }
    ActArgs a;
    a.x = q->x; a.s = q->s;
    a.xw = q->x_w; a.xh = q->x_h; a.xc = q->x_c; a.xn = q->x_n;
    a.sxw = q->x_stride_w; a.sxh = q->x_stride_h; a.sxc = q->x_stride_c; a.sxn = q->x_stride_n;
    a.sw = q->s_w; a.sh = q->s_h; a.sox = q->s_ofs_x; a.soy = q->s_ofs_y;
    a.gain = q->gain; a.slope = q->slope; a.clamp = q->clamp;
    cudaStream_t st = (cudaStream_t)stream;
    switch (q->dtype) {
        case IDE3D_F32: return launch_act<float>(a, q->write_signs, q->read_signs, st);
        case IDE3D_F16: return launch_act<__half>(a, q->write_signs, q->read_signs, st);
        case IDE3D_F64: return launch_act<double>(a, q->write_signs, q->read_signs, st);
    }
    IDE3D_FAIL(IDE3D_INVALID, "filtered_lrelu_act: unsupported dtype %d", q->dtype);
}

extern "C" int ide3d_filtered_lrelu(const ide3d_filtered_lrelu_params* q, ide3d_stream_t stream) {
    IDE3D_REQUIRE(q && q->x && q->y && q->fu && q->fd, "filtered_lrelu: null tensor");
    IDE3D_REQUIRE(q->dtype == IDE3D_F32 || q->dtype == IDE3D_F16, "x and b must be float16 or float32");
    IDE3D_REQUIRE(q->up >= 1 && q->down >= 1, "up and down must be at least 1");
    IDE3D_REQUIRE(q->x_c > 0 && q->x_n > 0 && q->y_w > 0 && q->y_h > 0, "filtered_lrelu: y is empty");
    IDE3D_REQUIRE(!(q->write_signs && q->read_signs), "filtered_lrelu: cannot read and write signs at once");
    // separable filters only (fu_h == 0), or 1x1 "full" filters when the factor is 1 (filtered_lrelu.py:178-181)
    const bool fu_ok = (q->fu_h == 0) || (q->fu_h == 1 && q->fu_w == 1);
    const bool fd_ok = (q->fd_h == 0) || (q->fd_h == 1 && q->fd_w == 1);
    if (!fu_ok || !fd_ok) IDE3D_FAIL(IDE3D_UNSUPPORTED, "filtered_lrelu: no fused kernel for 2-D filters %dx%d / %dx%d", q->fu_w, q->fu_h, q->fd_w, q->fd_h);
    if (q->write_signs || q->read_signs) {
        IDE3D_REQUIRE(q->s != nullptr && q->s_w > 0 && q->s_h > 0 && (q->s_w & 3) == 0, "signs tensor missing or malformed");
        if (q->write_signs) IDE3D_REQUIRE((q->s_w & 15) == 0 && (reinterpret_cast<uintptr_t>(q->s) & 3) == 0, "written signs need 16-element rows, 4-byte alignment");
    }
    FlFusedArgs a;
    a.x = q->x; a.b = q->b; a.fu = q->fu; a.fd = q->fd; a.y = q->y; a.s = q->s;
    a.px0 = q->pad_x0; a.py0 = q->pad_y0; a.flip = q->flip;
    a.gain = q->gain; a.slope = q->slope; a.clamp = q->clamp;
    a.xw = q->x_w; a.xh = q->x_h; a.xc = q->x_c; a.xn = q->x_n;
    a.sxw = q->x_stride_w; a.sxh = q->x_stride_h; a.sxc = q->x_stride_c; a.sxn = q->x_stride_n;
    a.yw = q->y_w; a.yh = q->y_h;
    a.syw = q->y_stride_w; a.syh = q->y_stride_h; a.syc = q->y_stride_c; a.syn = q->y_stride_n;
    a.sw = q->s_w; a.sh = q->s_h; a.sox = q->s_ofs_x; a.soy = q->s_ofs_y;
    a.mode = q->write_signs ? 1 : (q->read_signs ? 2 : 0);
    a.one_u = (q->fu_h == 1 && q->fu_w == 1); a.one_d = (q->fd_h == 1 && q->fd_w == 1);   // value applied once, not per axis
    cudaStream_t st = (cudaStream_t)stream;
    if (q->write_signs) IDE3D_CUDA(cudaMemsetAsync(q->s, 0, (size_t)q->x_n * q->x_c * q->s_h * (q->s_w >> 2), st));
    // channels-last tensors (unit channel stride, more than one channel) take the channel-blocked tiling
    a.channels_last = (q->x_stride_c == 1 && q->x_c > 1 && q->x_stride_w != 1) ? 1 : 0;
    return launch_filtered_lrelu_fused(a, q->dtype, q->up, q->down, q->fu_w, q->fd_w, st);
}
