// bias_act for sm_90a: y = clamp(gain * act(x + b)) plus the 1st/2nd-order gradient forms.
// Replaces bias_act_kernel<T,A> (torch_utils/ops/bias_act.cu:23-147) behind the same parameter set
// (bias_act.h:12-31).  Pure HBM stream: 2 * size_x * sizeof(T) algorithmic bytes (+ aux tensors for
// the gradient forms).  128-bit loads/stores, 4 vectors in flight per thread, 64-bit indexing, grid
// sized to the SM count (grid-stride loop).
#include "common.cuh"

namespace ide3d {

struct BiasActArgs {
    const void *x, *b, *xref, *yref, *dy;
    void* y;
    int grad;
    float alpha, gain, clamp;
    long long size_x, size_b, step_b;
};

template <typename T> struct Acc { using type = float; };
template <> struct Acc<double> { using type = double; };

template <typename S> __device__ __forceinline__ S exp_(S v);
template <> __device__ __forceinline__ float exp_<float>(float v) { return __expf(v); }
template <> __device__ __forceinline__ double exp_<double>(double v) { return exp(v); }
template <typename S> __device__ __forceinline__ S log_(S v);
template <> __device__ __forceinline__ float log_<float>(float v) { return __logf(v); }
template <> __device__ __forceinline__ double log_<double>(double v) { return log(v); }

// One element.  G = 0 forward; G = 1: x carries dy, result is dx; G = 2: second-order term.
// Case analysis follows bias_act.cu:57-129 (expRange 80, halfExpRange 40, selu constants).
template <typename S, int A>
__device__ __forceinline__ S eval(S x, S b, S xref, S yref, S dy, int G, S alpha, S gain, S clamp) {
    const S one = (S)1, two = (S)2, expRange = (S)80, halfExpRange = (S)40;
    const S seluScale = (S)1.0507009873554804934193349852946, seluAlpha = (S)1.6732632423543772848170429916717;
    const S yy = (gain != (S)0) ? yref / gain : (S)0;
    S y = 0;
    if (G == 0) x += b; else xref += b;
    if (A == 1) { y = x; if (G == 2) y = 0; }
    if (A == 2) { if (G == 0) y = (x > 0) ? x : 0; if (G == 1) y = (yy > 0) ? x : 0; }
    if (A == 3) { if (G == 0) y = (x > 0) ? x : x * alpha; if (G == 1) y = (yy > 0) ? x : x * alpha; }
    if (A == 4) {
        if (G == 0) { const S c = exp_(x), d = one / c; y = (x < -expRange) ? -one : (x > expRange) ? one : (c - d) / (c + d); }
        if (G == 1) y = x * (one - yy * yy);
        if (G == 2) y = x * (one - yy * yy) * (-two * yy);
    }
    if (A == 5) {
        if (G == 0) y = (x < -expRange) ? 0 : one / (exp_(-x) + one);
        if (G == 1) y = x * yy * (one - yy);
        if (G == 2) y = x * yy * (one - yy) * (one - two * yy);
    }
    if (A == 6) {
        if (G == 0) y = (x >= 0) ? x : exp_(x) - one;
        if (G == 1) y = (yy >= 0) ? x : x * (yy + one);
        if (G == 2) y = (yy >= 0) ? 0 : x * (yy + one);
    }
    if (A == 7) {
        if (G == 0) y = (x >= 0) ? seluScale * x : (seluScale * seluAlpha) * (exp_(x) - one);
        if (G == 1) y = (yy >= 0) ? x * seluScale : x * (yy + seluScale * seluAlpha);
        if (G == 2) y = (yy >= 0) ? 0 : x * (yy + seluScale * seluAlpha);
    }
    if (A == 8) {
        if (G == 0) y = (x > expRange) ? x : log_(exp_(x) + one);
        if (G == 1) y = x * (one - exp_(-yy));
        if (G == 2) { const S c = exp_(-yy); y = x * c * (one - c); }
    }
    if (A == 9) {
        if (G == 0) {
            y = (x < -expRange) ? 0 : x / (exp_(-x) + one);
        } else {
            const S c = exp_(xref), d = c + one;
            if (G == 1) y = (xref > halfExpRange) ? x : x * c * (xref + d) / (d * d);
            else y = (xref > halfExpRange) ? 0 : x * c * (xref * (two - d) + two * d) / (d * d * d);
            yref = (xref < -expRange) ? 0 : xref / (exp_(-xref) + one) * gain;
        }
    }
    y *= gain * dy;
    if (clamp >= 0) {
        if (G == 0) y = (y > -clamp & y < clamp) ? y : (y >= 0) ? clamp : -clamp;
        else y = (yref > -clamp & yref < clamp) ? y : 0;
    }
    return y;
}

// bias index of flat element e; 32-bit division whenever the tensor allows it
__device__ __forceinline__ long long bias_index(long long e, const BiasActArgs& p, bool small) {
    if (small) return (long long)(((unsigned)e / (unsigned)p.step_b) % (unsigned)p.size_b);
    return (e / p.step_b) % p.size_b;
}

template <typename T> struct Vec;
template <> struct Vec<float> { static constexpr int N = 4; using type = float4; };
template <> struct Vec<__half> { static constexpr int N = 8; using type = uint4; };
template <> struct Vec<double> { static constexpr int N = 2; using type = double2; };

template <typename T> __device__ __forceinline__ typename Acc<T>::type to_acc(T v) { return (typename Acc<T>::type)v; }
template <> __device__ __forceinline__ float to_acc<__half>(__half v) { return __half2float(v); }
template <typename T> __device__ __forceinline__ T from_acc(typename Acc<T>::type v) { return (T)v; }
template <> __device__ __forceinline__ __half from_acc<__half>(float v) { return __float2half(v); }

// one 16-byte vector <-> N accumulator-typed registers (explicit unpacking: no local-memory round trip)
__device__ __forceinline__ void load_vec(const float* p, long long v, float (&o)[4]) {
    const float4 t = __ldcs(reinterpret_cast<const float4*>(p) + v);
    o[0] = t.x; o[1] = t.y; o[2] = t.z; o[3] = t.w;
}
__device__ __forceinline__ void load_vec(const double* p, long long v, double (&o)[2]) {
    const double2 t = __ldcs(reinterpret_cast<const double2*>(p) + v);
    o[0] = t.x; o[1] = t.y;
}
__device__ __forceinline__ void load_vec(const __half* p, long long v, float (&o)[8]) {
    const uint4 t = __ldcs(reinterpret_cast<const uint4*>(p) + v);
    const unsigned w[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
        o[2 * i] = f.x; o[2 * i + 1] = f.y;
    }
}
__device__ __forceinline__ void store_vec(float* p, long long v, const float (&o)[4]) {
    __stcs(reinterpret_cast<float4*>(p) + v, make_float4(o[0], o[1], o[2], o[3]));
}
__device__ __forceinline__ void store_vec(double* p, long long v, const double (&o)[2]) {
    __stcs(reinterpret_cast<double2*>(p) + v, make_double2(o[0], o[1]));
}
__device__ __forceinline__ void store_vec(__half* p, long long v, const float (&o)[8]) {
    unsigned w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const __half2 h = __floats2half2_rn(o[2 * i], o[2 * i + 1]);
        w[i] = *reinterpret_cast<const unsigned*>(&h);
    }
    __stcs(reinterpret_cast<uint4*>(p) + v, make_uint4(w[0], w[1], w[2], w[3]));
}

// Vectorised kernel: every thread handles whole 16-byte vectors; the tail (size_x % N) is scalar.
// Bias addressing per vector: BMODE 0 = none, 1 = one bias for the whole vector (step_b % N == 0: NCHW),
// 2 = consecutive biases (step_b == 1 and size_b % N == 0: channels_last / [M, C] matrices), 3 = per element.
template <typename T, int A, int UNROLL, bool kFwd>
__global__ void __launch_bounds__(256) bias_act_kernel(const BiasActArgs p, const int bmode) {
    using S = typename Acc<T>::type;
    constexpr int N = Vec<T>::N;
    const S alpha = (S)p.alpha, gain = (S)p.gain, clamp = (S)p.clamp;
    const int G = kFwd ? 0 : p.grad;          // forward-only instantiation: the gradient forms fold away
    const T* x = (const T*)p.x;
    const T* b = (const T*)p.b;
    const T* xref = (const T*)p.xref;
    const T* yref = (const T*)p.yref;
    const T* dy = (const T*)p.dy;
    T* y = (T*)p.y;
    const long long nvec = p.size_x / N;
    const long long stride = (long long)gridDim.x * blockDim.x;
    const bool small = p.size_x <= 0x7fffffffll;

    for (long long v0 = (long long)blockIdx.x * blockDim.x + threadIdx.x; v0 < nvec; v0 += stride * UNROLL) {
        S vx[UNROLL][N];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const long long v = v0 + u * stride;
            if (v < nvec) load_vec(x, v, vx[u]);                              // all loads of the unrolled group first
        }
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const long long v = v0 + u * stride;
            if (v >= nvec) continue;
            const long long e0 = v * N;
            S exr[N], eyr[N], edy[N], out[N], bb[N];
            if (xref) load_vec(xref, v, exr);
            if (yref) load_vec(yref, v, eyr);
            if (dy) load_vec(dy, v, edy);
            if (bmode == 1) {
                const S t = to_acc<T>(b[bias_index(e0, p, small)]);
#pragma unroll
                for (int j = 0; j < N; ++j) bb[j] = t;
            } else if (bmode == 2) {
                const long long i0 = small ? (long long)((unsigned)e0 % (unsigned)p.size_b) : e0 % p.size_b;
#pragma unroll
                for (int j = 0; j < N; ++j) bb[j] = to_acc<T>(b[i0 + j]);
            } else {
#pragma unroll
                for (int j = 0; j < N; ++j) bb[j] = (bmode == 3) ? to_acc<T>(b[bias_index(e0 + j, p, small)]) : (S)0;
            }
#pragma unroll
            for (int j = 0; j < N; ++j)
                out[j] = eval<S, A>(vx[u][j], bb[j], xref ? exr[j] : (S)0, yref ? eyr[j] : (S)0, dy ? edy[j] : (S)1, G, alpha, gain, clamp);
            store_vec(y, v, out);
        }
    }
    // scalar tail
    const long long tail0 = nvec * N;
    for (long long e = tail0 + (long long)blockIdx.x * blockDim.x + threadIdx.x; e < p.size_x; e += stride) {
        const S bb = b ? to_acc<T>(b[bias_index(e, p, small)]) : (S)0;
        y[e] = from_acc<T>(eval<S, A>(to_acc<T>(x[e]), bb, xref ? to_acc<T>(xref[e]) : (S)0,
                                      yref ? to_acc<T>(yref[e]) : (S)0, dy ? to_acc<T>(dy[e]) : (S)1, G, alpha,
                                      gain, clamp));
    }
}

// Planar fast path (no bias, or NCHW-style bias with step_b >= 1024 elements): the work is cut into
// (plane, chunk) items so that the bias is BLOCK-uniform -- no per-thread index arithmetic beyond an add.
template <typename T, int A, int UNROLL, bool kFwd>
__global__ void __launch_bounds__(256) bias_act_planar_kernel(const BiasActArgs p, long long plane_elems, long long chunks_per_plane,
                                                             long long items) {
    using S = typename Acc<T>::type;
    constexpr int N = Vec<T>::N;
    const S alpha = (S)p.alpha, gain = (S)p.gain, clamp = (S)p.clamp;
    const int G = kFwd ? 0 : p.grad;          // forward-only instantiation: the gradient forms fold away
    const T* b = (const T*)p.b;
    const long long plane_vecs = plane_elems / N;
    for (long long item = blockIdx.x; item < items; item += gridDim.x) {
        const long long plane = item / chunks_per_plane;
        const long long chunk = item - plane * chunks_per_plane;
        const S bias = b ? to_acc<T>(b[plane % p.size_b]) : (S)0;
        const long long vbase = plane * plane_vecs;                       // first vector of the plane
        const long long v0 = chunk * (256 * UNROLL) + threadIdx.x;       // vector index inside the plane
        S vx[UNROLL][N];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u)
            if (v0 + u * 256 < plane_vecs) load_vec((const T*)p.x, vbase + v0 + u * 256, vx[u]);
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const long long vi = v0 + u * 256;
            if (vi >= plane_vecs) continue;
            const long long v = vbase + vi;
            S exr[N], eyr[N], edy[N], out[N];
            if (p.xref) load_vec((const T*)p.xref, v, exr);
            if (p.yref) load_vec((const T*)p.yref, v, eyr);
            if (p.dy) load_vec((const T*)p.dy, v, edy);
#pragma unroll
            for (int j = 0; j < N; ++j)
                out[j] = eval<S, A>(vx[u][j], bias, p.xref ? exr[j] : (S)0, p.yref ? eyr[j] : (S)0, p.dy ? edy[j] : (S)1, G, alpha, gain, clamp);
            store_vec((T*)p.y, v, out);
        }
    }
}

template <typename T, int A>
static int launch_bias_act(const BiasActArgs& p, cudaStream_t st) {
    constexpr int UNROLL = 4;
    constexpr int N = Vec<T>::N;
    const long long nvec = p.size_x / N;
    long long blocks = ceil_div<long long>(nvec > 0 ? nvec : 1, 256ll * UNROLL);
    const long long cap = (long long)sm_count() * 8;            // 8 resident blocks of 256 threads per SM
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    int bmode = 0;
    if (p.b != nullptr) bmode = (p.step_b % N == 0) ? 1 : ((p.step_b == 1 && p.size_b % N == 0) ? 2 : 3);
    // planar fast path: whole planes of >= 1024 elements share one bias (or there is no bias at all)
    const long long plane_elems = (p.b == nullptr) ? p.size_x : p.step_b;
    if ((p.b == nullptr || bmode == 1) && plane_elems >= 1024 && plane_elems % N == 0 && p.size_x % plane_elems == 0) {
        const long long cpp = ceil_div<long long>(plane_elems / N, 256ll * UNROLL);
        const long long items = (p.size_x / plane_elems) * cpp;
        long long g = items < cap ? items : cap;
        if (p.grad == 0) bias_act_planar_kernel<T, A, UNROLL, true><<<(unsigned)g, 256, 0, st>>>(p, plane_elems, cpp, items);
        else bias_act_planar_kernel<T, A, UNROLL, false><<<(unsigned)g, 256, 0, st>>>(p, plane_elems, cpp, items);
        IDE3D_CHECK_LAUNCH("bias_act_planar_kernel");
        return IDE3D_OK;
    }
    if (p.grad == 0) bias_act_kernel<T, A, UNROLL, true><<<(unsigned)blocks, 256, 0, st>>>(p, bmode);
    else bias_act_kernel<T, A, UNROLL, false><<<(unsigned)blocks, 256, 0, st>>>(p, bmode);
    IDE3D_CHECK_LAUNCH("bias_act_kernel");
    return IDE3D_OK;
}

template <typename T>
static int dispatch_act(const BiasActArgs& p, int act, cudaStream_t st) {
    switch (act) {
        case 1: return launch_bias_act<T, 1>(p, st);
        case 2: return launch_bias_act<T, 2>(p, st);
        case 3: return launch_bias_act<T, 3>(p, st);
        case 4: return launch_bias_act<T, 4>(p, st);
        case 5: return launch_bias_act<T, 5>(p, st);
        case 6: return launch_bias_act<T, 6>(p, st);
        case 7: return launch_bias_act<T, 7>(p, st);
        case 8: return launch_bias_act<T, 8>(p, st);
        case 9: return launch_bias_act<T, 9>(p, st);
    }
    IDE3D_FAIL(IDE3D_INVALID, "bias_act: unknown activation index %d", act);
}

}  // namespace ide3d

using namespace ide3d;

extern "C" int ide3d_bias_act(const void* x, const void* b, const void* xref, const void* yref, const void* dy,
                              void* y, int dtype, int grad, int act, float alpha, float gain, float clamp,
                              int64_t size_x, int64_t size_b, int64_t step_b, ide3d_stream_t stream) {
    IDE3D_REQUIRE(size_x >= 0, "bias_act: negative size");
    if (size_x == 0) return IDE3D_OK;
    IDE3D_REQUIRE(x && y, "bias_act: null x/y");
    IDE3D_REQUIRE(grad >= 0 && grad <= 2, "bias_act: grad must be 0, 1 or 2");
    IDE3D_REQUIRE(b == nullptr || (size_b > 0 && step_b > 0), "bias_act: bad bias geometry");
    const uintptr_t all = (uintptr_t)x | (uintptr_t)y | (uintptr_t)xref | (uintptr_t)yref | (uintptr_t)dy;
    IDE3D_REQUIRE((all & 15) == 0, "bias_act: tensors must be 16-byte aligned");
    BiasActArgs p{x, b, xref, yref, dy, y, grad, alpha, gain, clamp, size_x, size_b > 0 ? size_b : 1,
                  step_b > 0 ? step_b : 1};
    cudaStream_t st = (cudaStream_t)stream;
    switch (dtype) {
        case IDE3D_F32: return dispatch_act<float>(p, act, st);
        case IDE3D_F16: return dispatch_act<__half>(p, act, st);
        case IDE3D_F64: return dispatch_act<double>(p, act, st);
    }
    IDE3D_FAIL(IDE3D_INVALID, "bias_act: unsupported dtype %d", dtype);
}

// ------------------------------------------------------------------------------------------------------------------
// Fused epilogue of an activation-scaled ("non-fused") modulated convolution (inversion/networks.py:97-111 followed by
// :512):   y = bias_act(x * scale[n,c] + noise[(n),h,w], b[c])   in ONE pass instead of fma.fma + bias_act (two).
// No counterpart among the reference plugins; forward only (the Python wrapper composes the two reference ops whenever
// autograd is involved).
namespace ide3d {

struct EpiArgs {
    const void *x, *scale, *noise, *b;
    void* y;                              // may be NULL when only y2 is wanted
    const void* scale2;                   // optional second output y2 = y * scale2[n,c]: the NEXT layer's style modulation
    void* y2;
    float alpha, gain, clamp;
    long long n, c, hw;
    int noise_batch;                      // 1: one noise map for the whole batch, n: one per sample
};

template <typename T> __device__ __forceinline__ void load_vec_keep(const T* p, long long v, typename Acc<T>::type (&o)[Vec<T>::N]);
template <> __device__ __forceinline__ void load_vec_keep<float>(const float* p, long long v, float (&o)[4]) {
    const float4 t = __ldg(reinterpret_cast<const float4*>(p) + v);
    o[0] = t.x; o[1] = t.y; o[2] = t.z; o[3] = t.w;
}
template <> __device__ __forceinline__ void load_vec_keep<double>(const double* p, long long v, double (&o)[2]) {
    const double2 t = __ldg(reinterpret_cast<const double2*>(p) + v);
    o[0] = t.x; o[1] = t.y;
}
template <> __device__ __forceinline__ void load_vec_keep<__half>(const __half* p, long long v, float (&o)[8]) {
    const uint4 t = __ldg(reinterpret_cast<const uint4*>(p) + v);
    const unsigned w[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
        o[2 * i] = f.x; o[2 * i + 1] = f.y;
    }
}

// NCHW: (plane, chunk) work items, scale and bias are block-uniform, the noise map is read through L1/L2 (it is shared by
// every channel of the sample).
template <typename T, int A, int UNROLL>
__global__ void __launch_bounds__(256) modconv_epilogue_planar_kernel(const EpiArgs p, long long chunks_per_plane, long long items) {
    using S = typename Acc<T>::type;
    constexpr int N = Vec<T>::N;
    const S alpha = (S)p.alpha, gain = (S)p.gain, clamp = (S)p.clamp;
    const long long plane_vecs = p.hw / N;
    for (long long item = blockIdx.x; item < items; item += gridDim.x) {
        const long long plane = item / chunks_per_plane;
        const long long chunk = item - plane * chunks_per_plane;
        const long long smp = plane / p.c;
        const S d = p.scale ? to_acc<T>(((const T*)p.scale)[plane]) : (S)1;
        const S bias = p.b ? to_acc<T>(((const T*)p.b)[plane - smp * p.c]) : (S)0;
        const S d2 = p.y2 ? to_acc<T>(((const T*)p.scale2)[plane]) : (S)1;
        const long long vbase = plane * plane_vecs;
        const long long nbase = (p.noise_batch == 1 ? 0 : smp) * plane_vecs;
        const long long v0 = chunk * (256 * UNROLL) + threadIdx.x;
        S vx[UNROLL][N], vn[UNROLL][N];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u)
            if (v0 + u * 256 < plane_vecs) {
                load_vec((const T*)p.x, vbase + v0 + u * 256, vx[u]);
                if (p.noise) load_vec_keep<T>((const T*)p.noise, nbase + v0 + u * 256, vn[u]);
            }
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const long long vi = v0 + u * 256;
            if (vi >= plane_vecs) continue;
            S out[N];
#pragma unroll
            for (int j = 0; j < N; ++j) {
                const S t = p.noise ? vx[u][j] * d + vn[u][j] : vx[u][j] * d;
                out[j] = eval<S, A>(t, bias, (S)0, (S)0, (S)1, 0, alpha, gain, clamp);
            }
            if (p.y) store_vec((T*)p.y, vbase + vi, out);
            if (p.y2) {
#pragma unroll
                for (int j = 0; j < N; ++j) out[j] *= d2;
                store_vec((T*)p.y2, vbase + vi, out);
            }
        }
    }
}

// channels_last: one 16-byte vector = N consecutive channels of one pixel; scale / bias are vectors, the noise a scalar.
// Work items are (sample, chunk of 256*UNROLL vectors): the sample index is block-uniform and the position inside the
// sample fits 32 bits, so the per-vector index math is one shift/mask (power-of-two channel counts) or one 32-bit division
// -- the first version spent 3/4 of its issue slots on 64-bit div/mod.
template <typename T, int A, int UNROLL>
__global__ void __launch_bounds__(256) modconv_epilogue_cl_kernel(const EpiArgs p, unsigned chunks_per_sample, long long items, int cv_shift) {
    using S = typename Acc<T>::type;
    constexpr int N = Vec<T>::N;
    const S alpha = (S)p.alpha, gain = (S)p.gain, clamp = (S)p.clamp;
    const unsigned cv = (unsigned)(p.c / N);                     // vectors per pixel
    const unsigned svec = (unsigned)p.hw * cv;                   // vectors per sample (host guarantees < 2^31)
    for (long long item = blockIdx.x; item < items; item += gridDim.x) {
        const unsigned smp = (unsigned)(item / chunks_per_sample);
        const unsigned chunk = (unsigned)(item - (long long)smp * chunks_per_sample);
        const long long vbase = (long long)smp * svec;
        const unsigned v0 = chunk * (256u * UNROLL) + threadIdx.x;
        S vx[UNROLL][N];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u)
            if (v0 + u * 256u < svec) load_vec((const T*)p.x, vbase + v0 + u * 256u, vx[u]);
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const unsigned vi = v0 + u * 256u;
            if (vi >= svec) continue;
            unsigned pix, c0;
            if (cv_shift >= 0) { pix = vi >> cv_shift; c0 = vi & (cv - 1u); }
            else { pix = vi / cv; c0 = vi - pix * cv; }
            S d[N], bb[N], out[N];
            if (p.scale) load_vec_keep<T>((const T*)p.scale, (long long)smp * cv + c0, d);
            if (p.b) load_vec_keep<T>((const T*)p.b, c0, bb);
            const S nz = p.noise ? to_acc<T>(__ldg((const T*)p.noise + (p.noise_batch == 1 ? (long long)pix : (long long)smp * p.hw + pix))) : (S)0;
#pragma unroll
            for (int j = 0; j < N; ++j) {
                S t = p.scale ? vx[u][j] * d[j] : vx[u][j];
                if (p.noise) t = p.scale ? vx[u][j] * d[j] + nz : vx[u][j] + nz;
                out[j] = eval<S, A>(t, p.b ? bb[j] : (S)0, (S)0, (S)0, (S)1, 0, alpha, gain, clamp);
            }
            if (p.y) store_vec((T*)p.y, vbase + vi, out);
            if (p.y2) {
                S d2[N];
                load_vec_keep<T>((const T*)p.scale2, (long long)smp * cv + c0, d2);
#pragma unroll
                for (int j = 0; j < N; ++j) out[j] *= d2[j];
                store_vec((T*)p.y2, vbase + vi, out);
            }
        }
    }
}

template <typename T, int A>
static int launch_epilogue(const EpiArgs& p, int channels_last, cudaStream_t st) {
    constexpr int UNROLL = 4;
    constexpr int N = Vec<T>::N;
    const long long cap = (long long)sm_count() * 8;
    if (channels_last) {
        if (p.c % N != 0) IDE3D_FAIL(IDE3D_UNSUPPORTED, "modconv_epilogue: channels_last needs C %% %d == 0", N);
        const long long svec = p.hw * (p.c / N);
        if (svec >= (1ll << 31)) IDE3D_FAIL(IDE3D_UNSUPPORTED, "modconv_epilogue: more than 2^31 vectors per sample");
        const long long cps = ceil_div<long long>(svec, 256ll * UNROLL);
        const long long items = p.n * cps;
        const long long blocks = items < cap ? items : cap;
        const long long cvn = p.c / N;
        int cv_shift = -1;
        if ((cvn & (cvn - 1)) == 0) { cv_shift = 0; while ((1ll << cv_shift) < cvn) ++cv_shift; }
        modconv_epilogue_cl_kernel<T, A, UNROLL><<<(unsigned)blocks, 256, 0, st>>>(p, (unsigned)cps, items, cv_shift);
        IDE3D_CHECK_LAUNCH("modconv_epilogue_cl_kernel");
        return IDE3D_OK;
    }
    if (p.hw % N != 0) IDE3D_FAIL(IDE3D_UNSUPPORTED, "modconv_epilogue: H*W must be a multiple of %d", N);
    const long long cpp = ceil_div<long long>(p.hw / N, 256ll * UNROLL);
    const long long items = p.n * p.c * cpp;
    const long long g = items < cap ? items : cap;
    modconv_epilogue_planar_kernel<T, A, UNROLL><<<(unsigned)g, 256, 0, st>>>(p, cpp, items);
    IDE3D_CHECK_LAUNCH("modconv_epilogue_planar_kernel");
    return IDE3D_OK;
}

template <typename T>
static int dispatch_epilogue(const EpiArgs& p, int act, int channels_last, cudaStream_t st) {
    switch (act) {
        case 1: return launch_epilogue<T, 1>(p, channels_last, st);
        case 2: return launch_epilogue<T, 2>(p, channels_last, st);
        case 3: return launch_epilogue<T, 3>(p, channels_last, st);
        case 4: return launch_epilogue<T, 4>(p, channels_last, st);
        case 5: return launch_epilogue<T, 5>(p, channels_last, st);
        case 6: return launch_epilogue<T, 6>(p, channels_last, st);
        case 7: return launch_epilogue<T, 7>(p, channels_last, st);
        case 8: return launch_epilogue<T, 8>(p, channels_last, st);
        case 9: return launch_epilogue<T, 9>(p, channels_last, st);
    }
    IDE3D_FAIL(IDE3D_INVALID, "modconv_epilogue: unknown activation index %d", act);
}

}  // namespace ide3d

extern "C" int ide3d_modconv_epilogue(const void* x, const void* scale, const void* noise, const void* b, void* y,
                                      const void* scale2, void* y2, int dtype, int act, float alpha, float gain, float clamp,
                                      int64_t n, int64_t c, int64_t hw, int64_t noise_batch, int channels_last,
                                      ide3d_stream_t stream) {
    IDE3D_REQUIRE(n >= 0 && c >= 0 && hw >= 0, "modconv_epilogue: negative size");
    if (n * c * hw == 0) return IDE3D_OK;
    IDE3D_REQUIRE(x && (y || y2), "modconv_epilogue: null x / no output");
    IDE3D_REQUIRE((y2 == nullptr) == (scale2 == nullptr), "modconv_epilogue: scale2 and y2 go together");
    IDE3D_REQUIRE(noise == nullptr || noise_batch == 1 || noise_batch == n, "modconv_epilogue: noise batch must be 1 or n");
    const uintptr_t all = (uintptr_t)x | (uintptr_t)y | (uintptr_t)scale | (uintptr_t)noise | (uintptr_t)b | (uintptr_t)scale2 | (uintptr_t)y2;
    IDE3D_REQUIRE((all & 15) == 0, "modconv_epilogue: tensors must be 16-byte aligned");
    ide3d::EpiArgs p{x, scale, noise, b, y, scale2, y2, alpha, gain, clamp, n, c, hw, (int)noise_batch};
    cudaStream_t st = (cudaStream_t)stream;
    switch (dtype) {
        case IDE3D_F32: return ide3d::dispatch_epilogue<float>(p, act, channels_last, st);
        case IDE3D_F16: return ide3d::dispatch_epilogue<__half>(p, act, channels_last, st);
        case IDE3D_F64: return ide3d::dispatch_epilogue<double>(p, act, channels_last, st);
    }
    IDE3D_FAIL(IDE3D_INVALID, "modconv_epilogue: unsupported dtype %d", dtype);
}
