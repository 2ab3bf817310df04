// Element and vector access of the streaming kernels (upfirdn2d, bias_act and the modulated-convolution epilogues,
// filtered_lrelu): scalar conversion to and from the accumulation type, and 16-byte (8-byte for 4 fp16 values) vector loads
// and stores that unpack to / pack from accumulator registers.  The cache policy of each vector access is in its name:
//   load_vec_cs   streaming load (__ldcs): data read once
//   load_vec_ro   read-only load (__ldg): data other threads read again (noise maps, per-channel operands, FIR windows)
//   load_vec      plain load: shared memory reached through a generic pointer (TMA-staged tiles)
//   store_vec_cs  streaming store (__stcs); fp16 values are rounded once each (__floats2half2_rn)
#pragma once

#include <cuda_fp16.h>

namespace ide3d {

// accumulation type: float for float and __half, double for double
template <typename T> struct Acc { using type = float; };
template <> struct Acc<double> { using type = double; };

template <typename T> __device__ __forceinline__ typename Acc<T>::type to_acc(T v) { return (typename Acc<T>::type)v; }
template <> __device__ __forceinline__ float to_acc<__half>(__half v) { return __half2float(v); }
template <typename T> __device__ __forceinline__ T from_acc(typename Acc<T>::type v) { return (T)v; }
template <> __device__ __forceinline__ __half from_acc<__half>(float v) { return __float2half(v); }

// float for every T, double included: kernels that compute in float32 whatever the storage type
template <typename T> __device__ __forceinline__ float load_f32(const T* p) { return (float)(*p); }
template <> __device__ __forceinline__ float load_f32<__half>(const __half* p) { return __half2float(*p); }
template <typename T> __device__ __forceinline__ void store_f32(T* p, float v) { *p = (T)v; }
template <> __device__ __forceinline__ void store_f32<__half>(__half* p, float v) { *p = __float2half(v); }
template <typename T> __device__ __forceinline__ T zero_of() { return (T)0.f; }
template <> __device__ __forceinline__ __half zero_of<__half>() { return __float2half(0.f); }

// elements of T per 16-byte vector
template <typename T> struct Vec;
template <> struct Vec<float> { static constexpr int N = 4; };
template <> struct Vec<__half> { static constexpr int N = 8; };
template <> struct Vec<double> { static constexpr int N = 2; };

// K elements of T as one machine word (`raw`), unpacked to / packed from accumulator registers
template <typename T, int K> struct VecIO;
template <> struct VecIO<float, 4> {
    using raw = float4;
    static __device__ __forceinline__ void unpack(const float4 t, float (&o)[4]) { o[0] = t.x; o[1] = t.y; o[2] = t.z; o[3] = t.w; }
    static __device__ __forceinline__ float4 pack(const float (&o)[4]) { return make_float4(o[0], o[1], o[2], o[3]); }
};
template <> struct VecIO<double, 2> {
    using raw = double2;
    static __device__ __forceinline__ void unpack(const double2 t, double (&o)[2]) { o[0] = t.x; o[1] = t.y; }
    static __device__ __forceinline__ double2 pack(const double (&o)[2]) { return make_double2(o[0], o[1]); }
};
template <> struct VecIO<__half, 4> {
    using raw = uint2;
    static __device__ __forceinline__ void unpack(const uint2 t, float (&o)[4]) {
        const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&t.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&t.y));
        o[0] = a.x; o[1] = a.y; o[2] = b.x; o[3] = b.y;
    }
    static __device__ __forceinline__ uint2 pack(const float (&o)[4]) {
        const __half2 a = __floats2half2_rn(o[0], o[1]), b = __floats2half2_rn(o[2], o[3]);
        return make_uint2(*reinterpret_cast<const unsigned*>(&a), *reinterpret_cast<const unsigned*>(&b));
    }
};
template <> struct VecIO<__half, 8> {
    using raw = uint4;
    static __device__ __forceinline__ void unpack(const uint4 t, float (&o)[8]) {
        const unsigned w[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
            o[2 * i] = f.x; o[2 * i + 1] = f.y;
        }
    }
    static __device__ __forceinline__ uint4 pack(const float (&o)[8]) {
        unsigned w[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const __half2 h = __floats2half2_rn(o[2 * i], o[2 * i + 1]);
            w[i] = *reinterpret_cast<const unsigned*>(&h);
        }
        return make_uint4(w[0], w[1], w[2], w[3]);
    }
};

// vector v of K elements at p (p aligned to the vector; v = 0 for the vector at p) <-> K accumulator registers
template <typename T, int K>
__device__ __forceinline__ void load_vec_cs(const T* p, long long v, typename Acc<T>::type (&o)[K]) {
    VecIO<T, K>::unpack(__ldcs(reinterpret_cast<const typename VecIO<T, K>::raw*>(p) + v), o);
}
template <typename T, int K>
__device__ __forceinline__ void load_vec_ro(const T* p, long long v, typename Acc<T>::type (&o)[K]) {
    VecIO<T, K>::unpack(__ldg(reinterpret_cast<const typename VecIO<T, K>::raw*>(p) + v), o);
}
template <typename T, int K>
__device__ __forceinline__ void load_vec(const T* p, long long v, typename Acc<T>::type (&o)[K]) {
    VecIO<T, K>::unpack(*(reinterpret_cast<const typename VecIO<T, K>::raw*>(p) + v), o);
}
template <typename T, int K>
__device__ __forceinline__ void store_vec_cs(T* p, long long v, const typename Acc<T>::type (&o)[K]) {
    const typename VecIO<T, K>::raw t = VecIO<T, K>::pack(o);
    __stcs(reinterpret_cast<typename VecIO<T, K>::raw*>(p) + v, t);
}

}  // namespace ide3d
