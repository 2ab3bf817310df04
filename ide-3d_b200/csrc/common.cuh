// Shared helpers for libide3d_b200.so (sm_90a).  No torch, no global device state.
#pragma once

#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "../../include/ide3d_b200.h"

namespace ide3d {

// thread-local error message, returned by ide3d_last_error()
char* error_buffer();
void count_launch(int n = 1);

#define IDE3D_FAIL(code, ...)                                   \
    do {                                                        \
        snprintf(ide3d::error_buffer(), 512, __VA_ARGS__);      \
        return (code);                                          \
    } while (0)

#define IDE3D_REQUIRE(cond, ...)                                \
    do {                                                        \
        if (!(cond)) IDE3D_FAIL(IDE3D_INVALID, __VA_ARGS__);    \
    } while (0)

// call after every launch: surfaces launch-configuration errors without synchronising
#define IDE3D_CHECK_LAUNCH(what)                                                               \
    do {                                                                                       \
        cudaError_t e__ = cudaGetLastError();                                                  \
        if (e__ != cudaSuccess)                                                                \
            IDE3D_FAIL(IDE3D_CUDA_ERROR, "%s: %s", (what), cudaGetErrorString(e__));           \
        ide3d::count_launch();                                                                 \
    } while (0)

#define IDE3D_CUDA(call)                                                                       \
    do {                                                                                       \
        cudaError_t e__ = (call);                                                              \
        if (e__ != cudaSuccess)                                                                \
            IDE3D_FAIL(IDE3D_CUDA_ERROR, "%s: %s", #call, cudaGetErrorString(e__));            \
    } while (0)

// Experiment switches (IDE3D_* environment variables) are compiled in only with -DIDE3D_TUNING (IDE3D_BUILD_TUNING=1 python
// ide-3d_b200/build.py -- what the A/B scripts under scripts/ use).  The product build never reads the environment.
inline const char* tuning_env(const char* name) {
#ifdef IDE3D_TUNING
    return getenv(name);
#else
    (void)name;
    return nullptr;
#endif
}

inline int sm_count() {
    static thread_local int cached_dev = -1, cached = 0;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (dev != cached_dev) {
        cudaDeviceGetAttribute(&cached, cudaDevAttrMultiProcessorCount, dev);
        cached_dev = dev;
        if (cached <= 0) cached = 132;
    }
    return cached;
}

template <typename T>
__host__ __device__ inline T ceil_div(T a, T b) { return (a + b - 1) / b; }

// Grid of a persistent kernel: as many CTAs of `threads` threads and `smem` bytes of dynamic shared memory as are resident on
// the device at once, at most `max_ctas` (the CTAs that have work).  Raises the kernel's dynamic shared-memory limit to `smem`
// when `smem` exceeds the 48 KB every kernel may use without it.
template <typename Kernel>
inline int persistent_grid(Kernel kern, int threads, size_t smem, long long max_ctas, int& grid) {
    if (smem > 48 * 1024) IDE3D_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 1;
    IDE3D_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem));
    if (per_sm < 1) per_sm = 1;
    const long long resident = (long long)sm_count() * per_sm;
    grid = (int)(resident < max_ctas ? resident : max_ctas);
    if (grid < 1) grid = 1;
    return IDE3D_OK;
}

// torch's float -> uint8 conversion on the device after (v * 127.5 + 128).clamp(0, 255): two rounded float ops, clamp lets NaN through,
// and the cast goes float -> int64 -> uint8 (the conversion of save_image_u8 in strips.cu).
__device__ __forceinline__ unsigned char torch_u8(float v) {
    float y = __fadd_rn(__fmul_rn(v, 127.5f), 128.f);
    if (y == y) y = fminf(fmaxf(y, 0.f), 255.f);
    return (unsigned char)(long long)y;
}

// floor division for possibly negative numerators
__host__ __device__ inline int floor_div(int a, int b) {
    int q = a / b;
    return (a % b != 0 && ((a < 0) != (b < 0))) ? q - 1 : q;
}

}  // namespace ide3d
