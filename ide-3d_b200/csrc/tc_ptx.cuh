// Thin inline-PTX wrappers for the Hopper (sm_90a) tensor-core path: warpgroup MMA (wgmma.mma_async with the A operand in
// shared memory or in registers, fp32 accumulators in registers), its fences, proxy fences, named barriers and the shared-memory
// matrix descriptor.  Bit layouts follow the PTX ISA "wgmma" chapter (matrix descriptor, register fragments) as used by CUTLASS'
// cute::GMMA.
#pragma once

#include <cuda_bf16.h>
#include <stdint.h>

#include "tma.cuh"

namespace ide3d {
namespace tc {

// ---------------------------------------------------------------------------------------- fences / barriers
// generic-proxy shared-memory writes -> visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// named barrier over `threads` threads (id 1..15; 0 is __syncthreads)
__device__ __forceinline__ void bar_sync(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

// wgmma ordering: fence before the first MMA that touches accumulator / A registers written by ordinary instructions;
// commit closes a group of MMAs; wait_group<N> returns when at most N groups are still in flight
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// the accumulators are written asynchronously: keep the compiler from moving their reads across the wait
template <int R> __device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// ---------------------------------------------------------------------------------------- descriptors
// Shared-memory matrix descriptor for a K-major operand stored as 128-byte rows with the 128B swizzle
// (8-row x 128-byte atoms, 16-byte chunks XORed with row % 8; atoms 1024 bytes apart along M/N):
//   [0,14) start address >> 4   [16,30) leading byte offset >> 4 (unused for swizzled K-major: 1)
//   [32,46) stride byte offset >> 4 (1024 B between 8-row groups)   [49,52) base offset (0: atoms 1024-byte aligned)
//   [62,64) layout = 1 (SWIZZLE_128B)
// Moving along K inside the 128-byte row: + (bytes >> 4) on the start address.
__device__ __forceinline__ uint64_t make_sdesc_sw128(uint32_t smem_addr) {
    return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | (1ull << 16) | ((uint64_t)(1024u >> 4) << 32) | (1ull << 62);
}

// byte offset of 16-byte chunk `c` (0..7) of row `r` inside a swizzle-128B tile
__device__ __forceinline__ uint32_t sw128_offset(int r, int c) {
    return (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + (((c ^ r) & 7) << 4));
}

// ---------------------------------------------------------------------------------------- warpgroup MMA, M = 64, K = 16 bf16
// Issued by all 128 threads of a warpgroup.  Accumulator fragment of thread t (warp w = t / 32, lane l): rows 16w + l/4 and
// 16w + l/4 + 8, columns 8j + 2(l%4) + {0, 1}: d[4j + 0..1] (first row), d[4j + 2..3] (second row).  The register A fragment of a
// K = 16 step has the same row / column ownership: a[0] = (row, k 2(l%4)..+1), a[1] = (row + 8, same k), a[2] / a[3] = k + 8.
template <int N> struct Wgmma;

template <> struct Wgmma<16> {
    // D[64 x 16] (+)= A[smem] . B[smem]^T
    __device__ __forceinline__ static void ss(float* d, uint64_t a_desc, uint64_t b_desc, int scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
            : "l"(a_desc), "l"(b_desc), "r"(scale_d));
    }
    // D[64 x 16] += A[registers] . B[smem]^T
    __device__ __forceinline__ static void rs(float* d, const uint32_t (&a)[4], uint64_t b_desc) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1, 0;\n\t}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(1));
    }
};

template <> struct Wgmma<32> {
    // D[64 x 32] (+)= A[smem] . B[smem]^T
    __device__ __forceinline__ static void ss(float* d, uint64_t a_desc, uint64_t b_desc, int scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(a_desc), "l"(b_desc), "r"(scale_d));
    }
    // D[64 x 32] += A[registers] . B[smem]^T
    __device__ __forceinline__ static void rs(float* d, const uint32_t (&a)[4], uint64_t b_desc) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, 0;\n\t}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(1));
    }
};

template <> struct Wgmma<48> {
    // D[64 x 48] (+)= A[smem] . B[smem]^T
    __device__ __forceinline__ static void ss(float* d, uint64_t a_desc, uint64_t b_desc, int scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p, 1, 1, 0, 0;\n\t}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
            : "l"(a_desc), "l"(b_desc), "r"(scale_d));
    }
    // D[64 x 48] += A[registers] . B[smem]^T
    __device__ __forceinline__ static void rs(float* d, const uint32_t (&a)[4], uint64_t b_desc) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %29, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, {%24, %25, %26, %27}, %28, p, 1, 1, 0;\n\t}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(1));
    }
};

template <> struct Wgmma<64> {
    // D[64 x 64] (+)= A[smem] . B[smem]^T
    __device__ __forceinline__ static void ss(float* d, uint64_t a_desc, uint64_t b_desc, int scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "l"(a_desc), "l"(b_desc), "r"(scale_d));
    }
    // D[64 x 64] += A[registers] . B[smem]^T
    __device__ __forceinline__ static void rs(float* d, const uint32_t (&a)[4], uint64_t b_desc) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(1));
    }
};

// ---------------------------------------------------------------------------------------- warpgroup MMA, M = 64, N = 128, K = 16 fp16
// D[64 x 128] (+)= A[smem] . B[smem]^T with both operands K-major fp16 (same descriptors and fragment layout as above, j = 0..15).
__device__ __forceinline__ void wgmma_f16_m64n128_ss(float* d, uint64_t a_desc, uint64_t b_desc, int scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a_desc), "l"(b_desc), "r"(scale_d));
}

// fp32 -> (hi, lo) bf16 pair with hi + lo ~= x to 16 mantissa bits
__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
    hi = __float2bfloat16_rn(x);
    lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}
// four fp32 -> packed bf16 hi pairs and lo pairs (hi = rn(x), lo = rn(x - hi)) with the two-element conversion
// (F2FP.BF16.F32.PACK_AB) instead of four scalar F2F per half
__device__ __forceinline__ void split4_bf16(const float (&f)[4], uint2& hi, uint2& lo) {
    const __nv_bfloat162 h01 = __floats2bfloat162_rn(f[0], f[1]), h23 = __floats2bfloat162_rn(f[2], f[3]);
    const float2 b01 = __bfloat1622float2(h01), b23 = __bfloat1622float2(h23);
    const __nv_bfloat162 l01 = __floats2bfloat162_rn(f[0] - b01.x, f[1] - b01.y), l23 = __floats2bfloat162_rn(f[2] - b23.x, f[3] - b23.y);
    hi = make_uint2(*reinterpret_cast<const uint32_t*>(&h01), *reinterpret_cast<const uint32_t*>(&h23));
    lo = make_uint2(*reinterpret_cast<const uint32_t*>(&l01), *reinterpret_cast<const uint32_t*>(&l23));
}
// two fp32 -> one packed bf16 hi pair and one lo pair
__device__ __forceinline__ void split2_bf16(float x0, float x1, uint32_t& hi, uint32_t& lo) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(x0, x1);
    const float2 b = __bfloat1622float2(h);
    const __nv_bfloat162 l = __floats2bfloat162_rn(x0 - b.x, x1 - b.y);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = *reinterpret_cast<const uint32_t*>(&l);
}

}  // namespace tc
}  // namespace ide3d
