// Density queries on the tensor cores: sigma for 64 points per warpgroup tile (extract_shapes.py:99-150, the 256^3 grid of config 4,
// and renderer.sample_voxel(..., sigma_only) with explicit points), for decoders whose density head reads the shape planes alone
// (the generator's three-head decoder).  The machinery of raymarch_tc.cu without the march:
//   gather   every warp: its 16 points -> 3 x 4 bilinear taps of the SHAPE tri-plane only (8 lanes x LDG.128 per texel), blend,
//            bf16 hi / lo, swizzled A tile (columns 32..63 of the [64 x 64] tile)
//   layer 1  D1[64 x 64] = A . W1_sigma^T, wgmma (both operands in shared memory), three bf16 products per K step
//   epilog   + b1 -> softplus -> 64 -> 1 second layer as FFMA over the lane's 16 hidden columns, 4-lane reduction -> + b2 -> out
// No per-point intermediate touches HBM; the only global traffic is the texel gather (L1 / L2 hits for a coherent grid) and 4 bytes
// out per point.  The CUDA-core kernel of voxel.cu remains for every other decoder / layout.
#include "raymarch_tc_shared.cuh"

namespace ide3d {
namespace vtc {

constexpr int kW1Bytes = 64 * 128;                                           // [64 hidden x 64 K] bf16, K columns 32..63 used

struct Args : VoxelArgs {
    const float* w1; const float* b1; const float* w2; const float* b2;     // sigma head: [64,32], [64], [1,64], [1]
    long long tiles_per_item, num_tiles;
};

__global__ void __launch_bounds__(kTcThreads) sigma_tc_kernel(const Args a) {
    extern __shared__ unsigned char smem_raw[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    unsigned char* w_hi = smem;
    unsigned char* w_lo = smem + kW1Bytes;
    unsigned char* tile_base = smem + 2 * kW1Bytes;
    float* b1s = reinterpret_cast<float*>(tile_base + kWarpgroups * kStageBytes);     // [64] x log2e
    float* wsig = b1s + 64;                                                            // [64] x ln2

    const int tid = threadIdx.x, lane = tid & 31;
    for (int i = tid; i < 64 * 32; i += kTcThreads) {
        const int j = i >> 5, k = i & 31;
        __nv_bfloat16 hi, lo;
        tc::split_bf16(a.w1[j * 32 + k] * 1.4426950408889634f, hi, lo);
        tile_store_bf16(w_hi, j, 32 + k, hi);
        tile_store_bf16(w_lo, j, 32 + k, lo);
    }
    if (tid < 64) { b1s[tid] = a.b1[tid] * 1.4426950408889634f; wsig[tid] = a.w2[tid] * 0.6931471805599453f; }
    tc::fence_async_smem();
    __syncthreads();

    const int wg = tid >> 7, w = (tid >> 5) & 3;
    const int g = lane >> 2, c = lane & 3;
    const int q4 = lane & 7, grp = lane >> 3, l16 = lane & 15;
    const int shb = (int)(a.seg.sh * 4), swb = (int)(a.seg.sw * 4);
    const int W = a.seg.w, H = a.seg.h;
    unsigned char* a_hi = tile_base + wg * kStageBytes;
    unsigned char* a_lo = a_hi + kTileBytes;
    const uint64_t ah = tc::make_sdesc_sw128(smem_u32(a_hi)), al = tc::make_sdesc_sw128(smem_u32(a_lo));
    const uint64_t wh = tc::make_sdesc_sw128(smem_u32(w_hi)), wl = tc::make_sdesc_sw128(smem_u32(w_lo));
    const float sig_b = a.b2[0];
    const long long stride = (long long)kWarpgroups * gridDim.x;

    for (long long tile = (long long)blockIdx.x * kWarpgroups + wg; tile < a.num_tiles; tile += stride) {
        const int n = (int)(tile / a.tiles_per_item);
        const long long p0 = (tile - (long long)n * a.tiles_per_item) * 64 + w * 16;       // first point of this warp's 16 rows
        {
            const long long p = p0 + l16;
            float cx = 4.f, cy = 4.f, cz = 4.f;
            if (p < a.P) {
                if (a.points == nullptr) grid_point(a, a.first + p, cx, cy, cz);
                else { const float* pt = a.points + ((long long)n * a.P + p) * 3; cx = pt[0]; cy = pt[1]; cz = pt[2]; }
                cx *= a.box_scale; cy *= a.box_scale; cz *= a.box_scale;
            }
            const AxisFoot fx = axis_foot(cx, W), fyr = axis_foot(cy, H), fyc = axis_foot(cy, W), fz = axis_foot(cz, H);
            const AxisTaps mX = axis_taps(fx.i0, fx.f, W, swb), mYr = axis_taps(fyr.i0, fyr.f, H, shb);
            const AxisTaps mYc = axis_taps(fyc.i0, fyc.f, W, swb), mZ = axis_taps(fz.i0, fz.f, H, shb);
            const char* sb = reinterpret_cast<const char*>(a.seg.base + (long long)n * a.seg.sn);
#pragma unroll 1
            for (int it = 0; it < 4; ++it) {
                const int src = it * 4 + grp;
                AxisTaps X = shfl_taps(mX, src), Yc = shfl_taps(mYc, src);
                const AxisTaps Yr = shfl_taps(mYr, src), Z = shfl_taps(mZ, src);
                X.lo += q4 * 16; X.hi += q4 * 16; Yc.lo += q4 * 16; Yc.hi += q4 * 16;
                const uint32_t o_seg = tc::sw128_offset(w * 16 + src, 4 + (q4 >> 1)) + (q4 & 1) * 8;
                float f[4];
                uint2 hi, lo;
                gather12(sb, X, Yr, Yc, Z, f);
                tc::split4_bf16(f, hi, lo);
                if (it == 0) tc::bar_sync(1 + wg, 128);                        // every warp is past the MMAs of the previous tile
                *reinterpret_cast<uint2*>(a_hi + o_seg) = hi;
                *reinterpret_cast<uint2*>(a_lo + o_seg) = lo;
            }
            tc::fence_async_smem();
            tc::bar_sync(1 + wg, 128);
        }
        float d1[32];
        tc::wgmma_fence();
#pragma unroll
        for (int ks = 2; ks < 4; ++ks) {                                       // K columns 32..63 (the shape features)
            tc::Wgmma<64>::ss(d1, ah + ks * 2, wh + ks * 2, ks > 2);
            tc::Wgmma<64>::ss(d1, ah + ks * 2, wl + ks * 2, 1);
            tc::Wgmma<64>::ss(d1, al + ks * 2, wh + ks * 2, 1);
        }
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::fence_regs(d1);
        float sig[2] = {0.f, 0.f};                                             // rows g and g + 8
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int col = 8 * j + 2 * c + e;
#pragma unroll
                for (int r = 0; r < 2; ++r) sig[r] = fmaf(softplus2(d1[4 * j + 2 * r + e] + b1s[col]), wsig[col], sig[r]);
            }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            float v = sig[r];
            v += __shfl_xor_sync(kFull, v, 1); v += __shfl_xor_sync(kFull, v, 2);
            const long long p = p0 + g + 8 * r;
            if (c == 0 && p < a.P) a.out[(long long)n * a.P + p] = v + sig_b;
        }
    }
}

}  // namespace vtc

// entry used by voxel.cu: sigma-only queries with a three-head style decoder on channels-last planes.  `handled` = false when the
// decoder has no density head of its own over the shape planes (the CUDA-core kernel then runs).
int launch_sigma_tc(const VoxelArgs& v, cudaStream_t st, bool& handled) {
    handled = false;
    const ide3d_mlp_head* H = nullptr;
    for (int h = 0; h < v.dec.num_heads; ++h) {
        const ide3d_mlp_head& c = v.dec.heads[h];
        if (c.out_offset <= kOut - 1 && c.out_offset + c.out_count > kOut - 1) {        // the head that produces sigma
            if (c.out_count != 1 || c.hidden != 64 || c.in_sel != 1) return IDE3D_OK;
            H = &c;
        }
    }
    if (H == nullptr) return IDE3D_OK;
    if (!plane_fits_32bit(v.seg)) return IDE3D_OK;
    if (tuning_env("IDE3D_VOXEL_SIMT") != nullptr) return IDE3D_OK;
    handled = true;
    vtc::Args a;
    static_cast<VoxelArgs&>(a) = v;
    a.w1 = H->w1; a.b1 = H->b1; a.w2 = H->w2; a.b2 = H->b2;
    a.tiles_per_item = (v.P + 63) / 64;
    a.num_tiles = a.tiles_per_item * v.n;
    const int smem = 2 * vtc::kW1Bytes + kWarpgroups * kStageBytes + 128 * 4 + 1024;
    int grid, rc;
    if ((rc = persistent_grid(vtc::sigma_tc_kernel, kTcThreads, smem, ceil_div<long long>(a.num_tiles, kWarpgroups), grid)) != IDE3D_OK) return rc;
    vtc::sigma_tc_kernel<<<grid, kTcThreads, smem, st>>>(a);
    IDE3D_CHECK_LAUNCH("sigma_tc_kernel");
    return IDE3D_OK;
}

}  // namespace ide3d
