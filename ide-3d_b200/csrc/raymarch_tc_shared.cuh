// Pieces shared by the tensor-core kernels (raymarch_tc.cu: the fused renderer; voxel_tc.cu: density queries): tile geometry,
// per-ray set-up, the tri-plane gather that feeds the swizzled A tiles, and the host-side hidden-block program.
#pragma once
#include <stdlib.h>

#include "raymarch_common.cuh"
#include "tc_ptx.cuh"

namespace ide3d {

constexpr int kWarpgroups = 2;                                          // warpgroups per CTA; each marches its own units
constexpr int kTcThreads = 128 * kWarpgroups;
constexpr int kTcMaxBlocks = 3;
constexpr int kTileBytes = 64 * 128;                                     // [64 rows x 64 bf16], one warpgroup's tile
constexpr int kStageBytes = 2 * kTileBytes;                              // hi + lo
constexpr int kUnitW = 4, kUnitH = 2, kTileDepth = 8;                    // unit = 4 x 2 rays; tile = 8 depth samples of the unit

struct TcBlock {
    const float* w1; int w1_ld, k0, kcount;        // W1 rows of this hidden block; inputs land at A columns [k0, k0+kcount)
    const float* b1;
    const float* w2; int w2_ld, out0, outc;        // W2[out, hidden cols of this block]; rows feed outputs [out0, out0+outc)
    int w1_off;                                    // byte offset of the [64 x 64] W1 tile inside a weight part (shared by two 32-input blocks)
    int w2_off, w2_row0, w2_rows;                  // byte offset of the W2 row block; it feeds output columns [w2_row0, w2_row0 + w2_rows)
};
struct TcProgram {
    int nblocks;
    TcBlock blk[kTcMaxBlocks];
    int wpart;                                     // bytes of one weight part (hi or lo), multiple of 1024
};

struct TcArgs {
    PlaneView tex, seg;
    ide3d_decoder dec;
    TcProgram prog;
    const float* cam2world;
    int n, res_w, res_h, steps;
    float cam_z, ray_start, ray_end, box_scale;
    int jitter_mode;
    const float* jitter_u;
    uint32_t seed_lo, seed_hi;
    int clamp_mode, last_back, white_back, fill_weight;
    float max_depth, noise_std;
    const float* noise;
    float *out_feat, *out_depth, *out_weights;
    int units_x, units_y, num_units, tiles_per_unit;
};

// log2(1 + 2^t): the hidden softplus in base-2 units (log2e folded into W1 / b1, ln2 into W2 at set-up).  ex2 of the clamped
// argument cannot overflow; for t >= 24 the sum rounds to 2^t and lg2 returns t itself, max(., t) keeps t beyond the clamp.
__device__ __forceinline__ float softplus2(float t) {
    float e, l;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(fminf(t, 126.f)));
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(l) : "f"(1.f + e));
    return fmaxf(l, t);
}

__device__ __forceinline__ void tile_store_bf16(unsigned char* tile, int row, int k, __nv_bfloat16 v) {
    *reinterpret_cast<__nv_bfloat16*>(tile + tc::sw128_offset(row, k >> 3) + (k & 7) * 2) = v;
}

// per-ray constants
struct RaySetup {
    int n, ray;
    bool ok;
    float dx, dy, dz, dnorm, spacing;
    long long sample_base;
};
__device__ __forceinline__ RaySetup ray_setup(const TcArgs& a, int unit, int rx, int ry) {
    RaySetup r;
    const int per_frame = a.units_x * a.units_y;
    r.n = unit / per_frame;
    const int t = unit - r.n * per_frame;
    const int px = (t % a.units_x) * kUnitW + rx;
    const int py = (t / a.units_x) * kUnitH + ry;
    r.ok = (px < a.res_w) && (py < a.res_h);
    r.ray = r.ok ? py * a.res_w + px : 0;
    const float x = linspace_at(-1.f, 1.f, a.res_w, px);
    const float y = linspace_at(1.f, -1.f, a.res_h, py);
    const float inv = 1.f / sqrtf(x * x + y * y + a.cam_z * a.cam_z);
    r.dx = x * inv; r.dy = y * inv; r.dz = a.cam_z * inv;
    r.dnorm = sqrtf(r.dx * r.dx + r.dy * r.dy + r.dz * r.dz);
    const int S = a.steps;
    r.spacing = (S > 1) ? linspace_at(a.ray_start, a.ray_end, S, 1) - linspace_at(a.ray_start, a.ray_end, S, 0) : 0.f;
    r.sample_base = ((long long)r.n * (a.res_w * a.res_h) + r.ray) * S;
    return r;
}
// jittered depth of sample s and of sample s+1 (z1, only meaningful when s+1 < S), and the jitter offset of s
__device__ __forceinline__ void sample_depths(const TcArgs& a, const RaySetup& r, int s, float& z0, float& off0, float& z1) {
    const int S = a.steps;
    z0 = linspace_at(a.ray_start, a.ray_end, S, s);
    z1 = (s + 1 < S) ? linspace_at(a.ray_start, a.ray_end, S, s + 1) : 0.f;
    off0 = 0.f;
    if (a.jitter_mode == IDE3D_JITTER_TENSOR) {
        off0 = (a.jitter_u[r.sample_base + s] - 0.5f) * r.spacing;
        if (s + 1 < S) z1 += (a.jitter_u[r.sample_base + s + 1] - 0.5f) * r.spacing;
    } else if (a.jitter_mode == IDE3D_JITTER_HASH) {
        const uint32_t gi = (uint32_t)(r.sample_base + s);
        off0 = (jitter_hash(gi, a.seed_lo, a.seed_hi) - 0.5f) * r.spacing;
        if (s + 1 < S) z1 += (jitter_hash(gi + 1u, a.seed_lo, a.seed_hi) - 0.5f) * r.spacing;
    } else if (a.jitter_mode == IDE3D_JITTER_ZVALS) {                  // depths given per sample (hierarchical second pass)
        z0 = a.jitter_u[r.sample_base + s];
        z1 = (s + 1 < S) ? a.jitter_u[r.sample_base + s + 1] : 0.f;
    }
}

// one tri-plane's contribution to 4 channels of one sample: 12 LDG.128 in flight, then the blend (plane by plane, taps in the
// order (col lo,row lo) (col hi,row lo) (col lo,row hi) (col hi,row hi) -- the arithmetic of gather_chunk_axes)
// Offsets are 32-bit BYTE offsets (tap = row role + column role + plane * 128 B; the lane's channel quad is already folded into the
// column roles), added to a 64-bit per-frame base: 3 integer instructions per load.
__device__ __forceinline__ float4 ldg_at(const char* __restrict__ base, unsigned byte_off) {
    return __ldg(reinterpret_cast<const float4*>(base + byte_off));
}
__device__ __forceinline__ void gather12(const char* __restrict__ base, const AxisTaps& X, const AxisTaps& Yr, const AxisTaps& Yc,
                                         const AxisTaps& Z, float (&out)[4]) {
    float4 v[12];
#define IDE3D_LD(k, C, R)                                                                                         \
    v[4 * k + 0] = ldg_at(base, (unsigned)(R.lo + C.lo + k * (kFeat * 4))); v[4 * k + 1] = ldg_at(base, (unsigned)(R.lo + C.hi + k * (kFeat * 4))); \
    v[4 * k + 2] = ldg_at(base, (unsigned)(R.hi + C.lo + k * (kFeat * 4))); v[4 * k + 3] = ldg_at(base, (unsigned)(R.hi + C.hi + k * (kFeat * 4)));
    IDE3D_LD(0, X, Yr)
    IDE3D_LD(1, Yc, Z)
    IDE3D_LD(2, X, Z)
#undef IDE3D_LD
    out[0] = out[1] = out[2] = out[3] = 0.f;
#define IDE3D_BLEND(k, C, R)                                                                                      \
    {                                                                                                             \
        const float w4[4] = {C.wlo * R.wlo, C.whi * R.wlo, C.wlo * R.whi, C.whi * R.whi};                         \
        float p[4] = {0.f, 0.f, 0.f, 0.f};                                                                        \
        _Pragma("unroll") for (int tap = 0; tap < 4; ++tap) {                                                     \
            const float4 t4 = v[k * 4 + tap];                                                                     \
            const float w_ = w4[tap];                                                                             \
            p[0] += t4.x * w_; p[1] += t4.y * w_; p[2] += t4.z * w_; p[3] += t4.w * w_;                           \
        }                                                                                                         \
        _Pragma("unroll") for (int j = 0; j < 4; ++j) out[j] += p[j];                                             \
    }
    IDE3D_BLEND(0, X, Yr)
    IDE3D_BLEND(1, Yc, Z)
    IDE3D_BLEND(2, X, Z)
#undef IDE3D_BLEND
}

__device__ __forceinline__ AxisTaps shfl_taps(const AxisTaps& t, int src) {
    AxisTaps r;
    r.lo = __shfl_sync(kFull, t.lo, src); r.hi = __shfl_sync(kFull, t.hi, src);
    r.wlo = __shfl_sync(kFull, t.wlo, src); r.whi = __shfl_sync(kFull, t.whi, src);
    return r;
}


// Build the hidden-block program from the head list and lay the weight tiles out compactly.  Returns false when the decoder does
// not fit (hidden not a multiple of 64, more than kTcMaxBlocks blocks, outputs beyond 64 columns).
inline bool build_program(const ide3d_decoder& d, TcProgram& P) {
    P.nblocks = 0;
    for (int h = 0; h < d.num_heads; ++h) {
        const ide3d_mlp_head& H = d.heads[h];
        if (H.hidden <= 0 || H.hidden % 64 != 0) return false;
        if (H.out_offset < 0 || H.out_count <= 0 || H.out_offset + H.out_count > 64) return false;
        if (H.in_sel < 0 || H.in_sel > 2) return false;
        const int in = (H.in_sel == 2) ? 64 : 32;
        for (int c = 0; c < H.hidden / 64; ++c) {
            if (P.nblocks == kTcMaxBlocks) return false;
            TcBlock& B = P.blk[P.nblocks++];
            B.w1 = H.w1 + (size_t)c * 64 * in; B.w1_ld = in;
            B.k0 = (H.in_sel == 1) ? 32 : 0; B.kcount = in;
            B.b1 = H.b1 + c * 64;
            B.w2 = H.w2 + c * 64; B.w2_ld = H.hidden;
            B.out0 = H.out_offset; B.outc = H.out_count;
            // layer-2 column range in units of 16 (an N of 16..64 for the layer-2 MMA)
            const int g0 = H.out_offset / 16, g1 = (H.out_offset + H.out_count + 15) / 16;
            B.w2_row0 = g0 * 16;
            B.w2_rows = (g1 - g0) * 16;
        }
    }
    if (P.nblocks == 0) return false;
    // weight layout inside one part (hi or lo): W1 tiles of 8 KB ([64 hidden x 64 inputs]; two 32-input blocks with different k0
    // share a tile), then the W2 row blocks ((g1 - g0) * 16 rows x 128 bytes)
    int ntiles = 0, half_free[kTcMaxBlocks];          // half_free[t]: k0 of the half still free in tile t, or -1
    for (int b = 0; b < P.nblocks; ++b) {
        TcBlock& B = P.blk[b];
        int tile = -1;
        if (B.kcount == 32)
            for (int t = 0; t < ntiles; ++t) if (half_free[t] == B.k0) { tile = t; half_free[t] = -1; break; }
        if (tile < 0) {
            tile = ntiles++;
            half_free[tile] = (B.kcount == 32) ? (32 - B.k0) : -1;
        }
        B.w1_off = tile * 64 * 128;
    }
    int off = ntiles * 64 * 128;
    for (int b = 0; b < P.nblocks; ++b) {
        TcBlock& B = P.blk[b];
        B.w2_off = off;
        off += B.w2_rows * 128;
    }
    P.wpart = (off + 1023) & ~1023;
    return true;
}

}  // namespace ide3d
