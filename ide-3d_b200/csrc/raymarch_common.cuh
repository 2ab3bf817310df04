// Building blocks shared by the fused renderer kernels (raymarch*.cu, voxel*.cu): the ray-march parameter contract (validation,
// kernel arguments) and the device helpers of the gather, the decoder and the compositing.
//
// Data layout in HBM: a tri-plane tensor is [N, 96, H, W] fp32.  The fast path wants it
// channels-last ([N, H, W, 96]): one texel of one plane = 32 floats = one 128-byte line, fetched by
// eight lanes with one LDG.128 each (fully coalesced, 4 texels per warp instruction).
//
// Work mapping: one warp = one chunk of 32 consecutive samples.
//   gather : lane l serves sample (4*i + l/8) in sub-iteration i, channels 4*(l%8)..+3   (8 lanes/texel)
//   MLP    : lane l owns sample l (features transposed through a padded shared-memory row)
//   scan   : lane order = sample order along the ray, so compositing is a warp scan.
#pragma once

#include "common.cuh"

namespace ide3d {

constexpr int kFeat = 32;          // channels per plane
constexpr int kOut = 52;           // decoder outputs: 32 colour + 19 semantic + sigma
constexpr int kRow = 68;           // staging row stride in floats (64 + 4: conflict-free LDS.128/STS.128)
constexpr unsigned kFull = 0xffffffffu;

struct PlaneView {
    const float* base;
    long long sn, sc, sh, sw;      // element strides
    int h, w;
};

inline PlaneView make_view(const ide3d_triplane& t) {
    PlaneView v;
    v.base = t.data; v.sn = t.stride_n; v.sc = t.stride_c; v.sh = t.stride_h; v.sw = t.stride_w;
    v.h = t.h; v.w = t.w;
    return v;
}

// the fast gather's layout: [N, H, W, 96] with every texel on a 16-byte boundary (one LDG.128 per channel quad)
inline bool planes_channels_last(const ide3d_triplane& t) {
    return t.stride_c == 1 && (t.stride_w % 4 == 0) && (t.stride_h % 4 == 0) && (t.stride_n % 4 == 0) &&
           ((reinterpret_cast<uintptr_t>(t.data) & 15) == 0);
}

// ---------------------------------------------------------------------------------------------
// the ray-march parameter contract, shared by the forward kernels (raymarch.cu, raymarch_tc.cu) and the backward (raymarch_bwd.cu)

inline int check_planes(const ide3d_triplane& t, const char* name) {
    IDE3D_REQUIRE(t.data != nullptr, "%s: null data", name);
    IDE3D_REQUIRE(t.n > 0 && t.h > 0 && t.w > 0, "%s: empty tri-plane", name);
    return IDE3D_OK;
}

// Checks of ide3d_raymarch_params that every ray-march entry point needs before it reads the struct.
inline int check_raymarch_params(const ide3d_raymarch_params* p) {
    IDE3D_REQUIRE(p != nullptr, "raymarch: null params");
    int rc;
    if ((rc = check_planes(p->tex, "tex")) != IDE3D_OK) return rc;
    if ((rc = check_planes(p->seg, "seg")) != IDE3D_OK) return rc;
    IDE3D_REQUIRE(p->tex.h == p->seg.h && p->tex.w == p->seg.w, "raymarch: tex/seg plane sizes differ");
    IDE3D_REQUIRE(p->views >= 0, "raymarch: negative views");
    const long long views = p->views > 1 ? p->views : 1;
    IDE3D_REQUIRE(p->n > 0 && (long long)p->tex.n * views == p->n && (long long)p->seg.n * views == p->n, "raymarch: batch mismatch");
    IDE3D_REQUIRE(p->res_w > 0 && p->res_h > 0 && p->num_steps > 0, "raymarch: empty render");
    IDE3D_REQUIRE(p->cam2world != nullptr, "raymarch: null camera/output");
    IDE3D_REQUIRE(p->clamp_mode == IDE3D_CLAMP_SOFTPLUS || p->clamp_mode == IDE3D_CLAMP_RELU,
                  "Need to choose clamp mode");   // volumetric_rendering.py:51-52
    IDE3D_REQUIRE(p->jitter_mode >= 0 && p->jitter_mode <= 3, "raymarch: bad jitter mode");
    IDE3D_REQUIRE((p->jitter_mode != IDE3D_JITTER_TENSOR && p->jitter_mode != IDE3D_JITTER_ZVALS) || p->jitter_u, "raymarch: jitter / depth tensor missing");
    IDE3D_REQUIRE((long long)p->n * p->res_w * p->res_h * p->num_steps < (1ll << 32),
                  "raymarch: more than 2^32 samples per call");       // the jitter hash indexes samples with 32 bits
    return IDE3D_OK;
}

// Kernel arguments every ray-march kernel reads: RayArgs extends it, TcArgs and BwdArgs restate its fields.
struct MarchArgs {
    PlaneView tex, seg;
    ide3d_decoder dec;
    const float* cam2world;
    int n, res_w, res_h, steps;
    float cam_z;          // -1 / tan(fov/2)
    float ray_start, ray_end, box_scale;
    int jitter_mode;
    const float* jitter_u;
    uint32_t seed_lo, seed_hi;
    int clamp_mode, last_back, white_back, fill_weight;
    float max_depth, noise_std;
    const float* noise;   // null when noise_std == 0
    int views;            // frames per plane set (>= 1)
    const uint64_t* jitter_seeds;   // [n] per-frame HASH seeds, or null
};

// Args: MarchArgs or a struct with the same fields.  TcArgs and BwdArgs restate them instead of deriving from MarchArgs: as a
// derived kernel parameter the struct changes the code ptxas emits for those two kernels (3 more registers for raymarch_tc_kernel).
template <typename Args>
inline void fill_march_args(const ide3d_raymarch_params& p, Args& a) {
    a.tex = make_view(p.tex); a.seg = make_view(p.seg); a.dec = p.dec;
    a.cam2world = p.cam2world;
    a.n = p.n; a.res_w = p.res_w; a.res_h = p.res_h; a.steps = p.num_steps;
    a.cam_z = (float)(-1.0 / tan((2.0 * 3.14159265358979323846 * (double)p.fov_deg / 360.0) / 2.0));
    a.ray_start = p.ray_start; a.ray_end = p.ray_end; a.box_scale = p.box_scale;
    a.jitter_mode = p.jitter_mode; a.jitter_u = p.jitter_u;
    a.seed_lo = (uint32_t)(p.jitter_seed & 0xffffffffu); a.seed_hi = (uint32_t)(p.jitter_seed >> 32);
    a.clamp_mode = p.clamp_mode; a.last_back = p.last_back; a.white_back = p.white_back;
    a.fill_weight = p.fill_weight; a.max_depth = p.max_depth;
    a.noise_std = p.noise_std; a.noise = (p.noise_std != 0.f) ? p.noise : nullptr;
    a.views = p.views > 1 ? p.views : 1;
    a.jitter_seeds = p.jitter_seeds;
}

// The plane set frame n reads: `views` consecutive frames (the views of one latent) share one set.
__device__ __forceinline__ int plane_set(int n, int views) { return views > 1 ? n / views : n; }

// HASH jitter key of global sample index `sample` = (n * R + ray) * S + s of frame n: with per-frame seeds, jitter_seeds[n] and the
// frame-local index (frame n is then bit-identical to a one-frame launch with that seed); otherwise the launch's seed and the global
// index.  The hash indexes samples with 32 bits (check_raymarch_params bounds the launch).
struct HashKey {
    uint32_t idx, lo, hi;
};
template <typename Args>
__device__ __forceinline__ HashKey hash_key(const Args& a, int n, long long sample) {
    HashKey k;
    if (a.jitter_seeds != nullptr) {
        const unsigned long long seed = __ldg(reinterpret_cast<const unsigned long long*>(a.jitter_seeds) + n);
        k.idx = (uint32_t)(sample - (long long)n * a.res_w * a.res_h * a.steps);
        k.lo = (uint32_t)(seed & 0xffffffffull);
        k.hi = (uint32_t)(seed >> 32);
    } else {
        k.idx = (uint32_t)sample;
        k.lo = a.seed_lo;
        k.hi = a.seed_hi;
    }
    return k;
}

// ---------------------------------------------------------------------------------------------
// point queries (voxel.cu: CUDA cores; voxel_tc.cu: tensor cores, sigma only)

struct VoxelArgs {
    PlaneView tex, seg;
    ide3d_decoder dec;
    const float* points;      // [N, P, 3] or null (grid mode)
    long long P;              // points per batch item
    int n;
    float box_scale;
    int sigma_only;
    float* out;
    // grid mode (extract_shapes.create_samples)
    int grid_n;
    float voxel_size, org_x, org_y, org_z, pre_scale;
    long long first;
};

// ---------------------------------------------------------------------------------------------
// scalar helpers

// torch.linspace(start, end, steps)[i] for float32 (symmetric evaluation from both ends)
__device__ __forceinline__ float linspace_at(float start, float end, int steps, int i) {
    if (steps <= 1) return start;
    const float step = (end - start) / (float)(steps - 1);
    return (i < steps / 2) ? (start + step * (float)i) : (end - step * (float)(steps - 1 - i));
}

// counter-based uniform in [0,1); integer-exact twin of oracle.renderer.hash_uniform
__device__ __forceinline__ float jitter_hash(uint32_t idx, uint32_t lo, uint32_t hi) {
    uint32_t h = idx ^ lo;
    h *= 0x9E3779B1u;
    h ^= hi;
    h ^= h >> 16; h *= 0x21F0AAADu;
    h ^= h >> 15; h *= 0x735A2D97u;
    h ^= h >> 15;
    return (float)(h >> 8) * (1.0f / 16777216.0f);
}

// hidden-layer activation: |err| < 4e-7 absolute (MUFU ex2/lg2 on an argument in (1,2])
__device__ __forceinline__ float softplus_fast(float x) {
    return fmaxf(x, 0.f) + __logf(1.f + __expf(-fabsf(x)));
}
// density activation: full precision, matters because delta_last = 1e10 amplifies tiny values
__device__ __forceinline__ float softplus_precise(float x) {
    return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x)));
}

// coordinates of flat voxel index `idx`, bit-for-bit like extract_shapes.py:74-96 followed by `0.9 *`
__device__ __forceinline__ void grid_point(const VoxelArgs& a, long long idx, float& x, float& y, float& z) {
    const float N = (float)a.grid_n;
    const float fi = (float)idx;                                   // overall_index.float()
    const float s2 = (float)(idx % a.grid_n);                      // samples[:, 2] = index % N   (integer)
    const float q1 = __fdiv_rn(fi, N);
    const float s1 = fmodf(q1, N);                                 // (index.float() / N) % N      (fractional!)
    const float s0 = fmodf(__fdiv_rn(q1, N), N);                   // ((index.float() / N) / N) % N
    // column 0 uses voxel_origin[2], column 2 uses voxel_origin[0] (:91-93)
    x = __fmul_rn(__fadd_rn(__fmul_rn(s0, a.voxel_size), a.org_z), a.pre_scale);
    y = __fmul_rn(__fadd_rn(__fmul_rn(s1, a.voxel_size), a.org_y), a.pre_scale);
    z = __fmul_rn(__fadd_rn(__fmul_rn(s2, a.voxel_size), a.org_x), a.pre_scale);
}

// ---------------------------------------------------------------------------------------------
// bilinear footprint of one sample in one plane (align_corners=False, zeros padding)
struct Foot {
    int x0, y0;
    float fx, fy;
};
__device__ __forceinline__ Foot footprint(float u, float v, int W, int H) {
    Foot f;
    const float ix = ((u + 1.f) * (float)W - 1.f) * 0.5f;
    const float iy = ((v + 1.f) * (float)H - 1.f) * 0.5f;
    const float fx0 = floorf(ix), fy0 = floorf(iy);
    f.fx = ix - fx0;
    f.fy = iy - fy0;
    // clamp before the int conversion so that far-away points stay "out of range" instead of wrapping
    f.x0 = (int)fminf(fmaxf(fx0, -2.f), (float)W + 1.f);
    f.y0 = (int)fminf(fmaxf(fy0, -2.f), (float)H + 1.f);
    return f;
}

// Gather the features of the 32 samples of this warp's chunk from both tri-planes into the staging
// rows: stage[s*kRow + 0..31] = texture features, stage[s*kRow + 32..63] = shape features.
// (cx,cy,cz): this lane's own sample in plane grid units.  Inactive lanes pass any finite value.
// `store(sample, q, at, as)` receives, for sample `sample` (0..31 of the chunk), the texture / shape features of
// channels 4q..4q+3.
// kSkipTex: the caller only needs the shape features (sigma-only queries of a decoder whose sigma head reads the shape
// planes alone): the texture tri-plane is not touched at all.
template <bool kChannelsLast, bool kSkipTex = false, typename Store>
__device__ __forceinline__ void gather_chunk_to(const PlaneView& tex, const PlaneView& seg, int n, float cx,
                                                float cy, float cz, int lane, Store store) {
    const int W = tex.w, H = tex.h;
    // plane 0 samples (x,y), plane 1 (y,z), plane 2 (x,z)   (dnnlib/util.py:589-596)
    const Foot f0 = footprint(cx, cy, W, H);
    const Foot f1 = footprint(cy, cz, W, H);
    const Foot f2 = footprint(cx, cz, W, H);
    const int q = lane & 7;          // channel quad
    const int grp = lane >> 3;       // which of the 4 samples of a sub-iteration
    const float* tbase = tex.base + (long long)n * tex.sn;
    const float* sbase = seg.base + (long long)n * seg.sn;

#pragma unroll 1
    for (int it = 0; it < 8; ++it) {
        const int src = it * 4 + grp;
        float at[4] = {0.f, 0.f, 0.f, 0.f}, as[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const Foot& mine = (k == 0) ? f0 : (k == 1 ? f1 : f2);
            const int x0 = __shfl_sync(kFull, mine.x0, src);
            const int y0 = __shfl_sync(kFull, mine.y0, src);
            const float fx = __shfl_sync(kFull, mine.fx, src);
            const float fy = __shfl_sync(kFull, mine.fy, src);
            float pt[4] = {0.f, 0.f, 0.f, 0.f}, ps[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int tap = 0; tap < 4; ++tap) {
                const int xx = x0 + (tap & 1), yy = y0 + (tap >> 1);
                const bool ok = ((unsigned)xx < (unsigned)W) && ((unsigned)yy < (unsigned)H);
                const float wx = (tap & 1) ? fx : 1.f - fx;
                const float wy = (tap >> 1) ? fy : 1.f - fy;
                const float wgt = wx * wy;
                if (ok) {
                    if (kChannelsLast) {
                        const long long to = (long long)yy * tex.sh + (long long)xx * tex.sw + k * kFeat + q * 4;
                        const long long so = (long long)yy * seg.sh + (long long)xx * seg.sw + k * kFeat + q * 4;
                        const float4 b = __ldg(reinterpret_cast<const float4*>(sbase + so));
                        ps[0] += b.x * wgt; ps[1] += b.y * wgt; ps[2] += b.z * wgt; ps[3] += b.w * wgt;
                        if constexpr (!kSkipTex) {
                            const float4 a = __ldg(reinterpret_cast<const float4*>(tbase + to));
                            pt[0] += a.x * wgt; pt[1] += a.y * wgt; pt[2] += a.z * wgt; pt[3] += a.w * wgt;
                        }
                    } else {
                        const long long to = (long long)yy * tex.sh + (long long)xx * tex.sw;
                        const long long so = (long long)yy * seg.sh + (long long)xx * seg.sw;
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const int c = k * kFeat + q * 4 + j;
                            if constexpr (!kSkipTex) pt[j] += __ldg(tbase + to + (long long)c * tex.sc) * wgt;
                            ps[j] += __ldg(sbase + so + (long long)c * seg.sc) * wgt;
                        }
                    }
                }
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) { at[j] += pt[j]; as[j] += ps[j]; }
        }
        store(src, q, at, as);
    }
}

// Per-axis form of the same gather (tensor-core kernels): the three planes share their axes -- x is the column of planes 0 and
// 2, y the row of plane 0 and the column of plane 1, z the row of planes 1 and 2 -- so the floor / fraction / validity /
// clamp work is done once per axis role (4 roles) instead of once per tap (12 taps), and a tap's offset and weight are one
// add and one multiply.  Same arithmetic as the per-tap form above: w = (x-weight or 0) * (y-weight or 0), identical products.
// Taps whose weight is 0 (outside the plane) read a clamped, valid address -- no branches; all 24 LDG.128 of a pass are in flight.
struct AxisFoot {
    int i0;
    float f;
};
__device__ __forceinline__ AxisFoot axis_foot(float u, int D) {
    AxisFoot a;
    const float ix = ((u + 1.f) * (float)D - 1.f) * 0.5f;
    const float f0 = floorf(ix);
    a.f = ix - f0;
    a.i0 = (int)fminf(fmaxf(f0, -2.f), (float)D + 1.f);         // far-away points stay out of range instead of wrapping
    return a;
}
struct AxisTaps {
    int lo, hi;          // clamped indices, pre-multiplied by the stride of the role (float4 units)
    float wlo, whi;      // weights, 0 for an out-of-range tap
};
__device__ __forceinline__ AxisTaps axis_taps(int i0, float f, int D, int stride) {
    AxisTaps t;
    const bool lo_ok = (unsigned)i0 < (unsigned)D, hi_ok = (unsigned)(i0 + 1) < (unsigned)D;
    t.lo = min(max(i0, 0), D - 1) * stride;
    t.hi = min(max(i0 + 1, 0), D - 1) * stride;
    t.wlo = lo_ok ? 1.f - f : 0.f;
    t.whi = hi_ok ? f : 0.f;
    return t;
}
template <typename Store>
__device__ __forceinline__ void gather_chunk_axes(const PlaneView& tex, const PlaneView& seg, int n, float cx, float cy,
                                                  float cz, int lane, Store store) {
    const int W = tex.w, H = tex.h;
    const int sh4 = (int)(tex.sh >> 2), sw4 = (int)(tex.sw >> 2);      // strides in float4 units (multiples of 4 floats)
    const AxisFoot ax = axis_foot(cx, W), ayr = axis_foot(cy, H), ayc = axis_foot(cy, W), az = axis_foot(cz, H);
    const int q = lane & 7, grp = lane >> 3;
    const float4* tb = reinterpret_cast<const float4*>(tex.base + (long long)n * tex.sn) + q;
    const float4* sb = reinterpret_cast<const float4*>(seg.base + (long long)n * seg.sn) + q;

#pragma unroll 1
    for (int it = 0; it < 8; ++it) {
        const int src = it * 4 + grp;
        const AxisTaps X = axis_taps(__shfl_sync(kFull, ax.i0, src), __shfl_sync(kFull, ax.f, src), W, sw4);     // column of planes 0, 2
        const AxisTaps Yr = axis_taps(__shfl_sync(kFull, ayr.i0, src), __shfl_sync(kFull, ayr.f, src), H, sh4);  // row of plane 0
        const AxisTaps Yc = axis_taps(__shfl_sync(kFull, ayc.i0, src), __shfl_sync(kFull, ayc.f, src), W, sw4);  // column of plane 1
        const AxisTaps Z = axis_taps(__shfl_sync(kFull, az.i0, src), __shfl_sync(kFull, az.f, src), H, sh4);     // row of planes 1, 2
        // tap order inside a plane: (col lo,row lo) (col hi,row lo) (col lo,row hi) (col hi,row hi)
        float4 v[12], u[12];
#define IDE3D_PLANE_LOADS(k, C, R)                                                                                 \
        {                                                                                                         \
            const int o0 = R.lo + C.lo + k * (kFeat / 4), o1 = R.lo + C.hi + k * (kFeat / 4);                     \
            const int o2 = R.hi + C.lo + k * (kFeat / 4), o3 = R.hi + C.hi + k * (kFeat / 4);                     \
            v[4 * k + 0] = __ldg(tb + o0); v[4 * k + 1] = __ldg(tb + o1); v[4 * k + 2] = __ldg(tb + o2); v[4 * k + 3] = __ldg(tb + o3); \
            u[4 * k + 0] = __ldg(sb + o0); u[4 * k + 1] = __ldg(sb + o1); u[4 * k + 2] = __ldg(sb + o2); u[4 * k + 3] = __ldg(sb + o3); \
        }
        IDE3D_PLANE_LOADS(0, X, Yr)
        IDE3D_PLANE_LOADS(1, Yc, Z)
        IDE3D_PLANE_LOADS(2, X, Z)                                       // all 24 LDG.128 in flight
#undef IDE3D_PLANE_LOADS
        float at[4] = {0.f, 0.f, 0.f, 0.f}, as[4] = {0.f, 0.f, 0.f, 0.f};
#define IDE3D_PLANE_BLEND(k, C, R)                                                                                 \
        {                                                                                                         \
            const float w4[4] = {C.wlo * R.wlo, C.whi * R.wlo, C.wlo * R.whi, C.whi * R.whi};                     \
            float p[4] = {0.f, 0.f, 0.f, 0.f}, r[4] = {0.f, 0.f, 0.f, 0.f};                                       \
            _Pragma("unroll") for (int tap = 0; tap < 4; ++tap) {                                                 \
                const float4 a = v[k * 4 + tap], b = u[k * 4 + tap];                                              \
                const float w_ = w4[tap];                                                                         \
                p[0] += a.x * w_; p[1] += a.y * w_; p[2] += a.z * w_; p[3] += a.w * w_;                           \
                r[0] += b.x * w_; r[1] += b.y * w_; r[2] += b.z * w_; r[3] += b.w * w_;                           \
            }                                                                                                     \
            _Pragma("unroll") for (int j = 0; j < 4; ++j) { at[j] += p[j]; as[j] += r[j]; }                       \
        }
        IDE3D_PLANE_BLEND(0, X, Yr)
        IDE3D_PLANE_BLEND(1, Yc, Z)
        IDE3D_PLANE_BLEND(2, X, Z)
#undef IDE3D_PLANE_BLEND
        store(src, q, at, as);
    }
}

// staging-row flavour used by the SIMT kernels: stage[s*kRow + 0..31] = texture, [32..63] = shape features
template <bool kChannelsLast, bool kSkipTex = false>
__device__ __forceinline__ void gather_chunk(const PlaneView& tex, const PlaneView& seg, int n, float cx,
                                             float cy, float cz, float* __restrict__ stage, int lane) {
    gather_chunk_to<kChannelsLast, kSkipTex>(tex, seg, n, cx, cy, cz, lane, [stage](int src, int q, const float (&at)[4], const float (&as)[4]) {
        float* row = stage + src * kRow;
        if constexpr (!kSkipTex) *reinterpret_cast<float4*>(row + q * 4) = make_float4(at[0], at[1], at[2], at[3]);
        *reinterpret_cast<float4*>(row + kFeat + q * 4) = make_float4(as[0], as[1], as[2], as[3]);
    });
    __syncwarp();
}

// ---------------------------------------------------------------------------------------------
// decoder heads, lane-per-sample, weights broadcast from shared memory

template <int IN, int HID, int OUT>
struct HeadLayout {
    static constexpr int kW1 = 0;
    static constexpr int kB1 = HID * IN;
    static constexpr int kW2 = kB1 + HID;
    static constexpr int kB2 = kW2 + ((OUT * HID + 3) / 4) * 4;
    static constexpr int kSize = kB2 + ((OUT + 3) / 4) * 4;
};

// copy one head's parameters from global memory into the block's shared-memory image
template <int IN, int HID, int OUT>
__device__ __forceinline__ void load_head(const ide3d_mlp_head& h, float* __restrict__ dst) {
    using L = HeadLayout<IN, HID, OUT>;
    for (int i = threadIdx.x; i < HID * IN; i += blockDim.x) dst[L::kW1 + i] = h.w1[i];
    for (int i = threadIdx.x; i < HID; i += blockDim.x) dst[L::kB1 + i] = h.b1[i];
    for (int i = threadIdx.x; i < OUT * HID; i += blockDim.x) dst[L::kW2 + i] = h.w2[i];
    for (int i = threadIdx.x; i < OUT; i += blockDim.x) dst[L::kB2 + i] = h.b2[i];
}

// o = W2 softplus(W1 f + b1) + b2 for this lane's sample; f = IN floats at `frow` (shared memory)
template <int IN, int HID, int OUT>
__device__ __forceinline__ void mlp_head(const float* __restrict__ frow, const float* __restrict__ wsm,
                                         float (&o)[OUT]) {
    using L = HeadLayout<IN, HID, OUT>;
    float f[IN];
#pragma unroll
    for (int k = 0; k < IN; k += 4) {
        const float4 v = *reinterpret_cast<const float4*>(frow + k);
        f[k] = v.x; f[k + 1] = v.y; f[k + 2] = v.z; f[k + 3] = v.w;
    }
#pragma unroll
    for (int c = 0; c < OUT; ++c) o[c] = wsm[L::kB2 + c];

#pragma unroll 1
    for (int jc = 0; jc < HID; jc += 8) {
        float h[8];
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) h[jj] = wsm[L::kB1 + jc + jj];
#pragma unroll
        for (int k = 0; k < IN; k += 4) {
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                const float4 w = *reinterpret_cast<const float4*>(wsm + L::kW1 + (jc + jj) * IN + k);
                h[jj] = fmaf(w.x, f[k], h[jj]);
                h[jj] = fmaf(w.y, f[k + 1], h[jj]);
                h[jj] = fmaf(w.z, f[k + 2], h[jj]);
                h[jj] = fmaf(w.w, f[k + 3], h[jj]);
            }
        }
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) h[jj] = softplus_fast(h[jj]);
#pragma unroll
        for (int c = 0; c < OUT; ++c) {
            const float4 wa = *reinterpret_cast<const float4*>(wsm + L::kW2 + c * HID + jc);
            const float4 wb = *reinterpret_cast<const float4*>(wsm + L::kW2 + c * HID + jc + 4);
            float acc = o[c];
            acc = fmaf(wa.x, h[0], acc); acc = fmaf(wa.y, h[1], acc);
            acc = fmaf(wa.z, h[2], acc); acc = fmaf(wa.w, h[3], acc);
            acc = fmaf(wb.x, h[4], acc); acc = fmaf(wb.y, h[5], acc);
            acc = fmaf(wb.z, h[6], acc); acc = fmaf(wb.w, h[7], acc);
            o[c] = acc;
        }
    }
}

// decoder variants with a fused kernel
enum DecoderKind { kDense64 = 0, kDense128 = 1, kThreeHead64 = 2, kDecoderNone = -1 };

inline int classify_decoder(const ide3d_decoder& d) {
    if (d.num_heads == 1) {
        const ide3d_mlp_head& h = d.heads[0];
        if (h.in_sel == 2 && h.out_offset == 0 && h.out_count == kOut) {
            if (h.hidden == 64) return kDense64;
            if (h.hidden == 128) return kDense128;
        }
    } else if (d.num_heads == 3) {
        const ide3d_mlp_head *a = &d.heads[0], *b = &d.heads[1], *c = &d.heads[2];
        if (a->in_sel == 0 && a->out_offset == 0 && a->out_count == 32 && a->hidden == 64 &&
            b->in_sel == 1 && b->out_offset == 32 && b->out_count == 19 && b->hidden == 64 &&
            c->in_sel == 1 && c->out_offset == 51 && c->out_count == 1 && c->hidden == 64)
            return kThreeHead64;
    }
    return kDecoderNone;
}

template <int KIND> struct DecoderTraits;
template <> struct DecoderTraits<kDense64> { using H0 = HeadLayout<64, 64, 52>; static constexpr int kFloats = H0::kSize; };
template <> struct DecoderTraits<kDense128> { using H0 = HeadLayout<64, 128, 52>; static constexpr int kFloats = H0::kSize; };
template <> struct DecoderTraits<kThreeHead64> {
    using H0 = HeadLayout<32, 64, 32>;
    using H1 = HeadLayout<32, 64, 19>;
    using H2 = HeadLayout<32, 64, 1>;
    static constexpr int kOff1 = H0::kSize, kOff2 = H0::kSize + H1::kSize;
    static constexpr int kFloats = H0::kSize + H1::kSize + H2::kSize;
};

template <int KIND>
__device__ __forceinline__ void load_decoder(const ide3d_decoder& d, float* wsm) {
    if constexpr (KIND == kDense64) load_head<64, 64, 52>(d.heads[0], wsm);
    if constexpr (KIND == kDense128) load_head<64, 128, 52>(d.heads[0], wsm);
    if constexpr (KIND == kThreeHead64) {
        using T = DecoderTraits<kThreeHead64>;
        load_head<32, 64, 32>(d.heads[0], wsm);
        load_head<32, 64, 19>(d.heads[1], wsm + T::kOff1);
        load_head<32, 64, 1>(d.heads[2], wsm + T::kOff2);
    }
}

// sigma only (channel 51) for this lane's sample
template <int KIND>
__device__ __forceinline__ float decode_sigma(const float* row, const float* wsm) {
    if constexpr (KIND == kThreeHead64) {
        float s[1];
        mlp_head<32, 64, 1>(row + kFeat, wsm + DecoderTraits<kThreeHead64>::kOff2, s);
        return s[0];
    } else {
        float o[kOut];
        if constexpr (KIND == kDense64) mlp_head<64, 64, 52>(row, wsm, o);
        else mlp_head<64, 128, 52>(row, wsm, o);
        return o[kOut - 1];
    }
}

// all 52 channels for this lane's sample
template <int KIND>
__device__ __forceinline__ void decode_all(const float* row, const float* wsm, float (&o)[kOut]) {
    if constexpr (KIND == kThreeHead64) {
        using T = DecoderTraits<kThreeHead64>;
        float a[32], b[19], c[1];
        mlp_head<32, 64, 32>(row, wsm, a);
        mlp_head<32, 64, 19>(row + kFeat, wsm + T::kOff1, b);
        mlp_head<32, 64, 1>(row + kFeat, wsm + T::kOff2, c);
#pragma unroll
        for (int i = 0; i < 32; ++i) o[i] = a[i];
#pragma unroll
        for (int i = 0; i < 19; ++i) o[32 + i] = b[i];
        o[51] = c[0];
    } else if constexpr (KIND == kDense64) {
        mlp_head<64, 64, 52>(row, wsm, o);
    } else {
        mlp_head<64, 128, 52>(row, wsm, o);
    }
}

// warp product scan: returns the exclusive prefix product; `total` = product over all 32 lanes
__device__ __forceinline__ float warp_exclusive_product(float v, int lane, float& total) {
    float inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const float t = __shfl_up_sync(kFull, inc, d);
        if (lane >= d) inc *= t;
    }
    total = __shfl_sync(kFull, inc, 31);
    const float ex = __shfl_up_sync(kFull, inc, 1);
    return lane == 0 ? 1.f : ex;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(kFull, v, d);
    return v;
}

}  // namespace ide3d
