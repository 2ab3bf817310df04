// Fused volume renderer: rays -> jitter -> cam2world -> 2x tri-plane gather -> decoder MLP ->
// alpha compositing, one kernel, no per-sample intermediates in HBM.
//
// Replaces the chain the (absent) generator class runs per frame out of the reference's free
// functions: get_initial_rays_trig (training/volumetric_rendering.py:77-97), perturb_points (:99-105),
// transform_sampled_points (:108-136), sample_from_triplane x2 (dnnlib/util.py:580-617), decoder MLP,
// fancy_integration (:34-74).
//
// Algorithmic HBM bytes per frame: both tri-planes once (2*96*H*W*4) + outputs (R*(51+1)*4 [+R*S*4]).
// The practical limiter is the L1/L2 gather path: 24 texels * 128 B per sample.
//
// Mapping: persistent blocks of 8 warps; a block walks 4x2 pixel tiles (neighbouring rays share the
// yz / xz plane lines in L1), one warp per ray, 32 samples per chunk, compositing carried in registers.
#include <stdlib.h>

#include "raymarch_common.cuh"

namespace ide3d {

constexpr int kWarps = 8;
constexpr int kBlock = kWarps * 32;
constexpr int kTileX = 4, kTileY = 2;

struct RayArgs {
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
    const float* noise;
    float *out_feat, *out_depth, *out_weights;
    int tiles_x, tiles_y;
};

template <int KIND, bool kChannelsLast>
__global__ void __launch_bounds__(kBlock, 1) raymarch_kernel(const RayArgs a) {
    extern __shared__ __align__(16) float smem[];
    float* wsm = smem;                                                    // decoder image
    float* stage = smem + DecoderTraits<KIND>::kFloats + (threadIdx.x >> 5) * (32 * kRow);
    load_decoder<KIND>(a.dec, wsm);
    __syncthreads();

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int R = a.res_w * a.res_h, S = a.steps;
    const int tiles_per_frame = a.tiles_x * a.tiles_y;
    const int num_tiles = tiles_per_frame * a.n;
    const int chunks = (S + 31) >> 5;

    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int n = tile / tiles_per_frame;
        const int t = tile - n * tiles_per_frame;
        const int px = (t % a.tiles_x) * kTileX + (warp % kTileX);
        const int py = (t / a.tiles_x) * kTileY + (warp / kTileX);
        if (px >= a.res_w || py >= a.res_h) continue;          // warp-uniform
        const int ray = py * a.res_w + px;

        // --- ray in camera space (get_initial_rays_trig)
        const float x = linspace_at(-1.f, 1.f, a.res_w, px);
        const float y = linspace_at(1.f, -1.f, a.res_h, py);
        const float inv = 1.f / sqrtf(x * x + y * y + a.cam_z * a.cam_z);
        const float dx = x * inv, dy = y * inv, dz = a.cam_z * inv;
        const float dnorm = sqrtf(dx * dx + dy * dy + dz * dz);          // |rays_d_cam| in the delta scaling
        const float* M = a.cam2world + n * 16;
        const float m00 = M[0], m01 = M[1], m02 = M[2], m03 = M[3];
        const float m10 = M[4], m11 = M[5], m12 = M[6], m13 = M[7];
        const float m20 = M[8], m21 = M[9], m22 = M[10], m23 = M[11];
        const float zstep0 = linspace_at(a.ray_start, a.ray_end, S, 0);
        const float spacing = (S > 1) ? linspace_at(a.ray_start, a.ray_end, S, 1) - zstep0 : 0.f;
        const long long sample_base = ((long long)n * R + ray) * S;

        float acc[kOut - 1];
#pragma unroll
        for (int c = 0; c < kOut - 1; ++c) acc[c] = 0.f;
        float acc_w = 0.f, acc_d = 0.f, carry = 1.f;

        for (int ch = 0; ch < chunks; ++ch) {
            const int s = ch * 32 + lane;
            const bool live = s < S;
            // jittered depth of this sample and of the next one (for delta)
            float z0 = 0.f, z1 = 0.f, off0 = 0.f;
            if (live) {
                z0 = linspace_at(a.ray_start, a.ray_end, S, s);
                z1 = (s + 1 < S) ? linspace_at(a.ray_start, a.ray_end, S, s + 1) : 0.f;
                if (a.jitter_mode == IDE3D_JITTER_TENSOR) {
                    off0 = (a.jitter_u[sample_base + s] - 0.5f) * spacing;
                    if (s + 1 < S) z1 += (a.jitter_u[sample_base + s + 1] - 0.5f) * spacing;
                } else if (a.jitter_mode == IDE3D_JITTER_HASH) {
                    const uint32_t gi = (uint32_t)(sample_base + s);
                    off0 = (jitter_hash(gi, a.seed_lo, a.seed_hi) - 0.5f) * spacing;
                    if (s + 1 < S) z1 += (jitter_hash(gi + 1u, a.seed_lo, a.seed_hi) - 0.5f) * spacing;
                } else if (a.jitter_mode == IDE3D_JITTER_ZVALS) {          // depths given per sample (hierarchical second pass)
                    z0 = a.jitter_u[sample_base + s];
                    z1 = (s + 1 < S) ? a.jitter_u[sample_base + s + 1] : 0.f;
                }
            }
            const float zj = z0 + off0;
            // camera-space point = d*z + off*d, then cam2world, then world -> grid units
            const float pcx = dx * z0 + off0 * dx, pcy = dy * z0 + off0 * dy, pcz = dz * z0 + off0 * dz;
            float cx = (m00 * pcx + m01 * pcy + m02 * pcz + m03) * a.box_scale;
            float cy = (m10 * pcx + m11 * pcy + m12 * pcz + m13) * a.box_scale;
            float cz = (m20 * pcx + m21 * pcy + m22 * pcz + m23) * a.box_scale;
            if (!live) { cx = cy = cz = 4.f; }                // far outside: every tap masked, no loads

            gather_chunk<kChannelsLast>(a.tex, a.seg, n, cx, cy, cz, stage, lane);
            const float* row = stage + lane * kRow;

            // density first: it fixes the compositing weight of this sample
            float feat[kOut];
            float sigma;
            if constexpr (KIND == kThreeHead64) {
                sigma = decode_sigma<KIND>(row, wsm);
            } else {
                decode_all<KIND>(row, wsm, feat);
                sigma = feat[kOut - 1];
            }
            if (a.noise != nullptr && live) sigma += a.noise_std * a.noise[sample_base + s];
            const float delta = (s + 1 < S) ? (z1 - zj) * dnorm : 1e10f;
            const float dens = (a.clamp_mode == IDE3D_CLAMP_SOFTPLUS) ? softplus_precise(sigma) : fmaxf(sigma, 0.f);
            const float alpha = live ? 1.f - expf(-delta * dens) : 0.f;
            const float keep = live ? (1.f - alpha + 1e-10f) : 1.f;
            float total;
            const float T = warp_exclusive_product(keep, lane, total) * carry;
            carry *= total;
            float w = alpha * T;
            acc_w += w;                                        // per-lane partial of weights_sum
            if (a.last_back && ch == chunks - 1) {
                const float wsum = warp_sum(acc_w);            // weights.sum over the whole ray
                if (s == S - 1) { w += 1.f - wsum; }
            }
            if (a.out_weights != nullptr && live) a.out_weights[sample_base + s] = w;
            acc_d = fmaf(w, zj, acc_d);

            if constexpr (KIND == kThreeHead64) {
                using Tr = DecoderTraits<kThreeHead64>;
                {
                    float c0[32];
                    mlp_head<32, 64, 32>(row, wsm, c0);
#pragma unroll
                    for (int c = 0; c < 32; ++c) acc[c] = fmaf(w, c0[c], acc[c]);
                }
                {
                    float c1[19];
                    mlp_head<32, 64, 19>(row + kFeat, wsm + Tr::kOff1, c1);
#pragma unroll
                    for (int c = 0; c < 19; ++c) acc[32 + c] = fmaf(w, c1[c], acc[32 + c]);
                }
            } else {
#pragma unroll
                for (int c = 0; c < kOut - 1; ++c) acc[c] = fmaf(w, feat[c], acc[c]);
            }
            __syncwarp();                                      // staging rows are rewritten next chunk
        }

        // --- reduce over the 32 sample lanes and write the ray.  weights_sum is the sum BEFORE the
        // last_back correction (:56-59); white_back / max_depth / fill_mode use that value (:64-72).
        const float wsum = warp_sum(acc_w);
        float depth = warp_sum(acc_d);
        float mine0 = 0.f, mine1 = 0.f;
#pragma unroll
        for (int c = 0; c < kOut - 1; ++c) {
            const float v = warp_sum(acc[c]);
            if (c == lane) mine0 = v;
            if (c == lane + 32) mine1 = v;
        }
        if (a.white_back) { mine0 += 1.f - wsum; mine1 += 1.f - wsum; }
        if (a.max_depth != 0.f) depth += (1.f - wsum) * a.max_depth;
        if (a.fill_weight) { mine0 = wsum; mine1 = wsum; }
        float* of = a.out_feat + ((long long)n * R + ray) * (kOut - 1);
        of[lane] = mine0;
        if (lane + 32 < kOut - 1) of[lane + 32] = mine1;
        if (lane == 0) a.out_depth[(long long)n * R + ray] = depth;
    }
}

template <int KIND, bool CL>
static int launch_raymarch(const RayArgs& a, cudaStream_t st) {
    const size_t smem = (size_t)(DecoderTraits<KIND>::kFloats + kWarps * 32 * kRow) * sizeof(float);
    auto kern = raymarch_kernel<KIND, CL>;
    IDE3D_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 1;
    IDE3D_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kBlock, smem));
    if (per_sm < 1) per_sm = 1;
    const int num_tiles = a.tiles_x * a.tiles_y * a.n;
    int grid = sm_count() * per_sm;
    if (grid > num_tiles) grid = num_tiles;
    kern<<<grid, kBlock, smem, st>>>(a);
    IDE3D_CHECK_LAUNCH("raymarch_kernel");
    return IDE3D_OK;
}

int launch_raymarch_tc(const ide3d_raymarch_params* p, bool channels_last, cudaStream_t st);   // raymarch_tc.cu

}  // namespace ide3d

using namespace ide3d;

static int check_planes(const ide3d_triplane& t, const char* name) {
    IDE3D_REQUIRE(t.data != nullptr, "%s: null data", name);
    IDE3D_REQUIRE(t.n > 0 && t.h > 0 && t.w > 0, "%s: empty tri-plane", name);
    return IDE3D_OK;
}

static bool is_channels_last(const ide3d_triplane& t) {
    return t.stride_c == 1 && (t.stride_w % 4 == 0) && (t.stride_h % 4 == 0) && (t.stride_n % 4 == 0) &&
           ((reinterpret_cast<uintptr_t>(t.data) & 15) == 0);
}

extern "C" int ide3d_raymarch_fwd(const ide3d_raymarch_params* p, ide3d_stream_t stream) {
    IDE3D_REQUIRE(p != nullptr, "raymarch: null params");
    int rc;
    if ((rc = check_planes(p->tex, "tex")) != IDE3D_OK) return rc;
    if ((rc = check_planes(p->seg, "seg")) != IDE3D_OK) return rc;
    IDE3D_REQUIRE(p->tex.h == p->seg.h && p->tex.w == p->seg.w, "raymarch: tex/seg plane sizes differ");
    IDE3D_REQUIRE(p->n > 0 && p->tex.n == p->n && p->seg.n == p->n, "raymarch: batch mismatch");
    IDE3D_REQUIRE(p->res_w > 0 && p->res_h > 0 && p->num_steps > 0, "raymarch: empty render");
    IDE3D_REQUIRE(p->cam2world && p->out_feat && p->out_depth, "raymarch: null camera/output");
    IDE3D_REQUIRE(p->clamp_mode == IDE3D_CLAMP_SOFTPLUS || p->clamp_mode == IDE3D_CLAMP_RELU,
                  "Need to choose clamp mode");   // volumetric_rendering.py:51-52
    IDE3D_REQUIRE(p->jitter_mode >= 0 && p->jitter_mode <= 3, "raymarch: bad jitter mode");
    IDE3D_REQUIRE((p->jitter_mode != IDE3D_JITTER_TENSOR && p->jitter_mode != IDE3D_JITTER_ZVALS) || p->jitter_u, "raymarch: jitter / depth tensor missing");
    IDE3D_REQUIRE((long long)p->n * p->res_w * p->res_h * p->num_steps < (1ll << 32),
                  "raymarch: more than 2^32 samples per call");
    IDE3D_REQUIRE(p->precision >= IDE3D_PRECISION_AUTO && p->precision <= IDE3D_PRECISION_TC, "raymarch: bad precision");
    const bool planes_cl = is_channels_last(p->tex) && is_channels_last(p->seg);
    if (p->precision != IDE3D_PRECISION_FP32) {
        const int rc_tc = launch_raymarch_tc(p, planes_cl, (cudaStream_t)stream);
        if (rc_tc != IDE3D_UNSUPPORTED || p->precision == IDE3D_PRECISION_TC) return rc_tc;
    }
    const int kind = classify_decoder(p->dec);
    if (kind == kDecoderNone) IDE3D_FAIL(IDE3D_UNSUPPORTED, "raymarch: no fused kernel for this decoder shape");

    RayArgs a;
    a.tex = make_view(p->tex); a.seg = make_view(p->seg); a.dec = p->dec;
    a.cam2world = p->cam2world;
    a.n = p->n; a.res_w = p->res_w; a.res_h = p->res_h; a.steps = p->num_steps;
    a.cam_z = (float)(-1.0 / tan((2.0 * 3.14159265358979323846 * (double)p->fov_deg / 360.0) / 2.0));
    a.ray_start = p->ray_start; a.ray_end = p->ray_end; a.box_scale = p->box_scale;
    a.jitter_mode = p->jitter_mode; a.jitter_u = p->jitter_u;
    a.seed_lo = (uint32_t)(p->jitter_seed & 0xffffffffu); a.seed_hi = (uint32_t)(p->jitter_seed >> 32);
    a.clamp_mode = p->clamp_mode; a.last_back = p->last_back; a.white_back = p->white_back;
    a.fill_weight = p->fill_weight; a.max_depth = p->max_depth;
    a.noise_std = p->noise_std; a.noise = (p->noise_std != 0.f) ? p->noise : nullptr;
    a.out_feat = p->out_feat; a.out_depth = p->out_depth; a.out_weights = p->out_weights;
    a.tiles_x = ceil_div(p->res_w, kTileX); a.tiles_y = ceil_div(p->res_h, kTileY);
    const bool cl = planes_cl;
    cudaStream_t st = (cudaStream_t)stream;
    switch (kind) {
        case kDense64: return cl ? launch_raymarch<kDense64, true>(a, st) : launch_raymarch<kDense64, false>(a, st);
        case kDense128: return cl ? launch_raymarch<kDense128, true>(a, st) : launch_raymarch<kDense128, false>(a, st);
        default: return cl ? launch_raymarch<kThreeHead64, true>(a, st) : launch_raymarch<kThreeHead64, false>(a, st);
    }
}
