// Backward of the fused volume renderer (SURVEY.md §8f rank 1; PTI / encoder callers differentiate through G.synthesis,
// inversion/training/projectors/w_plus_projector_ide3d.py:115): gradients of (feat [N,R,51], depth [N,R]) w.r.t. the two tri-planes
// and the three decoder heads in ONE kernel -- the counterpart of aten::grid_sampler_2d_backward (grid_sample_gradfix.py:55-61) + the
// decoder / fancy_integration adjoints the reference gets from autograd, without materialising a single per-sample tensor.
//
// One warp = one ray, lane = sample (chunks of 32 along the ray), as in raymarch.cu.  Two passes over the ray:
//   pass 1  recompute  gather -> layer 1 -> softplus  and from it everything the compositing adjoint needs.  Because every sample of a
//           ray is hit by the SAME output gradient g, the layer-2 adjoint is rank-1:  q_s = g . o_s = (W2^T g) . h_s + g . b2, so only
//           the hidden activations are needed (gh = W2^T g once per ray).  alpha_s, T_s, w_s, q_s stay in shared memory (4 floats/sample).
//           Then the reverse scan of fancy_integration (volumetric_rendering.py:34-74):
//               dL/dw_s = q_s (+ white_back / max_depth / last_back / fill_weight terms),   B_s = sum_{t>s} w_t dL/dw_t,
//               dL/dalpha_s = T_s dL/dw_s - B_s / (1 - alpha_s + 1e-10),   dL/dsigma_s = dL/dalpha_s (1 - alpha_s) delta_s softplus'(sigma_s)
//   pass 2  recompute gather + layer 1 again, then per sample  dh = w'_s gh (colour / semantic heads) or dsigma_s W2_sigma,
//           da = dh * sigmoid(a),  df = W1^T da  -> scattered into the plane gradients with red.global.add.v4.f32 through the same
//           8-lanes-per-texel mapping as the forward gather;  dW1 += da (x) f  per 8-unit block through shared memory (the only true
//           per-sample outer product),  dW2 / db2 from per-ray sums  sum_s w'_s h_s  (rank-1 again),  db1 += da.
// Parameter gradients accumulate in a per-CTA shared-memory image of the decoder and are flushed with one atomicAdd per parameter per CTA.
// Camera gradient (kCam): a sample's grid point is c = b (M[:3,:3] p_cam + M[:3,3]) with p_cam = d_cam z, and neither z nor the
// compositing deltas depend on M, so  dL/dM[i][j] = b sum_s g_c[i] p_cam[j] (j < 3),  dL/dM[i][3] = b sum_s g_c[i].  g_c, the gradient
// w.r.t. the grid point, is grid_sampler_2d's grid gradient dotted with df: the scatter reads the plane value at every tap it visits.
// The 12 sums live in the sample's lane, are reduced per ray into shared memory per CTA and flushed to grad_cam2world[frame] when the
// CTA moves on to another frame's tiles (12 atomicAdds per frame per CTA, not per ray).
// Scope: channels-last fp32 planes, the three-head decoder (texture -> 32, shape -> 19, shape -> 1; 64 hidden each).
// Per-sample-weight gradients, other decoders and NCHW planes keep the composed-chain path of render_grad.py.
#include "raymarch_common.cuh"

namespace ide3d {

constexpr int kBWarps = 8;
constexpr int kBBlock = kBWarps * 32;
constexpr int kBTileX = 4, kBTileY = 2;
constexpr int kMaxSteps = 256;                      // per-ray shared-memory arrays

// the fields of MarchArgs (filled by fill_march_args), then the gradients and the tiling
struct BwdArgs {
    PlaneView tex, seg;
    ide3d_decoder dec;
    const float* cam2world;
    int n, res_w, res_h, steps;
    float cam_z, ray_start, ray_end, box_scale;
    int jitter_mode;
    const float* jitter_u;
    uint32_t seed_lo, seed_hi;
    int clamp_mode, last_back, white_back, fill_weight;
    float max_depth, noise_std;
    const float* noise;
    int views;                  // frames per plane set: the gradients of all views land in their shared set
    const uint64_t* jitter_seeds;
    const float* g_feat;        // [N, R, 51]
    const float* g_depth;       // [N, R] or null
    float* g_tex;               // same layout as tex (channels-last), zero-initialised, or null
    float* g_seg;
    float* g_param[3][4];       // per head: dW1, db1, dW2, db2 (dense, head shapes), or all null
    int tiles_x, tiles_y;
    float* g_cam;               // [N, 16] zero-initialised (rows 0..2 receive the gradient), or null
};

using T3 = DecoderTraits<kThreeHead64>;

__device__ __forceinline__ float sigmoid_from_softplus(float h) { return 1.f - __expf(-h); }   // sigmoid(a) = 1 - exp(-softplus(a))

// scatter 4 channel-quads of df (one sample per 8 lanes) into one tri-plane gradient, mirroring gather_chunk_to's taps.
// kCam: also add to gc[0..2] the gradient of this lane's own sample w.r.t. its grid point (cx, cy, cz) -- grid_sampler_2d's grid
// gradient (align_corners=False, zeros padding) from the plane values at the same taps, dotted with df.  gbase may then be null
// (camera-only request: the taps are read, nothing is scattered).
template <bool kCam = false>
__device__ __forceinline__ void scatter_chunk(const PlaneView& pv, float* __restrict__ gbase, int n, float cx, float cy, float cz,
                                              const float* __restrict__ stage, int col0, int lane, float (&gc)[3]) {
    const int W = pv.w, H = pv.h;
    const Foot f0 = footprint(cx, cy, W, H), f1 = footprint(cy, cz, W, H), f2 = footprint(cx, cz, W, H);
    const int q = lane & 7, grp = lane >> 3;
    float* base = gbase + (long long)n * pv.sn;
    const float* pbase = pv.base + (long long)n * pv.sn;
    const float hw = 0.5f * (float)W, hh = 0.5f * (float)H;                 // d ix / d u, d iy / d v
#pragma unroll 1
    for (int it = 0; it < 8; ++it) {
        const int src = it * 4 + grp;
        const float4 g = *reinterpret_cast<const float4*>(stage + src * kRow + col0 + q * 4);
        float gx = 0.f, gy = 0.f, gz = 0.f;                                 // sample src, this lane's 4 channels (kCam)
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const Foot& mine = (k == 0) ? f0 : (k == 1 ? f1 : f2);
            const int x0 = __shfl_sync(kFull, mine.x0, src), y0 = __shfl_sync(kFull, mine.y0, src);
            const float fx = __shfl_sync(kFull, mine.fx, src), fy = __shfl_sync(kFull, mine.fy, src);
            float gu = 0.f, gv = 0.f;
#pragma unroll
            for (int tap = 0; tap < 4; ++tap) {
                const int xx = x0 + (tap & 1), yy = y0 + (tap >> 1);
                const bool ok = ((unsigned)xx < (unsigned)W) && ((unsigned)yy < (unsigned)H);
                const float wgt = ((tap & 1) ? fx : 1.f - fx) * ((tap >> 1) ? fy : 1.f - fy);
                if (ok) {
                    if (!kCam || gbase != nullptr) {
                        float4* p = reinterpret_cast<float4*>(base + (long long)yy * pv.sh + (long long)xx * pv.sw + k * kFeat + q * 4);
                        atomicAdd(p, make_float4(g.x * wgt, g.y * wgt, g.z * wgt, g.w * wgt));
                    }
                    if (kCam) {
                        // d bil / d ix = sum_taps (+-1) wy P,  d bil / d iy = sum_taps wx (+-1) P
                        const float4 v = __ldg(reinterpret_cast<const float4*>(pbase + (long long)yy * pv.sh + (long long)xx * pv.sw + k * kFeat + q * 4));
                        const float dot = v.x * g.x + v.y * g.y + v.z * g.z + v.w * g.w;
                        const float wy = (tap >> 1) ? fy : 1.f - fy, wx = (tap & 1) ? fx : 1.f - fx;
                        gu += ((tap & 1) ? wy : -wy) * dot;
                        gv += ((tap >> 1) ? wx : -wx) * dot;
                    }
                }
            }
            // plane 0 samples (x, y), plane 1 (y, z), plane 2 (x, z)
            if (k == 0) { gx += hw * gu; gy += hh * gv; }
            else if (k == 1) { gy += hw * gu; gz += hh * gv; }
            else { gx += hw * gu; gz += hh * gv; }
        }
        if (kCam) {
            // sum over the 8 lanes of the texel, then hand the total to the lane that owns sample src (= it * 4 + grp)
#pragma unroll
            for (int d = 1; d < 8; d <<= 1) {
                gx += __shfl_xor_sync(kFull, gx, d); gy += __shfl_xor_sync(kFull, gy, d); gz += __shfl_xor_sync(kFull, gz, d);
            }
            const int from = (lane & 3) * 8;
            const float ox = __shfl_sync(kFull, gx, from), oy = __shfl_sync(kFull, gy, from), oz = __shfl_sync(kFull, gz, from);
            if ((lane >> 2) == it) { gc[0] += ox; gc[1] += oy; gc[2] += oz; }
        }
    }
}

// layer 1 of one head for this lane's sample, 8 hidden units at a time: a = W1 f + b1, h = softplus(a)
template <int IN>
__device__ __forceinline__ void hidden8(const float* __restrict__ w1, const float* __restrict__ b1, const float (&f)[IN], int jc, float (&h)[8]) {
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) h[jj] = b1[jc + jj];
#pragma unroll
    for (int k = 0; k < IN; k += 4) {
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
            const float4 w = *reinterpret_cast<const float4*>(w1 + (jc + jj) * IN + k);
            h[jj] = fmaf(w.x, f[k], h[jj]); h[jj] = fmaf(w.y, f[k + 1], h[jj]);
            h[jj] = fmaf(w.z, f[k + 2], h[jj]); h[jj] = fmaf(w.w, f[k + 3], h[jj]);
        }
    }
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) h[jj] = softplus_fast(h[jj]);
}

template <bool kParams, bool kCam>
__global__ void __launch_bounds__(kBBlock, 1) raymarch_bwd_kernel(const BwdArgs a) {
    extern __shared__ __align__(16) float smem[];
    float* wsm = smem;                                                      // decoder image (HeadLayout x 3)
    float* gacc = wsm + T3::kFloats;                                        // parameter-gradient image, same layout
    float* per_warp = gacc + (kParams ? T3::kFloats : 0);
    constexpr int kPerWarp = 32 * kRow + 32 * 9 + 128 + 5 * kMaxSteps;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* stage = per_warp + warp * kPerWarp;                              // [32][kRow] features (pass 1 / 2), then df
    float* da8 = stage + 32 * kRow;                                         // [32][9] da of the current 8-unit block
    float* gh = da8 + 32 * 9;                                               // [128] W2^T g of the colour / semantic heads
    float* s_al = gh + 128;                                                 // per-sample: alpha, T, w, q, fac
    float* s_T = s_al + kMaxSteps; float* s_w = s_T + kMaxSteps; float* s_q = s_w + kMaxSteps; float* s_fac = s_q + kMaxSteps;
    float* cam_sm = per_warp + kBWarps * kPerWarp;                          // kCam: rows 0..2 of dL/dM of frame cam_frame, before * b
    load_decoder<kThreeHead64>(a.dec, wsm);
    if (kParams) for (int i = threadIdx.x; i < T3::kFloats; i += kBBlock) gacc[i] = 0.f;
    if (kCam && threadIdx.x < 12) cam_sm[threadIdx.x] = 0.f;
    __syncthreads();
    int cam_frame = -1;
    // all threads: add the CTA's camera sums of frame `frame` (if any) to the global gradient and clear them
    auto flush_cam = [&](int frame) {
        __syncthreads();
        if (frame >= 0 && threadIdx.x < 12) {
            atomicAdd(a.g_cam + (long long)frame * 16 + threadIdx.x, a.box_scale * cam_sm[threadIdx.x]);
            cam_sm[threadIdx.x] = 0.f;
        }
        __syncthreads();
    };
    using L0 = HeadLayout<32, 64, 32>; using L1 = HeadLayout<32, 64, 19>; using L2 = HeadLayout<32, 64, 1>;
    const float* w0 = wsm; const float* w1h = wsm + T3::kOff1; const float* w2h = wsm + T3::kOff2;

    const int R = a.res_w * a.res_h, S = a.steps;
    const int tiles_per_frame = a.tiles_x * a.tiles_y;
    const int num_tiles = tiles_per_frame * a.n;
    const int chunks = (S + 31) >> 5;

    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int n = tile / tiles_per_frame;
        if (kCam && n != cam_frame) { flush_cam(cam_frame); cam_frame = n; }      // CTA-uniform: every warp visits every tile
        const int set = plane_set(n, a.views);
        const int t = tile - n * tiles_per_frame;
        const int px = (t % a.tiles_x) * kBTileX + (warp % kBTileX);
        const int py = (t / a.tiles_x) * kBTileY + (warp / kBTileX);
        if (px >= a.res_w || py >= a.res_h) continue;                        // warp-uniform
        const int ray = py * a.res_w + px;
        const float x = linspace_at(-1.f, 1.f, a.res_w, px);
        const float y = linspace_at(1.f, -1.f, a.res_h, py);
        const float inv = 1.f / sqrtf(x * x + y * y + a.cam_z * a.cam_z);
        const float dx = x * inv, dy = y * inv, dz = a.cam_z * inv;
        const float dnorm = sqrtf(dx * dx + dy * dy + dz * dz);
        const float* M = a.cam2world + n * 16;
        const float zstep0 = linspace_at(a.ray_start, a.ray_end, S, 0);
        const float spacing = (S > 1) ? linspace_at(a.ray_start, a.ray_end, S, 1) - zstep0 : 0.f;
        const long long sample_base = ((long long)n * R + ray) * S;
        const long long ray_index = (long long)n * R + ray;

        // output gradient of this ray: lane c holds g[c] and g[c + 32]
        const float* gf = a.g_feat + ray_index * (kOut - 1);
        float g_lo = gf[lane], g_hi = (lane + 32 < kOut - 1) ? gf[lane + 32] : 0.f;
        const float gd = a.g_depth ? a.g_depth[ray_index] : 0.f;
        const float gsum = warp_sum(g_lo + g_hi);
        if (a.fill_weight) { g_lo = 0.f; g_hi = 0.f; }                      // feat = weights_sum: no path through the decoder outputs
        // gh = W2^T g (colour: outputs 0..31, hidden j = lane, lane + 32; semantic: outputs 32..50), gb = g . b2
        {
            float c0 = 0.f, c1 = 0.f, s0 = 0.f, s1 = 0.f;
            for (int o = 0; o < 32; ++o) {
                const float go = __shfl_sync(kFull, g_lo, o);
                c0 = fmaf(w0[L0::kW2 + o * 64 + lane], go, c0); c1 = fmaf(w0[L0::kW2 + o * 64 + lane + 32], go, c1);
            }
            for (int o = 0; o < 19; ++o) {
                const float go = __shfl_sync(kFull, g_hi, o);
                s0 = fmaf(w1h[L1::kW2 + o * 64 + lane], go, s0); s1 = fmaf(w1h[L1::kW2 + o * 64 + lane + 32], go, s1);
            }
            __syncwarp();
            gh[lane] = c0; gh[lane + 32] = c1; gh[64 + lane] = s0; gh[96 + lane] = s1;
            __syncwarp();
        }
        const float gb = warp_sum(g_lo * w0[L0::kB2 + lane] + ((lane < 19) ? g_hi * w1h[L1::kB2 + lane] : 0.f));

        // pc: the camera-space point p_cam whose transform gives (cx, cy, cz) / box_scale
        auto position = [&](int s, bool live, float& zj, float& z1, float& cx, float& cy, float& cz, float (&pc)[3]) {
            float z0 = 0.f, off0 = 0.f;
            z1 = 0.f;
            if (live) {
                z0 = linspace_at(a.ray_start, a.ray_end, S, s);
                z1 = (s + 1 < S) ? linspace_at(a.ray_start, a.ray_end, S, s + 1) : 0.f;
                if (a.jitter_mode == IDE3D_JITTER_TENSOR) {
                    off0 = (a.jitter_u[sample_base + s] - 0.5f) * spacing;
                    if (s + 1 < S) z1 += (a.jitter_u[sample_base + s + 1] - 0.5f) * spacing;
                } else if (a.jitter_mode == IDE3D_JITTER_HASH) {
                    const HashKey k = hash_key(a, n, sample_base + s);
                    off0 = (jitter_hash(k.idx, k.lo, k.hi) - 0.5f) * spacing;
                    if (s + 1 < S) z1 += (jitter_hash(k.idx + 1u, k.lo, k.hi) - 0.5f) * spacing;
                } else if (a.jitter_mode == IDE3D_JITTER_ZVALS) {
                    z0 = a.jitter_u[sample_base + s];
                    z1 = (s + 1 < S) ? a.jitter_u[sample_base + s + 1] : 0.f;
                }
            }
            zj = z0 + off0;
            const float pcx = dx * z0 + off0 * dx, pcy = dy * z0 + off0 * dy, pcz = dz * z0 + off0 * dz;
            cx = (M[0] * pcx + M[1] * pcy + M[2] * pcz + M[3]) * a.box_scale;
            cy = (M[4] * pcx + M[5] * pcy + M[6] * pcz + M[7]) * a.box_scale;
            cz = (M[8] * pcx + M[9] * pcy + M[10] * pcz + M[11]) * a.box_scale;
            pc[0] = pcx; pc[1] = pcy; pc[2] = pcz;
            if (!live) { cx = cy = cz = 4.f; }
        };

        // ------------------------------------------------------------------ pass 1: compositing quantities per sample
        float carry = 1.f, acc_w = 0.f;
        for (int ch = 0; ch < chunks; ++ch) {
            const int s = ch * 32 + lane;
            const bool live = s < S;
            float zj, z1, cx, cy, cz, pc[3];
            position(s, live, zj, z1, cx, cy, cz, pc);
            gather_chunk<true>(a.tex, a.seg, set, cx, cy, cz, stage, lane);
            const float* row = stage + lane * kRow;
            float q = gb + gd * zj, sigma = w2h[L2::kB2];
            {
                float f[32];
#pragma unroll
                for (int k = 0; k < 32; k += 4) { const float4 v = *reinterpret_cast<const float4*>(row + k); f[k] = v.x; f[k + 1] = v.y; f[k + 2] = v.z; f[k + 3] = v.w; }
#pragma unroll 1
                for (int jc = 0; jc < 64; jc += 8) {
                    float h[8];
                    hidden8<32>(w0 + L0::kW1, w0 + L0::kB1, f, jc, h);
#pragma unroll
                    for (int jj = 0; jj < 8; ++jj) q = fmaf(gh[jc + jj], h[jj], q);
                }
#pragma unroll
                for (int k = 0; k < 32; k += 4) { const float4 v = *reinterpret_cast<const float4*>(row + kFeat + k); f[k] = v.x; f[k + 1] = v.y; f[k + 2] = v.z; f[k + 3] = v.w; }
#pragma unroll 1
                for (int jc = 0; jc < 64; jc += 8) {
                    float h[8];
                    hidden8<32>(w1h + L1::kW1, w1h + L1::kB1, f, jc, h);
#pragma unroll
                    for (int jj = 0; jj < 8; ++jj) q = fmaf(gh[64 + jc + jj], h[jj], q);
                    hidden8<32>(w2h + L2::kW1, w2h + L2::kB1, f, jc, h);
#pragma unroll
                    for (int jj = 0; jj < 8; ++jj) sigma = fmaf(w2h[L2::kW2 + jc + jj], h[jj], sigma);
                }
            }
            if (a.noise != nullptr && live) sigma += a.noise_std * a.noise[sample_base + s];
            const float delta = (s + 1 < S) ? (z1 - zj) * dnorm : 1e10f;
            const bool sp = (a.clamp_mode == IDE3D_CLAMP_SOFTPLUS);
            const float dens = sp ? softplus_precise(sigma) : fmaxf(sigma, 0.f);
            const float ex = expf(-delta * dens);
            const float alpha = live ? 1.f - ex : 0.f;
            const float keep = live ? (1.f - alpha + 1e-10f) : 1.f;
            float total;
            const float T = warp_exclusive_product(keep, lane, total) * carry;
            carry *= total;
            const float w = alpha * T;
            acc_w += w;
            // d alpha / d sigma = exp(-delta dens) * delta * dens'(sigma)
            const float dd = sp ? 1.f / (1.f + expf(-sigma)) : (sigma > 0.f ? 1.f : 0.f);
            if (live) { s_al[s] = alpha; s_T[s] = T; s_w[s] = w; s_q[s] = q; s_fac[s] = ex * delta * dd; }
            __syncwarp();
        }
        const float wsum = warp_sum(acc_w);
        // extra dL/dw terms that do not go through o_s:  feat += 1 - W (white_back), depth += (1 - W) max_depth, feat = W (fill_weight)
        float u = 0.f;
        if (a.white_back && !a.fill_weight) u -= gsum;
        if (a.max_depth != 0.f) u -= gd * a.max_depth;
        if (a.fill_weight) u += gsum;
        const float q_last = a.last_back ? s_q[S - 1] : 0.f;                 // F = sum w_s o_s + (1 - W) o_last  ->  dL/dw_s = q_s - q_last
        // reverse scan: B_s = sum_{t > s} w_t dL/dw_t
        float suffix = 0.f;
        for (int ch = chunks - 1; ch >= 0; --ch) {
            const int s = ch * 32 + lane;
            const bool live = s < S;
            const float dw = live ? (s_q[s] - q_last + u) : 0.f;
            const float v = live ? s_w[s] * dw : 0.f;
            float inc = v;                                                    // inclusive suffix sum within the chunk (lanes above me)
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const float tv = __shfl_down_sync(kFull, inc, d);
                if (lane + d < 32) inc += tv;
            }
            const float B = inc - v + suffix;
            suffix += __shfl_sync(kFull, inc, 0);
            if (live) {
                const float al = s_al[s];
                const float dalpha = s_T[s] * dw - B / (1.f - al + 1e-10f);
                float wp = s_w[s];
                if (a.last_back && s == S - 1) wp += 1.f - wsum;
                s_q[s] = dalpha * s_fac[s];                                   // dL/dsigma_s
                s_w[s] = a.fill_weight ? 0.f : wp;                            // weight of g in dL/do_s
            }
            __syncwarp();
        }

        // ------------------------------------------------------------------ pass 2: decoder adjoint + scatter
        float hsum[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};                      // sum_s coef_s h_s[j] for j = lane + 32 m  (m: 0,1 colour; 2,3 semantic; 4,5 sigma)
        float wp_sum = 0.f, ds_sum = 0.f;
        float cam_acc[12];                                                    // kCam: sum_s g_c[i] p_cam[j] at 4 i + j, sum_s g_c[i] at 4 i + 3
#pragma unroll
        for (int i = 0; i < 12; ++i) cam_acc[i] = 0.f;
        for (int ch = 0; ch < chunks; ++ch) {
            const int s = ch * 32 + lane;
            const bool live = s < S;
            float zj, z1, cx, cy, cz, pc[3];
            position(s, live, zj, z1, cx, cy, cz, pc);
            gather_chunk<true>(a.tex, a.seg, set, cx, cy, cz, stage, lane);
            float* row = stage + lane * kRow;
            const float wp = live ? s_w[s] : 0.f, ds = live ? s_q[s] : 0.f;
            wp_sum += wp; ds_sum += ds;
            float f[32], df[32];
            // one head: hidden blocks of 8 -> da -> df, da8 -> dW1 / db1, coefficient-weighted hidden sums for dW2
            auto head = [&](const float* wimg, int w1off, int b1off, int col0, const float* ghp, const float* w2sig, float coef, float& hs_lo, float& hs_hi, int gbase) {
#pragma unroll 1
                for (int jc = 0; jc < 64; jc += 8) {
                    float h[8], da[8];
                    hidden8<32>(wimg + w1off, wimg + b1off, f, jc, h);
#pragma unroll
                    for (int jj = 0; jj < 8; ++jj) {
                        const float dh = (ghp != nullptr) ? coef * ghp[jc + jj] : coef * w2sig[jc + jj];
                        da[jj] = dh * sigmoid_from_softplus(h[jj]);
                    }
#pragma unroll
                    for (int k = 0; k < 32; k += 4) {
#pragma unroll
                        for (int jj = 0; jj < 8; ++jj) {
                            const float4 w = *reinterpret_cast<const float4*>(wimg + w1off + (jc + jj) * 32 + k);
                            df[k] = fmaf(w.x, da[jj], df[k]); df[k + 1] = fmaf(w.y, da[jj], df[k + 1]);
                            df[k + 2] = fmaf(w.z, da[jj], df[k + 2]); df[k + 3] = fmaf(w.w, da[jj], df[k + 3]);
                        }
                    }
                    if (kParams) {
                        // hidden sums for the rank-1 dW2: lane (j & 31) keeps the total of hidden unit j = jc + jj
#pragma unroll
                        for (int jj = 0; jj < 8; ++jj) {
                            const float tot = warp_sum(coef * h[jj]);
                            const int j = jc + jj;
                            if (lane == (j & 31)) { if (j < 32) hs_lo += tot; else hs_hi += tot; }
                        }
                        // dW1[j][k] += sum_s da[s][j] f[s][k]: lane (jj = lane & 7, kg = lane >> 3) owns 8 inputs of one hidden unit
#pragma unroll
                        for (int jj = 0; jj < 8; ++jj) da8[lane * 9 + jj] = da[jj];
                        __syncwarp();
                        const int jj = lane & 7, kg = lane >> 3;
                        float acc8[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
                        float accb = 0.f;
                        for (int ss = 0; ss < 32; ++ss) {
                            const float dv = da8[ss * 9 + jj];
                            const float4 fa = *reinterpret_cast<const float4*>(stage + ss * kRow + col0 + kg * 8);
                            const float4 fb = *reinterpret_cast<const float4*>(stage + ss * kRow + col0 + kg * 8 + 4);
                            acc8[0] = fmaf(dv, fa.x, acc8[0]); acc8[1] = fmaf(dv, fa.y, acc8[1]); acc8[2] = fmaf(dv, fa.z, acc8[2]); acc8[3] = fmaf(dv, fa.w, acc8[3]);
                            acc8[4] = fmaf(dv, fb.x, acc8[4]); acc8[5] = fmaf(dv, fb.y, acc8[5]); acc8[6] = fmaf(dv, fb.z, acc8[6]); acc8[7] = fmaf(dv, fb.w, acc8[7]);
                            accb += dv;
                        }
#pragma unroll
                        for (int i = 0; i < 8; ++i) atomicAdd(gacc + gbase + w1off + (jc + jj) * 32 + kg * 8 + i, acc8[i]);
                        if (kg == 0) atomicAdd(gacc + gbase + b1off + jc + jj, accb);
                        __syncwarp();
                    }
                }
            };
            // texture half -> colour head
#pragma unroll
            for (int k = 0; k < 32; k += 4) { const float4 v = *reinterpret_cast<const float4*>(row + k); f[k] = v.x; f[k + 1] = v.y; f[k + 2] = v.z; f[k + 3] = v.w; }
#pragma unroll
            for (int k = 0; k < 32; ++k) df[k] = 0.f;
            head(w0, L0::kW1, L0::kB1, 0, gh, nullptr, wp, hsum[0], hsum[1], 0);
            float dft[32];
#pragma unroll
            for (int k = 0; k < 32; ++k) dft[k] = df[k];
            // shape half -> semantic + sigma heads
#pragma unroll
            for (int k = 0; k < 32; k += 4) { const float4 v = *reinterpret_cast<const float4*>(row + kFeat + k); f[k] = v.x; f[k + 1] = v.y; f[k + 2] = v.z; f[k + 3] = v.w; }
#pragma unroll
            for (int k = 0; k < 32; ++k) df[k] = 0.f;
            head(w1h, L1::kW1, L1::kB1, kFeat, gh + 64, nullptr, wp, hsum[2], hsum[3], T3::kOff1);
            head(w2h, L2::kW1, L2::kB1, kFeat, nullptr, w2h + L2::kW2, ds, hsum[4], hsum[5], T3::kOff2);
            // df -> staging rows (the features are no longer needed), then scatter through the gather's lane mapping
            __syncwarp();
#pragma unroll
            for (int k = 0; k < 32; k += 4) {
                *reinterpret_cast<float4*>(row + k) = make_float4(dft[k], dft[k + 1], dft[k + 2], dft[k + 3]);
                *reinterpret_cast<float4*>(row + kFeat + k) = make_float4(df[k], df[k + 1], df[k + 2], df[k + 3]);
            }
            __syncwarp();
            float gc[3] = {0.f, 0.f, 0.f};
            if (kCam) {
                scatter_chunk<true>(a.tex, a.g_tex, set, cx, cy, cz, stage, 0, lane, gc);
                scatter_chunk<true>(a.seg, a.g_seg, set, cx, cy, cz, stage, kFeat, lane, gc);
#pragma unroll
                for (int i = 0; i < 3; ++i) {
#pragma unroll
                    for (int j = 0; j < 3; ++j) cam_acc[4 * i + j] = fmaf(gc[i], pc[j], cam_acc[4 * i + j]);
                    cam_acc[4 * i + 3] += gc[i];
                }
            } else {
                if (a.g_tex != nullptr) scatter_chunk(a.tex, a.g_tex, set, cx, cy, cz, stage, 0, lane, gc);
                if (a.g_seg != nullptr) scatter_chunk(a.seg, a.g_seg, set, cx, cy, cz, stage, kFeat, lane, gc);
            }
            __syncwarp();
        }
        if (kCam) {
#pragma unroll
            for (int i = 0; i < 12; ++i) {
                const float v = warp_sum(cam_acc[i]);
                if (lane == 0) atomicAdd(cam_sm + i, v);
            }
        }
        if (kParams) {
            // rank-1 layer-2 gradients of this ray:  dW2[o][j] += g_o * sum_s w'_s h_s[j];  db2[o] += g_o * sum_s w'_s;  sigma head: coefficient dsigma_s
            const float wps = warp_sum(wp_sum), dss = warp_sum(ds_sum);
            for (int o = 0; o < 32; ++o) {
                const float go = __shfl_sync(kFull, g_lo, o);
                atomicAdd(gacc + L0::kW2 + o * 64 + lane, go * hsum[0]); atomicAdd(gacc + L0::kW2 + o * 64 + lane + 32, go * hsum[1]);
            }
            for (int o = 0; o < 19; ++o) {
                const float go = __shfl_sync(kFull, g_hi, o);
                atomicAdd(gacc + T3::kOff1 + L1::kW2 + o * 64 + lane, go * hsum[2]); atomicAdd(gacc + T3::kOff1 + L1::kW2 + o * 64 + lane + 32, go * hsum[3]);
            }
            atomicAdd(gacc + T3::kOff2 + L2::kW2 + lane, hsum[4]); atomicAdd(gacc + T3::kOff2 + L2::kW2 + lane + 32, hsum[5]);
            atomicAdd(gacc + L0::kB2 + lane, g_lo * wps);
            if (lane < 19) atomicAdd(gacc + T3::kOff1 + L1::kB2 + lane, g_hi * wps);
            if (lane == 0) atomicAdd(gacc + T3::kOff2 + L2::kB2, dss);
        }
    }

    if (kCam) flush_cam(cam_frame);
    if (kParams) {
        __syncthreads();
        // flush the CTA's gradient image: head h, tensor t (W1, b1, W2, b2) -> dense global gradient
        const int off[3] = {0, T3::kOff1, T3::kOff2};
        const int outc[3] = {32, 19, 1};
        for (int h = 0; h < 3; ++h) {
            const int kB1 = 64 * 32, kW2 = kB1 + 64, kB2 = kW2 + ((outc[h] * 64 + 3) / 4) * 4;
            for (int i = threadIdx.x; i < 64 * 32; i += kBBlock) atomicAdd(a.g_param[h][0] + i, gacc[off[h] + i]);
            for (int i = threadIdx.x; i < 64; i += kBBlock) atomicAdd(a.g_param[h][1] + i, gacc[off[h] + kB1 + i]);
            for (int i = threadIdx.x; i < outc[h] * 64; i += kBBlock) atomicAdd(a.g_param[h][2] + i, gacc[off[h] + kW2 + i]);
            for (int i = threadIdx.x; i < outc[h]; i += kBBlock) atomicAdd(a.g_param[h][3] + i, gacc[off[h] + kB2 + i]);
        }
    }
}

}  // namespace ide3d

using namespace ide3d;

template <bool kParams, bool kCam>
static int launch_bwd(const BwdArgs& a, int grid, size_t smem, cudaStream_t st) {
    IDE3D_CUDA(cudaFuncSetAttribute(raymarch_bwd_kernel<kParams, kCam>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    raymarch_bwd_kernel<kParams, kCam><<<grid, kBBlock, smem, st>>>(a);
    return IDE3D_OK;
}

static int raymarch_bwd(const ide3d_raymarch_params* p, const float* grad_feat, const float* grad_depth, float* grad_tex,
                        float* grad_seg, float* const* grad_params, float* grad_cam2world, ide3d_stream_t stream) {
    int rc;
    if ((rc = check_raymarch_params(p)) != IDE3D_OK) return rc;
    IDE3D_REQUIRE(grad_feat != nullptr, "raymarch_bwd: null argument");
    if (p->num_steps > kMaxSteps) IDE3D_FAIL(IDE3D_UNSUPPORTED, "raymarch_bwd: more than %d samples per ray", kMaxSteps);
    if (classify_decoder(p->dec) != kThreeHead64) IDE3D_FAIL(IDE3D_UNSUPPORTED, "raymarch_bwd: only the three-head decoder has a backward kernel");
    if (!planes_channels_last(p->tex) || !planes_channels_last(p->seg)) IDE3D_FAIL(IDE3D_UNSUPPORTED, "raymarch_bwd: planes must be channels-last fp32");
    IDE3D_REQUIRE(((reinterpret_cast<uintptr_t>(grad_tex) | reinterpret_cast<uintptr_t>(grad_seg)) & 15) == 0, "raymarch_bwd: plane gradients must be 16-byte aligned");
    BwdArgs a;
    fill_march_args(*p, a);
    a.g_feat = grad_feat; a.g_depth = grad_depth; a.g_tex = grad_tex; a.g_seg = grad_seg;
    const bool params = grad_params != nullptr;
    for (int h = 0; h < 3; ++h)
        for (int t = 0; t < 4; ++t) {
            a.g_param[h][t] = params ? grad_params[h * 4 + t] : nullptr;
            IDE3D_REQUIRE(!params || a.g_param[h][t] != nullptr, "raymarch_bwd: parameter gradient %d of head %d missing", t, h);
        }
    a.tiles_x = ceil_div(p->res_w, kBTileX); a.tiles_y = ceil_div(p->res_h, kBTileY);
    a.g_cam = grad_cam2world;
    const bool cam = grad_cam2world != nullptr;
    constexpr int kPerWarp = 32 * kRow + 32 * 9 + 128 + 5 * kMaxSteps;
    const size_t smem = (size_t)(T3::kFloats * (params ? 2 : 1) + kBWarps * kPerWarp + (cam ? 16 : 0)) * sizeof(float);
    const int num_tiles = a.tiles_x * a.tiles_y * a.n;
    int grid = sm_count();
    if (grid > num_tiles) grid = num_tiles;
    cudaStream_t st = (cudaStream_t)stream;
    if (params) rc = cam ? launch_bwd<true, true>(a, grid, smem, st) : launch_bwd<true, false>(a, grid, smem, st);
    else rc = cam ? launch_bwd<false, true>(a, grid, smem, st) : launch_bwd<false, false>(a, grid, smem, st);
    if (rc != IDE3D_OK) return rc;
    IDE3D_CHECK_LAUNCH("raymarch_bwd_kernel");
    return IDE3D_OK;
}

extern "C" int ide3d_raymarch_bwd(const ide3d_raymarch_params* p, const float* grad_feat, const float* grad_depth, float* grad_tex,
                                  float* grad_seg, float* const* grad_params, ide3d_stream_t stream) {
    return raymarch_bwd(p, grad_feat, grad_depth, grad_tex, grad_seg, grad_params, nullptr, stream);
}

extern "C" int ide3d_raymarch_bwd_cam(const ide3d_raymarch_params* p, const float* grad_feat, const float* grad_depth, float* grad_tex,
                                      float* grad_seg, float* const* grad_params, float* grad_cam2world, ide3d_stream_t stream) {
    return raymarch_bwd(p, grad_feat, grad_depth, grad_tex, grad_seg, grad_params, grad_cam2world, stream);
}
