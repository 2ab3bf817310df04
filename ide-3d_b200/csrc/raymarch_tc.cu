// Fused volume renderer, tensor-core decoder: rays -> jitter -> cam2world -> 2x tri-plane gather -> decoder MLP -> alpha compositing
// in ONE kernel, no per-sample intermediate in HBM (training/volumetric_rendering.py:34-136, dnnlib/util.py:580-617 and the
// generator's decoder in one pass).
//
//   unit   = 4x2 neighbouring rays, marched front to back by one warpgroup; tile = 8 consecutive depth samples of the 8 rays = 64 rows
//            warp w of the warpgroup owns rows 16w..16w+15: rays (2(w%2), w/2) and (2(w%2)+1, w/2), row = 8 * ray + depth index.
//            That is the row ownership of the wgmma accumulator (lane l holds rows l/4 and l/4 + 8), so a lane holds the same depth
//            sample of both of its warp's rays and the 8 samples of a ray sit in the 8 lanes l%4 == const (compositing = 8-lane scan)
//   A      = gathered features [64 x 64] (texture 0..31 | shape 32..63), bf16 hi + lo, K-major, 128B-swizzled smem rows; every warp
//            gathers its own 16 rows (8 lanes per texel x LDG.128), one named barrier per tile hands the tile to the warpgroup MMA
//   layer 1: D1[64 x 64] per hidden block = A . W1_blk^T, wgmma with both operands in shared memory, fp32 accumulators in registers
//   epilog : + b1 -> softplus -> bf16 hi / lo, repacked in registers as the A fragments of layer 2 (accumulator and A fragment share
//            their row / column ownership): no shared-memory round trip between the layers
//   layer 2: D2[64 x n] += A2 . W2_blk^T, wgmma with the A operand in registers, over the output columns the block feeds
//   final  : + b2 -> sigma -> alpha -> 8-lane product scan (+ carried transmittance) -> weighted accumulation in registers; one
//            8-lane reduction per ray at the end of the march
// Every product is bf16 hi*hi + hi*lo + lo*hi with fp32 accumulation ("bf16x3": 16 mantissa bits per operand).
//
// CTA = two warpgroups that share the weight tiles in shared memory (compacted: 52 KB for the three-head decoder) and march
// independent units, so the gather latency of one is covered by the MMA / softplus / compositing work of the other and of the
// other resident CTAs.
#include "raymarch_tc_shared.cuh"

namespace ide3d {

// layer 2 of one hidden block into D2 columns [N0, N0 + N)
template <int N0, int N>
__device__ __forceinline__ void layer2(float (&d2)[32], const uint32_t (&ah)[4][4], const uint32_t (&al)[4][4], uint64_t wh, uint64_t wl) {
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
        tc::Wgmma<N>::rs(d2 + N0 / 2, ah[ks], wh + ks * 2);
        tc::Wgmma<N>::rs(d2 + N0 / 2, ah[ks], wl + ks * 2);
        tc::Wgmma<N>::rs(d2 + N0 / 2, al[ks], wh + ks * 2);
    }
}

__device__ __forceinline__ void layer2_cols(int n0, int n, float (&d2)[32], const uint32_t (&ah)[4][4], const uint32_t (&al)[4][4],
                                            uint64_t wh, uint64_t wl) {
    switch ((n0 >> 4) * 4 + (n >> 4) - 1) {
        case 0: layer2<0, 16>(d2, ah, al, wh, wl); break;
        case 1: layer2<0, 32>(d2, ah, al, wh, wl); break;
        case 2: layer2<0, 48>(d2, ah, al, wh, wl); break;
        case 3: layer2<0, 64>(d2, ah, al, wh, wl); break;
        case 4: layer2<16, 16>(d2, ah, al, wh, wl); break;
        case 5: layer2<16, 32>(d2, ah, al, wh, wl); break;
        case 6: layer2<16, 48>(d2, ah, al, wh, wl); break;
        case 8: layer2<32, 16>(d2, ah, al, wh, wl); break;
        case 9: layer2<32, 32>(d2, ah, al, wh, wl); break;
        case 12: layer2<48, 16>(d2, ah, al, wh, wl); break;
        default: break;                                                  // excluded by build_program (columns within 0..63)
    }
}

__device__ __forceinline__ void fence_frag(uint32_t (&f)[4][4]) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) asm volatile("" : "+r"(f[i][j])::"memory");
}

__global__ void __launch_bounds__(kTcThreads) raymarch_tc_kernel(const TcArgs a) {
    extern __shared__ unsigned char smem_raw[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const TcProgram& P = a.prog;
    unsigned char* w_hi = smem;
    unsigned char* w_lo = smem + P.wpart;
    unsigned char* tile_base = smem + 2 * P.wpart;
    float* b1s = reinterpret_cast<float*>(tile_base + kWarpgroups * kStageBytes);   // [3 x 64] hidden biases (x log2e)
    float* b2s = b1s + kTcMaxBlocks * 64;                                            // [64] output biases

    const int tid = threadIdx.x, lane = tid & 31;

    // ---------------- one-time setup: weights -> bf16 hi/lo swizzled tiles (compacted), biases
    for (int i = tid; i < (2 * P.wpart) / 16; i += kTcThreads) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
    __syncthreads();
    for (int i = tid; i < P.nblocks * 64 * 64; i += kTcThreads) {
        const int b = i >> 12, j = (i >> 6) & 63, k = i & 63;
        const TcBlock& B = P.blk[b];
        __nv_bfloat16 hi, lo;
        // hidden activation in base 2: softplus(x) = ln2 * log2(1 + 2^(x*log2e)); log2e goes into W1 / b1, ln2 into W2, once
        if (k < B.kcount) {                                                  // W1[hidden j][input k] -> column k0 + k
            tc::split_bf16(B.w1[j * B.w1_ld + k] * 1.4426950408889634f, hi, lo);
            tile_store_bf16(w_hi + B.w1_off, j, B.k0 + k, hi);
            tile_store_bf16(w_lo + B.w1_off, j, B.k0 + k, lo);
        }
        const int oc = B.w2_row0 + j;                                        // W2[output oc][hidden k] -> row j of the row block
        if (oc >= B.out0 && oc < B.out0 + B.outc) {
            tc::split_bf16(B.w2[(oc - B.out0) * B.w2_ld + k] * 0.6931471805599453f, hi, lo);
            tile_store_bf16(w_hi + B.w2_off, j, k, hi);
            tile_store_bf16(w_lo + B.w2_off, j, k, lo);
        }
    }
    for (int i = tid; i < kTcMaxBlocks * 64; i += kTcThreads) b1s[i] = (i < P.nblocks * 64) ? P.blk[i >> 6].b1[i & 63] * 1.4426950408889634f : 0.f;
    if (tid < 64) {
        float v = 0.f;
        for (int h = 0; h < a.dec.num_heads; ++h) {
            const ide3d_mlp_head& H = a.dec.heads[h];
            if (tid >= H.out_offset && tid < H.out_offset + H.out_count) v = H.b2[tid - H.out_offset];
        }
        b2s[tid] = v;
    }
    tc::fence_async_smem();
    __syncthreads();

    const int S = a.steps;
    const int wg = tid >> 7, w = (tid >> 5) & 3;
    const int g = lane >> 2, c = lane & 3;                               // accumulator rows g / g + 8, columns 8j + 2c + {0, 1}
    const int q4 = lane & 7, grp = lane >> 3, l16 = lane & 15;           // gather: channel quad, sample of the instruction, own row
    const int shb = (int)(a.tex.sh * 4), swb = (int)(a.tex.sw * 4);     // strides in bytes (32-bit: checked by the launcher)
    const int W = a.tex.w, H = a.tex.h;
    unsigned char* a_hi = tile_base + wg * kStageBytes;
    unsigned char* a_lo = a_hi + kTileBytes;
    const uint64_t ah0 = tc::make_sdesc_sw128(tc::smem_u32(a_hi)), al0 = tc::make_sdesc_sw128(tc::smem_u32(a_lo));
    const uint64_t wh0 = tc::make_sdesc_sw128(tc::smem_u32(w_hi)), wl0 = tc::make_sdesc_sw128(tc::smem_u32(w_lo));
    const int unit_stride = kWarpgroups * gridDim.x;

    for (int unit = blockIdx.x * kWarpgroups + wg; unit < a.num_units; unit += unit_stride) {
        const RaySetup rA = ray_setup(a, unit, (w & 1) * 2, w >> 1);
        const RaySetup rB = ray_setup(a, unit, (w & 1) * 2 + 1, w >> 1);
        const RaySetup rG = ray_setup(a, unit, (w & 1) * 2 + (l16 >> 3), w >> 1);      // the ray of this lane's gather row
        const char* tb = reinterpret_cast<const char*>(a.tex.base + (long long)rG.n * a.tex.sn);
        const char* sb = reinterpret_cast<const char*>(a.seg.base + (long long)rG.n * a.seg.sn);
        float acc[2][16];
#pragma unroll
        for (int i = 0; i < 16; ++i) acc[0][i] = acc[1][i] = 0.f;
        float acc_w[2] = {0.f, 0.f}, acc_d[2] = {0.f, 0.f}, T_in[2] = {1.f, 1.f};

        for (int step = 0; step < a.tiles_per_unit; ++step) {
            // ---- gather: this lane's sample position, per-axis bilinear footprints (dnnlib/util.py:589-596: plane 0 = (x,y),
            //      plane 1 = (y,z), plane 2 = (x,z)), computed once per sample; the 8 lanes that fetch a texel receive them by shuffle
            {
                const int s = step * kTileDepth + (l16 & 7);
                float cx = 4.f, cy = 4.f, cz = 4.f;                            // far outside the planes: every tap gets weight 0
                if (rG.ok && s < S) {
                    const float* M = a.cam2world + rG.n * 16;
                    float z0, off0, z1;
                    sample_depths(a, rG, s, z0, off0, z1);
                    const float pcx = rG.dx * z0 + off0 * rG.dx, pcy = rG.dy * z0 + off0 * rG.dy, pcz = rG.dz * z0 + off0 * rG.dz;
                    cx = (M[0] * pcx + M[1] * pcy + M[2] * pcz + M[3]) * a.box_scale;
                    cy = (M[4] * pcx + M[5] * pcy + M[6] * pcz + M[7]) * a.box_scale;
                    cz = (M[8] * pcx + M[9] * pcy + M[10] * pcz + M[11]) * a.box_scale;
                }
                const AxisFoot fx = axis_foot(cx, W), fyr = axis_foot(cy, H), fyc = axis_foot(cy, W), fz = axis_foot(cz, H);
                const AxisTaps mX = axis_taps(fx.i0, fx.f, W, swb), mYr = axis_taps(fyr.i0, fyr.f, H, shb);
                const AxisTaps mYc = axis_taps(fyc.i0, fyc.f, W, swb), mZ = axis_taps(fz.i0, fz.f, H, shb);
#pragma unroll 1
                for (int it = 0; it < 4; ++it) {
                    const int src = it * 4 + grp;                              // 4 depth-consecutive samples of one ray per instruction
                    AxisTaps X = shfl_taps(mX, src), Yc = shfl_taps(mYc, src);
                    const AxisTaps Yr = shfl_taps(mYr, src), Z = shfl_taps(mZ, src);
                    X.lo += q4 * 16; X.hi += q4 * 16; Yc.lo += q4 * 16; Yc.hi += q4 * 16;      // this lane's channel quad
                    const int row = w * 16 + src;
                    const uint32_t o_tex = tc::sw128_offset(row, q4 >> 1) + (q4 & 1) * 8;
                    const uint32_t o_seg = tc::sw128_offset(row, 4 + (q4 >> 1)) + (q4 & 1) * 8;
                    float f[4];
                    uint2 hi, lo;
                    gather12(tb, X, Yr, Yc, Z, f);
                    tc::split4_bf16(f, hi, lo);
                    // the tile is overwritten only when every warp of the warpgroup is past the MMAs of the previous tile; the first
                    // loads of this tile are already in flight
                    if (it == 0) tc::bar_sync(1 + wg, 128);
                    *reinterpret_cast<uint2*>(a_hi + o_tex) = hi;
                    *reinterpret_cast<uint2*>(a_lo + o_tex) = lo;
                    gather12(sb, X, Yr, Yc, Z, f);
                    tc::split4_bf16(f, hi, lo);
                    *reinterpret_cast<uint2*>(a_hi + o_seg) = hi;
                    *reinterpret_cast<uint2*>(a_lo + o_seg) = lo;
                }
                tc::fence_async_smem();                                        // my generic-proxy stores -> async proxy (wgmma)
                tc::bar_sync(1 + wg, 128);
            }

            // ---- decoder: per hidden block, layer 1 (smem x smem) -> softplus -> layer 2 (registers x smem) into D2
            float d2[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) d2[i] = 0.f;
            for (int b = 0; b < P.nblocks; ++b) {
                const TcBlock& B = P.blk[b];
                float d1[32];
                tc::wgmma_fence();
                {
                    const uint64_t wh = wh0 + (B.w1_off >> 4), wl = wl0 + (B.w1_off >> 4);
                    const int ks0 = B.k0 >> 4, ks1 = ks0 + (B.kcount >> 4);
                    for (int ks = ks0; ks < ks1; ++ks) {
                        const uint64_t off = (uint64_t)(ks * 2);               // 16 bf16 = 32 bytes along K, same column in A and W1
                        tc::Wgmma<64>::ss(d1, ah0 + off, wh + off, ks > ks0);
                        tc::Wgmma<64>::ss(d1, ah0 + off, wl + off, 1);
                        tc::Wgmma<64>::ss(d1, al0 + off, wh + off, 1);
                    }
                }
                tc::wgmma_commit();
                tc::wgmma_wait<0>();
                tc::fence_regs(d1);
                uint32_t ah[4][4], al[4][4];
                const float* bb = b1s + b * 64;
#pragma unroll
                for (int ks = 0; ks < 4; ++ks)
#pragma unroll
                    for (int q = 0; q < 4; ++q) {                              // q: (n8 tile 2ks + q/2, row g + 8 (q%2))
                        const int j = 2 * ks + (q >> 1), e = 4 * j + 2 * (q & 1);
                        const float h0 = softplus2(d1[e] + bb[8 * j + 2 * c]);
                        const float h1 = softplus2(d1[e + 1] + bb[8 * j + 2 * c + 1]);
                        tc::split2_bf16(h0, h1, ah[ks][q], al[ks][q]);
                    }
                tc::wgmma_fence();
                const uint64_t wh = wh0 + (B.w2_off >> 4), wl = wl0 + (B.w2_off >> 4);
                layer2_cols(B.w2_row0, B.w2_rows, d2, ah, al, wh, wl);
                tc::wgmma_commit();
                tc::wgmma_wait<0>();
                tc::fence_regs(d2);
                fence_frag(ah);
                fence_frag(al);
            }

            // ---- sigma (column 51 = n8 tile 6, lane c == 1, second element), compositing weights of this lane's two samples
            const float sig_row[2] = {__shfl_sync(kFull, d2[25], (lane & ~3) | 1), __shfl_sync(kFull, d2[27], (lane & ~3) | 1)};
            const int s = step * kTileDepth + g;
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const RaySetup& R = r ? rB : rA;
                const bool live = R.ok && (s < S);
                float z0 = 0.f, off0 = 0.f, z1 = 0.f;
                if (live) sample_depths(a, R, s, z0, off0, z1);
                const float zj = z0 + off0;
                float sigma = sig_row[r] + b2s[kOut - 1];
                if (a.noise != nullptr && live) sigma += a.noise_std * a.noise[R.sample_base + s];
                const float delta = (s + 1 < S) ? (z1 - zj) * R.dnorm : 1e10f;
                const float dens = (a.clamp_mode == IDE3D_CLAMP_SOFTPLUS) ? softplus_precise(sigma) : fmaxf(sigma, 0.f);
                const float alpha = live ? 1.f - expf(-delta * dens) : 0.f;
                const float keep = live ? (1.f - alpha + 1e-10f) : 1.f;
                // exclusive product over the 8 samples of the ray in sample order, times the transmittance carried in
                float tr = T_in[r], mine = T_in[r];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float kj = __shfl_sync(kFull, keep, 4 * j + c);
                    if (j == g) mine = tr;
                    tr *= kj;
                }
                T_in[r] = tr;
                float wt = alpha * mine;
                acc_w[r] += wt;
                if (a.last_back && step == a.tiles_per_unit - 1) {
                    float ws = acc_w[r];
                    ws += __shfl_xor_sync(kFull, ws, 4); ws += __shfl_xor_sync(kFull, ws, 8); ws += __shfl_xor_sync(kFull, ws, 16);
                    if (s == S - 1) wt += 1.f - ws;
                }
                if (a.out_weights != nullptr && live && c == 0) a.out_weights[R.sample_base + s] = wt;
                acc_d[r] = fmaf(wt, zj, acc_d[r]);
#pragma unroll
                for (int j = 0; j < 8; ++j)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int col = 8 * j + 2 * c + e;
                        if (col < kOut - 1) acc[r][2 * j + e] = fmaf(wt, d2[4 * j + 2 * r + e] + b2s[col], acc[r][2 * j + e]);
                    }
            }
        }

        // ---- per-ray reduction over the 8 depth lanes and store (weights_sum is the sum BEFORE the last_back correction,
        //      volumetric_rendering.py:56-72)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const RaySetup& R = r ? rB : rA;
            float wsum = acc_w[r], depth = acc_d[r];
#pragma unroll
            for (int m = 4; m < 32; m <<= 1) { wsum += __shfl_xor_sync(kFull, wsum, m); depth += __shfl_xor_sync(kFull, depth, m); }
            if (a.max_depth != 0.f) depth += (1.f - wsum) * a.max_depth;
            const long long ray_index = (long long)R.n * (a.res_w * a.res_h) + R.ray;
            float* of = a.out_feat + ray_index * (kOut - 1);
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    float v = acc[r][2 * j + e];
                    v += __shfl_xor_sync(kFull, v, 4); v += __shfl_xor_sync(kFull, v, 8); v += __shfl_xor_sync(kFull, v, 16);
                    if (a.white_back) v += 1.f - wsum;
                    if (a.fill_weight) v = wsum;
                    const int col = 8 * j + 2 * c + e;
                    if (R.ok && g == 0 && col < kOut - 1) of[col] = v;
                }
            if (R.ok && lane == 0) a.out_depth[ray_index] = depth;
        }
    }
}

// entry used by ide3d_raymarch_fwd (raymarch.cu); IDE3D_UNSUPPORTED when this decoder / layout has no TC kernel
int launch_raymarch_tc(const ide3d_raymarch_params* p, bool channels_last, cudaStream_t st) {
    if (!channels_last) IDE3D_FAIL(IDE3D_UNSUPPORTED, "raymarch_tc: planes must be channels-last");
    if (p->tex.stride_h != p->seg.stride_h || p->tex.stride_w != p->seg.stride_w)
        IDE3D_FAIL(IDE3D_UNSUPPORTED, "raymarch_tc: tex and seg planes must share strides");
    if (((long long)p->tex.h * p->tex.stride_h + (long long)p->tex.w * p->tex.stride_w + 96) * 4 >= (1ll << 31))
        IDE3D_FAIL(IDE3D_UNSUPPORTED, "raymarch_tc: plane too large for 32-bit byte offsets");
    TcArgs a;
    if (!build_program(p->dec, a.prog)) IDE3D_FAIL(IDE3D_UNSUPPORTED, "raymarch_tc: decoder shape not supported");
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
    a.units_x = ceil_div(p->res_w, kUnitW); a.units_y = ceil_div(p->res_h, kUnitH);
    a.num_units = a.units_x * a.units_y * a.n;
    a.tiles_per_unit = ceil_div(p->num_steps, kTileDepth);
    const int smem = 2 * a.prog.wpart + kWarpgroups * kStageBytes + (kTcMaxBlocks * 64 + 64) * 4 + 1024;
    IDE3D_CUDA(cudaFuncSetAttribute(raymarch_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    int per_sm = 1;
    IDE3D_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, raymarch_tc_kernel, kTcThreads, smem));
    if (per_sm < 1) per_sm = 1;
    int grid = sm_count() * per_sm;
    if (grid * kWarpgroups > a.num_units) grid = ceil_div(a.num_units, kWarpgroups);
    raymarch_tc_kernel<<<grid, kTcThreads, smem, st>>>(a);
    IDE3D_CHECK_LAUNCH("raymarch_tc_kernel");
    return IDE3D_OK;
}

}  // namespace ide3d
