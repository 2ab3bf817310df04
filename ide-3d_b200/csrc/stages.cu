// Stand-alone renderer stages: the reference's free functions on materialised tensors.
//   ide3d_initial_rays      get_initial_rays_trig      training/volumetric_rendering.py:77-97
//   ide3d_transform_points  perturb_points + transform_sampled_points (camera given)  :99-136
//   ide3d_sample_triplane   sample_from_triplane       dnnlib/util.py:580-617
//   ide3d_integrate         fancy_integration          training/volumetric_rendering.py:34-74
//   ide3d_sample_pdf        sample_pdf                 :224-265
// All are HBM streams (read inputs once, write outputs once); the fused kernel in raymarch.cu is the
// fast path, these exist so that callers of the individual functions keep working unchanged.
#include "raymarch_common.cuh"

namespace ide3d {

// ------------------------------------------------------------------------------- rays
__global__ void __launch_bounds__(256) rays_kernel(int n, int S, float cam_z, int W, int H, float rs, float re,
                                                   float* __restrict__ points, float* __restrict__ zv,
                                                   float* __restrict__ dirs) {
    const long long R = (long long)W * H;
    const long long total = (long long)n * R * S;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int s = (int)(i % S);
        const long long nr = i / S;
        const int ray = (int)(nr % R);
        const int px = ray % W, py = ray / W;
        const float x = linspace_at(-1.f, 1.f, W, px);
        const float y = linspace_at(1.f, -1.f, H, py);
        const float inv = 1.f / sqrtf(x * x + y * y + cam_z * cam_z);
        const float dx = x * inv, dy = y * inv, dz = cam_z * inv;
        const float z = linspace_at(rs, re, S, s);
        points[i * 3 + 0] = dx * z;
        points[i * 3 + 1] = dy * z;
        points[i * 3 + 2] = dz * z;
        zv[i] = z;
        if (s == 0) { dirs[nr * 3 + 0] = dx; dirs[nr * 3 + 1] = dy; dirs[nr * 3 + 2] = dz; }
    }
}

// ------------------------------------------------------------------------------- jitter + cam2world
__global__ void __launch_bounds__(256) transform_kernel(const float* __restrict__ points, const float* __restrict__ zv,
                                                        const float* __restrict__ dirs, const float* __restrict__ u,
                                                        const float* __restrict__ cam, int n, int R, int S,
                                                        float* __restrict__ pw, float* __restrict__ zo,
                                                        float* __restrict__ dw, float* __restrict__ ow) {
    const long long total = (long long)n * R * S;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int s = (int)(i % S);
        const long long nr = i / S;
        const int b = (int)(nr / R);
        const float* M = cam + b * 16;
        const float dx = dirs[nr * 3], dy = dirs[nr * 3 + 1], dz = dirs[nr * 3 + 2];
        float px = points[i * 3], py = points[i * 3 + 1], pz = points[i * 3 + 2];
        float z = zv[i];
        if (u != nullptr) {
            const float spacing = (S > 1) ? zv[nr * S + 1] - zv[nr * S] : 0.f;     // z_vals[:,:,1:2]-z_vals[:,:,0:1]
            const float off = (u[i] - 0.5f) * spacing;
            z += off;
            px += off * dx; py += off * dy; pz += off * dz;
        }
        pw[i * 3 + 0] = M[0] * px + M[1] * py + M[2] * pz + M[3];
        pw[i * 3 + 1] = M[4] * px + M[5] * py + M[6] * pz + M[7];
        pw[i * 3 + 2] = M[8] * px + M[9] * py + M[10] * pz + M[11];
        zo[i] = z;
        if (s == 0) {
            dw[nr * 3 + 0] = M[0] * dx + M[1] * dy + M[2] * dz;
            dw[nr * 3 + 1] = M[4] * dx + M[5] * dy + M[6] * dz;
            dw[nr * 3 + 2] = M[8] * dx + M[9] * dy + M[10] * dz;
            ow[nr * 3 + 0] = M[3]; ow[nr * 3 + 1] = M[7]; ow[nr * 3 + 2] = M[11];
        }
    }
}

// ------------------------------------------------------------------------------- tri-plane gather
// 8 lanes per point (one float4 of the 32 channels each), 4 points per warp instruction.
template <bool kChannelsLast>
__global__ void __launch_bounds__(256) triplane_kernel(PlaneView pl, const float* __restrict__ coords, int n,
                                                       long long P, float* __restrict__ out) {
    const long long total = (long long)n * P;
    const int q = threadIdx.x & 7;
    for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 3; i < total;
         i += ((long long)gridDim.x * blockDim.x) >> 3) {
        const int b = (int)(i / P);
        const float cx = coords[i * 3], cy = coords[i * 3 + 1], cz = coords[i * 3 + 2];
        const float* base = pl.base + (long long)b * pl.sn;
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const Foot f = footprint(k == 1 ? cy : cx, k == 0 ? cy : cz, pl.w, pl.h);
            float part[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int tap = 0; tap < 4; ++tap) {
                const int xx = f.x0 + (tap & 1), yy = f.y0 + (tap >> 1);
                if (((unsigned)xx < (unsigned)pl.w) && ((unsigned)yy < (unsigned)pl.h)) {
                    const float wgt = ((tap & 1) ? f.fx : 1.f - f.fx) * ((tap >> 1) ? f.fy : 1.f - f.fy);
                    const long long o = (long long)yy * pl.sh + (long long)xx * pl.sw;
                    if (kChannelsLast) {
                        const float4 v = __ldg(reinterpret_cast<const float4*>(base + o + k * kFeat + q * 4));
                        part[0] += v.x * wgt; part[1] += v.y * wgt; part[2] += v.z * wgt; part[3] += v.w * wgt;
                    } else {
#pragma unroll
                        for (int j = 0; j < 4; ++j) part[j] += __ldg(base + o + (long long)(k * kFeat + q * 4 + j) * pl.sc) * wgt;
                    }
                }
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[j] += part[j];
        }
        *reinterpret_cast<float4*>(out + i * kFeat + q * 4) = make_float4(acc[0], acc[1], acc[2], acc[3]);
    }
}

// ------------------------------------------------------------------------------- compositing
// one warp per ray; lanes stride the samples, channels are looped (generic C)
__global__ void __launch_bounds__(256) integrate_kernel(const float* __restrict__ rgb_sigma, const float* __restrict__ dirs,
                                                        const float* __restrict__ zv, const float* __restrict__ noise,
                                                        float noise_std, long long rays, int S, int C, int clamp_mode,
                                                        int last_back, int white_back, float max_depth, int fill_weight,
                                                        float* __restrict__ rgb, float* __restrict__ depth,
                                                        float* __restrict__ weights) {
    const int lane = threadIdx.x & 31;
    const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    const int chunks = (S + 31) >> 5;
    for (long long r = warp0; r < rays; r += nwarps) {
        const float dx = dirs[r * 3], dy = dirs[r * 3 + 1], dz = dirs[r * 3 + 2];
        const float dnorm = sqrtf(dx * dx + dy * dy + dz * dz);
        const float* rs = rgb_sigma + r * (long long)S * C;
        const float* z = zv + r * (long long)S;
        float* wout = weights + r * (long long)S;
        float carry = 1.f, acc_w = 0.f, acc_d = 0.f;
        // pass 1: weights (and depth); pass 2: channels, re-reading the weights just written
        for (int ch = 0; ch < chunks; ++ch) {
            const int s = ch * 32 + lane;
            const bool live = s < S;
            float alpha = 0.f, zj = 0.f;
            if (live) {
                zj = z[s];
                float sigma = rs[(long long)s * C + (C - 1)];
                if (noise != nullptr) sigma += noise_std * noise[r * (long long)S + s];
                const float delta = (s + 1 < S) ? (z[s + 1] - zj) * dnorm : 1e10f;
                const float dens = (clamp_mode == IDE3D_CLAMP_SOFTPLUS) ? softplus_precise(sigma) : fmaxf(sigma, 0.f);
                alpha = 1.f - expf(-delta * dens);
            }
            const float keep = live ? (1.f - alpha + 1e-10f) : 1.f;
            float total;
            const float T = warp_exclusive_product(keep, lane, total) * carry;
            carry *= total;
            float w = alpha * T;
            acc_w += w;
            if (last_back && ch == chunks - 1) {
                const float wsum_all = warp_sum(acc_w);
                if (s == S - 1) w += 1.f - wsum_all;
            }
            if (live) wout[s] = w;
            acc_d = fmaf(w, zj, acc_d);
        }
        const float wsum = warp_sum(acc_w);
        float d = warp_sum(acc_d);
        if (max_depth != 0.f) d += (1.f - wsum) * max_depth;
        if (lane == 0) depth[r] = d;
        __syncwarp();
        // channels: lane = channel, loop samples (weights come back through L1)
        for (int c0 = 0; c0 < C - 1; c0 += 32) {
            const int c = c0 + lane;
            float a = 0.f;
            if (c < C - 1) {
                for (int s = 0; s < S; ++s) a = fmaf(wout[s], rs[(long long)s * C + c], a);
                if (white_back) a += 1.f - wsum;
                if (fill_weight) a = wsum;
                rgb[r * (long long)(C - 1) + c] = a;
            }
        }
        __syncwarp();
    }
}

// ------------------------------------------------------------------------------- importance pdf
// one warp per ray: cdf by warp scan into shared memory, then each lane resolves its samples
__global__ void __launch_bounds__(256) pdf_kernel(const float* __restrict__ bins, const float* __restrict__ weights,
                                                  const float* __restrict__ u, int rays, int nb, int nimp, float eps,
                                                  float* __restrict__ out) {
    extern __shared__ float sm[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* cdf = sm + warp * (nb + 1);
    const int warps = blockDim.x >> 5;
    for (int r = blockIdx.x * warps + warp; r < rays; r += gridDim.x * warps) {
        const float* w = weights + (long long)r * nb;
        const float* b = bins + (long long)r * (nb + 1);
        float part = 0.f;
        for (int i = lane; i < nb; i += 32) part += w[i] + eps;
        const float tot = warp_sum(part);
        // sequential-order cumulative sum of pdf in chunks of 32 (inclusive scan + carry)
        float carry = 0.f;
        if (lane == 0) cdf[0] = 0.f;
        for (int i0 = 0; i0 < nb; i0 += 32) {
            const int i = i0 + lane;
            float v = (i < nb) ? (w[i] + eps) / tot : 0.f;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const float t = __shfl_up_sync(kFull, v, d);
                if (lane >= d) v += t;
            }
            v += carry;
            if (i < nb) cdf[i + 1] = v;
            carry = __shfl_sync(kFull, v, 31);
        }
        __syncwarp();
        for (int k = lane; k < nimp; k += 32) {
            const float uu = u[(long long)r * nimp + k];
            // searchsorted(cdf, u, right=False): first index with cdf[idx] >= u
            int lo = 0, hi = nb + 1;
            while (lo < hi) { const int mid = (lo + hi) >> 1; if (cdf[mid] < uu) lo = mid + 1; else hi = mid; }
            const int below = max(lo - 1, 0), above = min(lo, nb);
            float den = cdf[above] - cdf[below];
            if (den < eps) den = 1.f;
            out[(long long)r * nimp + k] = b[below] + (uu - cdf[below]) / den * (b[above] - b[below]);
        }
        __syncwarp();
    }
}

}  // namespace ide3d

using namespace ide3d;

extern "C" int ide3d_initial_rays(int n, int num_steps, float fov_deg, int res_w, int res_h, float ray_start,
                                  float ray_end, float* points, float* z_vals, float* rays_d_cam,
                                  ide3d_stream_t stream) {
    IDE3D_REQUIRE(n > 0 && num_steps > 0 && res_w > 0 && res_h > 0, "initial_rays: empty request");
    IDE3D_REQUIRE(points && z_vals && rays_d_cam, "initial_rays: null output");
    const float cam_z = (float)(-1.0 / tan((2.0 * 3.14159265358979323846 * (double)fov_deg / 360.0) / 2.0));
    const long long total = (long long)n * res_w * res_h * num_steps;
    const unsigned grid = capped_grid(ceil_div<long long>(total, 256), 16);
    rays_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(n, num_steps, cam_z, res_w, res_h, ray_start,
                                                        ray_end, points, z_vals, rays_d_cam);
    IDE3D_CHECK_LAUNCH("rays_kernel");
    return IDE3D_OK;
}

extern "C" int ide3d_transform_points(const float* points, const float* z_vals, const float* dirs, const float* u,
                                      const float* cam2world, int n, int num_rays, int num_steps, float* points_world,
                                      float* z_out, float* dirs_world, float* origins, ide3d_stream_t stream) {
    IDE3D_REQUIRE(n > 0 && num_rays > 0 && num_steps > 0, "transform_points: empty request");
    IDE3D_REQUIRE(points && z_vals && dirs && cam2world && points_world && z_out && dirs_world && origins,
                  "transform_points: null pointer");
    const long long total = (long long)n * num_rays * num_steps;
    transform_kernel<<<capped_grid(ceil_div<long long>(total, 256), 16), 256, 0, (cudaStream_t)stream>>>(
        points, z_vals, dirs, u, cam2world, n, num_rays, num_steps, points_world, z_out, dirs_world, origins);
    IDE3D_CHECK_LAUNCH("transform_kernel");
    return IDE3D_OK;
}

extern "C" int ide3d_sample_triplane(const ide3d_triplane* planes, const float* coords, int64_t num_points,
                                     float* out, ide3d_stream_t stream) {
    IDE3D_REQUIRE(planes && planes->data, "sample_triplane: null planes");
    IDE3D_REQUIRE(planes->n > 0 && planes->h > 0 && planes->w > 0, "sample_triplane: empty planes");
    IDE3D_REQUIRE(num_points >= 0, "sample_triplane: negative point count");
    if (num_points == 0) return IDE3D_OK;
    IDE3D_REQUIRE(coords && out, "sample_triplane: null coords/out");
    IDE3D_REQUIRE((reinterpret_cast<uintptr_t>(out) & 15) == 0, "sample_triplane: out must be 16-byte aligned");
    const PlaneView v = make_view(*planes);
    const bool cl = planes->stride_c == 1 && planes->stride_w % 4 == 0 && planes->stride_h % 4 == 0 &&
                    planes->stride_n % 4 == 0 && (reinterpret_cast<uintptr_t>(planes->data) & 15) == 0;
    const long long threads = (long long)planes->n * num_points * 8;
    const unsigned grid = capped_grid(ceil_div<long long>(threads, 256), 16);
    if (cl) triplane_kernel<true><<<grid, 256, 0, (cudaStream_t)stream>>>(v, coords, planes->n, num_points, out);
    else triplane_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>(v, coords, planes->n, num_points, out);
    IDE3D_CHECK_LAUNCH("triplane_kernel");
    return IDE3D_OK;
}

extern "C" int ide3d_integrate(const float* rgb_sigma, const float* rays_d_cam, const float* z_vals, const float* noise,
                               float noise_std, int n, int num_rays, int num_steps, int channels, int clamp_mode,
                               int last_back, int white_back, float max_depth, int fill_weight, float* rgb,
                               float* depth, float* weights, ide3d_stream_t stream) {
    IDE3D_REQUIRE(clamp_mode == IDE3D_CLAMP_SOFTPLUS || clamp_mode == IDE3D_CLAMP_RELU, "Need to choose clamp mode");
    IDE3D_REQUIRE(n > 0 && num_rays > 0 && num_steps > 0 && channels >= 1, "integrate: empty request");
    IDE3D_REQUIRE(rgb_sigma && rays_d_cam && z_vals && rgb && depth && weights, "integrate: null pointer");
    const long long rays = (long long)n * num_rays;
    integrate_kernel<<<capped_grid(ceil_div<long long>(rays * 32, 256), 16), 256, 0, (cudaStream_t)stream>>>(
        rgb_sigma, rays_d_cam, z_vals, (noise_std != 0.f) ? noise : nullptr, noise_std, rays, num_steps, channels,
        clamp_mode, last_back, white_back, max_depth, fill_weight, rgb, depth, weights);
    IDE3D_CHECK_LAUNCH("integrate_kernel");
    return IDE3D_OK;
}

extern "C" int ide3d_sample_pdf(const float* bins, const float* weights, const float* u, int num_rays, int num_bins,
                                int n_importance, float eps, float* samples, ide3d_stream_t stream) {
    IDE3D_REQUIRE(num_rays >= 0 && num_bins > 0 && n_importance > 0, "sample_pdf: bad sizes");
    if (num_rays == 0) return IDE3D_OK;
    IDE3D_REQUIRE(bins && weights && u && samples, "sample_pdf: null pointer");
    const int warps = 8;
    const size_t smem = (size_t)warps * (num_bins + 1) * sizeof(float);
    IDE3D_REQUIRE(smem <= 48 * 1024, "sample_pdf: too many bins for one block");
    const unsigned grid = capped_grid(ceil_div(num_rays, warps), 8);
    pdf_kernel<<<grid, warps * 32, smem, (cudaStream_t)stream>>>(bins, weights, u, num_rays, num_bins, n_importance,
                                                                eps, samples);
    IDE3D_CHECK_LAUNCH("pdf_kernel");
    return IDE3D_OK;
}

// ------------------------------------------------------------------------------------------------------------------
// mask2color (dnnlib/seg_tools.py:75-82): argmax over the class logits + colour look-up, one thread per pixel.
namespace ide3d {
template <typename O>
__global__ void __launch_bounds__(256) mask2color_kernel(const float* __restrict__ m, int c, int h, int w, long long sn, long long sc,
                                                         long long sh, long long sw, const float* __restrict__ lut, O* __restrict__ out,
                                                         long long total) {
    const long long hw = (long long)h * w;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long n = i / hw, r = i - n * hw;
        const int y = (int)(r / w), x = (int)(r - (long long)y * w);
        const float* p = m + n * sn + y * sh + x * sw;
        float best = p[0];
        int arg = 0;
        for (int k = 1; k < c; ++k) {
            const float v = p[k * sc];
            if (v > best || (v != v && best == best)) { best = v; arg = k; }      // first maximum; NaN counts as maximal (torch.argmax)
        }
#pragma unroll
        for (int j = 0; j < 3; ++j) out[(n * 3 + j) * hw + r] = (O)lut[arg * 3 + j];
    }
}
}  // namespace ide3d

extern "C" int ide3d_mask2color(const float* masks, int n, int c, int h, int w, int64_t stride_n, int64_t stride_c, int64_t stride_h,
                                int64_t stride_w, const float* lut, void* out, int out_u8, ide3d_stream_t stream) {
    IDE3D_REQUIRE(n >= 0 && c >= 1 && h >= 0 && w >= 0, "mask2color: bad sizes");
    const long long total = (long long)n * h * w;
    if (total == 0) return IDE3D_OK;
    IDE3D_REQUIRE(masks && lut && out, "mask2color: null tensor");
    const unsigned grid = ide3d::capped_grid(ide3d::ceil_div<long long>(total, 256), 16);
    cudaStream_t st = (cudaStream_t)stream;
    if (out_u8) ide3d::mask2color_kernel<unsigned char><<<grid, 256, 0, st>>>(masks, c, h, w, stride_n, stride_c, stride_h, stride_w, lut, (unsigned char*)out, total);
    else ide3d::mask2color_kernel<float><<<grid, 256, 0, st>>>(masks, c, h, w, stride_n, stride_c, stride_h, stride_w, lut, (float*)out, total);
    IDE3D_CHECK_LAUNCH("mask2color_kernel");
    return IDE3D_OK;
}
