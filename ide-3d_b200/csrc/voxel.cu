// Point queries against the two tri-planes + decoder:
//   ide3d_sample_voxel   renderer.sample_voxel(img_v, seg_v, points) -> [N,P,52]   (extract_shapes.py:146)
//   ide3d_sigma_grid     the whole density-grid loop of extract_shapes.py:99-150 with the points of
//                        0.9*create_samples() generated in the kernel (no 201 MB point tensor)
//   ide3d_planes_to_nhwc layout conversion feeding the fast gather path
#include "raymarch_common.cuh"

namespace ide3d {

constexpr int kVWarps = 8;
constexpr int kVBlock = kVWarps * 32;

template <int KIND, bool kChannelsLast, bool kGrid>
__global__ void __launch_bounds__(kVBlock, 1) voxel_kernel(const VoxelArgs a) {
    extern __shared__ __align__(16) float smem[];
    float* wsm = smem;
    float* stage = smem + DecoderTraits<KIND>::kFloats + (threadIdx.x >> 5) * (32 * kRow);
    load_decoder<KIND>(a.dec, wsm);
    __syncthreads();

    const int lane = threadIdx.x & 31;
    const long long chunks_per_item = (a.P + 31) >> 5;
    const long long total = chunks_per_item * a.n;
    const long long warp_global = (long long)blockIdx.x * kVWarps + (threadIdx.x >> 5);
    const long long warp_stride = (long long)gridDim.x * kVWarps;

    for (long long chunk = warp_global; chunk < total; chunk += warp_stride) {
        const int n = (int)(chunk / chunks_per_item);
        const long long p0 = (chunk - (long long)n * chunks_per_item) << 5;
        const long long p = p0 + lane;
        const bool live = p < a.P;
        float x = 4.f, y = 4.f, z = 4.f;
        if (live) {
            if (kGrid) {
                grid_point(a, a.first + p, x, y, z);
            } else {
                const float* pt = a.points + ((long long)n * a.P + p) * 3;
                x = pt[0]; y = pt[1]; z = pt[2];
            }
            x *= a.box_scale; y *= a.box_scale; z *= a.box_scale;
        }
        // sigma of the three-head decoder reads the shape planes only: skip the texture tri-plane (half of the gather)
        if (KIND == kThreeHead64 && a.sigma_only) gather_chunk<kChannelsLast, true>(a.tex, a.seg, n, x, y, z, stage, lane);
        else gather_chunk<kChannelsLast>(a.tex, a.seg, n, x, y, z, stage, lane);
        const float* row = stage + lane * kRow;
        if (a.sigma_only) {
            const float sg = decode_sigma<KIND>(row, wsm);
            if (live) a.out[(long long)n * a.P + p] = sg;
            __syncwarp();
        } else {
            float o[kOut];
            decode_all<KIND>(row, wsm, o);
            __syncwarp();                                   // everyone is done reading the feature rows
            float* wrow = stage + lane * kRow;
#pragma unroll
            for (int c = 0; c < kOut; c += 4)
                *reinterpret_cast<float4*>(wrow + c) = make_float4(o[c], o[c + 1], o[c + 2], o[c + 3]);
            __syncwarp();
            // the 32 rows are contiguous in the output ([P][52]): copy them out coalesced
            const long long valid = min((long long)32, a.P - p0);
            float* dst = a.out + ((long long)n * a.P + p0) * kOut;
            for (int i = lane; i < (int)valid * kOut; i += 32) dst[i] = stage[(i / kOut) * kRow + (i % kOut)];
            __syncwarp();
        }
    }
}

template <int KIND, bool CL, bool GRID>
static int launch_voxel(const VoxelArgs& a, cudaStream_t st) {
    const size_t smem = (size_t)(DecoderTraits<KIND>::kFloats + kVWarps * 32 * kRow) * sizeof(float);
    auto kern = voxel_kernel<KIND, CL, GRID>;
    int grid, rc;
    if ((rc = persistent_grid(kern, kVBlock, smem, ceil_div<long long>(((a.P + 31) >> 5) * a.n, kVWarps), grid)) != IDE3D_OK) return rc;
    kern<<<grid, kVBlock, smem, st>>>(a);
    IDE3D_CHECK_LAUNCH("voxel_kernel");
    return IDE3D_OK;
}

template <bool GRID>
static int dispatch_voxel(const VoxelArgs& a, bool cl, int kind, cudaStream_t st) {
    switch (kind) {
        case kDense64: return cl ? launch_voxel<kDense64, true, GRID>(a, st) : launch_voxel<kDense64, false, GRID>(a, st);
        case kDense128: return cl ? launch_voxel<kDense128, true, GRID>(a, st) : launch_voxel<kDense128, false, GRID>(a, st);
        default: return cl ? launch_voxel<kThreeHead64, true, GRID>(a, st) : launch_voxel<kThreeHead64, false, GRID>(a, st);
    }
}

// [N,C,H,W] strided -> [N,H,W,C] dense, 32x32 tiles through shared memory
__global__ void __launch_bounds__(256) nhwc_kernel(const float* __restrict__ src, float* __restrict__ dst, int C,
                                                   long long HW, int W, long long sn, long long sc,
                                                   long long sh, long long sw) {
    __shared__ float tile[32][33];
    const int n = blockIdx.z;
    const long long p0 = (long long)blockIdx.x * 32;
    const int c0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;      // 32 x 8
#pragma unroll
    for (int j = 0; j < 32; j += 8) {
        const int c = c0 + ty + j;
        const long long p = p0 + tx;
        if (c < C && p < HW) {
            const long long yy = p / W, xx = p - yy * W;
            tile[ty + j][tx] = src[n * sn + c * sc + yy * sh + xx * sw];
        }
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 32; j += 8) {
        const long long p = p0 + ty + j;
        const int c = c0 + tx;
        if (c < C && p < HW) dst[((long long)n * HW + p) * C + c] = tile[tx][ty + j];
    }
}

static int fill_common(VoxelArgs& a, const ide3d_triplane* tex, const ide3d_triplane* seg, const ide3d_decoder* dec,
                       int& kind, bool& cl) {
    IDE3D_REQUIRE(tex && seg && dec, "voxel: null argument");
    IDE3D_REQUIRE(tex->data && seg->data, "voxel: null plane data");
    IDE3D_REQUIRE(tex->n == seg->n && tex->n > 0, "voxel: batch mismatch");
    IDE3D_REQUIRE(tex->h == seg->h && tex->w == seg->w && tex->h > 0 && tex->w > 0, "voxel: plane sizes differ");
    kind = classify_decoder(*dec);
    if (kind == kDecoderNone) IDE3D_FAIL(IDE3D_UNSUPPORTED, "voxel: no fused kernel for this decoder shape");
    a.tex = make_view(*tex); a.seg = make_view(*seg); a.dec = *dec; a.n = tex->n;
    cl = planes_channels_last(*tex) && planes_channels_last(*seg);
    return IDE3D_OK;
}

// voxel_tc.cu: sigma-only queries on the tensor cores (decoders with a density head over the shape planes, channels-last planes)
int launch_sigma_tc(const VoxelArgs& a, cudaStream_t st, bool& handled);

}  // namespace ide3d

using namespace ide3d;

extern "C" int ide3d_sample_voxel(const ide3d_triplane* tex, const ide3d_triplane* seg, const ide3d_decoder* dec,
                                  const float* points, int64_t num_points, float box_scale, int sigma_only,
                                  float* out, ide3d_stream_t stream) {
    VoxelArgs a{};
    int kind; bool cl;
    int rc = fill_common(a, tex, seg, dec, kind, cl);
    if (rc != IDE3D_OK) return rc;
    IDE3D_REQUIRE(num_points >= 0, "sample_voxel: negative point count");
    if (num_points == 0) return IDE3D_OK;
    IDE3D_REQUIRE(points && out, "sample_voxel: null points/out");
    a.points = points; a.P = num_points; a.box_scale = box_scale; a.sigma_only = sigma_only; a.out = out;
    if (sigma_only && cl) {
        bool handled = false;
        rc = launch_sigma_tc(a, (cudaStream_t)stream, handled);
        if (handled) return rc;
    }
    return dispatch_voxel<false>(a, cl, kind, (cudaStream_t)stream);
}

extern "C" int ide3d_sigma_grid(const ide3d_triplane* tex, const ide3d_triplane* seg, const ide3d_decoder* dec,
                                int grid_n, const float voxel_origin[3], float cube_length, float pre_scale,
                                float box_scale, int64_t first, int64_t count, float* out, ide3d_stream_t stream) {
    VoxelArgs a{};
    int kind; bool cl;
    int rc = fill_common(a, tex, seg, dec, kind, cl);
    if (rc != IDE3D_OK) return rc;
    IDE3D_REQUIRE(grid_n >= 2, "sigma_grid: grid_n must be >= 2");
    const long long total = (long long)grid_n * grid_n * grid_n;
    IDE3D_REQUIRE(first >= 0 && count >= 0 && first + count <= total, "sigma_grid: range outside the grid");
    if (count == 0) return IDE3D_OK;
    IDE3D_REQUIRE(out && voxel_origin, "sigma_grid: null argument");
    // create_samples (extract_shapes.py:76-78) evaluates these in float64 and the tensor ops round to fp32
    const double half = (double)cube_length / 2.0;
    a.grid_n = grid_n;
    a.voxel_size = (float)((double)cube_length / (double)(grid_n - 1));
    a.org_x = (float)((double)voxel_origin[0] - half);
    a.org_y = (float)((double)voxel_origin[1] - half);
    a.org_z = (float)((double)voxel_origin[2] - half);
    a.pre_scale = pre_scale;
    a.first = first; a.P = count; a.box_scale = box_scale; a.sigma_only = 1; a.out = out; a.points = nullptr;
    if (cl) {
        bool handled = false;
        rc = launch_sigma_tc(a, (cudaStream_t)stream, handled);
        if (handled) return rc;
    }
    return dispatch_voxel<true>(a, cl, kind, (cudaStream_t)stream);
}

extern "C" int ide3d_planes_to_nhwc(const float* src, int n, int c, int h, int w, int64_t stride_n, int64_t stride_c,
                                    int64_t stride_h, int64_t stride_w, float* dst, ide3d_stream_t stream) {
    IDE3D_REQUIRE(src && dst, "planes_to_nhwc: null pointer");
    IDE3D_REQUIRE(n > 0 && c > 0 && h > 0 && w > 0, "planes_to_nhwc: empty tensor");
    IDE3D_REQUIRE(n <= 65535 && ceil_div(c, 32) <= 65535, "planes_to_nhwc: tensor too large");
    const long long HW = (long long)h * w;
    dim3 grid((unsigned)ceil_div<long long>(HW, 32), (unsigned)ceil_div(c, 32), (unsigned)n);
    nhwc_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(src, dst, c, HW, w, stride_n, stride_c, stride_h, stride_w);
    IDE3D_CHECK_LAUNCH("nhwc_kernel");
    return IDE3D_OK;
}
