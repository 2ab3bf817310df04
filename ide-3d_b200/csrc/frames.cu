// Video frames of gen_videos.py's image_seg / image_depth modes (gen_videos.py:129-139 + layout_grid's uint8 conversion :29-30),
// straight from the synthesis outputs to uint8 CHW frames.  Kernels, in launch order:
//   IDE3D_FRAMES_IMAGE_SEG    frames_seg_kernel      output pixel -> image bytes | bilinear class logits -> argmax -> COLOR_MAP bytes
//   IDE3D_FRAMES_IMAGE_DEPTH  frames_minmax_kernel   (frame, block) -> partial min / max of -image
//                             frames_depth_kernel    frame's min / max from the partials, then pixel -> normalised -> bytes
// Every float operation is explicitly rounded (__fmul_rn / __fadd_rn / __fsub_rn / __fdiv_rn): the reference runs each as its own torch
// op, so a contracted FMA would round differently.  The 512^2 logits are never materialised: each pixel interpolates its classes from
// the render-resolution logits (any strides: the strided channel view of the ray-march output is read in place).
#include "seg_common.cuh"

namespace ide3d {

constexpr int kTileX = 64, kTileY = 4;           // 256 threads, one output pixel each

// layout_grid: (x * 127.5 + 128).clamp(0, 255).to(torch.uint8).  clamp lets NaN through and the cast goes float -> int64 -> uint8,
// as torch's clamp and c10's float -> uint8 conversion do, so a NaN pixel gets the byte torch writes for it.
__device__ __forceinline__ unsigned char to_u8(float v) {
    float y = __fadd_rn(__fmul_rn(v, 127.5f), 128.f);
    if (y == y) y = fminf(fmaxf(y, 0.f), 255.f);
    return (unsigned char)(long long)y;
}

// NaN-propagating min / max (torch.min / torch.max return NaN when any element is NaN)
__device__ __forceinline__ float nan_min(float a, float b) { return a != a ? a : (b != b ? b : fminf(a, b)); }
__device__ __forceinline__ float nan_max(float a, float b) { return a != a ? a : (b != b ? b : fmaxf(a, b)); }

__global__ void __launch_bounds__(kTileX * kTileY) frames_seg_kernel(ide3d_frames_params p) {
    const int x = blockIdx.x * kTileX + threadIdx.x, y = blockIdx.y * kTileY + threadIdx.y, n = blockIdx.z;
    if (x >= p.width || y >= p.height) return;
    const long long W2 = 2LL * p.width, plane = (long long)p.height * W2;
    unsigned char* o = p.out + (long long)n * 3 * plane + (long long)y * W2 + x;
    const float* im = p.image + n * p.image_stride_n + y * p.image_stride_h + x * p.image_stride_w;
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c * plane] = to_u8(__ldg(im + c * p.image_stride_c));

    // seg half: class of the bilinearly upsampled logits -> COLOR_MAP bytes
    const int arg = seg_class_at(p.seg + n * p.seg_stride_n, p.seg_c, p.seg_h, p.seg_w, p.seg_stride_c, p.seg_stride_h, p.seg_stride_w,
                                 x, y, p.height, p.width);
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c * plane + p.width] = (unsigned char)__ldg(p.lut + arg * 3 + c);
}

__global__ void __launch_bounds__(256) frames_minmax_kernel(ide3d_frames_params p, float* __restrict__ partials) {
    const int n = blockIdx.y;
    const long long hw = (long long)p.height * p.width, total = 3 * hw;
    const float* im = p.image + n * p.image_stride_n;
    float mn = INFINITY, mx = -INFINITY;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long c = i / hw, r = i - c * hw;
        const int yy = (int)(r / p.width), xx = (int)(r - (long long)yy * p.width);
        const float t = -__ldg(im + c * p.image_stride_c + yy * p.image_stride_h + xx * p.image_stride_w);
        mn = nan_min(mn, t);
        mx = nan_max(mx, t);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        mn = nan_min(mn, __shfl_xor_sync(0xffffffffu, mn, off));
        mx = nan_max(mx, __shfl_xor_sync(0xffffffffu, mx, off));
    }
    __shared__ float smn[8], smx[8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { smn[warp] = mn; smx[warp] = mx; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int k = 1; k < 8; ++k) { mn = nan_min(mn, smn[k]); mx = nan_max(mx, smx[k]); }
        partials[(n * IDE3D_FRAMES_PARTIALS + blockIdx.x) * 2 + 0] = mn;
        partials[(n * IDE3D_FRAMES_PARTIALS + blockIdx.x) * 2 + 1] = mx;
    }
}

__global__ void __launch_bounds__(kTileX * kTileY) frames_depth_kernel(ide3d_frames_params p, const float* __restrict__ partials) {
    const int n = blockIdx.z;
    __shared__ float range[2];
    if (threadIdx.x == 0 && threadIdx.y == 0) {
        float mn = INFINITY, mx = -INFINITY;
        for (int k = 0; k < IDE3D_FRAMES_PARTIALS; ++k) {
            mn = nan_min(mn, partials[(n * IDE3D_FRAMES_PARTIALS + k) * 2 + 0]);
            mx = nan_max(mx, partials[(n * IDE3D_FRAMES_PARTIALS + k) * 2 + 1]);
        }
        range[0] = mn;
        range[1] = mx;
    }
    __syncthreads();
    const int x = blockIdx.x * kTileX + threadIdx.x, y = blockIdx.y * kTileY + threadIdx.y;
    if (x >= p.width || y >= p.height) return;
    const float mn = range[0], d = __fsub_rn(range[1], range[0]);
    const long long plane = (long long)p.height * p.width;
    unsigned char* o = p.out + (long long)n * 3 * plane + (long long)y * p.width + x;
    const float* im = p.image + n * p.image_stride_n + y * p.image_stride_h + x * p.image_stride_w;
    // gen_videos.py:131-132: img = -img; img = (img - img.min()) / (img.max() - img.min()) * 2 - 1
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float t = -__ldg(im + c * p.image_stride_c);
        const float q = __fdiv_rn(__fsub_rn(t, mn), d);
        o[c * plane] = to_u8(__fsub_rn(__fmul_rn(q, 2.f), 1.f));
    }
}

}  // namespace ide3d

extern "C" int ide3d_video_frames(const ide3d_frames_params* p, ide3d_stream_t stream) {
    IDE3D_REQUIRE(p, "video_frames: null params");
    IDE3D_REQUIRE(p->mode == IDE3D_FRAMES_IMAGE_SEG || p->mode == IDE3D_FRAMES_IMAGE_DEPTH, "video_frames: unknown mode %d", p->mode);
    IDE3D_REQUIRE(p->n >= 0 && p->n <= 65535 && p->height >= 1 && p->width >= 1 && p->height <= 65535 * ide3d::kTileY,
                  "video_frames: bad sizes (n %d, height %d, width %d)", p->n, p->height, p->width);
    const bool seg = p->mode == IDE3D_FRAMES_IMAGE_SEG;
    if (seg) IDE3D_REQUIRE(p->seg_c >= 1 && p->seg_h >= 1 && p->seg_w >= 1, "video_frames: bad logit sizes (%d, %d, %d)", p->seg_c, p->seg_h, p->seg_w);
    if (p->n == 0) return IDE3D_OK;
    IDE3D_REQUIRE(p->image && p->out, "video_frames: null image or output");
    if (seg) IDE3D_REQUIRE(p->seg && p->lut, "video_frames: null logits or colour table");
    else IDE3D_REQUIRE(p->scratch, "video_frames: null scratch");
    cudaStream_t st = (cudaStream_t)stream;
    const dim3 block(ide3d::kTileX, ide3d::kTileY);
    const dim3 grid((unsigned)ide3d::ceil_div(p->width, ide3d::kTileX), (unsigned)ide3d::ceil_div(p->height, ide3d::kTileY), (unsigned)p->n);
    if (seg) {
        ide3d::frames_seg_kernel<<<grid, block, 0, st>>>(*p);
        IDE3D_CHECK_LAUNCH("frames_seg_kernel");
        return IDE3D_OK;
    }
    ide3d::frames_minmax_kernel<<<dim3(IDE3D_FRAMES_PARTIALS, (unsigned)p->n), 256, 0, st>>>(*p, p->scratch);
    IDE3D_CHECK_LAUNCH("frames_minmax_kernel");
    ide3d::frames_depth_kernel<<<grid, block, 0, st>>>(*p, p->scratch);
    IDE3D_CHECK_LAUNCH("frames_depth_kernel");
    return IDE3D_OK;
}
