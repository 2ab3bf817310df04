// The two PNG strips of gen_images.py (gen_images.py:109-116): per seed, its views side by side as torchvision's make_grid lays them
// out, in the uint8 HWC bytes save_image(normalize=True, value_range=(-1, 1)) hands to PIL.  One kernel, one thread per strip pixel:
//   padding pixel -> 0 in both strips
//   view pixel    -> image bytes (the save_image chain) | bilinear class logits -> argmax -> COLOR_MAP bytes
// The seg strip needs no float chain: (colour / 255 - 0.5) / 0.5 followed by save_image's conversion returns every byte value unchanged.
#include "seg_common.cuh"

namespace ide3d {

constexpr int kStripTileX = 64, kStripTileY = 4;      // 256 threads, one strip pixel each

// save_image(normalize=True, value_range=(-1, 1)): make_grid's norm_ip (clamp_(-1, 1), sub_(-1), div_(2)), then
// mul(255).add_(0.5).clamp_(0, 255).to(uint8).  clamp lets NaN through and the cast goes float -> int64 -> uint8, as torch's device
// conversion does.
__device__ __forceinline__ unsigned char save_image_u8(float v) {
    float y = v == v ? fminf(fmaxf(v, -1.f), 1.f) : v;
    y = __fdiv_rn(__fsub_rn(y, -1.f), 2.f);
    y = __fadd_rn(__fmul_rn(y, 255.f), 0.5f);
    if (y == y) y = fminf(fmaxf(y, 0.f), 255.f);
    return (unsigned char)(long long)y;
}

__global__ void __launch_bounds__(kStripTileX * kStripTileY) image_strips_kernel(ide3d_strips_params p, int strip_h, int strip_w, int pad) {
    const int x = blockIdx.x * kStripTileX + threadIdx.x, y = blockIdx.y * kStripTileY + threadIdx.y, s = blockIdx.z;
    if (x >= strip_w || y >= strip_h) return;
    const long long o = (((long long)s * strip_h + y) * strip_w + x) * 3;
    // which view, and where in it: view j spans columns [pad + j * (width + pad), + width), rows [pad, pad + height)
    const int xr = x - pad, yr = y - pad;
    const int j = xr >= 0 ? xr / (p.width + pad) : -1;
    const int px = xr - j * (p.width + pad);
    if (xr < 0 || j >= p.views || px >= p.width || yr < 0 || yr >= p.height) {
#pragma unroll
        for (int c = 0; c < 3; ++c) { p.out_image[o + c] = 0; p.out_seg[o + c] = 0; }
        return;
    }
    const long long n = (long long)s * p.views + j;
    const float* im = p.image + n * p.image_stride_n + yr * p.image_stride_h + px * p.image_stride_w;
#pragma unroll
    for (int c = 0; c < 3; ++c) p.out_image[o + c] = save_image_u8(__ldg(im + c * p.image_stride_c));
    const int arg = seg_class_at(p.seg + n * p.seg_stride_n, p.seg_c, p.seg_h, p.seg_w, p.seg_stride_c, p.seg_stride_h, p.seg_stride_w,
                                 px, yr, p.height, p.width);
#pragma unroll
    for (int c = 0; c < 3; ++c) p.out_seg[o + c] = (unsigned char)__ldg(p.lut + arg * 3 + c);
}

}  // namespace ide3d

extern "C" int ide3d_image_strips(const ide3d_strips_params* p, ide3d_stream_t stream) {
    IDE3D_REQUIRE(p, "image_strips: null params");
    IDE3D_REQUIRE(p->seeds >= 0 && p->seeds <= 65535 && p->views >= 1 && p->views <= 8 && p->height >= 1 && p->width >= 1,
                  "image_strips: bad sizes (seeds %d, views %d, height %d, width %d)", p->seeds, p->views, p->height, p->width);
    IDE3D_REQUIRE(p->seg_c >= 1 && p->seg_h >= 1 && p->seg_w >= 1, "image_strips: bad logit sizes (%d, %d, %d)", p->seg_c, p->seg_h, p->seg_w);
    const int pad = p->views > 1 ? 2 : 0;
    const long long strip_h = (long long)p->height + 2 * pad, strip_w = (long long)p->views * (p->width + pad) + pad;
    IDE3D_REQUIRE(strip_w <= (1 << 30) && strip_h <= 65535LL * ide3d::kStripTileY, "image_strips: strip too large (%lld x %lld)", strip_h, strip_w);
    if (p->seeds == 0) return IDE3D_OK;
    IDE3D_REQUIRE(p->image && p->seg && p->lut, "image_strips: null image, logits or colour table");
    IDE3D_REQUIRE(p->out_image && p->out_seg, "image_strips: null output");
    const dim3 block(ide3d::kStripTileX, ide3d::kStripTileY);
    const dim3 grid((unsigned)ide3d::ceil_div((int)strip_w, ide3d::kStripTileX), (unsigned)ide3d::ceil_div((int)strip_h, ide3d::kStripTileY),
                    (unsigned)p->seeds);
    ide3d::image_strips_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(*p, (int)strip_h, (int)strip_w, pad);
    IDE3D_CHECK_LAUNCH("image_strips_kernel");
    return IDE3D_OK;
}
