// The style-mixing grid of style_mixing.py:139-153 in the uint8 HWC bytes PIL pastes: a black top-left cell, the column seeds along the
// top, the row seeds down the left, the mixed cells inside.  One kernel, one thread per canvas pixel, every view in one launch:
//   canvas pixel -> grid slot (g, j) = (y / height, x / width) -> cell g * (cols + 1) + j - 1 (canvas order), or black for slot (0, 0)
//   cell pixel   -> (v * 127.5 + 128).clamp(0, 255).to(uint8) per channel (style_mixing.py:101)
#include "common.cuh"

namespace ide3d {

constexpr int kGridTileX = 64, kGridTileY = 4;      // 256 threads, one canvas pixel each

__global__ void __launch_bounds__(kGridTileX * kGridTileY)
style_grid_kernel(const float* __restrict__ cells, int first_row, int cols, int views, int height, int width, long long first_cell,
                  long long stride_n, long long stride_c, long long stride_h, long long stride_w, unsigned char* __restrict__ out,
                  long long out_stride_row, long long out_stride_view, int canvas_h, int canvas_w) {
    const int x = blockIdx.x * kGridTileX + threadIdx.x, y = blockIdx.y * kGridTileY + threadIdx.y, v = blockIdx.z;
    if (x >= canvas_w || y >= canvas_h) return;
    const int gi = y / height, yy = y - gi * height, j = x / width, xx = x - j * width;
    const long long g = (long long)first_row + gi;
    unsigned char* o = out + gi * out_stride_row + v * out_stride_view + (long long)yy * canvas_w * 3 + (long long)x * 3;
    const long long slot = g * (cols + 1) + j;
    if (slot == 0) {
        o[0] = 0; o[1] = 0; o[2] = 0;
        return;
    }
    const long long n = (slot - 1 - first_cell) * views + v;
    const float* im = cells + n * stride_n + yy * stride_h + xx * stride_w;
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = torch_u8(__ldg(im + c * stride_c));
}

}  // namespace ide3d

extern "C" int ide3d_style_grid(const float* cells, int first_row, int rows, int cols, int views, int height, int width, int64_t stride_n,
                                int64_t stride_c, int64_t stride_h, int64_t stride_w, uint8_t* out, int64_t out_stride_row,
                                int64_t out_stride_view, ide3d_stream_t stream) {
    IDE3D_REQUIRE(first_row >= 0 && rows >= 0 && cols >= 1 && views >= 1 && views <= 65535 && height >= 1 && width >= 1,
                  "style_grid: bad sizes (first_row %d, rows %d, cols %d, views %d, height %d, width %d)", first_row, rows, cols, views,
                  height, width);
    const long long canvas_h = (long long)rows * height, canvas_w = ((long long)cols + 1) * width;
    IDE3D_REQUIRE(canvas_w * 3 <= (1LL << 30) && canvas_h <= 65535LL * ide3d::kGridTileY,
                  "style_grid: canvas too large (%lld x %lld)", canvas_h, canvas_w);
    if (rows == 0) return IDE3D_OK;
    IDE3D_REQUIRE(cells && out, "style_grid: null cells or output");
    const long long first_cell = first_row == 0 ? 0 : (long long)first_row * (cols + 1) - 1;
    const dim3 block(ide3d::kGridTileX, ide3d::kGridTileY);
    const dim3 grid((unsigned)ide3d::ceil_div(canvas_w, (long long)ide3d::kGridTileX),
                    (unsigned)ide3d::ceil_div(canvas_h, (long long)ide3d::kGridTileY), (unsigned)views);
    ide3d::style_grid_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(cells, first_row, cols, views, height, width, first_cell, stride_n,
                                                                      stride_c, stride_h, stride_w, out, out_stride_row, out_stride_view,
                                                                      (int)canvas_h, (int)canvas_w);
    IDE3D_CHECK_LAUNCH("style_grid_kernel");
    return IDE3D_OK;
}
