// Arguments of the fused filtered_lrelu kernel (filtered_lrelu_fused.cu), filled in by ide3d_filtered_lrelu (filtered_lrelu.cu).
#pragma once

#include <cuda_runtime.h>

namespace ide3d {

struct FlFusedArgs {
    const void* x; const void* b; const float* fu; const float* fd; void* y; unsigned char* s;
    int px0, py0, flip;
    float gain, slope, clamp;
    int xw, xh, xc, xn;
    long long sxw, sxh, sxc, sxn;
    int yw, yh;
    long long syw, syh, syc, syn;
    int sw, sh, sox, soy, mode;          // mode 0: plain, 1: write signs, 2: read signs
    int one_u, one_d;                    // 1x1 "full" filters carry their value once, not once per axis
    int channels_last;
};

// IDE3D_UNSUPPORTED when no fused kernel covers (up, down, fu, fd); dtype IDE3D_F32 or IDE3D_F16
int launch_filtered_lrelu_fused(const FlFusedArgs& a, int dtype, int up, int down, int fu, int fd, cudaStream_t st);

}  // namespace ide3d
