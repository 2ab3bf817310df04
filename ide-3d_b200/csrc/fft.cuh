// Float64 radix-2 FFT in shared memory: the building blocks of the power spectra (spectra.cu) and the visualizer's FFT panel (viz.cu).
//
// A tile holds kTile complex values: kTile / N sequences of length N side by side, rows padded by one element against bank conflicts.
// Twiddles come from a per-CTA table of w_P^j, j < P, for some multiple P of N (w_N^k = w_P^{k P / N}).
#pragma once

#include "common.cuh"

namespace ide3d {

__device__ __forceinline__ double2 cmul(double2 a, double2 b) { return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }

// tw[j] = w_P^j = exp(-2 pi i j / P), j < P
template <int kThreads>
__device__ __forceinline__ void twiddle_table(double2* tw, int P) {
    for (int j = threadIdx.x; j < P; j += kThreads) {
        double s, c;
        sincospi(2.0 * j / P, &s, &c);
        tw[j] = make_double2(c, -s);
    }
}

// In-place radix-2 DIF over the tile: kTile / N sequences of length N = 2^logN at row stride N + 1; output in bit-reversed order.
template <int kThreads, int kTile>
__device__ __forceinline__ void dif_fft(double2* buf, const double2* tw, int N, int logN, int P) {
    constexpr int kPer = kTile / kThreads;
    const int half = N >> 1, logHalf = logN - 1;
    for (int logh = logN - 1; logh >= 0; --logh) {
        const int h = 1 << logh;
        const int tstep = P >> (logh + 1);                   // w_N^{j N / 2h} = w_P^{j P / 2h}
#pragma unroll
        for (int k = 0; k < kPer / 2; ++k) {
            const int t = threadIdx.x + k * kThreads;
            const int f = t >> logHalf, q = t & (half - 1);
            const int j = q & (h - 1);
            const int i = ((q >> logh) << (logh + 1)) + j;
            double2* p = buf + f * (N + 1) + i;
            const double2 x = p[0], y = p[h];
            p[0] = make_double2(x.x + y.x, x.y + y.y);
            p[h] = cmul(make_double2(x.x - y.x, x.y - y.y), tw[j * tstep]);
        }
        __syncthreads();
    }
}

__device__ __forceinline__ int bitrev(int m, int logN) { return (int)(__brev((unsigned)m) >> (32 - logN)); }

inline int log2_exact(int v) {
    int l = 0;
    while ((1 << l) < v) ++l;
    return (1 << l) == v ? l : -1;
}

}  // namespace ide3d
