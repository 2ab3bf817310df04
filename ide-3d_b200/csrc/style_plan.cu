// All style vectors and demodulation coefficients of one synthesis call in TWO launches.
//
// The reference evaluates, per modulated convolution, `styles = affine(w)` (FullyConnectedLayer, inversion/networks.py:136-165,
// :476) and `dcoefs = rsqrt(sum_{i,k} (W[o,i,k] s[n,i])^2 + 1e-8)` (:89-90); with 18 layers that was ~150 tiny library launches
// per step (addmm / square / sum / rsqrt / mul; about 10 % of the step in the first measured profile).  Both are
// independent of the activations, so they are computed up front:
//   styles[l][n, i] = ((A_l[i, :] . ws[n, w_index_l, :]) * w_gain_l + b_l[i] * b_gain_l) * out_scale_l        (one warp per row i)
//   dcoefs[l][n, o] = rsqrt(sum_i styles[l][n, i]^2 * Wsq_l[o, i] + 1e-8),  Wsq_l[o, i] = sum_k W_l[o, i, k]^2   (one warp per o)
// Wsq is a constant of the weights (cached by the host).  fp32 throughout.
#include "common.cuh"

namespace ide3d {

constexpr int kMaxStyleLayers = 32;
constexpr int kStyleBatch = 8;           // batch entries handled per pass (accumulators per lane)

struct StylePlanArgs {
    ide3d_style_layer layer[kMaxStyleLayers];
    int row_start[kMaxStyleLayers + 1];   // prefix sums of in_ch (styles) or out_ch (dcoefs)
    int num_layers;
    const float* ws;
    int n, num_ws, w_dim;
    float* styles;
    float* dcoefs;
};

__device__ __forceinline__ int find_layer(const int* row_start, int num_layers, int row) {
    int lo = 0, hi = num_layers;          // largest l with row_start[l] <= row
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (row_start[mid] <= row) lo = mid; else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(256) style_affine_kernel(const __grid_constant__ StylePlanArgs a) {
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= a.row_start[a.num_layers]) return;
    const int l = find_layer(a.row_start, a.num_layers, row);
    const ide3d_style_layer& L = a.layer[l];
    const int i = row - a.row_start[l];
    const float* arow = L.affine_w + (long long)i * a.w_dim;
    const float bias = L.affine_b ? L.affine_b[i] * L.b_gain : 0.f;
    for (int n0 = 0; n0 < a.n; n0 += kStyleBatch) {
        float acc[kStyleBatch];
#pragma unroll
        for (int j = 0; j < kStyleBatch; ++j) acc[j] = 0.f;
        for (int k = lane; k < a.w_dim; k += 32) {           // (unrolling by 4 measured slower: 68 vs 42 us)
            const float av = arow[k];
#pragma unroll
            for (int j = 0; j < kStyleBatch; ++j)
                if (n0 + j < a.n) acc[j] = fmaf(av, a.ws[((long long)(n0 + j) * a.num_ws + L.w_index) * a.w_dim + k], acc[j]);
        }
#pragma unroll
        for (int j = 0; j < kStyleBatch; ++j) {
            float v = acc[j];
#pragma unroll
            for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
            if (lane == j && n0 + j < a.n) a.styles[L.style_off + (long long)(n0 + j) * L.in_ch + i] = (v * L.w_gain + bias) * L.out_scale;
        }
    }
}

__global__ void __launch_bounds__(256) style_demod_kernel(const __grid_constant__ StylePlanArgs a) {
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= a.row_start[a.num_layers]) return;
    const int l = find_layer(a.row_start, a.num_layers, row);
    const ide3d_style_layer& L = a.layer[l];
    if (L.wsq == nullptr) return;
    const int o = row - a.row_start[l];
    const float* wrow = L.wsq + (long long)o * L.in_ch;
    for (int n0 = 0; n0 < a.n; n0 += kStyleBatch) {
        float acc[kStyleBatch];
#pragma unroll
        for (int j = 0; j < kStyleBatch; ++j) acc[j] = 0.f;
        for (int i = lane; i < L.in_ch; i += 32) {
            const float wv = wrow[i];
#pragma unroll
            for (int j = 0; j < kStyleBatch; ++j)
                if (n0 + j < a.n) {
                    const float s = a.styles[L.style_off + (long long)(n0 + j) * L.in_ch + i];
                    acc[j] = fmaf(s * s, wv, acc[j]);
                }
        }
#pragma unroll
        for (int j = 0; j < kStyleBatch; ++j) {
            float v = acc[j];
#pragma unroll
            for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
            if (lane == j && n0 + j < a.n) a.dcoefs[L.dcoef_off + (long long)(n0 + j) * L.out_ch + o] = rsqrtf(v + 1e-8f);
        }
    }
}

}  // namespace ide3d

using namespace ide3d;

extern "C" int ide3d_style_plan(const float* ws, int n, int num_ws, int w_dim, const ide3d_style_layer* layers, int num_layers,
                                float* styles, float* dcoefs, ide3d_stream_t stream) {
    IDE3D_REQUIRE(ws && layers && styles, "style_plan: null argument");
    IDE3D_REQUIRE(n > 0 && num_ws > 0 && w_dim > 0, "style_plan: empty ws");
    IDE3D_REQUIRE(num_layers > 0 && num_layers <= kMaxStyleLayers, "style_plan: between 1 and 32 layers");
    StylePlanArgs a;
    a.num_layers = num_layers; a.ws = ws; a.n = n; a.num_ws = num_ws; a.w_dim = w_dim; a.styles = styles; a.dcoefs = dcoefs;
    bool any_demod = false;
    a.row_start[0] = 0;
    for (int l = 0; l < num_layers; ++l) {
        const ide3d_style_layer& L = layers[l];
        IDE3D_REQUIRE(L.affine_w && L.in_ch > 0 && L.w_index >= 0 && L.w_index < num_ws, "style_plan: bad layer %d", l);
        IDE3D_REQUIRE(L.wsq == nullptr || (L.out_ch > 0 && dcoefs != nullptr), "style_plan: layer %d demodulates but has no output", l);
        a.layer[l] = L;
        a.row_start[l + 1] = a.row_start[l] + L.in_ch;
        any_demod |= (L.wsq != nullptr);
    }
    cudaStream_t st = (cudaStream_t)stream;
    style_affine_kernel<<<ceil_div(a.row_start[num_layers], 8), 256, 0, st>>>(a);
    IDE3D_CHECK_LAUNCH("style_affine_kernel");
    if (any_demod) {
        for (int l = 0; l < num_layers; ++l) a.row_start[l + 1] = a.row_start[l] + (layers[l].wsq ? layers[l].out_ch : 0);
        if (a.row_start[num_layers] > 0) {
            style_demod_kernel<<<ceil_div(a.row_start[num_layers], 8), 256, 0, st>>>(a);
            IDE3D_CHECK_LAUNCH("style_demod_kernel");
        }
    }
    return IDE3D_OK;
}
