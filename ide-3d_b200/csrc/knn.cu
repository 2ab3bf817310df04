// k-nearest-neighbour distances of the precision/recall metric (metrics/precision_recall.py): ide3d_knn_kth_dist and
// ide3d_knn_within.  Both are one Hopper GEMM main loop over fp16 features with the distance epilogue in registers:
//
//   CTA = 128 rows (two consumer warpgroups of 64) x all column tiles of its split (128 columns each).  A producer warp streams
//   the row tile's and the column tile's 64-wide K slices with tma_load_2d (128-byte swizzle) into a 4-stage
//   full / empty mbarrier ring; each consumer warpgroup runs wgmma m64n128k16 (fp16 operands, fp32 accumulators) over the ring
//   and turns its 64 x 128 dot products into squared distances max(|x|^2 + |y|^2 - 2 x.y, 0) with fp32 row norms of the same
//   fp16 values (knn_norms_kernel).  The R x C matrix is never stored.
//
//   kth_dist: each thread keeps the K smallest squared distances of its two rows over the columns it owns, sorted in registers;
//             at the end the four threads of a row merge their lists, and a second launch merges the column splits and takes
//             the kth one.
//   within:   a row's flag is set when some column j has d^2 <= radius[j]^2.  After every column tile the CTA votes; once all of
//             its rows have a hit it stops (the producer learns it one tile later, so the consumers drain the one tile already
//             in flight).
//
// Column tiles are walked in ascending order by every CTA, so the CTAs resident at the same time stream the same column tiles
// through L2.  Splitting the columns over several CTAs (when the row tiles alone do not fill the device) keeps that order inside
// each split.
#include "common.cuh"
#include "tc_ptx.cuh"
#include "tma.cuh"

namespace ide3d {
namespace {

constexpr int kBM = 128, kBN = 128, kBK = 64;         // kBK fp16 = one 128-byte swizzled row
constexpr int kStages = 4;
constexpr int kTileBytes = kBM * kBK * 2;             // A and B tiles are both 128 x 64 fp16
constexpr int kStageBytes = 2 * kTileBytes;
constexpr int kThreads = 288;                         // 2 consumer warpgroups + 1 producer warp
constexpr size_t kSmem = (size_t)kStages * kStageBytes + 1024 + 256;
static_assert(kBM == kBN, "one tensor-map box serves both operands");

struct KnnArgs {
    const float* row_norm;
    const float* col_norm;
    int64_t R, C;
    int kchunks, col_tiles, splits;
    const float* radius;     // within
    uint8_t* flags;          // within
    float* partial;          // kth_dist: [splits, R, K]
};

// sorted insertion into the K smallest seen so far (t ascending)
template <int K>
__device__ __forceinline__ void insert(float (&t)[K], float v) {
    if (v < t[K - 1]) {
#pragma unroll
        for (int i = 0; i < K; ++i) {
            const float lo = fminf(t[i], v);
            v = fmaxf(t[i], v);
            t[i] = lo;
        }
    }
}

// |x|^2 in fp32 of every fp16 row, one warp per row (D % 8 == 0, 16-byte aligned rows)
__global__ void __launch_bounds__(256) knn_norms_kernel(const __half* __restrict__ x, int64_t n, int D, float* __restrict__ out) {
    const int64_t row = (int64_t)blockIdx.x * 8 + threadIdx.x / 32;
    const int lane = threadIdx.x % 32;
    if (row >= n) return;
    const __half* p = x + row * D;
    float s = 0.f;
    for (int k = lane * 8; k < D; k += 256) {
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(p + k));
        const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 f = __half22float2(h[i]);
            s = fmaf(f.x, f.x, s);
            s = fmaf(f.y, f.y, s);
        }
    }
#pragma unroll
    for (int m = 16; m; m >>= 1) s += __shfl_xor_sync(~0u, s, m);
    if (lane == 0) out[row] = s;
}

template <int K, bool WITHIN>
__global__ void __launch_bounds__(kThreads, 1) knn_tile_kernel(const __grid_constant__ CUtensorMap rows_map,
                                                               const __grid_constant__ CUtensorMap cols_map, const KnnArgs a) {
    extern __shared__ unsigned char knn_raw[];
    unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(knn_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* full = reinterpret_cast<uint64_t*>(base + kStages * kStageBytes);
    uint64_t* empty = full + kStages;
    uint64_t* tile_done = empty + kStages;                                  // [2], within only: tile j's vote is posted
    volatile int* decision = reinterpret_cast<volatile int*>(tile_done + 2);  // [2]: tile j's vote (1 = every row has a hit)
    volatile int* warp_ok = decision + 2;                                   // [2][8]

    const int row_tile = blockIdx.x / a.splits, split = blockIdx.x % a.splits;
    const int row0 = row_tile * kBM;
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;

    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 8);                                        // lane 0 of each consumer warp
        }
        mbar_init(&tile_done[0], 1);
        mbar_init(&tile_done[1], 1);
        mbar_fence_init();
    }
    __syncthreads();

    if (warp == 8) {                                                        // producer
        if (lane == 0) {
            int it = 0, j = 0;
            for (int ct = split; ct < a.col_tiles; ct += a.splits, ++j) {
                if (WITHIN && j >= 2) {                                     // tile j is issued only if tile j - 2 left a row without a hit
                    mbar_wait(&tile_done[j & 1], ((j - 2) >> 1) & 1);
                    if (decision[j & 1]) break;
                }
                for (int kc = 0; kc < a.kchunks; ++kc, ++it) {
                    const int s = it % kStages;
                    if (it >= kStages) mbar_wait(&empty[s], (it / kStages - 1) & 1);
                    mbar_arrive_expect_tx(&full[s], kStageBytes);
                    unsigned char* st = base + s * kStageBytes;
                    tma_load_2d(st, &rows_map, &full[s], kc * kBK, row0);
                    tma_load_2d(st + kTileBytes, &cols_map, &full[s], kc * kBK, ct * kBN);
                }
            }
        }
        return;
    }

    // consumer: thread (warpgroup wg, warp w4, lane) owns rows r and r + 8, columns 8j + 2(lane % 4) + {0, 1} of each tile
    const int wg = warp / 4, w4 = warp % 4;
    const int64_t gr0 = row0 + wg * 64 + w4 * 16 + lane / 4, gr1 = gr0 + 8;
    const float nr0 = gr0 < a.R ? a.row_norm[gr0] : 0.f, nr1 = gr1 < a.R ? a.row_norm[gr1] : 0.f;
    float acc[64];
    float top0[K], top1[K];
#pragma unroll
    for (int i = 0; i < K; ++i) top0[i] = top1[i] = INFINITY;
    bool hit0 = false, hit1 = false;

    int it = 0, j = 0;
    for (int ct = split; ct < a.col_tiles; ct += a.splits, ++j) {
        for (int kc = 0; kc < a.kchunks; ++kc, ++it) {
            const int s = it % kStages;
            mbar_wait(&full[s], (it / kStages) & 1);
            const uint32_t a_addr = smem_u32(base + s * kStageBytes) + wg * 64 * 128;
            const uint32_t b_addr = smem_u32(base + s * kStageBytes + kTileBytes);
            tc::wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < kBK / 16; ++kk)
                tc::wgmma_f16_m64n128_ss(acc, tc::make_sdesc_sw128(a_addr + kk * 32), tc::make_sdesc_sw128(b_addr + kk * 32), (kc | kk) != 0);
            tc::wgmma_commit();
            tc::wgmma_wait<1>();
            if (kc > 0) {                                                   // the previous chunk's MMAs are done: release its stage
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[(it - 1) % kStages]);
            }
        }
        tc::wgmma_wait<0>();
        tc::fence_regs(acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[(it - 1) % kStages]);

        const int64_t cb = (int64_t)ct * kBN + 2 * (lane % 4);
#pragma unroll
        for (int jj = 0; jj < kBN / 8; ++jj) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int64_t c = cb + 8 * jj + e;
                const bool valid = c < a.C;
                const float nc = valid ? __ldg(a.col_norm + c) : 0.f;
                const float d0 = fmaxf(nr0 + nc - 2.f * acc[4 * jj + e], 0.f);
                const float d1 = fmaxf(nr1 + nc - 2.f * acc[4 * jj + 2 + e], 0.f);
                if constexpr (WITHIN) {
                    const float r = valid ? __ldg(a.radius + c) : -1.f;
                    const float r2 = r >= 0.f ? r * r : -1.f;
                    hit0 |= d0 <= r2;
                    hit1 |= d1 <= r2;
                } else if (valid) {
                    insert(top0, d0);
                    insert(top1, d1);
                }
            }
        }

        if constexpr (WITHIN) {
            hit0 |= __shfl_xor_sync(~0u, hit0, 1);
            hit0 |= __shfl_xor_sync(~0u, hit0, 2);
            hit1 |= __shfl_xor_sync(~0u, hit1, 1);
            hit1 |= __shfl_xor_sync(~0u, hit1, 2);
            const bool ok = __all_sync(~0u, (gr0 >= a.R || hit0) && (gr1 >= a.R || hit1));
            if (lane == 0) warp_ok[(j & 1) * 8 + warp] = ok;
            tc::bar_sync(1, 256);
            bool stop = true;
#pragma unroll
            for (int w = 0; w < 8; ++w) stop &= warp_ok[(j & 1) * 8 + w] != 0;
            if (threadIdx.x == 0) {
                decision[j & 1] = stop;
                mbar_arrive(&tile_done[j & 1]);
            }
            if (stop) {
                // the producer issued tile j + 1 before it could see this vote: take its chunks off the ring
                if (ct + a.splits < a.col_tiles) {
                    for (int kc = 0; kc < a.kchunks; ++kc, ++it) {
                        const int s = it % kStages;
                        mbar_wait(&full[s], (it / kStages) & 1);
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&empty[s]);
                    }
                }
                break;
            }
        }
    }

    if constexpr (WITHIN) {
        if (lane % 4 == 0) {
            if (gr0 < a.R && hit0) a.flags[gr0] = 1;
            if (gr1 < a.R && hit1) a.flags[gr1] = 1;
        }
    } else {
#pragma unroll
        for (int m = 1; m <= 2; m <<= 1) {
            float o0[K], o1[K];
#pragma unroll
            for (int i = 0; i < K; ++i) {
                o0[i] = __shfl_xor_sync(~0u, top0[i], m);
                o1[i] = __shfl_xor_sync(~0u, top1[i], m);
            }
#pragma unroll
            for (int i = 0; i < K; ++i) {
                insert(top0, o0[i]);
                insert(top1, o1[i]);
            }
        }
        if (lane % 4 == 0) {
            float* p = a.partial + ((int64_t)split * a.R) * K;
#pragma unroll
            for (int i = 0; i < K; ++i) {
                if (gr0 < a.R) p[gr0 * K + i] = top0[i];
                if (gr1 < a.R) p[gr1 * K + i] = top1[i];
            }
        }
    }
}

// out[r] = sqrt of the kth smallest squared distance over the splits' lists
template <int K>
__global__ void __launch_bounds__(256) knn_kth_merge_kernel(const float* __restrict__ partial, int splits, int64_t R, int kth, float* __restrict__ out) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    float t[K];
#pragma unroll
    for (int i = 0; i < K; ++i) t[i] = INFINITY;
    for (int s = 0; s < splits; ++s) {
        const float* p = partial + ((int64_t)s * R + r) * K;
#pragma unroll
        for (int i = 0; i < K; ++i) insert(t, p[i]);
    }
    float v = t[0];
#pragma unroll
    for (int i = 1; i < K; ++i)
        if (i == kth - 1) v = t[i];
    out[r] = sqrtf(v);
}

// [n, D] fp16 row-major, 128 x 64 boxes with the 128-byte swizzle; rows past n and K past D read as zero
int make_map(CUtensorMap* map, const void* x, int64_t n, int D) {
    if (encode_tiled() == nullptr) IDE3D_FAIL(IDE3D_UNSUPPORTED, "knn: the driver provides no tensor-map encoder");
    const cuuint64_t dims[2] = {(cuuint64_t)D, (cuuint64_t)n};
    const cuuint64_t strides[1] = {(cuuint64_t)D * 2};
    const cuuint32_t box[2] = {(cuuint32_t)kBK, (cuuint32_t)kBM};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = encode_tiled()(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(x), dims, strides, box, estr,
                                      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) IDE3D_FAIL(IDE3D_UNSUPPORTED, "knn: encoding the tensor map failed (%d)", (int)r);
    return IDE3D_OK;
}

// column splits: enough CTAs to give every SM one when the row tiles alone do not
int knn_splits(int64_t rows, int64_t cols) {
    const int64_t row_tiles = ceil_div<int64_t>(rows, kBM), col_tiles = ceil_div<int64_t>(cols, kBN);
    int64_t s = ceil_div<int64_t>(sm_count(), row_tiles < 1 ? 1 : row_tiles);
    if (s > col_tiles) s = col_tiles;
    return (int)(s < 1 ? 1 : s);
}

int kth_cap(int kth) { return kth <= 1 ? 1 : kth <= 4 ? 4 : 16; }

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

int check_operands(const char* fn, const void* a, int64_t n, const void* b, int64_t m, int D) {
    IDE3D_REQUIRE(a != nullptr && b != nullptr, "%s: null feature pointer", fn);
    IDE3D_REQUIRE(n >= 0 && m >= 1 && n <= 0x7fffffffLL && m <= 0x7fffffffLL, "%s: bad row counts %lld, %lld", fn, (long long)n, (long long)m);
    IDE3D_REQUIRE(D >= 8 && D % 8 == 0, "%s: feature dimension D = %d must be a positive multiple of 8", fn, D);
    IDE3D_REQUIRE((reinterpret_cast<uintptr_t>(a) & 15) == 0 && (reinterpret_cast<uintptr_t>(b) & 15) == 0,
                  "%s: feature pointers must be 16-byte aligned", fn);
    return IDE3D_OK;
}

template <int K, bool WITHIN>
int launch_tiles(const void* rows, int64_t R, const void* cols, int64_t C, int D, const KnnArgs& a, cudaStream_t st) {
    CUtensorMap rmap, cmap;
    int rc = make_map(&rmap, rows, R, D);
    if (rc != IDE3D_OK) return rc;
    rc = make_map(&cmap, cols, C, D);
    if (rc != IDE3D_OK) return rc;
    auto kern = knn_tile_kernel<K, WITHIN>;
    IDE3D_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmem));
    const long long grid = ceil_div<int64_t>(R, kBM) * a.splits;
    kern<<<(unsigned)grid, kThreads, kSmem, st>>>(rmap, cmap, a);
    IDE3D_CHECK_LAUNCH(WITHIN ? "knn_within_kernel" : "knn_kth_kernel");
    return IDE3D_OK;
}

int launch_norms(const void* x, int64_t n, int D, float* out, cudaStream_t st) {
    knn_norms_kernel<<<(unsigned)ceil_div<int64_t>(n, 8), 256, 0, st>>>(static_cast<const __half*>(x), n, D, out);
    IDE3D_CHECK_LAUNCH("knn_norms_kernel");
    return IDE3D_OK;
}

}  // namespace
}  // namespace ide3d

using namespace ide3d;

extern "C" int64_t ide3d_knn_kth_dist_scratch_bytes(int64_t R, int64_t C, int kth) {
    if (R < 0 || C < 1 || kth < 1 || kth > IDE3D_KNN_MAX_KTH) return IDE3D_INVALID;
    return (int64_t)(align256((size_t)(R + C) * 4) + (size_t)knn_splits(R, C) * R * kth_cap(kth) * 4);
}

extern "C" int ide3d_knn_kth_dist(const void* rows, int64_t R, const void* cols, int64_t C, int D, int kth, float* out, void* scratch,
                                  int64_t scratch_bytes, ide3d_stream_t stream) {
    int rc = check_operands("knn_kth_dist", rows, R, cols, C, D);
    if (rc != IDE3D_OK) return rc;
    IDE3D_REQUIRE(kth >= 1 && kth <= IDE3D_KNN_MAX_KTH, "knn_kth_dist: kth = %d outside [1, %d]", kth, IDE3D_KNN_MAX_KTH);
    IDE3D_REQUIRE(kth <= C, "knn_kth_dist: kth = %d exceeds the %lld columns", kth, (long long)C);
    IDE3D_REQUIRE(out != nullptr && scratch != nullptr, "knn_kth_dist: null output or scratch pointer");
    IDE3D_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 255) == 0, "knn_kth_dist: scratch must be 256-byte aligned");
    const int64_t need = ide3d_knn_kth_dist_scratch_bytes(R, C, kth);     // the one check that queries the device (its SM count)
    IDE3D_REQUIRE(scratch_bytes >= need, "knn_kth_dist: scratch of %lld bytes, %lld needed", (long long)scratch_bytes, (long long)need);
    if (R == 0) return IDE3D_OK;
    cudaStream_t st = (cudaStream_t)stream;
    float* rn = static_cast<float*>(scratch);
    float* cn = rn + R;
    KnnArgs a{};
    a.row_norm = rn;
    a.col_norm = cn;
    a.R = R;
    a.C = C;
    a.kchunks = ceil_div(D, kBK);
    a.col_tiles = (int)ceil_div<int64_t>(C, kBN);
    a.splits = knn_splits(R, C);
    a.partial = reinterpret_cast<float*>(static_cast<unsigned char*>(scratch) + align256((size_t)(R + C) * 4));
    if ((rc = launch_norms(rows, R, D, rn, st)) != IDE3D_OK) return rc;
    if ((rc = launch_norms(cols, C, D, cn, st)) != IDE3D_OK) return rc;
    const unsigned mgrid = (unsigned)ceil_div<int64_t>(R, 256);
    switch (kth_cap(kth)) {
    case 1:
        if ((rc = launch_tiles<1, false>(rows, R, cols, C, D, a, st)) != IDE3D_OK) return rc;
        knn_kth_merge_kernel<1><<<mgrid, 256, 0, st>>>(a.partial, a.splits, R, kth, out);
        break;
    case 4:
        if ((rc = launch_tiles<4, false>(rows, R, cols, C, D, a, st)) != IDE3D_OK) return rc;
        knn_kth_merge_kernel<4><<<mgrid, 256, 0, st>>>(a.partial, a.splits, R, kth, out);
        break;
    default:
        if ((rc = launch_tiles<16, false>(rows, R, cols, C, D, a, st)) != IDE3D_OK) return rc;
        knn_kth_merge_kernel<16><<<mgrid, 256, 0, st>>>(a.partial, a.splits, R, kth, out);
        break;
    }
    IDE3D_CHECK_LAUNCH("knn_kth_merge_kernel");
    return IDE3D_OK;
}

extern "C" int64_t ide3d_knn_within_scratch_bytes(int64_t Q, int64_t M) {
    if (Q < 0 || M < 1) return IDE3D_INVALID;
    return (int64_t)align256((size_t)(Q + M) * 4);
}

extern "C" int ide3d_knn_within(const void* probes, int64_t Q, const void* manifold, int64_t M, int D, const float* radius,
                                uint8_t* flags, void* scratch, int64_t scratch_bytes, ide3d_stream_t stream) {
    int rc = check_operands("knn_within", probes, Q, manifold, M, D);
    if (rc != IDE3D_OK) return rc;
    IDE3D_REQUIRE(radius != nullptr && flags != nullptr && scratch != nullptr, "knn_within: null radius, flags or scratch pointer");
    IDE3D_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 255) == 0, "knn_within: scratch must be 256-byte aligned");
    const int64_t need = ide3d_knn_within_scratch_bytes(Q, M);
    IDE3D_REQUIRE(scratch_bytes >= need, "knn_within: scratch of %lld bytes, %lld needed", (long long)scratch_bytes, (long long)need);
    if (Q == 0) return IDE3D_OK;
    cudaStream_t st = (cudaStream_t)stream;
    float* qn = static_cast<float*>(scratch);
    float* mn = qn + Q;
    KnnArgs a{};
    a.row_norm = qn;
    a.col_norm = mn;
    a.R = Q;
    a.C = M;
    a.kchunks = ceil_div(D, kBK);
    a.col_tiles = (int)ceil_div<int64_t>(M, kBN);
    a.splits = knn_splits(Q, M);
    a.radius = radius;
    a.flags = flags;
    IDE3D_CUDA(cudaMemsetAsync(flags, 0, (size_t)Q, st));
    if ((rc = launch_norms(probes, Q, D, qn, st)) != IDE3D_OK) return rc;
    if ((rc = launch_norms(manifold, M, D, mn, st)) != IDE3D_OK) return rc;
    return launch_tiles<1, true>(probes, Q, manifold, M, D, a, st);
}
