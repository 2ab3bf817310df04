// upfirdn2d for sm_90a: pad -> zero-upsample -> FIR -> decimate.
// Replaces upfirdn2d_kernel_small/_large (torch_utils/ops/upfirdn2d.cu:29-200) behind the field set of
// upfirdn2d_kernel_params (upfirdn2d.h:14-40).
//
//   y[oy,ox] = gain * sum_{ky,kx} F[ky,kx] * X[(oy*dy + ky - py0)/uy, (ox*dx + kx - px0)/ux]
//   over taps whose numerators are >= 0, divisible by the up factor and inside the image;
//   F = f flipped unless `flip` (true convolution by default).
//
// HBM roofline: (numel_in + numel_out) * sizeof(T).  Two kernels:
//   * patch kernel (W-contiguous tensors, the StyleGAN2/3 filter shapes): a 64x64 output tile per block,
//     input tile staged once in shared memory (out-of-image = 0), each thread produces a 4x4 output patch
//     from a register window.  Polyphase structure is resolved at COMPILE time: the phase of the
//     padding (pad mod up) is a template parameter, so every tap -> window index is a constant and there
//     are no divisions, no bounds checks and no wasted zero taps in the inner loop.
//   * generic kernel: any strides (channels_last included), any filter, one thread per output.
#include <cuda.h>
#include <stdlib.h>

#include "common.cuh"

namespace ide3d {

struct UpfirArgs {
    const void* x;
    const float* f;
    void* y;
    int ux, uy, dx, dy, px0, py0, flip;
    float gain;
    int in_w, in_h, in_c, in_n;
    long long isw, ish, isc, isn;
    int fw, fh;
    long long fsw, fsh;
    int out_w, out_h;
    long long osw, osh, osc, osn;
    // ide3d_upfirdn2d_add only (channels_last patch kernel): y = upfirdn2d(x) + add + bias[c]; add has stride_c == 1
    const void* add = nullptr;
    long long asw = 0, ash = 0, asn = 0;
    const void* bias = nullptr;
    // ide3d_upfirdn2d_epilogue only (channels_last patch kernel): the modulated-convolution tail applied to the FIR output
    //   v = act(fir * scale[n,c] + noise[(n),oy,ox] + bias[c]) * gain, clamped;  y = v (if y != NULL);  y2 = v * scale2[n,c]
    int epi = 0, act = 1, noise_batch = 1;
    float alpha = 0.f, act_gain = 1.f, clamp = -1.f;
    const void *scale = nullptr, *noise = nullptr, *scale2 = nullptr;
    void* y2 = nullptr;
};

template <typename T> struct AccT { using type = float; };
template <> struct AccT<double> { using type = double; };
template <typename T> __device__ __forceinline__ typename AccT<T>::type ld(const T* p) { return (typename AccT<T>::type)(*p); }
template <> __device__ __forceinline__ float ld<__half>(const __half* p) { return __half2float(*p); }
template <typename T> __device__ __forceinline__ void st(T* p, typename AccT<T>::type v) { *p = (T)v; }
template <> __device__ __forceinline__ void st<__half>(__half* p, float v) { *p = __float2half(v); }

// ------------------------------------------------------------------------------------------
// compile-time polyphase bookkeeping for one axis: U = up, D = down, F = taps, PH = pad0 mod U
constexpr int cmod(int a, int m) { return ((a % m) + m) % m; }
constexpr int cfloor(int a, int m) { return (a - cmod(a, m)) / m; }
constexpr int kPatch = 4;                                   // outputs per thread per axis
constexpr int kTile = 64;                                   // outputs per block per axis

template <int U, int D, int F, int PH>
struct Axis {
    // output j of a patch whose origin is a multiple of kPatch
    static constexpr int k0(int j) { return cmod(PH - j * D, U); }                       // first live tap
    static constexpr int taps(int j) { return k0(j) < F ? (F - k0(j) + U - 1) / U : 0; }
    static constexpr int off(int j) { return cfloor(j * D - PH + k0(j), U); }            // input index of that tap (minus runtime base)
    static constexpr int lo() {
        int m = 1 << 20;
        for (int j = 0; j < kPatch; ++j) if (taps(j) > 0 && off(j) < m) m = off(j);
        return m == (1 << 20) ? 0 : m;
    }
    static constexpr int hi() {
        int m = -(1 << 20);
        for (int j = 0; j < kPatch; ++j) if (taps(j) > 0 && off(j) + taps(j) - 1 > m) m = off(j) + taps(j) - 1;
        return m == -(1 << 20) ? 0 : m;
    }
    static constexpr int kWin = hi() - lo() + 1;                                         // window length per patch
    static constexpr int kStep = kPatch * D / U;                                         // window advance per patch
    static constexpr int kTileIn = (kTile / kPatch - 1) * kStep + kWin;                  // staged inputs per tile
    static_assert((kPatch * D) % U == 0, "patch origin must stay phase aligned");
};

// 4x4 output patch of this thread from the staged input tile (row pitch PITCH), polyphase indices all compile-time
template <typename T, typename TT, int UX, int UY, int DX, int DY, int FW, int FH, int PHX, int PHY, int PITCH>
__device__ __forceinline__ void patch_compute_store_impl(const UpfirArgs& p, const TT* __restrict__ tile,
                                                         const typename AccT<T>::type (&fk)[FH][FW], int n, int c, int ox_t, int oy_t) {
    using S = typename AccT<T>::type;
    using AX = Axis<UX, DX, FW, PHX>;
    using AY = Axis<UY, DY, FH, PHY>;
    constexpr int TIWP = PITCH;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const TT* wbase = tile + (ty * AY::kStep) * TIWP + tx * AX::kStep;
    S acc[kPatch][kPatch];
#pragma unroll
    for (int i = 0; i < kPatch; ++i)
#pragma unroll
        for (int j = 0; j < kPatch; ++j) acc[i][j] = 0;

#pragma unroll
    for (int r = 0; r < AY::kWin; ++r) {
        S win[AX::kWin];
#pragma unroll
        for (int q = 0; q < AX::kWin; ++q) win[q] = ld<TT>(wbase + r * TIWP + q);
#pragma unroll
        for (int i = 0; i < kPatch; ++i) {
#pragma unroll
            for (int ty_ = 0; ty_ < AY::taps(i); ++ty_) {
                if (AY::off(i) - AY::lo() + ty_ != r) continue;              // folded at compile time
                const int ky = AY::k0(i) + ty_ * UY;
#pragma unroll
                for (int j = 0; j < kPatch; ++j)
#pragma unroll
                    for (int tx_ = 0; tx_ < AX::taps(j); ++tx_)
                        acc[i][j] += fk[ky][AX::k0(j) + tx_ * UX] * win[AX::off(j) - AX::lo() + tx_];
            }
        }
    }

    const int ox0 = ox_t + tx * kPatch, oy0 = oy_t + ty * kPatch;
    T* yout = (T*)p.y + n * p.osn + c * p.osc;
#pragma unroll
    for (int i = 0; i < kPatch; ++i) {
        const int oy = oy0 + i;
        if (oy >= p.out_h) break;
        T* rowp = yout + oy * p.osh + ox0;
        if (sizeof(T) == 4 && ox0 + kPatch <= p.out_w && ((reinterpret_cast<uintptr_t>(rowp) & 15) == 0)) {
            __stcs(reinterpret_cast<float4*>(rowp), make_float4((float)acc[i][0], (float)acc[i][1], (float)acc[i][2], (float)acc[i][3]));
        } else {
#pragma unroll
            for (int j = 0; j < kPatch; ++j)
                if (ox0 + j < p.out_w) st<T>(rowp + j, acc[i][j]);
        }
    }
}

template <typename T, int UX, int UY, int DX, int DY, int FW, int FH, int PHX, int PHY, int PITCH>
__device__ __forceinline__ void patch_compute_store(const UpfirArgs& p, const typename AccT<T>::type* __restrict__ tile,
                                                    const typename AccT<T>::type (&fk)[FH][FW], int n, int c, int ox_t, int oy_t) {
    patch_compute_store_impl<T, typename AccT<T>::type, UX, UY, DX, DY, FW, FH, PHX, PHY, PITCH>(p, tile, fk, n, c, ox_t, oy_t);
}
template <int UX, int UY, int DX, int DY, int FW, int FH, int PHX, int PHY, int PITCH>
__device__ __forceinline__ void patch_compute_store_h(const UpfirArgs& p, const __half* __restrict__ tile, const float (&fk)[FH][FW],
                                                      int n, int c, int ox_t, int oy_t) {
    patch_compute_store_impl<__half, __half, UX, UY, DX, DY, FW, FH, PHX, PHY, PITCH>(p, tile, fk, n, c, ox_t, oy_t);
}

// kVec (fp32, 16-byte aligned rows, W % 4 == 0): the tile is staged with LDG.128 from the 4-aligned column at or before
// the tile origin; the 0..3 surplus columns are absorbed by the row pitch and the window base is shifted accordingly.
template <typename T, int UX, int UY, int DX, int DY, int FW, int FH, int PHX, int PHY, bool kVec>
__global__ void __launch_bounds__(256) upfirdn2d_patch_kernel(const UpfirArgs p, int tiles_x, int tiles_y) {
    using S = typename AccT<T>::type;
    using AX = Axis<UX, DX, FW, PHX>;
    using AY = Axis<UY, DY, FH, PHY>;
    constexpr int TIW = AX::kTileIn, TIH = AY::kTileIn;
    constexpr int TIWP = (kVec ? ((TIW + 3 + 3) / 4 * 4) : TIW) | 1;   // odd row pitch: spreads rows over banks
    constexpr int TIV = (TIW + 3 + 3) / 4;                   // float4 per staged row in the vector path
    extern __shared__ __align__(16) unsigned char smem_raw[];
    S* tile = reinterpret_cast<S*>(smem_raw);

    // filter taps to registers, flipped here once
    S fk[FH][FW];
#pragma unroll
    for (int ky = 0; ky < FH; ++ky)
#pragma unroll
        for (int kx = 0; kx < FW; ++kx) {
            const int sy = p.flip ? ky : FH - 1 - ky, sx = p.flip ? kx : FW - 1 - kx;
            fk[ky][kx] = (S)p.f[sy * p.fsh + sx * p.fsw] * (S)p.gain;
        }

    const int ax = floor_div(p.px0, UX), ay = floor_div(p.py0, UY);      // pad = U*a + PH
    const long long tiles_plane = (long long)tiles_x * tiles_y;
    const long long total = tiles_plane * p.in_c * p.in_n;

    for (long long blk = blockIdx.x; blk < total; blk += gridDim.x) {
        const long long plane = blk / tiles_plane;
        const int t = (int)(blk - plane * tiles_plane);
        const int n = (int)(plane / p.in_c), c = (int)(plane - (long long)n * p.in_c);
        const int ox_t = (t % tiles_x) * kTile, oy_t = (t / tiles_x) * kTile;
        const int ix_t = ox_t * DX / UX - ax + AX::lo();
        const int iy_t = oy_t * DY / UY - ay + AY::lo();
        const T* xin = (const T*)p.x + n * p.isn + c * p.isc;

        __syncthreads();                                      // previous tile fully consumed
        int shift = 0;
        if constexpr (kVec) {
            const int ixa = ix_t & ~3;                        // 4-aligned column at or left of the tile origin (also for negatives)
            shift = ix_t - ixa;
            for (int i = threadIdx.x; i < TIV * TIH; i += 256) {
                const int ty = i / TIV, tv = i - ty * TIV;
                const int gx = ixa + tv * 4, gy = iy_t + ty;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if ((unsigned)gx < (unsigned)p.in_w && (unsigned)gy < (unsigned)p.in_h)    // W % 4 == 0: a vector is all in or all out
                    v = __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(xin) + gy * p.ish + gx));
                S* d = tile + ty * TIWP + tv * 4;
                d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
            }
        } else {
            for (int i = threadIdx.x; i < TIW * TIH; i += 256) {
                const int ty = i / TIW, tx = i - ty * TIW;
                const int gx = ix_t + tx, gy = iy_t + ty;
                S v = 0;
                if ((unsigned)gx < (unsigned)p.in_w && (unsigned)gy < (unsigned)p.in_h) v = ld<T>(xin + gy * p.ish + gx);
                tile[ty * TIWP + tx] = v;
            }
        }
        __syncthreads();

        patch_compute_store<T, UX, UY, DX, DY, FW, FH, PHX, PHY, TIWP>(p, tile + shift, fk, n, c, ox_t, oy_t);
    }
}

// ------------------------------------------------------------------------------------------
// TMA-staged flavour of the patch kernel (fp32 / fp16, dense NCHW): the input tile is fetched by ONE
// cp.async.bulk.tensor (3-D map: W x H x planes, box = tile), out-of-image elements are zero-filled by the TMA unit
// (negative / overflowing coordinates included), two tiles are in flight per block (double buffer + mbarrier) so the
// load of tile i+1 overlaps the FIR of tile i, and no thread spends instructions on staging.
__device__ __forceinline__ unsigned smem_addr(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void tma_bar_init(unsigned long long* bar) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_addr(bar)) : "memory");
}
__device__ __forceinline__ void tma_load_tile(void* dst, const CUtensorMap* map, unsigned long long* bar, int x, int y, int z, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 ::"r"(smem_addr(dst)), "l"(map), "r"(smem_addr(bar)), "r"(x), "r"(y), "r"(z) : "memory");
}
__device__ __forceinline__ void tma_bar_wait(unsigned long long* bar, unsigned parity) {
    unsigned ok = 0;
    while (!ok) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
                     : "=r"(ok) : "r"(smem_addr(bar)), "r"(parity) : "memory");
    }
}

template <typename T, int UX, int UY, int DX, int DY, int FW, int FH, int PHX, int PHY>
struct TmaGeom {
    using AX = Axis<UX, DX, FW, PHX>;
    using AY = Axis<UY, DY, FH, PHY>;
    // The innermost box coordinate has to sit on a 16-byte boundary: UTMALDG raises "illegal instruction" for x = -1 or 31
    // (fp32) while x = 0 or 64 work.  The box therefore starts at the
    // 16-byte aligned column at or left of the tile origin and is up to kVec-1 columns wider; the window base is shifted.
    static constexpr int kVec = 16 / (int)sizeof(T);
    static constexpr int BW = (AX::kTileIn + kVec - 1 + kVec - 1) / kVec * kVec, BH = AY::kTileIn;
    static constexpr int kTileBytes = ((BW * BH * (int)sizeof(T) + 127) / 128) * 128;
    static constexpr int kSmem = 2 * kTileBytes + 128 + 128;                           // 2 tiles + barriers + alignment slack
};

template <typename T, int UX, int UY, int DX, int DY, int FW, int FH, int PHX, int PHY>
__global__ void __launch_bounds__(256) upfirdn2d_patch_tma_kernel(const UpfirArgs p, int tiles_x, int tiles_y,
                                                                  const __grid_constant__ CUtensorMap tmap) {
    using GM = TmaGeom<T, UX, UY, DX, DY, FW, FH, PHX, PHY>;
    using AX = typename GM::AX;
    using AY = typename GM::AY;
    static_assert(sizeof(T) == sizeof(typename AccT<T>::type) || sizeof(T) == 2, "fp32 / fp16 only");
    static_assert((kTile * DX / UX) % GM::kVec == 0, "tile origins must keep the 16-byte phase of the box origin");
    extern __shared__ unsigned char tma_raw[];
    unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(tma_raw) + 127) & ~(uintptr_t)127);
    T* tiles[2] = {reinterpret_cast<T*>(base), reinterpret_cast<T*>(base + GM::kTileBytes)};
    unsigned long long* bars = reinterpret_cast<unsigned long long*>(base + 2 * GM::kTileBytes);

    float fk[FH][FW];
#pragma unroll
    for (int ky = 0; ky < FH; ++ky)
#pragma unroll
        for (int kx = 0; kx < FW; ++kx) {
            const int sy = p.flip ? ky : FH - 1 - ky, sx = p.flip ? kx : FW - 1 - kx;
            fk[ky][kx] = p.f[sy * p.fsh + sx * p.fsw] * p.gain;
        }
    const int ax = floor_div(p.px0, UX), ay = floor_div(p.py0, UY);
    const long long tiles_plane = (long long)tiles_x * tiles_y;
    const long long total = tiles_plane * p.in_c * p.in_n;
    constexpr unsigned kBytes = GM::BW * GM::BH * sizeof(T);

    auto coords = [&](long long blk, int& plane, int& ox_t, int& oy_t) {
        const long long pl = blk / tiles_plane;
        const int t = (int)(blk - pl * tiles_plane);
        plane = (int)pl;
        ox_t = (t % tiles_x) * kTile; oy_t = (t / tiles_x) * kTile;
    };
    // tile origins advance by kTile*DX/UX columns (a multiple of 16), so the distance to the aligned box origin is one constant
    const int shift = (-ax + AX::lo()) & (GM::kVec - 1);
    auto issue = [&](long long blk, int buf) {
        int pl, ox_t, oy_t;
        coords(blk, pl, ox_t, oy_t);
        tma_load_tile(tiles[buf], &tmap, &bars[buf], ox_t * DX / UX - ax + AX::lo() - shift, oy_t * DY / UY - ay + AY::lo(), pl, kBytes);
    };
    if (threadIdx.x == 0) {
        tma_bar_init(&bars[0]); tma_bar_init(&bars[1]);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        if ((long long)blockIdx.x < total) issue(blockIdx.x, 0);
    }
    __syncthreads();

    int it = 0;
    for (long long blk = blockIdx.x; blk < total; blk += gridDim.x, ++it) {
        const int cur = it & 1;
        const long long nxt = blk + gridDim.x;
        if (threadIdx.x == 0 && nxt < total) issue(nxt, cur ^ 1);   // buffer cur^1 was released by the __syncthreads ending the previous iteration
        int plane, ox_t, oy_t;
        coords(blk, plane, ox_t, oy_t);
        const int n = plane / p.in_c, c = plane - n * p.in_c;
        tma_bar_wait(&bars[cur], (it >> 1) & 1);
        if constexpr (sizeof(T) == 4) {
            patch_compute_store<T, UX, UY, DX, DY, FW, FH, PHX, PHY, GM::BW>(p, reinterpret_cast<const float*>(tiles[cur]) + shift, fk, n, c, ox_t, oy_t);
        } else {
            // fp16: widen the staged tile in place is not possible (same buffer); convert through registers in the window loads
            patch_compute_store_h<UX, UY, DX, DY, FW, FH, PHX, PHY, GM::BW>(p, reinterpret_cast<const __half*>(tiles[cur]) + shift, fk, n, c, ox_t, oy_t);
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------
// generic: any strides / filter / factors.  Thread order follows the fastest-varying output stride.
template <typename T>
__global__ void __launch_bounds__(256) upfirdn2d_generic_kernel(const UpfirArgs p, int c_fastest) {
    using S = typename AccT<T>::type;
    const long long total = (long long)p.out_w * p.out_h * p.in_c * p.in_n;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        int ox, oy, c, n;
        long long r = i;
        if (c_fastest) { c = (int)(r % p.in_c); r /= p.in_c; ox = (int)(r % p.out_w); r /= p.out_w; oy = (int)(r % p.out_h); n = (int)(r / p.out_h); }
        else { ox = (int)(r % p.out_w); r /= p.out_w; oy = (int)(r % p.out_h); r /= p.out_h; c = (int)(r % p.in_c); n = (int)(r / p.in_c); }
        const int bx = ox * p.dx - p.px0, by = oy * p.dy - p.py0;
        const int kx0 = ((-bx) % p.ux + p.ux) % p.ux, ky0 = ((-by) % p.uy + p.uy) % p.uy;
        const T* xin = (const T*)p.x + n * p.isn + c * p.isc;
        S acc = 0;
        for (int ky = ky0; ky < p.fh; ky += p.uy) {
            const int iy = (by + ky) / p.uy;                    // exact
            if (iy < 0 || by + ky < 0) continue;
            if (iy >= p.in_h) break;
            const int sy = p.flip ? ky : p.fh - 1 - ky;
            for (int kx = kx0; kx < p.fw; kx += p.ux) {
                const int ix = (bx + kx) / p.ux;
                if (ix < 0 || bx + kx < 0) continue;
                if (ix >= p.in_w) break;
                const int sx = p.flip ? kx : p.fw - 1 - kx;
                acc += (S)p.f[sy * p.fsh + sx * p.fsw] * ld<T>(xin + iy * p.ish + ix * p.isw);
            }
        }
        st<T>((T*)p.y + n * p.osn + c * p.osc + oy * p.osh + ox * p.osw, acc * (S)p.gain);
    }
}

// ---- host side of the TMA path -----------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled() {
    static EncodeTiledFn fn = []() -> EncodeTiledFn {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qr) != cudaSuccess || qr != cudaDriverEntryPointSuccess) return nullptr;
        return (EncodeTiledFn)ptr;
    }();
    return fn;
}

// can the TMA unit describe this input?  dense NCHW (planes equally spaced), 16-byte aligned base and row pitch
template <typename T>
static bool tma_eligible(const UpfirArgs& p) {
    if (sizeof(T) > 4 || encode_tiled() == nullptr) return false;
    if (p.isw != 1 || p.osw != 1) return false;
    if (p.isn != p.isc * p.in_c) return false;                           // (n, c) must collapse into one plane index
    if ((reinterpret_cast<uintptr_t>(p.x) & 15) || (p.ish * sizeof(T)) % 16 || (p.isc * sizeof(T)) % 16) return false;
    if ((long long)p.in_c * p.in_n > 0x7fffffffll) return false;
    return true;
}

template <typename T, int UX, int UY, int DX, int DY, int FW, int FH, int PHX, int PHY>
static int launch_patch_tma(const UpfirArgs& p, cudaStream_t st_) {
    using GM = TmaGeom<T, UX, UY, DX, DY, FW, FH, PHX, PHY>;
    CUtensorMap map;
    const cuuint64_t dims[3] = {(cuuint64_t)p.in_w, (cuuint64_t)p.in_h, (cuuint64_t)p.in_c * p.in_n};
    const cuuint64_t strides[2] = {(cuuint64_t)p.ish * sizeof(T), (cuuint64_t)p.isc * sizeof(T)};
    const cuuint32_t box[3] = {(cuuint32_t)GM::BW, (cuuint32_t)GM::BH, 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    const CUresult r = encode_tiled()(&map, sizeof(T) == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3,
                                      const_cast<void*>(p.x), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                      CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) IDE3D_FAIL(IDE3D_UNSUPPORTED, "upfirdn2d: cuTensorMapEncodeTiled failed (%d)", (int)r);
    auto kern = upfirdn2d_patch_tma_kernel<T, UX, UY, DX, DY, FW, FH, PHX, PHY>;
    const size_t smem = GM::kSmem;
    if (smem > 48 * 1024) IDE3D_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int tiles_x = ceil_div(p.out_w, kTile), tiles_y = ceil_div(p.out_h, kTile);
    const long long total = (long long)tiles_x * tiles_y * p.in_c * p.in_n;
    int per_sm = 1;
    IDE3D_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 256, smem));
    if (per_sm < 1) per_sm = 1;
    long long grid = (long long)sm_count() * per_sm;
    if (grid > total) grid = total;
    kern<<<(unsigned)grid, 256, smem, st_>>>(p, tiles_x, tiles_y, map);
    IDE3D_CHECK_LAUNCH("upfirdn2d_patch_tma_kernel");
    return IDE3D_OK;
}

template <typename T, int UX, int UY, int DX, int DY, int FW, int FH, int PHX, int PHY>
static int launch_patch(const UpfirArgs& p, cudaStream_t st_) {
    if constexpr (sizeof(T) <= 4) {
        // One bulk-tensor copy per tile, double-buffered: both tiles have to fit the 227 KB of one SM.  IDE3D_TMA=0 selects
        // the thread-staged kernel below (kept for tensors the TMA unit cannot describe: unaligned base / row pitch).
        constexpr bool fits = TmaGeom<T, UX, UY, DX, DY, FW, FH, PHX, PHY>::kSmem <= 200 * 1024;
        const char* tma_env = tuning_env("IDE3D_TMA");
        if (fits && !(tma_env != nullptr && tma_env[0] == '0') && tma_eligible<T>(p)) {
            const int rc = launch_patch_tma<T, UX, UY, DX, DY, FW, FH, PHX, PHY>(p, st_);
            if (rc != IDE3D_UNSUPPORTED) return rc;
        }
    }
    using S = typename AccT<T>::type;
    using AX = Axis<UX, DX, FW, PHX>;
    using AY = Axis<UY, DY, FH, PHY>;
    bool vec = false;
    if constexpr (sizeof(T) == 4)
        vec = (p.in_w % 4 == 0) && (p.ish % 4 == 0) && (p.isc % 4 == 0) && (p.isn % 4 == 0) && ((reinterpret_cast<uintptr_t>(p.x) & 15) == 0);
    const int pitch = (vec ? ((AX::kTileIn + 6) / 4 * 4) : AX::kTileIn) | 1;
    const size_t smem = (size_t)pitch * AY::kTileIn * sizeof(S) + 16;
    void (*kern)(const UpfirArgs, int, int) = upfirdn2d_patch_kernel<T, UX, UY, DX, DY, FW, FH, PHX, PHY, false>;
    if constexpr (sizeof(T) == 4) { if (vec) kern = upfirdn2d_patch_kernel<T, UX, UY, DX, DY, FW, FH, PHX, PHY, true>; }
    if (smem > 48 * 1024) IDE3D_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int tiles_x = ceil_div(p.out_w, kTile), tiles_y = ceil_div(p.out_h, kTile);
    const long long total = (long long)tiles_x * tiles_y * p.in_c * p.in_n;
    int per_sm = 1;
    IDE3D_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 256, smem));
    if (per_sm < 1) per_sm = 1;
    long long grid = (long long)sm_count() * per_sm;
    if (grid > total) grid = total;
    kern<<<(unsigned)grid, 256, smem, st_>>>(p, tiles_x, tiles_y);
    IDE3D_CHECK_LAUNCH("upfirdn2d_patch_kernel");
    return IDE3D_OK;
}

// phase dispatch: PHX in [0,UX), PHY in [0,UY)
template <typename T, int UX, int UY, int DX, int DY, int FW, int FH>
static int dispatch_phase(const UpfirArgs& p, cudaStream_t s) {
    const int phx = p.px0 - floor_div(p.px0, UX) * UX, phy = p.py0 - floor_div(p.py0, UY) * UY;
    if constexpr (UX == 1 && UY == 1) return launch_patch<T, UX, UY, DX, DY, FW, FH, 0, 0>(p, s);
    if constexpr (UX == 2 && UY == 1) return phx ? launch_patch<T, UX, UY, DX, DY, FW, FH, 1, 0>(p, s) : launch_patch<T, UX, UY, DX, DY, FW, FH, 0, 0>(p, s);
    if constexpr (UX == 1 && UY == 2) return phy ? launch_patch<T, UX, UY, DX, DY, FW, FH, 0, 1>(p, s) : launch_patch<T, UX, UY, DX, DY, FW, FH, 0, 0>(p, s);
    if constexpr (UX == 2 && UY == 2) {
        if (phx == 0 && phy == 0) return launch_patch<T, 2, 2, DX, DY, FW, FH, 0, 0>(p, s);
        if (phx == 1 && phy == 0) return launch_patch<T, 2, 2, DX, DY, FW, FH, 1, 0>(p, s);
        if (phx == 0 && phy == 1) return launch_patch<T, 2, 2, DX, DY, FW, FH, 0, 1>(p, s);
        return launch_patch<T, 2, 2, DX, DY, FW, FH, 1, 1>(p, s);
    }
    IDE3D_FAIL(IDE3D_UNSUPPORTED, "upfirdn2d: no phase table");
}

// ------------------------------------------------------------------------------------------
// channels_last patch kernel (stride_c == 1, C % 4 == 0) for the StyleGAN2 4x4 filter shapes: a thread owns a 4x4 output
// patch x 4 consecutive channels.  Same compile-time polyphase tables as the planar patch kernel; the input window
// (kWin x kWin pixels, e.g. 7x7 for the up=1 FIR, 3x3 for 2x upsampling) is read with one vector load per pixel straight
// from L1/L2 -- consecutive threads take consecutive channel vectors of the same patch, so every load and store of a warp
// is one contiguous run along C.  No shared memory, no divisions / bounds checks per tap.
template <typename T> struct V4;
template <> struct V4<float> {
    static __device__ __forceinline__ void ld(const float* p, float (&o)[4]) { const float4 t = __ldg(reinterpret_cast<const float4*>(p)); o[0] = t.x; o[1] = t.y; o[2] = t.z; o[3] = t.w; }
    static __device__ __forceinline__ void st(float* p, const float (&o)[4]) { __stcs(reinterpret_cast<float4*>(p), make_float4(o[0], o[1], o[2], o[3])); }
};
template <> struct V4<__half> {
    static __device__ __forceinline__ void ld(const __half* p, float (&o)[4]) {
        const uint2 t = __ldg(reinterpret_cast<const uint2*>(p));
        const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&t.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&t.y));
        o[0] = a.x; o[1] = a.y; o[2] = b.x; o[3] = b.y;
    }
    static __device__ __forceinline__ void st(__half* p, const float (&o)[4]) {
        const __half2 a = __floats2half2_rn(o[0], o[1]), b = __floats2half2_rn(o[2], o[3]);
        __stcs(reinterpret_cast<uint2*>(p), make_uint2(*reinterpret_cast<const unsigned*>(&a), *reinterpret_cast<const unsigned*>(&b)));
    }
};

// One 4x4 output patch x 4 channels: accumulate from a window supplied by `load(r, q, out[4])` (global memory with bounds
// checks, or a TMA-staged shared-memory tile), then the optional skip-add / modconv tail, then the stores.
template <typename T, int UX, int UY, int DX, int DY, int FW, int FH, int PHX, int PHY, bool kEpi, typename LoadFn>
__device__ __forceinline__ void cl_patch_body(const UpfirArgs& p, const float (&fk)[FH][FW], int n, int cv, int ox0, int oy0, LoadFn load) {
    using AX = Axis<UX, DX, FW, PHX>;
    using AY = Axis<UY, DY, FH, PHY>;
    float acc[kPatch][kPatch][4];
#pragma unroll
    for (int a = 0; a < kPatch; ++a)
#pragma unroll
        for (int b = 0; b < kPatch; ++b)
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[a][b][c] = 0.f;
    if (p.add != nullptr) {
        // skip-connection form (upsample2d(img) + y + b): the accumulators START from the new contribution, so its 16 loads are in
        // flight together with the window loads instead of after the FIR (the kernel is latency bound) -- same registers, twice the
        // loads in flight
        const T* ain = (const T*)p.add + n * p.asn + cv * 4;
        float bv[4] = {0.f, 0.f, 0.f, 0.f};
        if (p.bias != nullptr) V4<T>::ld((const T*)p.bias + cv * 4, bv);
#pragma unroll
        for (int a = 0; a < kPatch; ++a) {
#pragma unroll
            for (int b = 0; b < kPatch; ++b)
                if (oy0 + a < p.out_h && ox0 + b < p.out_w) {
                    float av[4];
                    V4<T>::ld(ain + (oy0 + a) * p.ash + (ox0 + b) * p.asw, av);
#pragma unroll
                    for (int c = 0; c < 4; ++c) acc[a][b][c] = av[c] + bv[c];
                }
        }
    }

#pragma unroll
    for (int r = 0; r < AY::kWin; ++r) {
        float win[AX::kWin][4];
#pragma unroll
        for (int q = 0; q < AX::kWin; ++q) load(r, q, win[q]);
#pragma unroll
        for (int a = 0; a < kPatch; ++a) {
#pragma unroll
            for (int ty_ = 0; ty_ < AY::taps(a); ++ty_) {
                if (AY::off(a) - AY::lo() + ty_ != r) continue;              // folded at compile time
                const int ky = AY::k0(a) + ty_ * UY;
#pragma unroll
                for (int b = 0; b < kPatch; ++b)
#pragma unroll
                    for (int tx_ = 0; tx_ < AX::taps(b); ++tx_) {
                        const float w = fk[ky][AX::k0(b) + tx_ * UX];
#pragma unroll
                        for (int c = 0; c < 4; ++c) acc[a][b][c] = fmaf(w, win[AX::off(b) - AX::lo() + tx_][c], acc[a][b][c]);
                    }
            }
        }
    }
    T* yout = (T*)p.y + n * p.osn + cv * 4;
    if constexpr (kEpi) {
        float dv[4] = {1.f, 1.f, 1.f, 1.f}, bv[4] = {0.f, 0.f, 0.f, 0.f}, d2[4] = {1.f, 1.f, 1.f, 1.f};
        if (p.scale != nullptr) V4<T>::ld((const T*)p.scale + (long long)n * p.in_c + cv * 4, dv);
        if (p.bias != nullptr) V4<T>::ld((const T*)p.bias + cv * 4, bv);
        if (p.y2 != nullptr) V4<T>::ld((const T*)p.scale2 + (long long)n * p.in_c + cv * 4, d2);
        const T* nz = (p.noise != nullptr) ? (const T*)p.noise + (p.noise_batch == 1 ? 0ll : (long long)n * p.out_h * p.out_w) : nullptr;
        T* y2out = (p.y2 != nullptr) ? (T*)p.y2 + n * p.osn + cv * 4 : nullptr;
#pragma unroll
        for (int a = 0; a < kPatch; ++a) {
            if (oy0 + a >= p.out_h) break;
#pragma unroll
            for (int b = 0; b < kPatch; ++b) {
                if (ox0 + b >= p.out_w) continue;
                const float nv = nz ? ld<T>(nz + (long long)(oy0 + a) * p.out_w + (ox0 + b)) : 0.f;
                float v[4];
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    float t = nz ? fmaf(acc[a][b][c], dv[c], nv) : acc[a][b][c] * dv[c];
                    t += bv[c];
                    if (p.act == 3) t = (t > 0.f) ? t : t * p.alpha;
                    t *= p.act_gain;
                    if (p.clamp >= 0.f) t = fminf(fmaxf(t, -p.clamp), p.clamp);
                    v[c] = t;
                }
                const long long o = (long long)(oy0 + a) * p.osh + (long long)(ox0 + b) * p.osw;
                if (p.y != nullptr) V4<T>::st(yout + o, v);
                if (y2out != nullptr) {
#pragma unroll
                    for (int c = 0; c < 4; ++c) v[c] *= d2[c];
                    V4<T>::st(y2out + o, v);
                }
            }
        }
    } else {
#pragma unroll
        for (int a = 0; a < kPatch; ++a) {
            if (oy0 + a >= p.out_h) break;
#pragma unroll
            for (int b = 0; b < kPatch; ++b)
                if (ox0 + b < p.out_w) V4<T>::st(yout + (oy0 + a) * p.osh + (ox0 + b) * p.osw, acc[a][b]);
        }
    }
}

template <int FW, int FH>
__device__ __forceinline__ void load_filter(const UpfirArgs& p, float (&fk)[FH][FW]) {
#pragma unroll
    for (int ky = 0; ky < FH; ++ky)
#pragma unroll
        for (int kx = 0; kx < FW; ++kx) {
            const int sy = p.flip ? ky : FH - 1 - ky, sx = p.flip ? kx : FW - 1 - kx;
            fk[ky][kx] = p.f[sy * p.fsh + sx * p.fsw] * p.gain;
        }
}

template <typename T, int UX, int UY, int DX, int DY, int FW, int FH, int PHX, int PHY, bool kEpi>
__global__ void __launch_bounds__(256) upfirdn2d_cl_patch_kernel(const UpfirArgs p, int patches_x, int patches_y) {
    using AX = Axis<UX, DX, FW, PHX>;
    using AY = Axis<UY, DY, FH, PHY>;
    float fk[FH][FW];
    load_filter<FW, FH>(p, fk);
    const int ax = floor_div(p.px0, UX), ay = floor_div(p.py0, UY);
    const unsigned cvn = (unsigned)(p.in_c >> 2);
    const long long total = (long long)patches_x * patches_y * p.in_n * cvn;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        int cv, pxi, pyi, n;
        if (total <= 0xffffffffll) {                             // 32-bit index math (64-bit div/mod costs ~60 instructions each)
            const unsigned ii = (unsigned)i, r0 = ii / cvn, r1 = r0 / (unsigned)patches_x;
            cv = (int)(ii - r0 * cvn); pxi = (int)(r0 - r1 * (unsigned)patches_x);
            n = (int)(r1 / (unsigned)patches_y); pyi = (int)(r1 - (unsigned)n * (unsigned)patches_y);
        } else {
            const long long r0 = i / cvn, r1 = r0 / patches_x;
            cv = (int)(i - r0 * cvn); pxi = (int)(r0 % patches_x);
            pyi = (int)(r1 % patches_y); n = (int)(r1 / patches_y);
        }
        const int ox0 = pxi * kPatch, oy0 = pyi * kPatch;
        const int ix0 = ox0 * DX / UX - ax + AX::lo(), iy0 = oy0 * DY / UY - ay + AY::lo();
        const T* xin = (const T*)p.x + (long long)n * p.isn + cv * 4;
        cl_patch_body<T, UX, UY, DX, DY, FW, FH, PHX, PHY, kEpi>(p, fk, n, cv, ox0, oy0, [&](int r, int q, float (&w)[4]) {
            const int gy = iy0 + r, gx = ix0 + q;
            if ((unsigned)gy < (unsigned)p.in_h && (unsigned)gx < (unsigned)p.in_w) V4<T>::ld(xin + gy * p.ish + gx * p.isw, w);
            else { w[0] = 0.f; w[1] = 0.f; w[2] = 0.f; w[3] = 0.f; }
        });
    }
}

// TMA-staged channels_last flavour (C % 32 == 0): a block owns a 32 x 16 pixel output tile x 32 channels; the input box
// (channels x columns x rows of a 4-D tensor map, zero-filled outside the image by the TMA unit) arrives with ONE
// cp.async.bulk.tensor.4d per tile, double-buffered against the FIR of the previous tile.  Shared-memory pixels are 128-byte
// (fp32) runs of 32 channels, so the 8 lanes that share a patch read one contiguous line per window element.
// Tile shapes: CB channels x (PX x PY patches of 4 x 4 pixels), CB/4 * PX * PY = 256 threads.  The TMA unit is fed one
// innermost run (CB channels) per request, so wider channel blocks move more bytes per request: 64 channels x 16x16 pixels
// when C % 64 == 0, else 32 channels x 32x16 pixels.
template <typename T, int UX, int UY, int DX, int DY, int FW, int FH, int PHX, int PHY, int CB>
struct ClTmaGeom {
    using AX = Axis<UX, DX, FW, PHX>;
    using AY = Axis<UY, DY, FH, PHY>;
    static constexpr int kCB = CB, kCV = CB / 4;
    static constexpr int PX = (CB == 32) ? 8 : 4, PY = 256 / (kCV * PX);
    static constexpr int kTileW = PX * kPatch, kTileH = PY * kPatch;
    static constexpr int BW = (PX - 1) * AX::kStep + AX::kWin;
    static constexpr int BH = (PY - 1) * AY::kStep + AY::kWin;
    static constexpr int kTileBytes = ((BW * BH * CB * (int)sizeof(T) + 127) / 128) * 128;
    // Two blocks per SM (16 warps) hide the FIR's issue latency better than one block with a deeper ring (measured: one
    // 8-warp block issues 42 % of its slots): small boxes are double-buffered inside the block, large ones (the 92 KB box of
    // the up=1 FIR) rely on the co-resident block to overlap their load.
    static constexpr int kStages = (2 * kTileBytes + 256 <= 110 * 1024) ? 2 : 1;
    static constexpr int kSmem = kStages * kTileBytes + 128 + 128;
    static_assert(kCV * PX * PY == 256, "one thread per (channel vector, patch)");
};
__device__ __forceinline__ void tma_load_tile4(void* dst, const CUtensorMap* map, unsigned long long* bar, int c, int x, int y, int n, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                 ::"r"(smem_addr(dst)), "l"(map), "r"(smem_addr(bar)), "r"(c), "r"(x), "r"(y), "r"(n) : "memory");
}
template <typename T> struct V4s;
template <> struct V4s<float> {
    static __device__ __forceinline__ void ld(const float* p, float (&o)[4]) { const float4 t = *reinterpret_cast<const float4*>(p); o[0] = t.x; o[1] = t.y; o[2] = t.z; o[3] = t.w; }
};
template <> struct V4s<__half> {
    static __device__ __forceinline__ void ld(const __half* p, float (&o)[4]) {
        const uint2 t = *reinterpret_cast<const uint2*>(p);
        const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&t.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&t.y));
        o[0] = a.x; o[1] = a.y; o[2] = b.x; o[3] = b.y;
    }
};

template <typename T, int UX, int UY, int DX, int DY, int FW, int FH, int PHX, int PHY, bool kEpi, int CB>
__global__ void __launch_bounds__(256, 2) upfirdn2d_cl_tma_kernel(const UpfirArgs p, int tiles_x, int tiles_y, int cblocks,
                                                               const __grid_constant__ CUtensorMap tmap) {
    using GM = ClTmaGeom<T, UX, UY, DX, DY, FW, FH, PHX, PHY, CB>;
    constexpr int kClCB = CB, kClTileW = GM::kTileW, kClTileH = GM::kTileH;
    using AX = typename GM::AX;
    using AY = typename GM::AY;
    extern __shared__ unsigned char tma_raw[];
    unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(tma_raw) + 127) & ~(uintptr_t)127);
    constexpr int NST = GM::kStages;
    unsigned long long* bars = reinterpret_cast<unsigned long long*>(base + NST * GM::kTileBytes);
    float fk[FH][FW];
    load_filter<FW, FH>(p, fk);
    const int ax = floor_div(p.px0, UX), ay = floor_div(p.py0, UY);
    const long long total = (long long)tiles_x * tiles_y * cblocks * p.in_n;
    constexpr unsigned kBytes = GM::BW * GM::BH * kClCB * sizeof(T);

    // tile index -> (n, channel block, tile y, tile x); x fastest so that concurrently resident blocks share halo rows in L2
    auto coords = [&](long long t, int& n, int& cb, int& ox_t, int& oy_t) {
        const int tx = (int)(t % tiles_x); t /= tiles_x;
        const int ty = (int)(t % tiles_y); t /= tiles_y;
        cb = (int)(t % cblocks); n = (int)(t / cblocks);
        ox_t = tx * kClTileW; oy_t = ty * kClTileH;
    };
    auto issue = [&](long long t, int buf) {
        int n, cb, ox_t, oy_t;
        coords(t, n, cb, ox_t, oy_t);
        tma_load_tile4(base + buf * GM::kTileBytes, &tmap, &bars[buf], cb * kClCB, ox_t * DX / UX - ax + AX::lo(),
                       oy_t * DY / UY - ay + AY::lo(), n, kBytes);
    };
    if (threadIdx.x == 0) {
        for (int i = 0; i < NST; ++i) tma_bar_init(&bars[i]);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        for (int i = 0; i < NST; ++i)
            if ((long long)blockIdx.x + (long long)i * gridDim.x < total) issue((long long)blockIdx.x + (long long)i * gridDim.x, i);
    }
    __syncthreads();

    const int cvl = threadIdx.x % GM::kCV, pl = threadIdx.x / GM::kCV;       // channel vector inside the block, patch inside the tile
    const int ptx = pl % GM::PX, pty = pl / GM::PX;
    int it = 0;
    for (long long t = blockIdx.x; t < total; t += gridDim.x, ++it) {
        const int cur = it % NST;
        int n, cb, ox_t, oy_t;
        coords(t, n, cb, ox_t, oy_t);
        tma_bar_wait(&bars[cur], (it / NST) & 1);
        const T* tile = reinterpret_cast<const T*>(base + cur * GM::kTileBytes) + ((pty * AY::kStep) * GM::BW + ptx * AX::kStep) * kClCB + cvl * 4;
        const int ox0 = ox_t + ptx * kPatch, oy0 = oy_t + pty * kPatch;
        if (ox0 < p.out_w && oy0 < p.out_h)
            cl_patch_body<T, UX, UY, DX, DY, FW, FH, PHX, PHY, kEpi>(p, fk, n, cb * (kClCB / 4) + cvl, ox0, oy0, [&](int r, int q, float (&w)[4]) {
                V4s<T>::ld(tile + (r * GM::BW + q) * kClCB, w);
            });
        __syncthreads();                                                     // every thread is done with stage `cur`
        const long long nxt = t + (long long)NST * gridDim.x;
        if (threadIdx.x == 0 && nxt < total) issue(nxt, cur);
    }
}

template <typename T, int UX, int UY, int DX, int DY, int FW, int FH, int PHX, int PHY, int CB>
static int launch_cl_tma(const UpfirArgs& p, cudaStream_t st_) {
    using GM = ClTmaGeom<T, UX, UY, DX, DY, FW, FH, PHX, PHY, CB>;
    constexpr int kClCB = CB, kClTileW = GM::kTileW, kClTileH = GM::kTileH;
    CUtensorMap map;
    const cuuint64_t dims[4] = {(cuuint64_t)p.in_c, (cuuint64_t)p.in_w, (cuuint64_t)p.in_h, (cuuint64_t)p.in_n};
    const cuuint64_t strides[3] = {(cuuint64_t)p.isw * sizeof(T), (cuuint64_t)p.ish * sizeof(T), (cuuint64_t)p.isn * sizeof(T)};
    const cuuint32_t box[4] = {(cuuint32_t)kClCB, (cuuint32_t)GM::BW, (cuuint32_t)GM::BH, 1};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    const CUresult r = encode_tiled()(&map, sizeof(T) == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4,
                                      const_cast<void*>(p.x), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                      CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) IDE3D_FAIL(IDE3D_UNSUPPORTED, "upfirdn2d: cuTensorMapEncodeTiled (channels_last) failed (%d)", (int)r);
    void (*kern)(const UpfirArgs, int, int, int, const CUtensorMap) = p.epi ? upfirdn2d_cl_tma_kernel<T, UX, UY, DX, DY, FW, FH, PHX, PHY, true, CB>
                                                                            : upfirdn2d_cl_tma_kernel<T, UX, UY, DX, DY, FW, FH, PHX, PHY, false, CB>;
    const size_t smem = GM::kSmem;
    if (smem > 48 * 1024) IDE3D_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int tiles_x = ceil_div(p.out_w, kClTileW), tiles_y = ceil_div(p.out_h, kClTileH), cblocks = p.in_c / kClCB;
    const long long total = (long long)tiles_x * tiles_y * cblocks * p.in_n;
    int per_sm = 1;
    IDE3D_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 256, smem));
    if (per_sm < 1) per_sm = 1;
    long long grid = (long long)sm_count() * per_sm;
    if (grid > total) grid = total;
    kern<<<(unsigned)grid, 256, smem, st_>>>(p, tiles_x, tiles_y, cblocks, map);
    IDE3D_CHECK_LAUNCH("upfirdn2d_cl_tma_kernel");
    return IDE3D_OK;
}

template <typename T, int UX, int UY, int DX, int DY, int FW, int FH, int PHX, int PHY>
static int launch_cl_patch(const UpfirArgs& p, cudaStream_t st_) {
    // TMA-staged tiles when the tensor map can describe the input (C % 32 == 0, 16-byte aligned base and pitches) and two
    // input boxes fit one SM; IDE3D_TMA=0 keeps the L1-gather kernel below.
    // Measured (scripts/bench_ops.py, [1,512,512,512] fp32): the up=1 FIR runs at 87 % of the HBM peak from TMA tiles (46 % from
    // the L1-gather kernel); 2x upsampling has only 2x2 live taps per output and is faster straight from L1 (85 % vs 80 %).
    if constexpr (UX == 1 && UY == 1 && ClTmaGeom<T, UX, UY, DX, DY, FW, FH, PHX, PHY, 32>::kSmem <= 200 * 1024) {
        const char* tma_env = tuning_env("IDE3D_TMA");
        const char* cb_env = tuning_env("IDE3D_CL_CB");                         // experiments: force the 32-channel tile shape
        const bool ok = !(tma_env != nullptr && tma_env[0] == '0') && encode_tiled() != nullptr && p.in_c % 32 == 0 &&
                        (reinterpret_cast<uintptr_t>(p.x) & 15) == 0 && (p.isw * sizeof(T)) % 16 == 0 && (p.ish * sizeof(T)) % 16 == 0 &&
                        (p.isn * sizeof(T)) % 16 == 0 && p.out_w * (long long)p.out_h >= 64;
        if (ok) {
            int rc = IDE3D_UNSUPPORTED;
            if constexpr (ClTmaGeom<T, UX, UY, DX, DY, FW, FH, PHX, PHY, 64>::kSmem <= 200 * 1024) {
                if (p.in_c % 64 == 0 && !(cb_env != nullptr && cb_env[0] == '3')) rc = launch_cl_tma<T, UX, UY, DX, DY, FW, FH, PHX, PHY, 64>(p, st_);
            }
            if (rc == IDE3D_UNSUPPORTED) rc = launch_cl_tma<T, UX, UY, DX, DY, FW, FH, PHX, PHY, 32>(p, st_);
            if (rc != IDE3D_UNSUPPORTED) return rc;
        }
    }
    const int patches_x = ceil_div(p.out_w, kPatch), patches_y = ceil_div(p.out_h, kPatch);
    const long long total = (long long)patches_x * patches_y * p.in_n * (p.in_c >> 2);
    long long grid = ceil_div<long long>(total, 256);
    const long long cap = (long long)sm_count() * 8;
    if (grid > cap) grid = cap;
    if (p.epi) upfirdn2d_cl_patch_kernel<T, UX, UY, DX, DY, FW, FH, PHX, PHY, true><<<(unsigned)grid, 256, 0, st_>>>(p, patches_x, patches_y);
    else upfirdn2d_cl_patch_kernel<T, UX, UY, DX, DY, FW, FH, PHX, PHY, false><<<(unsigned)grid, 256, 0, st_>>>(p, patches_x, patches_y);
    IDE3D_CHECK_LAUNCH("upfirdn2d_cl_patch_kernel");
    return IDE3D_OK;
}

template <typename T, int UX, int UY, int DX, int DY, int FW, int FH>
static int dispatch_phase_cl(const UpfirArgs& p, cudaStream_t s) {
    const int phx = p.px0 - floor_div(p.px0, UX) * UX, phy = p.py0 - floor_div(p.py0, UY) * UY;
    if constexpr (UX == 1 && UY == 1) return launch_cl_patch<T, UX, UY, DX, DY, FW, FH, 0, 0>(p, s);
    if constexpr (UX == 2 && UY == 2) {
        if (phx == 0 && phy == 0) return launch_cl_patch<T, 2, 2, DX, DY, FW, FH, 0, 0>(p, s);
        if (phx == 1 && phy == 0) return launch_cl_patch<T, 2, 2, DX, DY, FW, FH, 1, 0>(p, s);
        if (phx == 0 && phy == 1) return launch_cl_patch<T, 2, 2, DX, DY, FW, FH, 0, 1>(p, s);
        return launch_cl_patch<T, 2, 2, DX, DY, FW, FH, 1, 1>(p, s);
    }
    IDE3D_FAIL(IDE3D_UNSUPPORTED, "upfirdn2d: no channels_last phase table");
}

// ------------------------------------------------------------------------------------------
// channels_last fallback (stride_c == 1): a thread owns one output pixel x 4 consecutive channels (one 16-byte vector for
// fp32, 8 bytes for fp16), walks the live polyphase taps and reads the neighbouring input pixels straight from L1/L2
// (adjacent outputs share them).  Any filter / factors; coalesced along C.
template <typename T>
__global__ void __launch_bounds__(256) upfirdn2d_cl_kernel(const UpfirArgs p) {
    using S = typename AccT<T>::type;
    const int c4n = p.in_c >> 2;
    const long long total = (long long)p.out_w * p.out_h * p.in_n * c4n;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % c4n);
        long long r = i / c4n;
        const int ox = (int)(r % p.out_w); r /= p.out_w;
        const int oy = (int)(r % p.out_h);
        const int n = (int)(r / p.out_h);
        const int bx = ox * p.dx - p.px0, by = oy * p.dy - p.py0;
        const int kx0 = ((-bx) % p.ux + p.ux) % p.ux, ky0 = ((-by) % p.uy + p.uy) % p.uy;
        const T* xin = (const T*)p.x + n * p.isn + c4 * 4;
        S a0 = 0, a1 = 0, a2 = 0, a3 = 0;
        for (int ky = ky0; ky < p.fh; ky += p.uy) {
            if (by + ky < 0) continue;
            const int iy = (by + ky) / p.uy;
            if (iy >= p.in_h) break;
            const int sy = p.flip ? ky : p.fh - 1 - ky;
            for (int kx = kx0; kx < p.fw; kx += p.ux) {
                if (bx + kx < 0) continue;
                const int ix = (bx + kx) / p.ux;
                if (ix >= p.in_w) break;
                const S w = (S)p.f[sy * p.fsh + (p.flip ? kx : p.fw - 1 - kx) * p.fsw];
                const T* px = xin + iy * p.ish + ix * p.isw;
                a0 += w * ld<T>(px); a1 += w * ld<T>(px + 1); a2 += w * ld<T>(px + 2); a3 += w * ld<T>(px + 3);
            }
        }
        T* py = (T*)p.y + n * p.osn + oy * p.osh + ox * p.osw + c4 * 4;
        const S g = (S)p.gain;
        st<T>(py, a0 * g); st<T>(py + 1, a1 * g); st<T>(py + 2, a2 * g); st<T>(py + 3, a3 * g);
    }
}

template <typename T>
static int launch_cl(const UpfirArgs& p, cudaStream_t s) {
    const long long total = (long long)p.out_w * p.out_h * p.in_n * (p.in_c >> 2);
    long long grid = ceil_div<long long>(total, 256);
    const long long cap = (long long)sm_count() * 16;
    if (grid > cap) grid = cap;
    upfirdn2d_cl_kernel<T><<<(unsigned)grid, 256, 0, s>>>(p);
    IDE3D_CHECK_LAUNCH("upfirdn2d_cl_kernel");
    return IDE3D_OK;
}

template <typename T>
static int launch_generic(const UpfirArgs& p, cudaStream_t s) {
    const long long total = (long long)p.out_w * p.out_h * p.in_c * p.in_n;
    long long grid = ceil_div<long long>(total, 256);
    const long long cap = (long long)sm_count() * 16;
    if (grid > cap) grid = cap;
    const int c_fastest = (p.osc == 1 && p.osw != 1) ? 1 : 0;
    upfirdn2d_generic_kernel<T><<<(unsigned)grid, 256, 0, s>>>(p, c_fastest);
    IDE3D_CHECK_LAUNCH("upfirdn2d_generic_kernel");
    return IDE3D_OK;
}

template <typename T>
static int dispatch_upfirdn2d(const UpfirArgs& p, cudaStream_t s) {
    const bool wcontig = (p.isw == 1 && p.osw == 1);
    if (wcontig && sizeof(T) <= 4 && p.add == nullptr && !p.epi) {
#define IDE3D_CASE(UX, UY, DX, DY, FW, FH)                                                              \
    if (p.ux == UX && p.uy == UY && p.dx == DX && p.dy == DY && p.fw == FW && p.fh == FH)                \
        return dispatch_phase<T, UX, UY, DX, DY, FW, FH>(p, s);
        IDE3D_CASE(1, 1, 1, 1, 4, 4)      // conv-up post filter (conv2d_resample.py:125)
        IDE3D_CASE(2, 2, 1, 1, 4, 4)      // upsample2d of the skip image (networks.py:841)
        IDE3D_CASE(1, 1, 2, 2, 4, 4)      // downsample2d
        IDE3D_CASE(2, 1, 1, 1, 12, 1)     // separable 12-tap passes (StyleGAN3 filters, filtered_lrelu fallback)
        IDE3D_CASE(1, 2, 1, 1, 1, 12)
        IDE3D_CASE(1, 1, 2, 1, 12, 1)
        IDE3D_CASE(1, 1, 1, 2, 1, 12)
        IDE3D_CASE(1, 1, 1, 1, 12, 1)
        IDE3D_CASE(1, 1, 1, 1, 1, 12)
#undef IDE3D_CASE
    }
    if (p.isc == 1 && p.osc == 1 && (p.in_c & 3) == 0 && p.isw != 1) {
        if constexpr (sizeof(T) <= 4) {
            const long long vb = 4 * (long long)sizeof(T);                      // one channel vector: 16 bytes (fp32) / 8 bytes (fp16)
            const bool aligned = ((reinterpret_cast<uintptr_t>(p.x) | reinterpret_cast<uintptr_t>(p.y)) % vb == 0) &&
                                 ((p.isw | p.ish | p.isn | p.osw | p.osh | p.osn) % 4 == 0);
            if (aligned) {
#define IDE3D_CASE_CL(UX, UY, DX, DY, FW, FH)                                                           \
    if (p.ux == UX && p.uy == UY && p.dx == DX && p.dy == DY && p.fw == FW && p.fh == FH)                \
        return dispatch_phase_cl<T, UX, UY, DX, DY, FW, FH>(p, s);
                IDE3D_CASE_CL(1, 1, 1, 1, 4, 4)
                IDE3D_CASE_CL(2, 2, 1, 1, 4, 4)
                IDE3D_CASE_CL(1, 1, 2, 2, 4, 4)
#undef IDE3D_CASE_CL
            }
        }
        if (p.add == nullptr && !p.epi) return launch_cl<T>(p, s);
    }
    if (p.add != nullptr || p.epi) IDE3D_FAIL(IDE3D_UNSUPPORTED, "upfirdn2d_add/_epilogue: needs channels_last tensors, C %% 4 == 0 and a 4x4 filter with up/down in {1,2}");
    return launch_generic<T>(p, s);
}

}  // namespace ide3d

using namespace ide3d;

static int upfirdn2d_entry(const ide3d_upfirdn2d_params* q, const void* add, int64_t asn, int64_t ash, int64_t asw, const void* bias,
                           ide3d_stream_t stream, const ide3d_fir_epilogue* e = nullptr) {
    IDE3D_REQUIRE(q != nullptr, "upfirdn2d: null params");
    IDE3D_REQUIRE(q->x && q->f && (q->y || (e && e->y2)), "upfirdn2d: null tensor");
    IDE3D_REQUIRE(q->up_x >= 1 && q->up_y >= 1 && q->down_x >= 1 && q->down_y >= 1, "upsampling and downsampling factors must be at least 1");
    IDE3D_REQUIRE(q->f_w >= 1 && q->f_h >= 1, "f must be at least 1x1");
    IDE3D_REQUIRE(q->in_w > 0 && q->in_h > 0 && q->in_c > 0 && q->in_n > 0, "x is empty");
    IDE3D_REQUIRE(q->out_w >= 1 && q->out_h >= 1, "output must be at least 1x1");
    UpfirArgs p;
    p.x = q->x; p.f = q->f; p.y = q->y;
    p.ux = q->up_x; p.uy = q->up_y; p.dx = q->down_x; p.dy = q->down_y; p.px0 = q->pad_x0; p.py0 = q->pad_y0;
    p.flip = q->flip; p.gain = q->gain;
    p.in_w = q->in_w; p.in_h = q->in_h; p.in_c = q->in_c; p.in_n = q->in_n;
    p.isw = q->in_stride_w; p.ish = q->in_stride_h; p.isc = q->in_stride_c; p.isn = q->in_stride_n;
    p.fw = q->f_w; p.fh = q->f_h; p.fsw = q->f_stride_w; p.fsh = q->f_stride_h;
    p.out_w = q->out_w; p.out_h = q->out_h;
    p.osw = q->out_stride_w; p.osh = q->out_stride_h; p.osc = q->out_stride_c; p.osn = q->out_stride_n;
    if (add != nullptr) {
        const uintptr_t vb = (q->dtype == IDE3D_F16) ? 8 : 16;
        IDE3D_REQUIRE(((uintptr_t)add % vb) == 0 && (bias == nullptr || ((uintptr_t)bias % vb) == 0) && (asn | ash | asw) % 4 == 0,
                      "upfirdn2d_add: add / bias must be aligned to one 4-channel vector");
        p.add = add; p.asn = asn; p.ash = ash; p.asw = asw; p.bias = bias;
    }
    if (e != nullptr) {
        const uintptr_t vb = (q->dtype == IDE3D_F16) ? 8 : 16;
        const uintptr_t all = (uintptr_t)e->scale | (uintptr_t)e->b | (uintptr_t)e->scale2 | (uintptr_t)e->y2;
        IDE3D_REQUIRE(all % vb == 0, "upfirdn2d_epilogue: scale / b / scale2 / y2 must be aligned to one 4-channel vector");
        IDE3D_REQUIRE((e->y2 == nullptr) == (e->scale2 == nullptr), "upfirdn2d_epilogue: scale2 and y2 go together");
        IDE3D_REQUIRE(e->noise == nullptr || e->noise_batch == 1 || e->noise_batch == q->in_n, "upfirdn2d_epilogue: noise batch must be 1 or n");
        if (e->act != 1 && e->act != 3) IDE3D_FAIL(IDE3D_UNSUPPORTED, "upfirdn2d_epilogue: only linear / lrelu are fused");
        if (q->dtype == IDE3D_F64) IDE3D_FAIL(IDE3D_UNSUPPORTED, "upfirdn2d_epilogue: fp64 is not fused");
        p.epi = 1; p.act = e->act; p.alpha = e->alpha; p.act_gain = e->gain; p.clamp = e->clamp; p.noise_batch = (int)e->noise_batch;
        p.scale = e->scale; p.noise = e->noise; p.bias = e->b; p.scale2 = e->scale2; p.y2 = e->y2;
    }
    cudaStream_t s = (cudaStream_t)stream;
    switch (q->dtype) {
        case IDE3D_F32: return dispatch_upfirdn2d<float>(p, s);
        case IDE3D_F16: return dispatch_upfirdn2d<__half>(p, s);
        case IDE3D_F64: return dispatch_upfirdn2d<double>(p, s);
    }
    IDE3D_FAIL(IDE3D_INVALID, "upfirdn2d: unsupported dtype %d", q->dtype);
}

extern "C" int ide3d_upfirdn2d(const ide3d_upfirdn2d_params* q, ide3d_stream_t stream) {
    return upfirdn2d_entry(q, nullptr, 0, 0, 0, nullptr, stream);
}

extern "C" int ide3d_upfirdn2d_add(const ide3d_upfirdn2d_params* q, const void* add, int64_t add_stride_n, int64_t add_stride_h,
                                   int64_t add_stride_w, const void* bias, ide3d_stream_t stream) {
    IDE3D_REQUIRE(add != nullptr, "upfirdn2d_add: null add tensor");
    return upfirdn2d_entry(q, add, add_stride_n, add_stride_h, add_stride_w, bias, stream);
}

extern "C" int ide3d_upfirdn2d_epilogue(const ide3d_upfirdn2d_params* q, const ide3d_fir_epilogue* e, ide3d_stream_t stream) {
    IDE3D_REQUIRE(e != nullptr, "upfirdn2d_epilogue: null epilogue");
    return upfirdn2d_entry(q, nullptr, 0, 0, 0, nullptr, stream, e);
}
