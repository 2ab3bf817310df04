// Fused filtered_lrelu for sm_90a: bias -> up-FIR -> gain * leaky ReLU * clamp (+ 2-bit signs) -> down-FIR in ONE kernel for
// separable filters (filtered_lrelu.cu:139-1099 of the reference; its CASE table :1248-1278).  Round-2 design.
//
// A CTA owns a TOW x TOH output tile of CB channels; the up^2-sized intermediate never leaves the SM.  The four separable
// passes are ordered  vertical-up, [horizontal-up -> activation -> horizontal-down], vertical-down  and the middle three run
// in REGISTERS: a thread owns one intermediate row segment, slides along it with the last TU input samples and the last FD
// activated samples in register rings, and emits one horizontally down-filtered sample per DOWN intermediate samples --
// one shared-memory load and one store per UP*TU + FD fused multiply-adds (0.08 accesses / FMA; the round-1 kernel spent
// 0.5 / FMA on shared-memory windows and was shared-memory bound at 5 % of the HBM roofline).
//
//   s_in [IH][BW][CB]   input tile in the tensor's own dtype, staged by ONE TMA box load per tile (cp.async.bulk.tensor, 3-D map
//                       W x H x planes for NCHW, 4-D map C x W x H x N for channels-last); out-of-image texels arrive as zeros
//                       (the TMA unit's out-of-bounds fill = the op's zero padding).  The load of tile i+1 is issued as soon as
//                       pass A of tile i has consumed the buffer and overlaps passes B and C.  Tensors the TMA unit cannot
//                       describe (unaligned pitch, 8-byte channel blocks) are staged by the threads instead -- same layout.
//   pass A  vertical up-FIR (+ bias inside the image):       s_in -> g1 [UH][G1P][CB] fp32       lanes walk along x (and c)
//   pass B  horizontal up-FIR, activation, signs, horizontal down-FIR, all in registers:  g1 -> w [UH][WP][CB]   lanes walk down rows
//   pass C  vertical down-FIR:                               w -> y (global, coalesced)          lanes walk along x (and c)
// Row pitches G1P / WP are odd so that both access directions are bank-conflict free; CB (1 for NCHW, 4 for channels-last)
// is the fastest index everywhere, which keeps channels-last global accesses at full sector width.
//
// Polyphase bookkeeping (per axis).  With q = u - pad0 the intermediate sample u is  sum_t f[r + UP t] x[ceil(q / UP) + t],
// r = (-q) mod UP  (f = the filter as applied: flipped unless `flip`).  A tile's intermediate origin is a multiple of UP, so the
// phase  ph = (-pad0) mod UP  is one constant per launch; "aligned" indices e = ph + (u - tile origin) make the input index
// ceil(e / UP) relative to the tile's input origin floor((u_origin - pad0) / UP).  A march starts at the aligned index
// e_start = UP * b0 - UP + 1 (b0 = ceil(e_first / UP)) and produces e_start + n for n = 0, 1, 2, ...; D = e_first - e_start is the
// number of leading samples to skip (< UP).  Loops run over blocks of P input samples, P chosen so that every ring slot, filter
// phase, down-sampling phase and sign-nibble position is a compile-time constant inside the unrolled block body.
#include <cuda.h>

#include "common.cuh"

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

namespace flf {

template <typename T> __device__ __forceinline__ float ldf(const T* p) { return (float)(*p); }
template <> __device__ __forceinline__ float ldf<__half>(const __half* p) { return __half2float(*p); }
template <typename T> __device__ __forceinline__ void stf(T* p, float v) { *p = (T)v; }
template <> __device__ __forceinline__ void stf<__half>(__half* p, float v) { *p = __float2half(v); }
template <typename T> __device__ __forceinline__ T zero_of() { return (T)0.f; }
template <> __device__ __forceinline__ __half zero_of<__half>() { return __float2half(0.f); }

__host__ __device__ constexpr int cgcd(int a, int b) { return b == 0 ? a : cgcd(b, a % b); }
__host__ __device__ constexpr int clcm(int a, int b) { return a / cgcd(a, b) * b; }
__host__ __device__ constexpr int cdiv(int a, int b) { return (a + b - 1) / b; }
__host__ __device__ constexpr int pmod(int a, int b) { return ((a % b) + b) % b; }

// per-axis geometry of a tile of TO outputs
template <int UP, int DOWN, int FU, int FD, int TO>
struct Axis {
    static constexpr int TU = cdiv(FU, UP);                         // up-FIR taps per polyphase branch
    static constexpr int UL = (TO - 1) * DOWN + FD;                 // intermediate samples the tile needs
    static constexpr int IL = cdiv(UL + UP - 2, UP) + TU;           // input samples (worst phase)
};

template <typename T, int UP, int DOWN, int FU, int FD, int CB>
struct Geom {
    // tile shape and work split (items per pass ~ thread count)
    static constexpr int TOW = (CB == 1) ? (DOWN >= 4 ? 32 : 64) : (DOWN >= 4 ? 16 : 32);
    static constexpr int TOH = (CB == 1) ? (DOWN >= 4 ? 32 : 64) : (DOWN >= 4 ? 8 : 16);
    static constexpr int kThreads = (CB == 1) ? 288 : 192;
    using AX = Axis<UP, DOWN, FU, FD, TOW>;
    using AY = Axis<UP, DOWN, FU, FD, TOH>;
    static constexpr int TU = AX::TU;
    static constexpr int UW = AX::UL, UH = AY::UL, IW = AX::IL, IH = AY::IL;
    static constexpr int kVec = 16 / (int)sizeof(T);                // elements per 16 bytes
    // NCHW: the TMA box must start on a 16-byte boundary of the row -> up to kVec-1 extra columns on the left
    static constexpr int BW = (CB == 1) ? cdiv(IW + kVec - 1, kVec) * kVec : IW;
    static constexpr int BH = IH;
    static constexpr int G1P = IW | 1, WP = TOW | 1;
    // block length of the marches: ring slots (TU inputs, FD intermediates), the down-sampling phase and the sign nibble repeat
    static constexpr int P = clcm(clcm(TU, FD / cgcd(FD, UP)), clcm(DOWN / cgcd(DOWN, UP), 4 / cgcd(4, UP)));
    static constexpr int NSB = (CB == 1) ? 2 : 1;                   // x segments of pass B
    static constexpr int NO = TOW / NSB;                            // outputs per segment
    static constexpr int NSA = (CB == 1) ? 3 : 1;                   // row segments of pass A
    static constexpr int RA = cdiv(UH, NSA);                        // intermediate rows per pass-A segment
    static constexpr int NSC = (CB == 1) ? 4 : 1;                   // row segments of pass C
    static constexpr int NOC = TOH / NSC;
    static constexpr int NB_B = cdiv((UP - 1 + (NO - 1) * DOWN + FD - 1) / UP + 1, P);      // blocks of a pass-B march
    static constexpr int NB_A = cdiv((UP - 1 + RA - 1) / UP + 1, P);                         // blocks of a pass-A march
    static constexpr int NB_C = cdiv((NOC - 1) * DOWN + FD, FD);                             // blocks (of FD rows) of a pass-C march
    static constexpr int kBoxBytes = BW * BH * CB * (int)sizeof(T);
    // The marches run in whole blocks, so each reads a little past the data it needs (values unused).  Every buffer is followed by
    // a zeroed slack region sized for its over-read -- no pass ever reads memory another thread is writing.
    static constexpr int kInBytes = (((BH + P + TU) * BW * CB * (int)sizeof(T) + 127) / 128) * 128;    // pass A over-reads rows
    static constexpr int kG1Floats = UH * G1P * CB, kG1Slack = (P + TU + 4) * CB;                        // pass B over-reads columns
    static constexpr int kWFloats = UH * WP * CB, kWSlack = (FD + DOWN) * WP * CB;                       // pass C over-reads rows
    static constexpr int kSmem = kInBytes + (kG1Floats + kG1Slack + kWFloats + kWSlack + 4 * 32) * 4 + 64 + 128;
    static_assert((TOW * DOWN) % UP == 0 && (TOH * DOWN) % UP == 0, "tile origins must keep the polyphase phase");
    static_assert((NO * DOWN) % UP == 0 && (NO * DOWN) % 4 == 0, "segment origins must keep phase and sign-byte alignment");
    static_assert((UP * P) % FD == 0 && (UP * P) % DOWN == 0 && (UP * P) % 4 == 0 && P % TU == 0 && FD % DOWN == 0, "march block");
    static_assert(CB == 1 || ((TOW * DOWN / UP) >= 1), "tile");
};

__device__ __forceinline__ unsigned smem_addr(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void bar_init(unsigned long long* bar) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_addr(bar)) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void bar_wait(unsigned long long* bar, unsigned parity) {
    unsigned ok = 0;
    while (!ok) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
                     : "=r"(ok) : "r"(smem_addr(bar)), "r"(parity) : "memory");
    }
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, unsigned long long* bar, int x, int y, int z, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 ::"r"(smem_addr(dst)), "l"(map), "r"(smem_addr(bar)), "r"(x), "r"(y), "r"(z) : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, unsigned long long* bar, int c, int x, int y, int n, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                 ::"r"(smem_addr(dst)), "l"(map), "r"(smem_addr(bar)), "r"(c), "r"(x), "r"(y), "r"(n) : "memory");
}

// -------------------------------------------------------------------------------------------------------------------------
// pass B of one item: intermediate row `row` (g1, element stride CB), x segment starting at output column o0.
// D = number of leading aligned samples to skip (compile time: ring and phase positions follow from it).
template <typename G, int UP, int DOWN, int FU, int FD, int CB, int MODE, int D, bool FAST>
__device__ __forceinline__ void pass_b_item(const FlFusedArgs& p, const float* __restrict__ src, float* __restrict__ dst,
                                            const float (&fh)[FU], const float (&fd)[FD], int ux0, int uy, bool own_row,
                                            bool tail_x, long long plane) {
    constexpr int TU = G::TU, P = G::P, NO = G::NO;
    constexpr int kNeeded = (NO - 1) * DOWN + FD;          // intermediate samples this segment consumes
    float hw[TU], uw[FD];
#pragma unroll
    for (int t = 0; t < TU - 1; ++t) hw[t] = src[t * CB];
#pragma unroll
    for (int t = 0; t < FD; ++t) uw[t] = 0.f;
    unsigned sacc = 0;
    const unsigned char* srow = nullptr;
    unsigned char* wrow = nullptr;
    if constexpr (MODE == 1) wrow = p.s + (long long)(p.sw >> 2) * (uy + (long long)p.sh * plane);
    if constexpr (MODE == 2) {
        const unsigned sy = (unsigned)(uy + p.soy);
        if (sy < (unsigned)p.sh) srow = p.s + (long long)(p.sw >> 2) * (sy + (long long)p.sh * plane);
    }
#pragma unroll 1
    for (int blk = 0; blk < G::NB_B; ++blk) {
        const int nb = blk * (UP * P);
#pragma unroll
        for (int ii = 0; ii < P; ++ii) {
            hw[(TU - 1 + ii) % TU] = src[(TU - 1 + blk * P + ii) * CB];
#pragma unroll
            for (int m = 0; m < UP; ++m) {
                const int r = UP - 1 - m;
                float acc = 0.f;
#pragma unroll
                for (int t = 0; t < TU; ++t)
                    if (r + UP * t < FU) acc = fmaf(fh[r + UP * t], hw[(ii + t) % TU], acc);
                const int ns = UP * ii + m;                   // position inside the block (compile time after unrolling)
                const int jrel = nb + ns - D;                 // intermediate column relative to the segment origin
                float val = acc;
                if constexpr (MODE == 2) {
                    const unsigned sx = (unsigned)(ux0 + jrel + p.sox);
                    if (srow != nullptr && jrel >= 0 && sx < (unsigned)p.sw) {
                        const unsigned sb = (unsigned)srow[sx >> 2] >> ((sx & 3) << 1);
                        if (sb & 1) val *= p.slope;
                        if (sb & 2) val = 0.f;
                    }
                } else if constexpr (MODE == 0 && FAST) {
                    // 0 <= slope <= 1: lrelu(v) = max(v, v * slope) and the clamp is a min / max pair -- the same values as the
                    // compare-and-select form below in 4 instructions instead of 7
                    val = fmaxf(val, val * p.slope);
                    val = fminf(fmaxf(val, -p.clamp), p.clamp);
                } else {
                    unsigned sg = 0;
                    if (val < 0.f) { val *= p.slope; sg = 1; }
                    if (fabsf(val) > p.clamp) { val = (val < 0.f) ? -p.clamp : p.clamp; sg = 2; }
                    if constexpr (MODE == 1) {
                        // a segment OWNS columns [0, NO*DOWN) of its march (the halo belongs to the neighbour), the last segment of the
                        // last tile column also its tail; bytes are 4-column aligned with the ownership boundaries
                        const int nib = pmod(ns - D, 4);
                        const bool valid = jrel >= 0 && jrel < kNeeded && (jrel < NO * DOWN || tail_x);
                        if (valid) sacc |= sg << (2 * nib);
                        if (nib == 3) {
                            const int ux = ux0 + jrel;
                            if (sacc != 0 && own_row && ux < p.sw) wrow[ux >> 2] = (unsigned char)sacc;
                            sacc = 0;
                        }
                    }
                }
                uw[ns % FD] = val;
                if (pmod(ns - D - (FD - 1), DOWN) == 0) {
                    const int num = nb + ns - D - (FD - 1);
                    if (num >= 0 && num < NO * DOWN) {        // uniform over the block's threads
                        float o = 0.f;
#pragma unroll
                        for (int k = 0; k < FD; ++k) o = fmaf(fd[k], uw[(ns + 1 + k) % FD], o);
                        dst[(num / DOWN) * CB] = o;
                    }
                }
            }
        }
    }
    if constexpr (MODE == 1) {
        constexpr int kLastNib = pmod(UP * P - 1 - D, 4);
        if (kLastNib != 3) {
            const int ux = ux0 + G::NB_B * UP * P - 1 - D;
            if (sacc != 0 && own_row && (ux & ~3) < p.sw) wrow[ux >> 2] = (unsigned char)sacc;
        }
    }
}

template <typename T, int UP, int DOWN, int FU, int FD, int CB, int MODE, bool FAST>
__global__ void __launch_bounds__((Geom<T, UP, DOWN, FU, FD, CB>::kThreads), (CB == 1 ? 2 : 3))
filtered_lrelu_fused2_kernel(const FlFusedArgs p, int tiles_x, int tiles_y, int cblocks, int use_tma, int shift_x,
                             const __grid_constant__ CUtensorMap tmap) {
    using G = Geom<T, UP, DOWN, FU, FD, CB>;
    constexpr int TU = G::TU, P = G::P, NT = G::kThreads;
    // no static shared memory in this kernel: the dynamic window starts at offset 0 of the CTA's shared memory, so the declared alignment
    // holds and every pointer below stays provably shared (LDS / STS instead of generic LD / ST: 7 % of the instructions in the first capture)
    extern __shared__ __align__(1024) unsigned char fl_raw[];
    unsigned char* base = fl_raw;
    T* s_in = reinterpret_cast<T*>(base);
    float* g1 = reinterpret_cast<float*>(base + G::kInBytes);
    float* w = g1 + G::kG1Floats + G::kG1Slack;
    float* taps = w + G::kWFloats + G::kWSlack;            // [4][32]: up (vertical), up (horizontal, * gains), down (horizontal), down (vertical)
    unsigned long long* bar = reinterpret_cast<unsigned long long*>(g1 + ((G::kG1Floats + G::kG1Slack + G::kWFloats + G::kWSlack + 4 * 32 + 3) / 4) * 4);    // 16-byte aligned: g1 starts on a 128-byte boundary
    const int tid = threadIdx.x;

    const float act_gain = p.gain * (float)(UP * UP) * (p.one_u ? 1.f / p.fu[0] : 1.f);
    const float fd_scale_y = p.one_d ? 1.f / p.fd[0] : 1.f;
    if (tid < 32) {
        const float u = (tid < FU) ? p.fu[p.flip ? tid : FU - 1 - tid] : 0.f;
        const float d = (tid < FD) ? p.fd[p.flip ? tid : FD - 1 - tid] : 0.f;
        taps[tid] = u; taps[32 + tid] = u * act_gain; taps[64 + tid] = d; taps[96 + tid] = d * fd_scale_y;
    }
    // slack regions (read by the block-rounded marches, values unused): zero once
    for (int i = tid; i < G::kG1Slack; i += NT) g1[G::kG1Floats + i] = 0.f;
    for (int i = tid; i < G::kWSlack; i += NT) w[G::kWFloats + i] = 0.f;
    for (int i = tid; i < (G::kInBytes - G::kBoxBytes) / (int)sizeof(T); i += NT) s_in[G::kBoxBytes / (int)sizeof(T) + i] = zero_of<T>();

    const int phx = pmod(-p.px0, UP), phy = pmod(-p.py0, UP);
    const int ix0 = floor_div(-p.px0, UP), iy0 = floor_div(-p.py0, UP);     // input origin of the tile at output (0, 0)
    const long long tiles_plane = (long long)tiles_x * tiles_y;
    const long long total = tiles_plane * cblocks * p.xn;
    constexpr unsigned kBoxBytes = G::kBoxBytes;

    // tile order: NCHW  plane-major (a plane's tiles are consecutive);  channels-last  channel block fastest, so that concurrently
    // running CTAs read neighbouring 16-byte channel groups of the same texels
    auto decode = [&](long long blk, int& n, int& cb, int& tx, int& ty) {
        if (CB == 1) {
            const long long pl = blk / tiles_plane;
            const int t = (int)(blk - pl * tiles_plane);
            n = (int)(pl / cblocks); cb = (int)(pl - (long long)n * cblocks);
            tx = t % tiles_x; ty = t / tiles_x;
        } else {
            cb = (int)(blk % cblocks);
            const long long r = blk / cblocks;
            const int t = (int)(r % tiles_plane);
            n = (int)(r / tiles_plane);
            tx = t % tiles_x; ty = t / tiles_x;
        }
    };
    auto issue = [&](long long blk) {
        int n, cb, tx, ty;
        decode(blk, n, cb, tx, ty);
        const int ix_t = tx * (G::TOW * DOWN / UP) + ix0, iy_t = ty * (G::TOH * DOWN / UP) + iy0;
        if (CB == 1) tma_load_3d(s_in, &tmap, bar, ix_t - shift_x, iy_t, n * p.xc + cb, kBoxBytes);
        else tma_load_4d(s_in, &tmap, bar, cb * CB, ix_t, iy_t, n, kBoxBytes);
    };
    if (tid == 0) {
        bar_init(bar);
        if (use_tma && (long long)blockIdx.x < total) issue(blockIdx.x);
    }
    __syncthreads();

    int it = 0;
    for (long long blk = blockIdx.x; blk < total; blk += gridDim.x, ++it) {
        int n, cb, tx, ty;
        decode(blk, n, cb, tx, ty);
        const int c0 = cb * CB;
        const int ox_t = tx * G::TOW, oy_t = ty * G::TOH;
        const int ux_t = ox_t * DOWN, uy_t = oy_t * DOWN;
        const int ix_t = tx * (G::TOW * DOWN / UP) + ix0, iy_t = ty * (G::TOH * DOWN / UP) + iy0;
        const int bx0 = ix_t - shift_x;                                       // global column of box column 0

        if (use_tma) {
            bar_wait(bar, it & 1);
        } else {
            // staged by the threads: same [row][col][c] layout, zeros outside the image / beyond the channel count
            const T* xin = (const T*)p.x + (long long)n * p.sxn;
            for (int i = tid; i < G::BH * G::BW * CB; i += NT) {
                const int c = i % CB, rc = i / CB;
                const int col = rc % G::BW, row = rc / G::BW;
                const int gx = bx0 + col, gy = iy_t + row, gc = c0 + c;
                T v = zero_of<T>();
                if ((unsigned)gx < (unsigned)p.xw && (unsigned)gy < (unsigned)p.xh && gc < p.xc)
                    v = xin[gc * p.sxc + (long long)gy * p.sxh + (long long)gx * p.sxw];
                s_in[i] = v;
            }
            __syncthreads();
        }

        // ---------------- pass A: vertical up-FIR.  item = (c, x, row segment); the thread walks down the input column
        {
            float fv[FU];
#pragma unroll
            for (int k = 0; k < FU; ++k) fv[k] = taps[k];
            for (int item = tid; item < CB * G::IW * G::NSA; item += NT) {
                const int c = item % CB, r2 = item / CB;
                const int x = r2 % G::IW, seg = r2 / G::IW;
                const int gx = ix_t + x, gc = c0 + c;
                const bool colok = (unsigned)gx < (unsigned)p.xw && gc < p.xc;
                const float bias = (colok && p.b) ? ldf<T>((const T*)p.b + gc) : 0.f;
                const int j0 = seg * G::RA;                                   // first intermediate row of the segment
                const int e0 = phy + j0;
                const int b0 = (e0 + UP - 1) / UP;
                const int dskip = e0 - (UP * b0 - UP + 1);
                const T* col = s_in + ((long long)b0 * G::BW + (x + shift_x)) * CB + c;
                float* out = g1 + ((long long)j0 * G::G1P + x) * CB + c;
                const int rows = min(G::RA, G::UH - j0);
                float hw[TU];
#pragma unroll
                for (int t = 0; t < TU - 1; ++t) {
                    const bool ok = colok && (unsigned)(iy_t + b0 + t) < (unsigned)p.xh;
                    hw[t] = ldf<T>(col + (long long)t * G::BW * CB) + (ok ? bias : 0.f);
                }
#pragma unroll 1
                for (int bk = 0; bk < G::NB_A; ++bk) {
#pragma unroll
                    for (int ii = 0; ii < P; ++ii) {
                        const int ip = bk * P + ii;
                        const bool ok = colok && (unsigned)(iy_t + b0 + TU - 1 + ip) < (unsigned)p.xh;
                        hw[(TU - 1 + ii) % TU] = ldf<T>(col + (long long)(TU - 1 + ip) * G::BW * CB) + (ok ? bias : 0.f);
#pragma unroll
                        for (int m = 0; m < UP; ++m) {
                            const int r = UP - 1 - m;
                            float acc = 0.f;
#pragma unroll
                            for (int t = 0; t < TU; ++t)
                                if (r + UP * t < FU) acc = fmaf(fv[r + UP * t], hw[(ii + t) % TU], acc);
                            const int jl = UP * ip + m - dskip;               // row inside the segment
                            if (jl >= 0 && jl < rows) out[(long long)jl * G::G1P * CB] = acc;
                        }
                    }
                }
            }
        }
        __syncthreads();                                                       // g1 complete, s_in free
        if (use_tma && tid == 0 && blk + gridDim.x < total) issue(blk + gridDim.x);

        // ---------------- pass B: horizontal up-FIR + activation (+ signs) + horizontal down-FIR in registers.  item = (c, row, x segment)
        {
            float fh[FU], fdh[FD];
#pragma unroll
            for (int k = 0; k < FU; ++k) fh[k] = taps[32 + k];
#pragma unroll
            for (int k = 0; k < FD; ++k) fdh[k] = taps[64 + k];
            const bool last_tx = (ox_t + G::TOW >= p.yw), last_ty = (oy_t + G::TOH >= p.yh);
            for (int item = tid; item < CB * G::UH * G::NSB; item += NT) {
                const int c = item % CB, r2 = item / CB;
                const int row = r2 % G::UH, seg = r2 / G::UH;
                const int o0 = seg * G::NO;
                const int e0 = phx + o0 * DOWN;
                const int b0 = (e0 + UP - 1) / UP;
                const float* src = g1 + ((long long)row * G::G1P + b0) * CB + c;
                float* dst = w + ((long long)row * G::WP + o0) * CB + c;
                const int uy = uy_t + row;
                const bool own_row = (row < G::TOH * DOWN || last_ty) && uy < p.sh && (c0 + c) < p.xc;
                const bool tail_x = last_tx && seg == G::NSB - 1;
                const long long plane = (long long)n * p.xc + c0 + c;
                const int ux0 = ux_t + o0 * DOWN;
                // D = (phx - 1) mod UP for every segment (segment origins are multiples of UP)
                if (UP == 1 || pmod(phx - 1, UP) == 0) pass_b_item<G, UP, DOWN, FU, FD, CB, MODE, 0, FAST>(p, src, dst, fh, fdh, ux0, uy, own_row, tail_x, plane);
                else if (UP == 2 || pmod(phx - 1, UP) == 1) pass_b_item<G, UP, DOWN, FU, FD, CB, MODE, (UP > 1 ? 1 : 0), FAST>(p, src, dst, fh, fdh, ux0, uy, own_row, tail_x, plane);
                else if (pmod(phx - 1, UP) == 2) pass_b_item<G, UP, DOWN, FU, FD, CB, MODE, (UP > 2 ? 2 : 0), FAST>(p, src, dst, fh, fdh, ux0, uy, own_row, tail_x, plane);
                else pass_b_item<G, UP, DOWN, FU, FD, CB, MODE, (UP > 3 ? 3 : 0), FAST>(p, src, dst, fh, fdh, ux0, uy, own_row, tail_x, plane);
            }
        }
        __syncthreads();                                                       // w complete

        // ---------------- pass C: vertical down-FIR -> global.  item = (c, x, row segment); the thread walks down its column of w
        {
            float fdv[FD];
#pragma unroll
            for (int k = 0; k < FD; ++k) fdv[k] = taps[96 + k];
            T* yout = (T*)p.y + (long long)n * p.syn;
            for (int item = tid; item < CB * G::TOW * G::NSC; item += NT) {
                const int c = item % CB, r2 = item / CB;
                const int x = r2 % G::TOW, seg = r2 / G::TOW;
                const int o0 = seg * G::NOC;
                const float* col = w + ((long long)(o0 * DOWN) * G::WP + x) * CB + c;
                const int ox = ox_t + x, gc = c0 + c;
                const bool colok = ox < p.yw && gc < p.xc;
                T* yc = yout + gc * p.syc + (long long)ox * p.syw;
                float uw[FD];
#pragma unroll
                for (int t = 0; t < FD; ++t) uw[t] = 0.f;
#pragma unroll 1
                for (int bk = 0; bk < G::NB_C; ++bk) {
#pragma unroll
                    for (int ii = 0; ii < FD; ++ii) {
                        const int nrow = bk * FD + ii;
                        uw[ii] = col[(long long)nrow * G::WP * CB];
                        if (pmod(ii - (FD - 1), DOWN) == 0) {
                            const int num = nrow - (FD - 1);
                            if (num >= 0 && num < G::NOC * DOWN) {
                                float o = 0.f;
#pragma unroll
                                for (int k = 0; k < FD; ++k) o = fmaf(fdv[k], uw[(ii + 1 + k) % FD], o);
                                const int oy = oy_t + o0 + num / DOWN;
                                if (colok && oy < p.yh) stf<T>(yc + (long long)oy * p.syh, o);
                            }
                        }
                    }
                }
            }
        }
        // no barrier here: the next tile's pass A writes g1 (last read before the barrier above) and reads s_in; its own barrier
        // orders this pass C's reads of w before the next pass B overwrites it.  The thread-staged path reloads s_in, which
        // pass A of THIS tile finished reading two barriers ago.
    }
}

// ---- host side --------------------------------------------------------------------------------------------------------------
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

template <typename T, int UP, int DOWN, int FU, int FD, int CB>
static bool make_map(const FlFusedArgs& a, CUtensorMap& map) {
    using G = Geom<T, UP, DOWN, FU, FD, CB>;
    memset(&map, 0, sizeof(map));
    if (encode_tiled() == nullptr) return false;
    if (tuning_env("IDE3D_FLRELU_NO_TMA") != nullptr) return false;
    if (reinterpret_cast<uintptr_t>(a.x) & 15) return false;
    const CUtensorMapDataType dt = sizeof(T) == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r;
    if (CB == 1) {
        if (a.sxw != 1 || a.sxn != a.sxc * a.xc) return false;                 // (n, c) must collapse into one plane index
        if ((a.sxh * sizeof(T)) % 16 || (a.sxc * sizeof(T)) % 16) return false;
        if ((long long)a.xc * a.xn > 0x7fffffffll) return false;
        const cuuint64_t dims[3] = {(cuuint64_t)a.xw, (cuuint64_t)a.xh, (cuuint64_t)a.xc * a.xn};
        const cuuint64_t strides[2] = {(cuuint64_t)a.sxh * sizeof(T), (cuuint64_t)a.sxc * sizeof(T)};
        const cuuint32_t box[3] = {(cuuint32_t)G::BW, (cuuint32_t)G::BH, 1};
        r = encode_tiled()(&map, dt, 3, const_cast<void*>(a.x), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    } else {
        if ((CB * sizeof(T)) % 16) return false;                                // innermost box extent must be a multiple of 16 bytes
        if (a.sxc != 1) return false;
        if ((a.sxw * sizeof(T)) % 16 || (a.sxh * sizeof(T)) % 16 || (a.sxn * sizeof(T)) % 16) return false;
        const cuuint64_t dims[4] = {(cuuint64_t)a.xc, (cuuint64_t)a.xw, (cuuint64_t)a.xh, (cuuint64_t)a.xn};
        const cuuint64_t strides[3] = {(cuuint64_t)a.sxw * sizeof(T), (cuuint64_t)a.sxh * sizeof(T), (cuuint64_t)a.sxn * sizeof(T)};
        const cuuint32_t box[4] = {(cuuint32_t)CB, (cuuint32_t)G::BW, (cuuint32_t)G::BH, 1};
        r = encode_tiled()(&map, dt, 4, const_cast<void*>(a.x), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    }
    return r == CUDA_SUCCESS;
}

template <typename T, int UP, int DOWN, int FU, int FD, int CB, int MODE, bool FAST = false>
static int launch_mode(const FlFusedArgs& a, cudaStream_t st) {
    using G = Geom<T, UP, DOWN, FU, FD, CB>;
    static_assert(G::kSmem <= 227 * 1024, "tile does not fit shared memory");
    CUtensorMap map;
    const bool tma = make_map<T, UP, DOWN, FU, FD, CB>(a, map);
    const int ix0 = floor_div(-a.px0, UP);
    const int shift = (CB == 1) ? pmod(ix0, G::kVec) : 0;
    auto kern = filtered_lrelu_fused2_kernel<T, UP, DOWN, FU, FD, CB, MODE, FAST>;
    const int smem = G::kSmem;
    IDE3D_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    const int tiles_x = ceil_div(a.yw, G::TOW), tiles_y = ceil_div(a.yh, G::TOH);
    const int cblocks = ceil_div(a.xc, CB);
    const long long total = (long long)tiles_x * tiles_y * cblocks * a.xn;
    int per_sm = 1;
    IDE3D_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, G::kThreads, smem));
    if (per_sm < 1) per_sm = 1;
    long long grid = (long long)sm_count() * per_sm;
    if (grid > total) grid = total;
    kern<<<(unsigned)grid, G::kThreads, smem, st>>>(a, tiles_x, tiles_y, cblocks, tma ? 1 : 0, shift, map);
    IDE3D_CHECK_LAUNCH("filtered_lrelu_fused2_kernel");
    return IDE3D_OK;
}

template <typename T, int UP, int DOWN, int FU, int FD>
static int launch_fused(const FlFusedArgs& a, cudaStream_t st) {
    const bool fast = (a.slope >= 0.f && a.slope <= 1.f);
    if (a.channels_last) {
        if (a.mode == 0) return fast ? launch_mode<T, UP, DOWN, FU, FD, 4, 0, true>(a, st) : launch_mode<T, UP, DOWN, FU, FD, 4, 0>(a, st);
        if (a.mode == 1) return launch_mode<T, UP, DOWN, FU, FD, 4, 1>(a, st);
        return launch_mode<T, UP, DOWN, FU, FD, 4, 2>(a, st);
    }
    if (a.mode == 0) return fast ? launch_mode<T, UP, DOWN, FU, FD, 1, 0, true>(a, st) : launch_mode<T, UP, DOWN, FU, FD, 1, 0>(a, st);
    if (a.mode == 1) return launch_mode<T, UP, DOWN, FU, FD, 1, 1>(a, st);
    return launch_mode<T, UP, DOWN, FU, FD, 1, 2>(a, st);
}

template <typename T>
static int dispatch_fused(const FlFusedArgs& a, int up, int down, int fu, int fd, cudaStream_t st) {
#define IDE3D_FL_CASE(UP, DOWN, FU, FD) if (up == UP && down == DOWN && fu == FU && fd == FD) return launch_fused<T, UP, DOWN, FU, FD>(a, st);
    IDE3D_FL_CASE(2, 2, 12, 12)     // StyleGAN3 default (filter_size 6), filtered_lrelu.cu:1262
    IDE3D_FL_CASE(2, 2, 8, 8)
    IDE3D_FL_CASE(2, 2, 16, 16)
    IDE3D_FL_CASE(4, 2, 24, 12)
    IDE3D_FL_CASE(4, 2, 16, 8)
    IDE3D_FL_CASE(2, 4, 12, 24)
    IDE3D_FL_CASE(2, 1, 12, 1)
    IDE3D_FL_CASE(2, 1, 8, 1)
    IDE3D_FL_CASE(1, 2, 1, 12)
    IDE3D_FL_CASE(1, 2, 1, 8)
    IDE3D_FL_CASE(1, 1, 1, 1)
#undef IDE3D_FL_CASE
    IDE3D_FAIL(IDE3D_UNSUPPORTED, "filtered_lrelu: no fused kernel for up=%d down=%d fu=%d fd=%d", up, down, fu, fd);
}

}  // namespace flf

// entry used by ide3d_filtered_lrelu (filtered_lrelu.cu)
int launch_filtered_lrelu_fused(const FlFusedArgs& a, int dtype, int up, int down, int fu, int fd, cudaStream_t st) {
    return (dtype == IDE3D_F32) ? flf::dispatch_fused<float>(a, up, down, fu, fd, st) : flf::dispatch_fused<__half>(a, up, down, fu, fd, st);
}

}  // namespace ide3d
