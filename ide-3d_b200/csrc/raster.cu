// Shaded turntable frames of a triangle mesh (the render step of render_mesh.py:44-67, which draws with pyrender / OpenGL offscreen;
// here a visibility buffer on the GPU, no graphics context).  Kernels, in launch order:
//   ide3d_mesh_normals    mesh_normals_kernel     vertex -> area-weighted sum of its faces' cross products (CSR order), normalised
//   ide3d_raster          raster_clear_kernel     key buffer := all ones, overflow counter := 0
//                         raster_transform_kernel (frame, vertex) -> 8-bit sub-pixel screen position, 1/w, valid flag
//                         raster_small_kernel     (frame, triangle) -> atomicMin(key) over its bounding box, or the overflow list
//                         raster_large_kernel     one CTA per overflow triangle, striding over its bounding box
//                         raster_resolve_kernel   pixel -> triangle -> perspective-correct normal -> shade -> RGB (+ id)
// Every float operation that decides a pixel or a colour is explicitly rounded (__fmul_rn / __fadd_rn / __fdiv_rn, no FMA
// contraction) in the order oracle/rasterizer.py uses, and the key (bits of the view depth w) << 32 | triangle resolves with a
// 64-bit atomicMin: the nearest surface wins, ties go to the lower triangle index, and the result does not depend on launch order.
#include "common.cuh"

namespace ide3d {

constexpr int kSub = 256;                         // fixed-point screen coordinates: 8 sub-pixel bits
constexpr float kGuardPx = 16384.f;               // a vertex further than this outside the viewport drops its triangles
constexpr long long kSmallBudget = 64;            // bounding boxes of more pixels go to raster_large_kernel
constexpr int kMaxRes = 16384;

__host__ __device__ inline int64_t align_up(int64_t v, int64_t a) { return (v + a - 1) / a * a; }

// scratch sections: keys u64 [F,H,W] | screen vertices int4 [F,V] | overflow counter u32 | overflow list int2 [F*T]
inline int64_t raster_layout(int64_t f, int64_t w, int64_t h, int64_t v, int64_t t, int64_t ofs[4]) {
    int64_t o = 0;
    ofs[0] = o; o = align_up(o + f * h * w * 8, 256);
    ofs[1] = o; o = align_up(o + f * v * 16, 256);
    ofs[2] = o; o = align_up(o + 4, 256);
    ofs[3] = o; o = align_up(o + f * t * 8, 256);
    return o;
}

__device__ __forceinline__ long long edge_fn(int ax, int ay, int bx, int by, int px, int py) {
    return (long long)(bx - ax) * (py - ay) - (long long)(by - ay) * (px - ax);
}

// One triangle in one frame, ready to evaluate at pixel centres.  The orientation is normalised (sgn) so that area > 0 and the edge
// functions are >= 0 inside; need[k] is 0 on a top or left edge (a centre exactly on it is covered) and 1 on the others.
struct TriSetup {
    int x[3], y[3];
    float iw[3];
    long long area;
    int sgn;
    int need[3];
};

__device__ __forceinline__ bool tri_setup(const int4* __restrict__ sv, long long V, int f, int i0, int i1, int i2, TriSetup& s) {
    const int4 a = sv[f * V + i0], b = sv[f * V + i1], c = sv[f * V + i2];
    if (!(a.w && b.w && c.w)) return false;
    s.x[0] = a.x; s.y[0] = a.y; s.iw[0] = __int_as_float(a.z);
    s.x[1] = b.x; s.y[1] = b.y; s.iw[1] = __int_as_float(b.z);
    s.x[2] = c.x; s.y[2] = c.y; s.iw[2] = __int_as_float(c.z);
    const long long area = edge_fn(s.x[0], s.y[0], s.x[1], s.y[1], s.x[2], s.y[2]);
    if (area == 0) return false;
    s.sgn = area > 0 ? 1 : -1;
    s.area = area > 0 ? area : -area;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int p = (k + 1) % 3, q = (k + 2) % 3;
        const int dx = (s.x[q] - s.x[p]) * s.sgn, dy = (s.y[q] - s.y[p]) * s.sgn;
        s.need[k] = (dy < 0 || (dy == 0 && dx > 0)) ? 0 : 1;        // top-left rule (screen y points down)
    }
    return true;
}

// exact integer barycentrics at the centre of pixel (i, j); true when the centre is covered
__device__ __forceinline__ bool tri_cover(const TriSetup& s, int i, int j, long long (&w)[3]) {
    const int px = i * kSub + kSub / 2, py = j * kSub + kSub / 2;
    bool in = true;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int p = (k + 1) % 3, q = (k + 2) % 3;
        w[k] = edge_fn(s.x[p], s.y[p], s.x[q], s.y[q], px, py) * s.sgn;
        in = in && (w[k] >= s.need[k]);
    }
    return in;
}

// q[k] = (w[k] / area) * (1/w_k): perspective weights before normalisation; returns their sum, 1/w at the pixel
__device__ __forceinline__ float tri_interp(const TriSetup& s, const long long (&w)[3], float (&q)[3]) {
    const float A = __ll2float_rn(s.area);
#pragma unroll
    for (int k = 0; k < 3; ++k) q[k] = __fmul_rn(__fdiv_rn(__ll2float_rn(w[k]), A), s.iw[k]);
    return __fadd_rn(__fadd_rn(q[0], q[1]), q[2]);
}

__device__ __forceinline__ void tri_bbox(const TriSetup& s, int W, int H, int& ilo, int& ihi, int& jlo, int& jhi) {
    const int xmin = min(s.x[0], min(s.x[1], s.x[2])), xmax = max(s.x[0], max(s.x[1], s.x[2]));
    const int ymin = min(s.y[0], min(s.y[1], s.y[2])), ymax = max(s.y[0], max(s.y[1], s.y[2]));
    ilo = max(0, floor_div(xmin - kSub / 2 + kSub - 1, kSub));
    ihi = min(W - 1, floor_div(xmax - kSub / 2, kSub));
    jlo = max(0, floor_div(ymin - kSub / 2 + kSub - 1, kSub));
    jhi = min(H - 1, floor_div(ymax - kSub / 2, kSub));
}

__device__ __forceinline__ void tri_plot(const TriSetup& s, unsigned int tri, int i, int j, unsigned long long* __restrict__ frame_keys,
                                         int W) {
    long long w[3];
    if (!tri_cover(s, i, j, w)) return;
    float q[3];
    const float depth = __fdiv_rn(1.f, tri_interp(s, w, q));          // the view depth w > 0: its bits sort nearest-first
    const unsigned long long key = ((unsigned long long)__float_as_uint(depth) << 32) | tri;
    atomicMin(frame_keys + (long long)j * W + i, key);
}

// ------------------------------------------------------------------------------------------------------------------- normals
__global__ void __launch_bounds__(256) mesh_normals_kernel(const float* __restrict__ vert, const int* __restrict__ tris, int64_t nv,
                                                           const int* __restrict__ adj_off, const int* __restrict__ adj_face,
                                                           float* __restrict__ normals) {
    for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < nv; v += (long long)gridDim.x * blockDim.x) {
        float sx = 0.f, sy = 0.f, sz = 0.f;
        for (int k = adj_off[v]; k < adj_off[v + 1]; ++k) {
            const long long f = adj_face[k];
            const float* p0 = vert + 3ll * tris[3 * f];
            const float* p1 = vert + 3ll * tris[3 * f + 1];
            const float* p2 = vert + 3ll * tris[3 * f + 2];
            const float ax = __fsub_rn(p1[0], p0[0]), ay = __fsub_rn(p1[1], p0[1]), az = __fsub_rn(p1[2], p0[2]);
            const float bx = __fsub_rn(p2[0], p0[0]), by = __fsub_rn(p2[1], p0[1]), bz = __fsub_rn(p2[2], p0[2]);
            sx = __fadd_rn(sx, __fsub_rn(__fmul_rn(ay, bz), __fmul_rn(az, by)));
            sy = __fadd_rn(sy, __fsub_rn(__fmul_rn(az, bx), __fmul_rn(ax, bz)));
            sz = __fadd_rn(sz, __fsub_rn(__fmul_rn(ax, by), __fmul_rn(ay, bx)));
        }
        const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(sx, sx), __fmul_rn(sy, sy)), __fmul_rn(sz, sz)));
        const bool ok = len > 0.f;
        normals[3 * v] = ok ? __fdiv_rn(sx, len) : 0.f;
        normals[3 * v + 1] = ok ? __fdiv_rn(sy, len) : 0.f;
        normals[3 * v + 2] = ok ? __fdiv_rn(sz, len) : 0.f;
    }
}

// ------------------------------------------------------------------------------------------------------------------- raster
__global__ void __launch_bounds__(256) raster_clear_kernel(unsigned long long* __restrict__ keys, long long n, unsigned int* overflow_count) {
    const long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i0 == 0) *overflow_count = 0u;
    for (long long i = i0; i < n; i += (long long)gridDim.x * blockDim.x) keys[i] = ~0ull;
}

// camera space = R^T (p - t) for the rigid cam2world [R | t]; OpenGL projection (camera looks down -z, +y up), w = -z_cam
__global__ void __launch_bounds__(256) raster_transform_kernel(const float* __restrict__ vert, int64_t nv, const float* __restrict__ c2w,
                                                               int F, int W, int H, float fx, float fy, float znear, int4* __restrict__ sv) {
    const long long total = (long long)F * nv;
    const float hw = 0.5f * (float)W, hh = 0.5f * (float)H;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const int f = (int)(idx / nv);
        const long long v = idx - (long long)f * nv;
        const float* M = c2w + 16 * f;
        const float d0 = __fsub_rn(vert[3 * v], M[3]), d1 = __fsub_rn(vert[3 * v + 1], M[7]), d2 = __fsub_rn(vert[3 * v + 2], M[11]);
        const float xc = __fadd_rn(__fadd_rn(__fmul_rn(M[0], d0), __fmul_rn(M[4], d1)), __fmul_rn(M[8], d2));
        const float yc = __fadd_rn(__fadd_rn(__fmul_rn(M[1], d0), __fmul_rn(M[5], d1)), __fmul_rn(M[9], d2));
        const float zc = __fadd_rn(__fadd_rn(__fmul_rn(M[2], d0), __fmul_rn(M[6], d1)), __fmul_rn(M[10], d2));
        const float w = -zc;
        int4 out = make_int4(0, 0, 0, 0);
        if (w >= znear) {                                                 // false for NaN too
            const float xn = __fdiv_rn(__fmul_rn(fx, xc), w), yn = __fdiv_rn(__fmul_rn(fy, yc), w);
            const float X = __fmul_rn(__fadd_rn(xn, 1.f), hw);            // pixels from the left edge
            const float Y = __fmul_rn(__fsub_rn(1.f, yn), hh);            // pixels from the top edge (row 0 at the top)
            if (X >= -kGuardPx && X <= (float)W + kGuardPx && Y >= -kGuardPx && Y <= (float)H + kGuardPx) {
                out.x = __float2int_rn(__fmul_rn(X, (float)kSub));       // round half to even
                out.y = __float2int_rn(__fmul_rn(Y, (float)kSub));
                out.z = __float_as_int(__fdiv_rn(1.f, w));
                out.w = 1;
            }
        }
        sv[idx] = out;
    }
}

__global__ void __launch_bounds__(128) raster_small_kernel(const int* __restrict__ tris, int64_t nt, int64_t nv, const int4* __restrict__ sv,
                                                           int F, int W, int H, unsigned long long* __restrict__ keys,
                                                           unsigned int* __restrict__ overflow_count, int2* __restrict__ overflow) {
    const long long total = (long long)F * nt;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const int f = (int)(idx / nt);
        const long long t = idx - (long long)f * nt;
        TriSetup s;
        if (!tri_setup(sv, nv, f, tris[3 * t], tris[3 * t + 1], tris[3 * t + 2], s)) continue;
        int ilo, ihi, jlo, jhi;
        tri_bbox(s, W, H, ilo, ihi, jlo, jhi);
        if (ilo > ihi || jlo > jhi) continue;
        if ((long long)(ihi - ilo + 1) * (jhi - jlo + 1) > kSmallBudget) {
            overflow[atomicAdd(overflow_count, 1u)] = make_int2(f, (int)t);
            continue;
        }
        unsigned long long* fk = keys + (long long)f * H * W;
        for (int j = jlo; j <= jhi; ++j)
            for (int i = ilo; i <= ihi; ++i) tri_plot(s, (unsigned int)t, i, j, fk, W);
    }
}

__global__ void __launch_bounds__(256) raster_large_kernel(const int* __restrict__ tris, int64_t nv, const int4* __restrict__ sv, int W, int H,
                                                           unsigned long long* __restrict__ keys, const unsigned int* __restrict__ overflow_count,
                                                           const int2* __restrict__ overflow) {
    const unsigned int n = *overflow_count;
    for (unsigned int k = blockIdx.x; k < n; k += gridDim.x) {
        const int2 e = overflow[k];
        const long long t = e.y;
        TriSetup s;
        tri_setup(sv, nv, e.x, tris[3 * t], tris[3 * t + 1], tris[3 * t + 2], s);      // valid: raster_small_kernel listed it
        int ilo, ihi, jlo, jhi;
        tri_bbox(s, W, H, ilo, ihi, jlo, jhi);
        const int bw = ihi - ilo + 1;
        const long long cnt = (long long)bw * (jhi - jlo + 1);
        unsigned long long* fk = keys + (long long)e.x * H * W;
        for (long long p = threadIdx.x; p < cnt; p += blockDim.x)
            tri_plot(s, (unsigned int)t, ilo + (int)(p % bw), jlo + (int)(p / bw), fk, W);
    }
}

// c = base * clamp(ambient + diffuse * |n.l|, 0, 1), l = the camera's view direction (a headlight), stored as round(255 c)
__global__ void __launch_bounds__(256) raster_resolve_kernel(const int* __restrict__ tris, int64_t nv, const float* __restrict__ normals,
                                                             const int4* __restrict__ sv, const float* __restrict__ c2w, int F, int W, int H,
                                                             float base, float ambient, float diffuse, int background,
                                                             const unsigned long long* __restrict__ keys, unsigned char* __restrict__ rgb,
                                                             int* __restrict__ ids) {
    const long long total = (long long)F * H * W;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const unsigned long long key = keys[idx];
        int value = background, id = -1;
        if (key != ~0ull) {
            const int f = (int)(idx / ((long long)H * W));
            const int pix = (int)(idx - (long long)f * H * W);
            const int j = pix / W, i = pix - j * W;
            id = (int)(unsigned int)(key & 0xffffffffull);
            const int v0 = tris[3ll * id], v1 = tris[3ll * id + 1], v2 = tris[3ll * id + 2];
            TriSetup s;
            tri_setup(sv, nv, f, v0, v1, v2, s);
            long long w[3];
            tri_cover(s, i, j, w);
            float q[3];
            const float iw = tri_interp(s, w, q);
            const float p0 = __fdiv_rn(q[0], iw), p1 = __fdiv_rn(q[1], iw), p2 = __fdiv_rn(q[2], iw);
            float n[3];
#pragma unroll
            for (int c = 0; c < 3; ++c)
                n[c] = __fadd_rn(__fadd_rn(__fmul_rn(p0, normals[3ll * v0 + c]), __fmul_rn(p1, normals[3ll * v1 + c])),
                                 __fmul_rn(p2, normals[3ll * v2 + c]));
            const float* M = c2w + 16 * f;
            const float lx = -M[2], ly = -M[6], lz = -M[10];
            const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(n[0], n[0]), __fmul_rn(n[1], n[1])), __fmul_rn(n[2], n[2])));
            const float dot = __fadd_rn(__fadd_rn(__fmul_rn(n[0], lx), __fmul_rn(n[1], ly)), __fmul_rn(n[2], lz));
            const float cosv = len > 0.f ? fminf(__fdiv_rn(fabsf(dot), len), 1.f) : 0.f;
            const float lit = fminf(fmaxf(__fadd_rn(ambient, __fmul_rn(diffuse, cosv)), 0.f), 1.f);
            value = min(255, max(0, __float2int_rn(__fmul_rn(255.f, __fmul_rn(base, lit)))));
        }
        rgb[3 * idx] = rgb[3 * idx + 1] = rgb[3 * idx + 2] = (unsigned char)value;
        if (ids) ids[idx] = id;
    }
}

}  // namespace ide3d

using namespace ide3d;

extern "C" int64_t ide3d_raster_scratch_bytes(int num_frames, int width, int height, int64_t num_vertices, int64_t num_triangles) {
    if (num_frames < 0 || width < 0 || height < 0 || num_vertices < 0 || num_triangles < 0) return -1;
    int64_t ofs[4];
    return raster_layout(num_frames, width, height, num_vertices, num_triangles, ofs);
}

extern "C" int ide3d_mesh_normals(const float* vertices, const int32_t* triangles, int64_t num_vertices, const int32_t* adj_offsets,
                                  const int32_t* adj_faces, float* normals, ide3d_stream_t stream) {
    IDE3D_REQUIRE(num_vertices >= 0, "mesh_normals: negative vertex count");
    if (num_vertices == 0) return IDE3D_OK;
    IDE3D_REQUIRE(vertices && triangles && adj_offsets && adj_faces && normals, "mesh_normals: null argument");
    const unsigned grid = capped_grid(ceil_div<long long>(num_vertices, 256), 16);
    mesh_normals_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(vertices, triangles, num_vertices, adj_offsets,
                                                                adj_faces, normals);
    IDE3D_CHECK_LAUNCH("mesh_normals_kernel");
    return IDE3D_OK;
}

extern "C" int ide3d_raster(const ide3d_raster_params* p, ide3d_stream_t stream) {
    IDE3D_REQUIRE(p, "raster: null params");
    IDE3D_REQUIRE(p->num_frames >= 0 && p->num_vertices >= 0 && p->num_triangles >= 0, "raster: negative count");
    IDE3D_REQUIRE(p->width >= 1 && p->height >= 1 && p->width <= kMaxRes && p->height <= kMaxRes,
                  "raster: resolution %d x %d outside 1..%d", p->width, p->height, kMaxRes);
    IDE3D_REQUIRE(p->num_triangles < (1ll << 31) && p->num_vertices < (1ll << 31), "raster: more than 2^31 - 1 vertices or triangles");
    IDE3D_REQUIRE((long long)p->num_frames * p->num_triangles < (1ll << 32), "raster: frames x triangles must stay below 2^32");
    IDE3D_REQUIRE(p->yfov_deg > 0.f && p->yfov_deg < 180.f, "raster: yfov %g outside (0, 180) degrees", p->yfov_deg);
    IDE3D_REQUIRE(p->znear > 0.f, "raster: znear must be positive");
    IDE3D_REQUIRE(p->background >= 0 && p->background <= 255, "raster: background must be 0..255");
    if (p->num_frames == 0) return IDE3D_OK;
    IDE3D_REQUIRE(p->cam2world && p->rgb && p->scratch, "raster: null cam2world, rgb or scratch");
    IDE3D_REQUIRE(p->num_triangles == 0 || (p->vertices && p->triangles && p->normals), "raster: null vertices, triangles or normals");
    int64_t ofs[4];
    const int64_t need = raster_layout(p->num_frames, p->width, p->height, p->num_vertices, p->num_triangles, ofs);
    IDE3D_REQUIRE(p->scratch_bytes >= need, "raster: scratch of %lld bytes, %lld needed (ide3d_raster_scratch_bytes)",
                  (long long)p->scratch_bytes, (long long)need);
    IDE3D_REQUIRE(((uintptr_t)p->scratch & 255) == 0, "raster: scratch must be 256-byte aligned");
    char* base = static_cast<char*>(p->scratch);
    auto* keys = reinterpret_cast<unsigned long long*>(base + ofs[0]);
    auto* sv = reinterpret_cast<int4*>(base + ofs[1]);
    auto* ocount = reinterpret_cast<unsigned int*>(base + ofs[2]);
    auto* olist = reinterpret_cast<int2*>(base + ofs[3]);
    const cudaStream_t s = (cudaStream_t)stream;
    const int F = p->num_frames, W = p->width, H = p->height;
    const long long npix = (long long)F * H * W;
    // projection: the same double-precision host arithmetic as oracle/rasterizer.py, rounded once to float
    const double fyd = 1.0 / tan(0.5 * ((double)p->yfov_deg * (3.141592653589793 / 180.0)));
    const float fy = (float)fyd, fx = (float)(fyd * H / W);

    const unsigned pix_grid = capped_grid(ceil_div<long long>(npix, 256), 16);
    raster_clear_kernel<<<pix_grid, 256, 0, s>>>(keys, npix, ocount);
    IDE3D_CHECK_LAUNCH("raster_clear_kernel");
    if (p->num_triangles > 0) {
        const unsigned vgrid = capped_grid(ceil_div<long long>((long long)F * p->num_vertices, 256), 16);
        raster_transform_kernel<<<vgrid, 256, 0, s>>>(p->vertices, p->num_vertices, p->cam2world,
                                                      F, W, H, fx, fy, p->znear, sv);
        IDE3D_CHECK_LAUNCH("raster_transform_kernel");
        const unsigned tgrid = capped_grid(ceil_div<long long>((long long)F * p->num_triangles, 128), 32);
        raster_small_kernel<<<tgrid, 128, 0, s>>>(p->triangles, p->num_triangles, p->num_vertices,
                                                  sv, F, W, H, keys, ocount, olist);
        IDE3D_CHECK_LAUNCH("raster_small_kernel");
        raster_large_kernel<<<(unsigned)sm_count() * 4, 256, 0, s>>>(p->triangles, p->num_vertices, sv, W, H, keys, ocount, olist);
        IDE3D_CHECK_LAUNCH("raster_large_kernel");
    }
    raster_resolve_kernel<<<pix_grid, 256, 0, s>>>(p->triangles, p->num_vertices, p->normals, sv, p->cam2world, F, W, H, p->base,
                                                   p->ambient, p->diffuse, p->background, keys, p->rgb, p->ids);
    IDE3D_CHECK_LAUNCH("raster_resolve_kernel");
    return IDE3D_OK;
}
