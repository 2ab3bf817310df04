// Marching cubes on the density grid (the step after extract_shapes' sigma grid: render_mesh.py:30-32 calls
// mcubes.marching_cubes(voxel_grid, sigma_threshold) on the host -- PyMCubes, a third-party dependency that is not in the reference
// tree; the algorithm is Lorensen & Cline's with the table generated in ide3d_b200/mesh.py).  Two kernels around one library scan:
//   ide3d_mc_classify  cell -> 8-bit corner configuration -> number of triangles               (1 byte per cell)
//   ide3d_mc_emit      cell -> its triangles: per vertex the global edge id (lower corner * 3 + axis) and the interpolated position,
//                      always evaluated from the edge's lower corner to its upper corner, so that the copies of a vertex emitted
//                      by the (up to four) cells sharing the edge are bit-identical and de-duplicate exactly by edge id.
// Volume [nx, ny, nz] fp32 dense, index = (x * ny + y) * nz + z; vertex coordinates are in index units, (x, y, z) order, like PyMCubes.
#include "common.cuh"

namespace ide3d {

__device__ __forceinline__ int mc_config(const float* __restrict__ v, int ny, int nz, int x, int y, int z, float iso, float (&val)[8]) {
    int cfg = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int cx = x + (i & 1), cy = y + ((i >> 1) & 1), cz = z + ((i >> 2) & 1);
        val[i] = v[((long long)cx * ny + cy) * nz + cz];
        cfg |= (val[i] < iso) ? 0 : (1 << i);                 // bit set = corner inside the surface (value >= threshold)
    }
    return cfg;
}

__global__ void __launch_bounds__(256) mc_classify_kernel(const float* __restrict__ v, int nx, int ny, int nz, float iso,
                                                          const int* __restrict__ ntri, unsigned char* __restrict__ counts) {
    const long long cells = (long long)(nx - 1) * (ny - 1) * (nz - 1);
    for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < cells; c += (long long)gridDim.x * blockDim.x) {
        const int z = (int)(c % (nz - 1));
        const long long r = c / (nz - 1);
        const int y = (int)(r % (ny - 1)), x = (int)(r / (ny - 1));
        float val[8];
        counts[c] = (unsigned char)ntri[mc_config(v, ny, nz, x, y, z, iso, val)];
    }
}

__global__ void __launch_bounds__(256) mc_emit_kernel(const float* __restrict__ v, int nx, int ny, int nz, float iso,
                                                      const signed char* __restrict__ tri, const int* __restrict__ edge_corner,
                                                      const unsigned char* __restrict__ counts, const long long* __restrict__ offsets,
                                                      long long* __restrict__ edge_ids, float* __restrict__ verts) {
    const long long cells = (long long)(nx - 1) * (ny - 1) * (nz - 1);
    for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < cells; c += (long long)gridDim.x * blockDim.x) {
        const int nt = counts[c];
        if (nt == 0) continue;
        const int z = (int)(c % (nz - 1));
        const long long r = c / (nz - 1);
        const int y = (int)(r % (ny - 1)), x = (int)(r / (ny - 1));
        float val[8];
        const int cfg = mc_config(v, ny, nz, x, y, z, iso, val);
        const long long first = offsets[c] - nt;                 // offsets = inclusive scan of counts
        for (int k = 0; k < 3 * nt; ++k) {
            const int e = tri[cfg * 16 + k];
            const int c0 = edge_corner[2 * e], c1 = edge_corner[2 * e + 1];          // c0 = lower corner, c1 = c0 | 1 << axis
            const int axis = e >> 2;
            const int px = x + (c0 & 1), py = y + ((c0 >> 1) & 1), pz = z + ((c0 >> 2) & 1);
            const float f0 = val[c0], f1 = val[c1];
            const float t = (f1 == f0) ? 0.5f : __fdiv_rn(__fsub_rn(iso, f0), __fsub_rn(f1, f0));
            float p[3] = {(float)px, (float)py, (float)pz};
            p[axis] = __fadd_rn(p[axis], t);
            const long long o = first * 3 + k;
            edge_ids[o] = (((long long)px * ny + py) * nz + pz) * 3 + axis;
            verts[o * 3] = p[0]; verts[o * 3 + 1] = p[1]; verts[o * 3 + 2] = p[2];
        }
    }
}

}  // namespace ide3d

using namespace ide3d;

extern "C" int ide3d_mc_classify(const float* volume, int nx, int ny, int nz, float threshold, const int* ntri_table,
                                 unsigned char* counts, ide3d_stream_t stream) {
    IDE3D_REQUIRE(volume && ntri_table && counts, "mc_classify: null argument");
    IDE3D_REQUIRE(nx >= 2 && ny >= 2 && nz >= 2, "mc_classify: the grid needs at least 2 points per axis");
    const long long cells = (long long)(nx - 1) * (ny - 1) * (nz - 1);
    mc_classify_kernel<<<capped_grid(ceil_div<long long>(cells, 256), 16), 256, 0, (cudaStream_t)stream>>>(volume, nx, ny, nz, threshold, ntri_table, counts);
    IDE3D_CHECK_LAUNCH("mc_classify_kernel");
    return IDE3D_OK;
}

extern "C" int ide3d_mc_emit(const float* volume, int nx, int ny, int nz, float threshold, const signed char* tri_table,
                             const int* edge_corner, const unsigned char* counts, const int64_t* offsets, int64_t* edge_ids,
                             float* verts, ide3d_stream_t stream) {
    IDE3D_REQUIRE(volume && tri_table && edge_corner && counts && offsets && edge_ids && verts, "mc_emit: null argument");
    IDE3D_REQUIRE(nx >= 2 && ny >= 2 && nz >= 2, "mc_emit: the grid needs at least 2 points per axis");
    const long long cells = (long long)(nx - 1) * (ny - 1) * (nz - 1);
    const unsigned grid = capped_grid(ceil_div<long long>(cells, 256), 16);
    mc_emit_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(volume, nx, ny, nz, threshold, tri_table, edge_corner, counts,
                                                           reinterpret_cast<const long long*>(offsets),
                                                           reinterpret_cast<long long*>(edge_ids), verts);
    IDE3D_CHECK_LAUNCH("mc_emit_kernel");
    return IDE3D_OK;
}
