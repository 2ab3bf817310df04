"""Marching cubes on the GPU: the step that follows extract_shapes' sigma grid (render_mesh.py:30-32,
`vertices, triangles = mcubes.marching_cubes(voxel_grid, sigma_threshold)`; dnnlib/geometry.py:282-286 calls it the same way).

PyMCubes (environment.yml:29, unpinned) is a third-party dependency that is not part of the reference tree, so this is a restatement of
the published algorithm (Lorensen & Cline 1987), not of PyMCubes' source: cell configuration from the 8 corner signs, triangles from a
256-entry table, vertices by linear interpolation along the cut edges, one indexed mesh (vertices shared between cells).  The table is
GENERATED here from first principles (`build_tables`) rather than typed in: per configuration the cut edges are linked into closed loops
face by face and fan-triangulated; the ambiguous faces (two diagonal inside corners) always separate the inside corners, the same rule
for both cells that share the face, which makes the surface watertight.  The generated table has the classic shape (820 triangles over
the 256 configurations, at most 5 per cell).  Conventions: volume indexed [x, y, z] and vertices in index units (as PyMCubes documents),
a corner is inside where value >= threshold, triangle normals point out of the inside region.  PyMCubes' own vertex / triangle order and its
choices on ambiguous faces are not recoverable here, so parity with it is unpinned; the tests pin the geometry instead (watertightness,
Euler characteristic, vertices on the iso-level, area / volume of analytic shapes) and the CUDA kernels against the numpy oracle bit for bit.

    vertices, triangles = marching_cubes(volume, threshold)      # volume: CUDA tensor [nx, ny, nz] (any float dtype)

The rest of render_mesh.py (:36-67, a shaded turntable drawn with pyrender) is `render_turntable`: smooth normals (`vertex_normals`) and
the frames (`rasterize`, csrc/raster.cu) on the device, the camera path of the reference (`turntable_poses`).
"""

import ctypes as C
import math

import numpy as np
import torch

from . import _lib as L


def build_tables():
    """-> tri [256,16] int8 (edge triples, -1 terminated), ntri [256] int32, edge_corner [12,2] int32.
    corner i = (i & 1, i >> 1 & 1, i >> 2 & 1); edge e = axis * 4 + k joins corner c0 (bit `axis` clear, k-th such corner) and c0 | 1 << axis."""
    corners = np.array([[i & 1, (i >> 1) & 1, (i >> 2) & 1] for i in range(8)])
    edge_corner = [(c0, c0 | (1 << a)) for a in range(3) for c0 in range(8) if not (c0 >> a) & 1]
    edge_of = {frozenset(ec): e for e, ec in enumerate(edge_corner)}
    faces = []
    for a in range(3):
        b, c = [(1, 2), (0, 2), (0, 1)][a]
        for val in (0, 1):
            cyc = []
            for vb, vc in ((0, 0), (1, 0), (1, 1), (0, 1)):
                p = [0, 0, 0]
                p[a], p[b], p[c] = val, vb, vc
                cyc.append(p[0] | (p[1] << 1) | (p[2] << 2))
            faces.append(cyc)
    tri = -np.ones((256, 16), np.int8)
    ntri = np.zeros(256, np.int32)
    for cfg in range(256):
        inside = [(cfg >> i) & 1 for i in range(8)]
        adj = {}
        for cyc in faces:
            fl = [inside[c] for c in cyc]
            fe = [edge_of[frozenset((cyc[k], cyc[(k + 1) % 4]))] for k in range(4)]
            cross = [k for k in range(4) if fl[k] != fl[(k + 1) % 4]]
            pairs = []
            if len(cross) == 2:
                pairs = [(fe[cross[0]], fe[cross[1]])]
            elif len(cross) == 4:                                   # ambiguous face: cut off each inside corner on its own
                pairs = [(fe[(k - 1) % 4], fe[k]) for k in range(4) if fl[k]]
            for e1, e2 in pairs:
                adj.setdefault(e1, []).append(e2)
                adj.setdefault(e2, []).append(e1)
        seen, out = set(), []
        for e0 in sorted(adj):
            if e0 in seen:
                continue
            loop, prev, cur = [e0], None, e0
            seen.add(e0)
            while True:
                n = adj[cur][0] if prev is None else [x for x in adj[cur] if x != prev][0]
                if n == e0:
                    break
                loop.append(n)
                seen.add(n)
                prev, cur = cur, n
            # orientation: the loop normal points from the inside corners to the outside ones
            mid = np.array([(corners[edge_corner[e][0]] + corners[edge_corner[e][1]]) / 2.0 for e in loop])
            g = np.zeros(3)
            for e in loop:
                c0, c1 = edge_corner[e]
                g += (corners[c1] - corners[c0]) * (1 if inside[c0] else -1)
            nrm = sum(np.cross(mid[i], mid[(i + 1) % len(loop)]) for i in range(len(loop)))
            if np.dot(nrm, g) < 0:
                loop = loop[::-1]
            for i in range(1, len(loop) - 1):
                out += [loop[0], loop[i], loop[i + 1]]
        assert len(out) <= 15
        tri[cfg, :len(out)] = out
        ntri[cfg] = len(out) // 3
    return tri, ntri, np.array(edge_corner, np.int32)


_tables = {}


def _device_tables(device):
    key = str(device)
    if key not in _tables:
        tri, ntri, ec = build_tables()
        _tables[key] = (torch.from_numpy(tri).to(device), torch.from_numpy(ntri).to(device), torch.from_numpy(ec).to(device).contiguous())
    return _tables[key]


@torch.no_grad()
def marching_cubes(volume, threshold):
    """volume [nx, ny, nz] on a CUDA device -> (vertices [V, 3] float32 in index units (x, y, z), triangles [T, 3] int64).
    Inside = value >= threshold; triangle normals point from inside to outside.  Vertices are shared between the cells that cut the same
    grid edge (de-duplicated exactly by edge id) and ordered by that id; triangles are ordered by cell."""
    L.require_cuda(volume)
    if volume.ndim != 3:
        raise ValueError('marching_cubes: volume must be a 3-D array')
    v = volume.detach().to(torch.float32).contiguous()
    nx, ny, nz = v.shape
    if min(nx, ny, nz) < 2:
        raise ValueError('marching_cubes: the grid needs at least 2 points per axis')
    dev = v.device
    tri, ntri, ec = _device_tables(dev)
    cells = (nx - 1) * (ny - 1) * (nz - 1)
    counts = torch.empty(cells, dtype=torch.uint8, device=dev)
    lib = L.get_lib()
    with torch.cuda.device(dev):
        L.check(lib.ide3d_mc_classify(L.ptr(v), nx, ny, nz, float(threshold), L.ptr(ntri), L.ptr(counts), L.stream_ptr(dev)))
        offsets = torch.cumsum(counts, 0, dtype=torch.int64)                       # the one library call: an inclusive scan
        total = int(offsets[-1].item()) if cells else 0
        if total == 0:
            return torch.zeros(0, 3, device=dev), torch.zeros(0, 3, dtype=torch.int64, device=dev)
        edge_ids = torch.empty(total * 3, dtype=torch.int64, device=dev)
        verts = torch.empty(total * 3, 3, dtype=torch.float32, device=dev)
        L.check(lib.ide3d_mc_emit(L.ptr(v), nx, ny, nz, float(threshold), L.ptr(tri), L.ptr(ec), L.ptr(counts), L.ptr(offsets),
                                  L.ptr(edge_ids), L.ptr(verts), L.stream_ptr(dev)))
    uniq, inverse = torch.unique(edge_ids, return_inverse=True)                     # vertex = cut grid edge
    vertices = torch.empty(uniq.numel(), 3, dtype=torch.float32, device=dev)
    vertices[inverse] = verts                                                       # duplicates are bit-identical by construction
    return vertices, inverse.reshape(total, 3)


@torch.no_grad()
def mesh_from_sigma_grid(sigma, size=None, sigma_threshold=10.0):
    """render_mesh.py:29-32 on the device: clamp the density grid at 0, marching cubes at `sigma_threshold`, vertices scaled by 1/size.
    sigma: [n, n, n] (or flat n^3, the layout extract_shapes.py writes) CUDA tensor.  -> (vertices [V,3] in [0,1), triangles [T,3])."""
    if sigma.ndim == 1:
        n = round(sigma.numel() ** (1 / 3))
        sigma = sigma.reshape(n, n, n)
    size = sigma.shape[0] if size is None else size
    vertices, triangles = marching_cubes(torch.clamp_min(sigma, 0), sigma_threshold)
    return vertices / float(size), triangles


# ---------------------------------------------------------------------------------------------------------------- rendering
# render_mesh.py:36-67 draws the mesh with pyrender (OpenGL offscreen, which needs a GL context).  Here: csrc/raster.cu, a visibility
# buffer resolved by 64-bit atomics, one call per batch of frames.  The camera path and projection are the reference's; the shading is
# this project's stated choice (DESIGN.md §3): grey, two-sided Lambert headlight plus ambient, no anti-aliasing, no culling.
MATERIAL = dict(base=0.85, ambient=0.25, diffuse=0.75, background=255)


def _check_mesh(vertices, triangles):
    L.require_cuda(vertices, triangles)
    if vertices.ndim != 2 or vertices.shape[1] != 3 or triangles.ndim != 2 or triangles.shape[1] != 3:
        raise ValueError('mesh: vertices must be [V, 3] and triangles [T, 3]')
    if vertices.shape[0] >= 2 ** 31 or triangles.shape[0] >= 2 ** 31:
        raise ValueError('mesh: at most 2^31 - 1 vertices and triangles')
    v = vertices.detach().to(torch.float32).contiguous()
    t = triangles.detach().to(device=v.device, dtype=torch.int32).contiguous()
    if t.numel() and (int(t.min()) < 0 or int(t.max()) >= v.shape[0]):
        raise ValueError('mesh: triangle index out of range')
    return v, t


@torch.no_grad()
def vertex_normals(vertices, triangles):
    """Smooth vertex normals (trimesh's, used by pyrender with smooth=True): per vertex the sum of its faces' cross products
    (area-weighted), normalised; (0, 0, 0) where the sum vanishes.  The vertex -> face adjacency is sorted here once, so the
    kernel sums in a fixed order and the result is the same on every run.  -> [V, 3] float32 on the vertices' device."""
    v, t = _check_mesh(vertices, triangles)
    V = v.shape[0]
    normals = torch.zeros(V, 3, dtype=torch.float32, device=v.device)
    if V == 0 or t.shape[0] == 0:
        return normals
    flat = t.reshape(-1).long()
    faces = (torch.sort(flat, stable=True)[1] // 3).to(torch.int32)               # stable: ascending face index per vertex
    offsets = torch.zeros(V + 1, dtype=torch.int32, device=v.device)
    offsets[1:] = torch.cumsum(torch.bincount(flat, minlength=V), 0)
    L.check(L.get_lib().ide3d_mesh_normals(L.ptr(v), L.ptr(t), V, L.ptr(offsets), L.ptr(faces), L.ptr(normals), L.stream_ptr(v.device)))
    return normals


def turntable_poses(w_frames=240, radius=2.7):
    """render_mesh.py:44-55: cam2world [F, 4, 4] float32 (CPU) of the turntable that circles the unit-cube mesh, looking at its
    centre (0.5, 0.5, 0.5).  Computed as the reference does, per frame with sample_camera_positions / create_cam2world_matrix."""
    from .training.volumetric_rendering import create_cam2world_matrix, sample_camera_positions
    poses = []
    for i in range(w_frames):
        yaw = math.pi * (0.5 + 0.15 * math.cos(2 * math.pi * i / w_frames))
        pitch = math.pi * (0.5 - 0.05 * math.sin(2 * math.pi * i / w_frames))
        p, _, _ = sample_camera_positions(None, n=1, r=radius, horizontal_mean=yaw, vertical_mean=pitch, mode=None)
        P = create_cam2world_matrix(-p, p, device=None).reshape(-1, 4, 4)[0].clone()
        P[:3, 3] += 0.5
        poses.append(P)
    return torch.stack(poses) if poses else torch.zeros(0, 4, 4)


@torch.no_grad()
def rasterize(vertices, triangles, cam2world, resolution=512, yfov=18.0, znear=0.05, normals=None, return_ids=False, **material):
    """Shaded frames of one mesh, one per camera: pyrender's PerspectiveCamera(yfov) on an OffscreenRenderer (OpenGL axes, aspect
    W / H, row 0 at the top) with a headlight.  vertices [V,3], triangles [T,3] on a CUDA device; cam2world [F,4,4] or [F,16], rigid;
    resolution: int or (W, H); material: base, ambient, diffuse (floats) and background (0..255), defaults MATERIAL.
    -> rgb uint8 [F,H,W,3] (and ids int32 [F,H,W], the visible triangle or -1, with return_ids)."""
    unknown = set(material) - set(MATERIAL)
    if unknown:
        raise TypeError(f'rasterize: unknown material keys {sorted(unknown)}')
    mat = dict(MATERIAL, **material)
    v, t = _check_mesh(vertices, triangles)
    dev = v.device
    W, H = (resolution, resolution) if isinstance(resolution, int) else (int(resolution[0]), int(resolution[1]))
    c2w = torch.as_tensor(cam2world).detach().to(device=dev, dtype=torch.float32).reshape(-1, 16).contiguous()
    F = c2w.shape[0]
    n = vertex_normals(v, t) if normals is None else normals.detach().to(device=dev, dtype=torch.float32).contiguous()
    if n.shape != v.shape:
        raise ValueError('rasterize: normals must be [V, 3] like the vertices')
    rgb = torch.empty(F, H, W, 3, dtype=torch.uint8, device=dev)
    ids = torch.empty(F, H, W, dtype=torch.int32, device=dev) if return_ids else None
    lib = L.get_lib()
    need = int(lib.ide3d_raster_scratch_bytes(F, W, H, v.shape[0], t.shape[0]))
    if need < 0:
        raise ValueError(f'rasterize: bad sizes (frames {F}, resolution {W} x {H})')
    scratch = torch.empty(max(need, 1), dtype=torch.uint8, device=dev)          # caching-allocator blocks are 512-byte aligned
    p = L.RasterParams(L.ptr(v), L.ptr(t), L.ptr(n), L.ptr(c2w), v.shape[0], t.shape[0], F, W, H, float(yfov), float(znear),
                       float(mat['base']), float(mat['ambient']), float(mat['diffuse']), int(mat['background']),
                       L.ptr(rgb), L.ptr(ids), L.ptr(scratch), scratch.numel())
    L.check(lib.ide3d_raster(C.byref(p), L.stream_ptr(dev)))
    return (rgb, ids) if return_ids else rgb


@torch.no_grad()
def render_turntable(sigma, size=None, sigma_threshold=10.0, w_frames=240, resolution=512, batch=8, **material):
    """render_mesh.render on the device: marching cubes of the clamped density grid (mesh_from_sigma_grid), the normals once, then
    the turntable frames rasterised `batch` at a time.  sigma: [n,n,n] (or flat n^3) CUDA tensor.  -> uint8 [F, H, W, 3] on its device."""
    vertices, triangles = mesh_from_sigma_grid(sigma, size=size, sigma_threshold=sigma_threshold)
    normals = vertex_normals(vertices, triangles)
    poses = turntable_poses(w_frames)
    frames = [rasterize(vertices, triangles, poses[k:k + batch], resolution=resolution, normals=normals, **material)
              for k in range(0, w_frames, batch)]
    if not frames:
        W, H = (resolution, resolution) if isinstance(resolution, int) else resolution
        return torch.zeros(0, H, W, 3, dtype=torch.uint8, device=sigma.device)
    return torch.cat(frames)
