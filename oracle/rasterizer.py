"""Oracle (test infrastructure): the mesh renderer of ide3d_b200.mesh (csrc/raster.cu) restated in numpy, for bit-for-bit comparison.

render_mesh.py:36-67 draws the marching-cubes mesh with pyrender (OpenGL offscreen, a PBR shader).  That renderer is third-party code
that is absent here, so PARITY UNPINNED for its pixel values; what is pinned by the reference is the camera path, the projection
(PerspectiveCamera(yfov), aspect = width / height, OpenGL axes, row 0 at the top, pixel centres at half-integers) and the image size.
The rules below are this project's, stated once in DESIGN.md §3 and followed operation for operation by the CUDA kernels:

  - camera space = R^T (p - t) for the rigid cam2world [R | t]; w = -z_cam; clip x = fx x_cam, y = fy y_cam with
    fy = 1 / tan(yfov / 2), fx = fy * H / W computed in double and rounded once to float32;
  - screen X = (x / w + 1) * W/2, Y = (1 - y / w) * H/2, snapped to 1/256 pixel (round half to even); a triangle is dropped when a
    vertex has w < znear or lies more than 16384 pixels outside the viewport;
  - coverage: exact int64 edge functions at the pixel centres, top-left fill rule (orientation normalised first);
  - depth at a covered centre: 1 / sum_k (w_k / area) * (1 / w_k) in float32, key = bits(depth) << 32 | triangle, minimum wins;
  - shading: perspective-correct normal, c = base * clamp(ambient + diffuse * |n . l|, 0, 1), l = the camera's view direction,
    stored as round(255 c) (round half to even).
Every float32 operation is a numpy float32 array operation (each one rounded, no fused multiply-add), in the CUDA kernels' order.
Never imported by the product package."""

import math

import numpy as np

SUB = 256
GUARD = np.float32(16384.0)
F32 = np.float32
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)


def projection(yfov_deg, width, height):
    """-> (fx, fy) float32, the host arithmetic of ide3d_raster."""
    fyd = 1.0 / math.tan(0.5 * (float(np.float32(yfov_deg)) * (3.141592653589793 / 180.0)))
    return np.float32(fyd * height / width), np.float32(fyd)


def vertex_normals(vertices, triangles):
    """Area-weighted smooth normals: per vertex the cross products of its faces summed in ascending face order, normalised."""
    v = np.asarray(vertices, np.float32)
    t = np.asarray(triangles, np.int64).reshape(-1, 3)
    V = len(v)
    out = np.zeros((V, 3), np.float32)
    if len(t) == 0 or V == 0:
        return out
    p0, p1, p2 = v[t[:, 0]], v[t[:, 1]], v[t[:, 2]]
    a, b = p1 - p0, p2 - p0
    fn = np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2], a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)
    flat = t.reshape(-1)
    faces = np.argsort(flat, kind='stable') // 3                         # CSR: the faces of each vertex in ascending order
    counts = np.bincount(flat, minlength=V)
    offs = np.concatenate([[0], np.cumsum(counts)])
    s = np.zeros((V, 3), np.float32)
    for k in range(int(counts.max())):
        m = counts > k
        s[m] = s[m] + fn[faces[offs[:-1][m] + k]]
    ln = np.sqrt((s[:, 0] * s[:, 0] + s[:, 1] * s[:, 1]) + s[:, 2] * s[:, 2])
    ok = ln > 0
    out[ok] = s[ok] / ln[ok, None]
    return out


def screen_vertices(vertices, cam2world, width, height, yfov_deg, znear):
    """One frame: -> (X, Y int64 fixed point, 1/w float32, valid bool) per vertex."""
    v = np.asarray(vertices, np.float32)
    M = np.asarray(cam2world, np.float32).reshape(4, 4)
    fx, fy = projection(yfov_deg, width, height)
    d = v - M[:3, 3]
    cam = [(M[0, c] * d[:, 0] + M[1, c] * d[:, 1]) + M[2, c] * d[:, 2] for c in range(3)]
    w = -cam[2]
    with np.errstate(all='ignore'):
        valid = w >= F32(znear)
        X = ((fx * cam[0]) / w + F32(1)) * F32(0.5 * width)
        Y = (F32(1) - (fy * cam[1]) / w) * F32(0.5 * height)
        valid &= (X >= -GUARD) & (X <= F32(width) + GUARD) & (Y >= -GUARD) & (Y <= F32(height) + GUARD)
        xs = np.where(valid, np.rint(X * F32(SUB)), 0).astype(np.int64)
        ys = np.where(valid, np.rint(Y * F32(SUB)), 0).astype(np.int64)
        iw = np.where(valid, F32(1) / w, F32(0)).astype(np.float32)
    return xs, ys, iw, valid


def _setup(sv, tris):
    """Per triangle: fixed-point corners [T,3], 1/w [T,3], |area|, orientation sign, top-left need [T,3], ok."""
    xs, ys, iw, valid = sv
    x, y, q = xs[tris], ys[tris], iw[tris]
    ok = valid[tris].all(1)
    area = (x[:, 1] - x[:, 0]) * (y[:, 2] - y[:, 0]) - (y[:, 1] - y[:, 0]) * (x[:, 2] - x[:, 0])
    ok &= area != 0
    sgn = np.where(area > 0, 1, -1).astype(np.int64)
    need = np.zeros(x.shape, np.int64)
    for k in range(3):
        p, r = (k + 1) % 3, (k + 2) % 3
        dx, dy = (x[:, r] - x[:, p]) * sgn, (y[:, r] - y[:, p]) * sgn
        need[:, k] = np.where((dy < 0) | ((dy == 0) & (dx > 0)), 0, 1)
    return x, y, q, np.abs(area), sgn, need, ok


def _edges(x, y, sgn, px, py):
    return [((x[:, (k + 2) % 3] - x[:, (k + 1) % 3]) * (py - y[:, (k + 1) % 3])
             - (y[:, (k + 2) % 3] - y[:, (k + 1) % 3]) * (px - x[:, (k + 1) % 3])) * sgn for k in range(3)]


def _interp(w, area, q):
    A = area.astype(np.float32)
    qq = [(w[k].astype(np.float32) / A) * q[:, k] for k in range(3)]
    return qq, (qq[0] + qq[1]) + qq[2]


def raster_keys(vertices, triangles, cam2world, width, height, yfov_deg=18.0, znear=0.05):
    """One frame -> (keys uint64 [H*W], screen vertices)."""
    tris = np.asarray(triangles, np.int64).reshape(-1, 3)
    sv = screen_vertices(vertices, cam2world, width, height, yfov_deg, znear)
    keys = np.full(height * width, EMPTY, np.uint64)
    if len(tris) == 0:
        return keys, sv
    x, y, q, area, sgn, need, ok = _setup(sv, tris)
    ilo = np.maximum(0, (x.min(1) - SUB // 2 + SUB - 1) // SUB)
    ihi = np.minimum(width - 1, (x.max(1) - SUB // 2) // SUB)
    jlo = np.maximum(0, (y.min(1) - SUB // 2 + SUB - 1) // SUB)
    jhi = np.minimum(height - 1, (y.max(1) - SUB // 2) // SUB)
    ok &= (ilo <= ihi) & (jlo <= jhi)
    t = np.nonzero(ok)[0]
    if len(t) == 0:
        return keys, sv
    bw = (ihi - ilo + 1)[t]
    n = bw * (jhi - jlo + 1)[t]
    tt = np.repeat(t, n)
    local = np.arange(int(n.sum()), dtype=np.int64) - np.repeat(np.cumsum(n) - n, n)
    i = ilo[tt] + local % np.repeat(bw, n)
    j = jlo[tt] + local // np.repeat(bw, n)
    w = _edges(x[tt], y[tt], sgn[tt], i * SUB + SUB // 2, j * SUB + SUB // 2)
    cov = (w[0] >= need[tt, 0]) & (w[1] >= need[tt, 1]) & (w[2] >= need[tt, 2])
    tt, i, j, w = tt[cov], i[cov], j[cov], [e[cov] for e in w]
    _, iwp = _interp(w, area[tt], q[tt])
    depth = F32(1) / iwp
    key = (depth.view(np.uint32).astype(np.uint64) << np.uint64(32)) | tt.astype(np.uint64)
    np.minimum.at(keys, j * width + i, key)
    return keys, sv


def rasterize(vertices, triangles, cam2world, resolution=512, yfov=18.0, znear=0.05, normals=None, return_ids=False,
              base=0.85, ambient=0.25, diffuse=0.75, background=255):
    """vertices [V,3], triangles [T,3], cam2world [F,4,4] or [F,16] -> rgb uint8 [F,H,W,3] (and ids int32 [F,H,W], -1 = background).
    resolution: int (square) or (W, H)."""
    W, H = (resolution, resolution) if np.isscalar(resolution) else (int(resolution[0]), int(resolution[1]))
    v = np.asarray(vertices, np.float32).reshape(-1, 3)
    tris = np.asarray(triangles, np.int64).reshape(-1, 3)
    nrm = vertex_normals(v, tris) if normals is None else np.asarray(normals, np.float32).reshape(-1, 3)
    c2w = np.asarray(cam2world, np.float32).reshape(-1, 16)
    rgb = np.empty((len(c2w), H, W, 3), np.uint8)
    ids = np.empty((len(c2w), H, W), np.int32)
    for f, M in enumerate(c2w):
        keys, sv = raster_keys(v, tris, M, W, H, yfov, znear)
        value = np.full(H * W, background, np.int64)
        idf = np.full(H * W, -1, np.int64)
        pix = np.nonzero(keys != EMPTY)[0]
        if len(pix):
            tt = (keys[pix] & np.uint64(0xFFFFFFFF)).astype(np.int64)
            x, y, q, area, sgn, need, _ = _setup(sv, tris[tt])
            w = _edges(x, y, sgn, (pix % W) * SUB + SUB // 2, (pix // W) * SUB + SUB // 2)
            qq, iwp = _interp(w, area, q)
            p = [qq[k] / iwp for k in range(3)]
            nv = [nrm[tris[tt, k]] for k in range(3)]
            n = [(p[0] * nv[0][:, c] + p[1] * nv[1][:, c]) + p[2] * nv[2][:, c] for c in range(3)]
            l = -M.reshape(4, 4)[:3, 2]
            ln = np.sqrt((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2])
            dot = (n[0] * l[0] + n[1] * l[1]) + n[2] * l[2]
            with np.errstate(all='ignore'):
                cos = np.where(ln > 0, np.minimum(np.abs(dot) / ln, F32(1)), F32(0)).astype(np.float32)
            lit = np.clip(F32(ambient) + F32(diffuse) * cos, F32(0), F32(1))
            value[pix] = np.clip(np.rint(F32(255) * (F32(base) * lit)), 0, 255).astype(np.int64)
            idf[pix] = tt
        rgb[f] = value.reshape(H, W, 1).astype(np.uint8)
        ids[f] = idf.reshape(H, W)
    return (rgb, ids) if return_ids else rgb
