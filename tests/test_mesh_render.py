"""Mesh rendering (render_mesh.py:44-67: a shaded turntable of the marching-cubes mesh).  pyrender's PBR pixels are third-party and
unpinned; pinned are the camera path (golden poses from the reference), the projection and image orientation, the fill and visibility
rules (oracle properties, CPU) and the CUDA kernels against oracle/rasterizer.py bit for bit (GPU)."""

import math
import os

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import marching_cubes as omc
from oracle import rasterizer as ora

FY18 = 1.0 / math.tan(math.radians(9.0))


def _sphere_field(n, r, centre):
    g = np.arange(n, dtype=np.float32)
    x, y, z = np.meshgrid(g, g, g, indexing='ij')
    return (r - np.sqrt((x - centre) ** 2 + (y - centre) ** 2 + (z - centre) ** 2)).astype(np.float32)


def _eye():
    return np.eye(4, dtype=np.float32)[None]                      # camera at the origin looking down -z, +y up


def _from_screen(points, W, H, yfov=18.0):
    """(X, Y, w) screen position in pixels (row 0 at the top) and view depth -> camera-space point (identity camera)."""
    fy = 1.0 / math.tan(math.radians(yfov) / 2)
    fx = fy * H / W
    out = []
    for X, Y, w in points:
        out.append([(X / (W / 2) - 1) * w / fx, (1 - Y / (H / 2)) * w / fy, -w])
    return np.array(out, np.float32)


def _disc_area(radius_world, dist, H, yfov=18.0):
    r_px = math.tan(math.asin(radius_world / dist)) / math.tan(math.radians(yfov) / 2) * H / 2
    return math.pi * r_px ** 2, r_px


# ----------------------------------------------------------------------------------------------------------------- CPU
def test_turntable_poses_equal_the_reference_golden():
    from ide3d_b200 import mesh
    g = load_golden('mesh_turntable')
    P = mesh.turntable_poses(int(g['w_frames']), float(g['radius']))
    assert P.dtype == torch.float32 and P.shape == (240, 4, 4)
    assert np.abs(P.numpy() - g['poses']).max() <= 1e-6
    # every camera looks at the centre of the unit cube from 2.7 away
    c = P.numpy()[:, :3, 3] - 0.5
    assert np.allclose(np.linalg.norm(c, axis=1), 2.7, atol=1e-5)
    assert np.allclose(np.einsum('fi,fi->f', -P.numpy()[:, :3, 2], -c / 2.7), 1.0, atol=1e-5)


def test_oracle_shared_edge_covers_each_pixel_exactly_once():
    W = H = 64
    # the diagonal A-C runs through the pixel centres (k + .5, k + .5): the fill rule must give each of them to one triangle
    A, B, C, D = (10.5, 10.5, 3.0), (52.3, 14.1, 3.5), (50.5, 50.5, 4.0), (12.2, 47.7, 2.8)
    v = _from_screen([A, B, C, D], W, H)
    quad = np.array([[0, 1, 2], [0, 2, 3]])
    cov = []
    for t in ([quad[0]], [quad[1]]):
        _, ids = ora.rasterize(v, np.array(t), _eye(), resolution=W, return_ids=True)
        cov.append(ids[0] >= 0)
    _, ids = ora.rasterize(v, quad, _eye(), resolution=W, return_ids=True)
    assert not (cov[0] & cov[1]).any()
    assert np.array_equal(cov[0] | cov[1], ids[0] >= 0)
    assert np.array_equal(ids[0] == 0, cov[0]) and np.array_equal(ids[0] == 1, cov[1])
    # the union is the quad's set of pixel centres (exact: integer edge functions on the snapped corners); the only centres on its
    # outline are the corners A and C themselves, which the fill rule may give or not
    xs, ys, _, _ = ora.screen_vertices(v, _eye()[0], W, H, 18.0, 0.05)
    jj, ii = np.mgrid[0:H, 0:W]
    px, py = ii * 256 + 128, jj * 256 + 128
    e = [(xs[(k + 1) % 4] - xs[k]) * (py - ys[k]) - (ys[(k + 1) % 4] - ys[k]) * (px - xs[k]) for k in range(4)]
    closed = np.all([ek >= 0 for ek in e], 0) | np.all([ek <= 0 for ek in e], 0)
    inside = np.all([ek > 0 for ek in e], 0) | np.all([ek < 0 for ek in e], 0)
    assert sorted(zip(*np.nonzero(closed & ~inside))) == [(10, 10), (50, 50)]
    covered = ids[0] >= 0
    assert covered[inside].all() and not covered[~closed].any()
    diag = [(k, k) for k in range(11, 50)]
    assert all(ids[0][j, i] >= 0 for i, j in diag)


def _small_sphere(n=16, r=5.3, size=None, centre=None):
    c = (n / 2.0) if centre is None else centre
    v, t = omc.marching_cubes(_sphere_field(n, r, c), 0.0)
    return v / float(size or n), t


def test_oracle_triangle_order_does_not_change_the_image():
    v, t = _small_sphere()
    poses = load_golden('mesh_turntable')['poses'][[0, 70]]
    rgb, ids = ora.rasterize(v, t, poses, resolution=(48, 40), return_ids=True)
    assert (ids >= 0).sum() > 400
    perm = np.random.RandomState(0).permutation(len(t))
    rgb2, ids2 = ora.rasterize(v, t[perm], poses, resolution=(48, 40), return_ids=True)
    assert np.array_equal(rgb, rgb2)
    assert np.array_equal(np.where(ids2 >= 0, perm[np.maximum(ids2, 0)], -1), ids)


def test_oracle_occlusion_nearest_wins_and_ties_go_to_the_lower_index():
    W = H = 48
    near = _from_screen([(8.3, 8.3, 3.0), (30.7, 8.3, 3.0), (30.7, 30.7, 3.0), (8.3, 30.7, 3.0)], W, H)
    far = _from_screen([(18.2, 18.2, 4.0), (40.6, 18.2, 4.0), (40.6, 40.6, 4.0), (18.2, 40.6, 4.0)], W, H)
    q = np.array([[0, 1, 2], [0, 2, 3]])
    for first, second, near_ids in ((near, far, (0, 1)), (far, near, (2, 3))):
        v = np.concatenate([first, second])
        _, ids = ora.rasterize(v, np.concatenate([q, q + 4]), _eye(), resolution=W, return_ids=True)
        overlap = ids[0, 19:30, 19:30]
        assert np.isin(overlap, near_ids).all()
        assert np.isin(ids[0, 35:40, 35:40], [t for t in range(4) if t not in near_ids]).all()
    # the same quad twice: equal depth everywhere, the lower triangle index wins
    v = np.concatenate([near, near])
    _, ids = ora.rasterize(v, np.concatenate([q, q + 4]), _eye(), resolution=W, return_ids=True)
    assert set(np.unique(ids[0])) == {-1, 0, 1}


def test_oracle_projection_matches_the_opengl_camera():
    W, H = 96, 64                                         # non-square: an x/y swap moves the points
    fy = FY18
    fx = fy * H / W
    P = load_golden('mesh_turntable')['poses'][37]
    for xc, yc, zc in ((0.1, 0.05, -2.5), (-0.2, -0.11, -3.1), (0.0, 0.0, -2.0), (0.3, 0.2, -4.0)):
        X = (fx * xc / -zc + 1) * W / 2
        Y = (1 - fy * yc / -zc) * H / 2
        world = (P @ np.array([xc, yc, zc, 1.0]))[:3].astype(np.float32)
        xs, ys, iw, ok = ora.screen_vertices(world[None], P, W, H, 18.0, 0.05)
        assert ok[0] and abs(xs[0] / 256 - X) < 2e-3 and abs(ys[0] / 256 - Y) < 2e-3 and abs(1 / iw[0] + zc) < 1e-5
        # a small triangle around the point lands on the expected pixels
        d = 0.012 * -zc
        tri = np.array([[xc - d, yc - d, zc, 1], [xc + d, yc - d, zc, 1], [xc, yc + 2 * d, zc, 1]]) @ P.T.astype(np.float64)   # centroid: the point
        _, ids = ora.rasterize(tri[:, :3].astype(np.float32), np.array([[0, 1, 2]]), P[None], resolution=(W, H), return_ids=True)
        jj, ii = np.nonzero(ids[0] == 0)
        assert len(ii) > 0 and abs(ii.mean() + 0.5 - X) < 1.0 and abs(jj.mean() + 0.5 - Y) < 1.0
    # world +y appears toward row 0, world +x (the camera's right for the identity pose) toward the last column
    pts = np.array([[0, 0.3, -3], [0.3, 0, -3]], np.float32)
    xs, ys, _, _ = ora.screen_vertices(pts, _eye()[0], W, H, 18.0, 0.05)
    assert ys[0] < H / 2 * 256 and xs[1] > W / 2 * 256
    # behind the near plane: dropped
    assert not ora.screen_vertices(np.array([[0, 0, -0.01]], np.float32), _eye()[0], W, H, 18.0, 0.05)[3][0]


def test_oracle_shading_of_a_quad_facing_the_camera():
    W = H = 32
    v = _from_screen([(4.3, 4.3, 3.0), (27.7, 4.3, 3.0), (27.7, 27.7, 3.0), (4.3, 27.7, 3.0)], W, H)
    q = np.array([[0, 1, 2], [0, 2, 3]])
    n = ora.vertex_normals(v, q)
    assert np.array_equal(np.abs(n), np.tile([[0, 0, 1]], (4, 1)).astype(np.float32))
    rgb, ids = ora.rasterize(v, q, _eye(), resolution=W, return_ids=True)
    face = rgb[0][ids[0] >= 0]
    assert len(face) > 400 and (face == round(255 * 0.85 * (0.25 + 0.75))).all()
    assert (rgb[0][ids[0] < 0] == 255).all()
    # facing away is shaded the same (two-sided); diffuse = 0: uniform ambient colour everywhere on the mesh
    rgb2 = ora.rasterize(v, q[:, ::-1], _eye(), resolution=W)
    assert np.array_equal(rgb, rgb2)
    vs, ts = _small_sphere()
    rgb3, ids3 = ora.rasterize(vs, ts, load_golden('mesh_turntable')['poses'][:1], resolution=40, return_ids=True, diffuse=0.0,
                               background=7)
    assert (rgb3[0][ids3[0] >= 0] == int(np.rint(np.float32(255) * (np.float32(0.85) * np.float32(0.25))))).all()
    assert (rgb3[0][ids3[0] < 0] == 7).all() and (ids3 >= 0).sum() > 100


def test_oracle_silhouette_of_a_marching_cubes_sphere():
    n, R = 64, 0.3
    v, t = omc.marching_cubes(_sphere_field(n, R * n, n / 2), 0.0)
    v = v / n                                               # centred at 0.5: on the optical axis of every turntable pose
    poses = load_golden('mesh_turntable')['poses'][[0, 100]]
    _, ids = ora.rasterize(v, t, poses, resolution=128, return_ids=True)
    area, r_px = _disc_area(R, 2.7, 128)
    for f in range(2):
        assert abs((ids[f] >= 0).sum() / area - 1) < 0.02
        jj, ii = np.nonzero(ids[f] >= 0)
        assert np.hypot(ii + 0.5 - 64, jj + 0.5 - 64).max() < r_px + 1


def test_raster_struct_size_and_invalid_arguments(lib):
    import ctypes
    from ide3d_b200 import _lib
    assert lib.ide3d_raster(None, None) == _lib.INVALID and b'null params' in lib.ide3d_last_error()
    p = _lib.RasterParams(num_frames=1, width=8, height=8, yfov_deg=18.0, znear=0.05, num_triangles=1, num_vertices=3)
    assert lib.ide3d_raster(ctypes.byref(p), None) == _lib.INVALID and b'null' in lib.ide3d_last_error()
    p.width = 0
    assert lib.ide3d_raster(ctypes.byref(p), None) == _lib.INVALID and b'resolution' in lib.ide3d_last_error()
    assert lib.ide3d_mesh_normals(None, None, 4, None, None, None, None) == _lib.INVALID
    assert lib.ide3d_mesh_normals(None, None, 0, None, None, None, None) == _lib.OK                 # no vertices: no-op
    assert lib.ide3d_raster_scratch_bytes(2, 16, 8, 10, 5) >= 2 * 16 * 8 * 8 + 2 * 10 * 16 + 2 * 5 * 8
    assert lib.ide3d_raster_scratch_bytes(-1, 16, 8, 10, 5) == -1


# ----------------------------------------------------------------------------------------------------------------- GPU
def _gpu_vs_oracle(v, t, poses, resolution, **kw):
    from ide3d_b200 import mesh
    rgb, ids = mesh.rasterize(torch.from_numpy(v).cuda(), torch.from_numpy(t).cuda(), torch.from_numpy(np.asarray(poses)), resolution=resolution,
                              return_ids=True, **kw)
    rgb_o, ids_o = ora.rasterize(v, t, poses, resolution=resolution, return_ids=True, **kw)
    ids, rgb = ids.cpu().numpy(), rgb.cpu().numpy()
    assert np.array_equal(ids, ids_o), f'{(ids != ids_o).sum()} pixels show a different triangle'
    assert np.abs(rgb.astype(np.int16) - rgb_o).max() <= 1
    return rgb, ids


def _soup(seed, n=1500):
    """Triangles in the view of the identity camera, with degenerate, off-screen, border-straddling and near-plane cases."""
    rng = np.random.RandomState(seed)
    c = rng.uniform([-0.55, -0.4, -4.0], [0.55, 0.4, -1.0], size=(n, 1, 3))
    tri = c + rng.normal(scale=0.06, size=(n, 3, 3))
    tri[:20, 1] = tri[:20, 0]                                       # two equal corners
    tri[20:40, 2] = 0.5 * (tri[20:40, 0] + tri[20:40, 1])           # collinear
    tri[40:80, :, :2] += np.array([1.5, 0.0])                       # off screen
    tri[80:160, :, 0] += 0.6 * -tri[80:160, :, 2] * 0.1584          # straddling the right border
    tri[160:200, 0, 2] = rng.uniform(-0.04, 0.5, size=40)           # a corner behind the near plane
    tri[200:240, 0, :2] *= 3000                                     # a corner far outside the guard band
    v = tri.reshape(-1, 3).astype(np.float32)
    return v, np.arange(len(v), dtype=np.int64).reshape(-1, 3)


@pytest.mark.gpu
@pytest.mark.parametrize('case', ['sphere', 'nonsquare', 'soup', 'fullscreen'])
def test_cuda_raster_matches_oracle(case):
    poses = load_golden('mesh_turntable')['poses']
    if case == 'sphere':
        v, t = _small_sphere(32, 9.7)
        _gpu_vs_oracle(v, t, poses[[0, 60, 150]], 128)
    elif case == 'nonsquare':
        v, t = _small_sphere(32, 9.7)
        _, ids = _gpu_vs_oracle(v, t, poses[[20, 200]], (96, 64))
        assert (ids >= 0).sum() > 2000
    elif case == 'soup':
        v, t = _soup(0)
        _, ids = _gpu_vs_oracle(v, t, _eye(), (96, 64), ambient=0.1, diffuse=0.9, base=1.0, background=0)
        assert len(np.unique(ids)) > 300
    else:                                                           # both triangles exceed the small-triangle budget
        v = _from_screen([(-3.0, -2.0, 3.0), (70.0, -2.5, 3.5), (69.0, 67.0, 4.0), (-2.0, 66.0, 2.5)], 64, 64)
        _, ids = _gpu_vs_oracle(v, np.array([[0, 1, 2], [0, 2, 3]]), _eye(), 64)
        assert (ids >= 0).all()


@pytest.mark.gpu
def test_cuda_vertex_normals_match_oracle():
    from ide3d_b200 import mesh
    v, t = _small_sphere(32, 9.7)
    t = np.concatenate([t, [[0, 0, 1]]])                            # a degenerate face adds nothing
    n = mesh.vertex_normals(torch.from_numpy(v).cuda(), torch.from_numpy(t).cuda()).cpu().numpy()
    assert np.array_equal(n, ora.vertex_normals(v, t))
    assert np.allclose(np.linalg.norm(n, axis=1), 1, atol=1e-6)
    # outward on a sphere
    assert (np.einsum('ij,ij->i', n, v - v.mean(0)) > 0).all()


@pytest.mark.gpu
def test_cuda_raster_is_deterministic_and_independent_of_triangle_order():
    from ide3d_b200 import mesh
    n = 96
    vol = torch.from_numpy(_sphere_field(n, 30.1, 48.3)).cuda() + torch.from_numpy(
        np.random.RandomState(3).randn(n, n, n).astype(np.float32)).cuda() * 0.7
    v, t = mesh.marching_cubes(vol, 0.0)
    v = v / n
    poses = mesh.turntable_poses(240)[::30]
    nrm = mesh.vertex_normals(v, t)
    rgb, ids = mesh.rasterize(v, t, poses, resolution=256, normals=nrm, return_ids=True)
    rgb2, ids2 = mesh.rasterize(v, t, poses, resolution=256, normals=nrm, return_ids=True)
    assert torch.equal(rgb, rgb2) and torch.equal(ids, ids2)
    perm = torch.randperm(t.shape[0], generator=torch.Generator().manual_seed(0)).cuda()
    rgb3, ids3 = mesh.rasterize(v, t[perm], poses, resolution=256, normals=nrm, return_ids=True)
    assert torch.equal(rgb, rgb3)
    assert (ids >= 0).sum() > 8 * 10000
    # the visible triangle is the same one, except where two triangles reach a pixel centre at exactly the same depth (the front and
    # back faces meeting on a silhouette edge): there the lower index wins, in either numbering
    remapped = torch.where(ids3 >= 0, perm[ids3.clamp_min(0).long()].int(), -1)
    diff = remapped != ids
    assert torch.equal(ids >= 0, remapped >= 0) and diff.sum() < 1e-3 * (ids >= 0).sum()
    inv = torch.empty_like(perm)
    inv[perm] = torch.arange(perm.numel(), device=perm.device)
    a, b = ids[diff].long(), remapped[diff].long()
    assert (a < b).all() and (inv[b] < inv[a]).all()


def _sphere_grid_cuda(n, r):
    g = torch.arange(n, dtype=torch.float32, device='cuda')
    x, y, z = torch.meshgrid(g, g, g, indexing='ij')
    return 10.0 + 4.0 * (r - torch.sqrt((x - n / 2) ** 2 + (y - n / 2) ** 2 + (z - n / 2) ** 2))     # sigma = 10 on the sphere


@pytest.mark.gpu
def test_render_turntable_full_size_sphere():
    from ide3d_b200 import mesh
    n, R = 256, 0.3
    frames = mesh.render_turntable(_sphere_grid_cuda(n, R * n))
    assert frames.shape == (240, 512, 512, 3) and frames.dtype == torch.uint8
    area, r_px = _disc_area(R, 2.7, 512)
    fg = (frames[..., 0] != 255)
    counts = fg.sum((1, 2)).double().cpu()
    assert ((counts / area - 1).abs() < 5e-3).all(), (counts.min().item(), counts.max().item(), area)
    jj, ii = torch.meshgrid(torch.arange(512, device='cuda'), torch.arange(512, device='cuda'), indexing='ij')
    outside = torch.hypot(ii + 0.5 - 256, jj + 0.5 - 256) > r_px + 1
    assert not fg[:, outside].any()
    assert torch.equal(frames[..., 0], frames[..., 2])             # grey


@pytest.mark.gpu
def test_render_mesh_cli_writes_the_frames(tmp_path):
    from PIL import Image
    from ide3d_b200 import mesh, render_mesh
    grid = _sphere_grid_cuda(64, 0.3 * 64)
    np.save(tmp_path / '7.npy', grid.cpu().numpy())
    out = render_mesh.main(['--fname', str(tmp_path / '7.npy'), '--outdir', str(tmp_path / 'out'), '--size', '64', '--w-frames', '4'])
    assert sorted(os.listdir(out)) == ['000.png', '001.png', '002.png', '003.png'] and out == str(tmp_path / 'out' / '7')
    frames = mesh.render_turntable(grid, size=64, w_frames=4)
    first = np.asarray(Image.open(os.path.join(out, '000.png')))
    assert np.array_equal(first, frames[0].cpu().numpy())
