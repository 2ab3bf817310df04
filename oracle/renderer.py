"""Oracle (test infrastructure): CPU restatement of the IDE-3D volume-rendering path.

torch-CPU fp32, written from the reference's Python functions (cited per function).  Used only as
the checker for the CUDA kernels and as the CPU baseline leg of bench.py -- never shipped.
The render chain follows the dtype and device of its inputs (the planes for render_frames), so the
same functions give a float64 reference on the GPU; fp32 CPU inputs take exactly the fp32 CPU ops.

Reference files followed (relative to the reference tree):
  training/volumetric_rendering.py   rays :77-97, jitter :99-105, world transform :108-136,
                                     compositing :34-74, importance pdf :224-265
  dnnlib/util.py                     tri-plane gather :580-617
  torch_utils/ops/grid_sample_gradfix.py:26-29   bilinear / zeros padding / align_corners=False
  extract_shapes.py                  :74-96 create_samples, :131-147 default render kwargs, 52-ch layout
The decoder MLP and the world->grid scale live in the (absent) generator class; their restatement
is this project's own and is documented in DESIGN.md ("parity unpinned" for those two pieces).
"""

import math

import numpy as np
import torch
import torch.nn.functional as F

N_FEAT = 32      # channels per plane (tri-plane tensor has 3*32 = 96)
N_OUT = 52       # 32 colour features + 19 semantic logits + 1 sigma (extract_shapes.py:146-147)


# ----------------------------------------------------------------------------- rays (a1)

def initial_rays(n, num_steps, fov, resolution, ray_start, ray_end, dtype=None, device=None):
    """get_initial_rays_trig, volumetric_rendering.py:77-97.

    Pixel i = py*W + px; x sweeps -1..1 along px, y sweeps +1..-1 along py (the reference builds a
    meshgrid with default 'ij' indexing and then transposes, :83-86).  Returns
    points [n,HW,S,3], z_vals [n,HW,S,1], rays_d_cam [n,HW,3] of the given dtype and device (None: torch's defaults)."""
    W, H = resolution
    xs = torch.linspace(-1, 1, W, dtype=dtype, device=device)
    ys = torch.linspace(1, -1, H, dtype=dtype, device=device)
    x = xs.reshape(1, W).expand(H, W).reshape(-1)
    y = ys.reshape(H, 1).expand(H, W).reshape(-1)
    z = -torch.ones_like(x) / np.tan((2 * math.pi * fov / 360) / 2)
    d = torch.stack([x, y, z], -1)
    d = d / torch.norm(d, dim=-1, keepdim=True)
    zv = torch.linspace(ray_start, ray_end, num_steps, dtype=dtype, device=device).reshape(1, num_steps, 1).repeat(W * H, 1, 1)
    pts = d.unsqueeze(1).repeat(1, num_steps, 1) * zv
    return (pts.unsqueeze(0).repeat(n, 1, 1, 1).contiguous(),
            zv.unsqueeze(0).repeat(n, 1, 1, 1).contiguous(),
            d.unsqueeze(0).repeat(n, 1, 1).contiguous())


# ----------------------------------------------------------------------------- jitter (a2)

def hash_uniform(index, seed):
    """Counter-based uniform in [0,1) shared bit-for-bit with the CUDA kernel
    (csrc/raymarch.cu: jitter_hash).  ``index`` = flat (n, ray, step) sample index (uint32 wrap),
    ``seed`` = 64-bit integer.  Integer arithmetic only, so numpy reproduces the device exactly."""
    idx = np.asarray(index, dtype=np.uint64) & np.uint64(0xFFFFFFFF)
    lo = np.uint64(int(seed) & 0xFFFFFFFF)
    hi = np.uint64((int(seed) >> 32) & 0xFFFFFFFF)
    m32 = np.uint64(0xFFFFFFFF)
    h = (idx ^ lo) & m32
    h = (h * np.uint64(0x9E3779B1)) & m32
    h = h ^ hi
    h = h ^ (h >> np.uint64(16))
    h = (h * np.uint64(0x21F0AAAD)) & m32
    h = h ^ (h >> np.uint64(15))
    h = (h * np.uint64(0x735A2D97)) & m32
    h = h ^ (h >> np.uint64(15))
    return ((h >> np.uint64(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)).astype(np.float32)


def perturb(points, z_vals, dirs, u):
    """perturb_points, volumetric_rendering.py:99-105, with the uniform draw ``u`` [n,HW,S,1]
    injected (the reference calls torch.rand in place).  u=None means "no jitter" (the behaviour of
    ide3d-nada's DEBUG_PERTURB switch, ide3d-nada/training/volumetric_rendering.py:118-119)."""
    if u is None:
        return points, z_vals
    dist = z_vals[:, :, 1:2, :] - z_vals[:, :, 0:1, :]
    off = (u - 0.5) * dist
    return points + off * dirs.unsqueeze(2), z_vals + off


# ----------------------------------------------------------------------------- world transform (a3)

def to_world(points, dirs, cam2world):
    """transform_sampled_points, volumetric_rendering.py:122-134 (camera given => sampled pose is
    discarded, :119-120).  Returns points_world [n,HW,S,3], dirs_world [n,HW,3], origins [n,HW,3]."""
    n, R, S, _ = points.shape
    hom = torch.ones((n, R, S, 4), dtype=cam2world.dtype, device=cam2world.device)
    hom[..., :3] = points
    pw = torch.bmm(cam2world, hom.reshape(n, -1, 4).permute(0, 2, 1)).permute(0, 2, 1).reshape(n, R, S, 4)
    dw = torch.bmm(cam2world[..., :3, :3], dirs.reshape(n, -1, 3).permute(0, 2, 1)).permute(0, 2, 1).reshape(n, R, 3)
    ho = torch.zeros((n, 4, R), dtype=cam2world.dtype, device=cam2world.device)
    ho[:, 3, :] = 1
    ow = torch.bmm(cam2world, ho).permute(0, 2, 1).reshape(n, R, 4)[..., :3]
    return pw[..., :3], dw, ow


# ----------------------------------------------------------------------------- tri-plane gather (a5)

def bilinear_zeros(plane, u, v):
    """Restatement of aten::grid_sampler_2d(bilinear, zeros, align_corners=False) as pinned by
    grid_sample_gradfix.py:29.  plane [N,C,H,W]; u (-> W axis), v (-> H axis) [N,P] in [-1,1] grid
    units.  Returns [N,P,C]."""
    N, C, H, W = plane.shape
    ix = ((u + 1) * W - 1) / 2
    iy = ((v + 1) * H - 1) / 2
    x0 = torch.floor(ix)
    y0 = torch.floor(iy)
    fx = ix - x0
    fy = iy - y0
    x0 = x0.long()
    y0 = y0.long()
    flat = plane.reshape(N, C, H * W)
    out = torch.zeros((N, u.shape[1], C), dtype=plane.dtype, device=plane.device)
    taps = ((0, 0, (1 - fx) * (1 - fy)), (0, 1, fx * (1 - fy)), (1, 0, (1 - fx) * fy), (1, 1, fx * fy))
    for dy, dx, w in taps:
        xx = x0 + dx
        yy = y0 + dy
        ok = (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H)
        lin = (yy.clamp(0, H - 1) * W + xx.clamp(0, W - 1))            # [N,P]
        val = torch.gather(flat, 2, lin.unsqueeze(1).expand(N, C, -1))  # [N,C,P]
        out = out + (val.permute(0, 2, 1) * (w * ok.to(plane.dtype)).unsqueeze(-1))
    return out


def sample_triplane(coords, grid):
    """sample_from_triplane, dnnlib/util.py:580-599: plane0 at (x,y), plane1 at (y,z), plane2 at
    (x,z); features are SUMMED (:599).  coords [N,P,3] in grid units, grid [N,3C,H,W].
    Returns [N*P, C] (batch folded into rows, :616)."""
    N, C3, H, W = grid.shape
    g = grid.reshape(N, 3, C3 // 3, H, W)
    x, y, z = coords[..., 0], coords[..., 1], coords[..., 2]
    f = bilinear_zeros(g[:, 0], x, y)
    f = f + bilinear_zeros(g[:, 1], y, z)
    f = f + bilinear_zeros(g[:, 2], x, z)
    return f.reshape(N * coords.shape[1], C3 // 3)


def sample_triplane_torch(coords, grid):
    """Same gather through torch's own grid_sample -- the arithmetic the reference actually runs."""
    N, C3, H, W = grid.shape
    g = grid.reshape(N, 3, C3 // 3, H, W)
    out = 0
    for k, idx in enumerate(([0, 1], [1, 2], [0, 2])):
        s = F.grid_sample(g[:, k], coords[..., idx].reshape(N, -1, 1, 2), mode='bilinear',
                          padding_mode='zeros', align_corners=False)
        out = out + s.permute(0, 3, 2, 1).reshape(-1, C3 // 3)
    return out


# ----------------------------------------------------------------------------- decoder (a6)

class Decoder:
    """Two-layer per-sample MLP over the concatenated features [tex(32); seg(32)]:

        h = softplus(W1 @ f + b1)      W1 [HID,64]
        o = W2 @ h + b2                W2 [52,HID]     o = (32 colour, 19 semantic, 1 sigma)

    The generator's three heads (texture->colour, shape->semantic, shape->sigma) are block-sparse
    instances of this dense form (see ide3d_b200.training.triplane.TriPlaneDecoder.packed()).
    Floating-point torch tensors keep their dtype and device; anything else becomes fp32 on the CPU."""

    def __init__(self, w1, b1, w2, b2):
        dtype = w1.dtype if torch.is_tensor(w1) and w1.is_floating_point() else torch.float32
        self.w1, self.b1, self.w2, self.b2 = [torch.as_tensor(t, dtype=dtype) for t in (w1, b1, w2, b2)]
        assert self.w1.shape[1] == 2 * N_FEAT and self.w2.shape == (N_OUT, self.w1.shape[0])

    def to(self, dtype=None, device=None):
        return Decoder(*[t.to(dtype=dtype, device=device) for t in (self.w1, self.b1, self.w2, self.b2)])

    @staticmethod
    def random(hidden=64, seed=0, three_head=True):
        g = torch.Generator().manual_seed(seed)
        if not three_head:
            w1 = torch.randn(hidden, 2 * N_FEAT, generator=g) / math.sqrt(N_FEAT)
            w2 = torch.randn(N_OUT, hidden, generator=g) / math.sqrt(hidden)
            return Decoder(w1, 0.1 * torch.randn(hidden, generator=g), w2, 0.1 * torch.randn(N_OUT, generator=g))
        H = hidden
        w1 = torch.zeros(3 * H, 2 * N_FEAT)
        w2 = torch.zeros(N_OUT, 3 * H)
        w1[0:H, 0:N_FEAT] = torch.randn(H, N_FEAT, generator=g) / math.sqrt(N_FEAT)          # tex -> colour
        w1[H:2 * H, N_FEAT:] = torch.randn(H, N_FEAT, generator=g) / math.sqrt(N_FEAT)       # seg -> semantic
        w1[2 * H:, N_FEAT:] = torch.randn(H, N_FEAT, generator=g) / math.sqrt(N_FEAT)        # seg -> sigma
        w2[0:32, 0:H] = torch.randn(32, H, generator=g) / math.sqrt(H)
        w2[32:51, H:2 * H] = torch.randn(19, H, generator=g) / math.sqrt(H)
        w2[51:52, 2 * H:] = torch.randn(1, H, generator=g) / math.sqrt(H)
        return Decoder(w1, 0.1 * torch.randn(3 * H, generator=g), w2, 0.1 * torch.randn(N_OUT, generator=g))

    def __call__(self, f_tex, f_seg):
        f = torch.cat([f_tex, f_seg], dim=-1)
        h = F.softplus(f @ self.w1.t() + self.b1)
        return h @ self.w2.t() + self.b2


# ----------------------------------------------------------------------------- compositing (a7)

def composite(rgb_sigma, rays_d_cam, z_vals, noise=None, noise_std=0.0, last_back=False, white_back=False,
              max_depth=None, clamp_mode=None, fill_mode=None):
    """fancy_integration, volumetric_rendering.py:34-74.  ``noise`` (standard normal, sigma-shaped)
    is injected instead of drawn (:45); None / noise_std=0 => no noise."""
    rgbs = rgb_sigma[..., :-1]
    sigmas = rgb_sigma[..., -1:]
    deltas = z_vals[:, :, 1:] - z_vals[:, :, :-1]
    deltas = deltas * torch.norm(rays_d_cam, p=2, dim=-1, keepdim=True).unsqueeze(2)
    deltas = torch.cat([deltas, 1e10 * torch.ones_like(deltas[:, :, :1])], -2)
    if noise is not None and noise_std != 0:
        sigmas = sigmas + noise * noise_std
    if clamp_mode == 'softplus':
        alphas = 1 - torch.exp(-deltas * F.softplus(sigmas))
    elif clamp_mode == 'relu':
        alphas = 1 - torch.exp(-deltas * F.relu(sigmas))
    else:
        raise ValueError("Need to choose clamp mode")     # reference raises a str (:51-52)
    shifted = torch.cat([torch.ones_like(alphas[:, :, :1]), 1 - alphas + 1e-10], -2)
    weights = alphas * torch.cumprod(shifted, -2)[:, :, :-1]
    wsum = weights.sum(2)
    if last_back:
        weights = weights.clone()
        weights[:, :, -1] += (1 - wsum)
    rgb = torch.sum(weights * rgbs, -2)
    depth = torch.sum(weights * z_vals, -2)
    if white_back:
        rgb = rgb + 1 - wsum
    if max_depth:
        depth = depth + (1 - wsum) * max_depth
    if fill_mode == 'weight':
        rgb = wsum.expand_as(rgb)
    return rgb, depth, weights


# ----------------------------------------------------------------------------- importance pdf (a8)

def sample_pdf(bins, weights, n_importance, det=False, eps=1e-5, u=None):
    """sample_pdf, volumetric_rendering.py:224-265.  ``u`` injects the uniform draws for det=False."""
    n_rays, n_s = weights.shape
    weights = weights + eps
    pdf = weights / torch.sum(weights, -1, keepdim=True)
    cdf = torch.cumsum(pdf, -1)
    cdf = torch.cat([torch.zeros_like(cdf[:, :1]), cdf], -1)
    if det:
        u = torch.linspace(0, 1, n_importance, dtype=weights.dtype, device=weights.device).expand(n_rays, n_importance)
    assert u is not None
    u = u.contiguous()
    inds = torch.searchsorted(cdf, u)
    below = torch.clamp_min(inds - 1, 0)
    above = torch.clamp_max(inds, n_s)
    cdf_lo, cdf_hi = torch.gather(cdf, 1, below), torch.gather(cdf, 1, above)
    bin_lo, bin_hi = torch.gather(bins, 1, below), torch.gather(bins, 1, above)
    denom = cdf_hi - cdf_lo
    denom = torch.where(denom < eps, torch.ones_like(denom), denom)
    return bin_lo + (u - cdf_lo) / denom * (bin_hi - bin_lo)


# ----------------------------------------------------------------------------- composed path

def sample_voxel(planes_tex, planes_seg, decoder, points, box_scale=2.0):
    """renderer.sample_voxel(img_v, seg_v, points) -> [N,P,52] (extract_shapes.py:146)."""
    N, P, _ = points.shape
    c = points.float() * box_scale
    f_tex = sample_triplane(c, planes_tex)
    f_seg = sample_triplane(c, planes_seg)
    return decoder(f_tex, f_seg).reshape(N, P, N_OUT)


def render_frames(planes_tex, planes_seg, decoder, cam2world, fov=18.0, num_steps=48, ray_start=2.25,
                  ray_end=3.3, resolution=(64, 64), box_scale=2.0, jitter_u=None, jitter_seed=None,
                  clamp_mode='softplus', last_back=False, white_back=False, max_depth=None,
                  fill_mode=None, noise=None, noise_std=0.0, return_stages=False, gather=sample_triplane):
    """a1 -> a2 -> a3 -> a5 x2 -> a6 -> a7, the chain the absent generator class runs per frame.
    jitter_u: explicit [N,HW,S,1] uniforms; jitter_seed: use hash_uniform(seed); neither: no jitter.
    Rays and camera take the planes' dtype and device; jitter_u and noise are moved to that device.
    gather: sample_triplane (the explicit restatement) or sample_triplane_torch (F.grid_sample, whose
    autograd saves the grid instead of four [N,C,P] gathers per plane: the memory-light form for a
    float64 reference at full size)."""
    N = planes_tex.shape[0]
    W, H = resolution
    dtype, dev = planes_tex.dtype, planes_tex.device
    pts, zv, d = initial_rays(N, num_steps, fov, resolution, ray_start, ray_end, dtype=dtype, device=dev)
    if jitter_u is None and jitter_seed is not None:
        idx = np.arange(N * W * H * num_steps, dtype=np.uint64)
        jitter_u = torch.from_numpy(hash_uniform(idx, jitter_seed)).reshape(N, W * H, num_steps, 1)
    if jitter_u is not None:
        jitter_u = jitter_u.to(device=dev)
    if noise is not None:
        noise = noise.to(device=dev)
    pts, zv = perturb(pts, zv, d, jitter_u)
    pw, dw, ow = to_world(pts, d, cam2world.to(device=dev, dtype=dtype))
    coords = pw.reshape(N, -1, 3) * box_scale
    f_tex = gather(coords, planes_tex)
    f_seg = gather(coords, planes_seg)
    out = decoder(f_tex, f_seg).reshape(N, W * H, num_steps, N_OUT)
    rgb, depth, weights = composite(out, d, zv, noise=noise, noise_std=noise_std, last_back=last_back,
                                    white_back=white_back, max_depth=max_depth, clamp_mode=clamp_mode,
                                    fill_mode=fill_mode)
    if return_stages:
        return dict(points_world=pw, z_vals=zv, f_tex=f_tex, f_seg=f_seg, raw=out, rgb=rgb, depth=depth,
                    weights=weights)
    return rgb, depth, weights


def render_frames_hierarchical(planes_tex, planes_seg, decoder, cam2world, fov=18.0, num_steps=48, n_importance=None,
                               ray_start=2.25, ray_end=3.3, resolution=(64, 64), box_scale=2.0, jitter_u=None,
                               jitter_seed=None, importance_u=None, det=False, clamp_mode='softplus', last_back=False,
                               white_back=False, max_depth=None):
    """Two-pass render around the reference's own sample_pdf (volumetric_rendering.py:224-265).  The reference tree holds the
    function but no caller (the generator class is absent, SURVEY.md a8), so the COMPOSITION is the one the function's
    docstring prescribes (bins = midpoints of the coarse depths, weights = coarse weights[1:-1]; nerf_pl / pi-GAN order):
    coarse chain -> weights (+1e-5) -> sample_pdf -> fine points = origin + direction * z -> decode -> merge by sorted depth
    -> composite over all samples.  Parity of the ORDER is therefore unpinned; every stage in it is a pinned one, and tests/golden/chain_hier.npz
    records this order executed with the reference's own stage functions (make_golden.py g_chain_hier).
    importance_u [N*HW, n_importance] injects the uniform draws of sample_pdf (det=True: linspace)."""
    N = planes_tex.shape[0]
    W, H = resolution
    S = num_steps
    n_imp = S if n_importance is None else n_importance
    st = render_frames(planes_tex, planes_seg, decoder, cam2world, fov=fov, num_steps=S, ray_start=ray_start, ray_end=ray_end,
                       resolution=resolution, box_scale=box_scale, jitter_u=jitter_u, jitter_seed=jitter_seed,
                       clamp_mode=clamp_mode, return_stages=True)
    zv, w = st['z_vals'], st['weights']                                   # [N,HW,S,1]
    dtype, dev = planes_tex.dtype, planes_tex.device
    _, _, d = initial_rays(N, S, fov, resolution, ray_start, ray_end, dtype=dtype, device=dev)
    _, dw, ow = to_world(torch.zeros(N, W * H, 1, 3, dtype=dtype, device=dev), d, cam2world.to(device=dev, dtype=dtype))
    z = zv.reshape(N * W * H, S)
    z_mid = 0.5 * (z[:, :-1] + z[:, 1:])
    fine = sample_pdf(z_mid, w.reshape(N * W * H, S)[:, 1:-1] + 1e-5, n_imp, det=det, u=importance_u).reshape(N, W * H, n_imp, 1)
    fine_pts = ow.unsqueeze(2) + dw.unsqueeze(2) * fine
    coords = fine_pts.reshape(N, -1, 3) * box_scale
    out_f = decoder(sample_triplane(coords, planes_tex), sample_triplane(coords, planes_seg)).reshape(N, W * H, n_imp, N_OUT)
    all_z = torch.cat([zv, fine], -2)
    all_out = torch.cat([st['raw'], out_f], -2)
    all_z, idx = torch.sort(all_z, dim=-2)
    all_out = torch.gather(all_out, -2, idx.expand(-1, -1, -1, N_OUT))
    rgb, depth, weights = composite(all_out, d, all_z, last_back=last_back, white_back=white_back, max_depth=max_depth,
                                    clamp_mode=clamp_mode)
    return rgb, depth, weights, all_z


def create_samples(N=512, voxel_origin=(0, 0, 0), cube_length=2.0):
    """extract_shapes.py:74-96 including the float-division index quirk (:84-86): the y and x voxel
    indices are computed with true division, so they are fractional."""
    origin = np.array(voxel_origin) - cube_length / 2
    voxel_size = cube_length / (N - 1)
    idx = torch.arange(0, N ** 3, 1, dtype=torch.long)
    s = torch.zeros(N ** 3, 3)
    s[:, 2] = idx % N
    s[:, 1] = (idx.float() / N) % N
    s[:, 0] = ((idx.float() / N) / N) % N
    s[:, 0] = (s[:, 0] * voxel_size) + origin[2]
    s[:, 1] = (s[:, 1] * voxel_size) + origin[1]
    s[:, 2] = (s[:, 2] * voxel_size) + origin[0]
    return s.unsqueeze(0), origin, voxel_size
