"""Volume-rendering free functions with the reference's names and signatures
(training/volumetric_rendering.py), computed by the sm_90a stage kernels in csrc/stages.cu.

    fancy_integration          :34    -> ide3d_integrate
    get_initial_rays_trig      :77    -> ide3d_initial_rays
    perturb_points             :99    -> ide3d_transform_points (identity camera)
    transform_sampled_points   :108   -> ide3d_transform_points
    sample_pdf                 :224   -> ide3d_sample_pdf
    sample_camera_positions :147, create_cam2world_matrix :195, LookAtPoseSampler :268
                               -> tiny pose helpers, plain torch on whatever device the caller asks for
                                  (gen_images.py:104-105, gen_videos.py:120 call them directly)

The generator does NOT chain these: it calls the fused kernel (renderer.TriPlaneRenderer / ide3d_raymarch_fwd),
which never materialises points, features or per-sample outputs.  These functions exist so that code written
against the reference module keeps working; they are CUDA-only (the CPU restatement is oracle/renderer.py).
"""

import math
import random

import numpy as np
import torch

from .. import _lib as L


def _cuda_only(*ts):
    L.require_cuda(*ts)


def _f32(t):
    return t.to(torch.float32).contiguous()


# ----------------------------------------------------------------------------------------------- small helpers
def transform_vectors(matrix: torch.Tensor, vectors4: torch.Tensor) -> torch.Tensor:
    """Left-multiplies MxM @ NxM. Returns NxM."""
    return torch.matmul(vectors4, matrix.T)


def normalize_vecs(vectors: torch.Tensor) -> torch.Tensor:
    return vectors / (torch.norm(vectors, dim=-1, keepdim=True))


def torch_dot(x: torch.Tensor, y: torch.Tensor):
    return (x * y).sum(-1)


# ----------------------------------------------------------------------------------------------- compositing
def fancy_integration(rgb_sigma, rays_d_cam, z_vals, device, noise_std=0.5, last_back=False, white_back=False,
                      max_depth=None, clamp_mode=None, fill_mode=None):
    """NeRF alpha compositing of rgb_sigma [N,R,S,C] (sigma last) -> (rgb [N,R,C-1], depth [N,R,1], weights [N,R,S,1])."""
    if clamp_mode not in ('softplus', 'relu'):
        raise ValueError('Need to choose clamp mode')      # the reference raises a bare string (:51-52)
    if fill_mode == 'debug':
        raise NotImplementedError("fill_mode='debug' paints 3-channel pixels and cannot apply to feature maps")
    _cuda_only(rgb_sigma, rays_d_cam, z_vals)
    L.forbid_grad('fancy_integration', rgb_sigma, rays_d_cam, z_vals)
    n, R, S, Cc = rgb_sigma.shape
    rs, d, z = _f32(rgb_sigma), _f32(rays_d_cam), _f32(z_vals)
    noise = torch.randn([n, R, S], device=rs.device, dtype=torch.float32) if noise_std else None
    rgb = torch.empty([n, R, Cc - 1], device=rs.device, dtype=torch.float32)
    depth = torch.empty([n, R, 1], device=rs.device, dtype=torch.float32)
    weights = torch.empty([n, R, S, 1], device=rs.device, dtype=torch.float32)
    rc = L.get_lib().ide3d_integrate(L.ptr(rs), L.ptr(d), L.ptr(z), L.ptr(noise), float(noise_std or 0.0), n, R, S, Cc,
                                     L.CLAMP_SOFTPLUS if clamp_mode == 'softplus' else L.CLAMP_RELU,
                                     int(bool(last_back)), int(bool(white_back)), float(max_depth or 0.0),
                                     int(fill_mode == 'weight'), L.ptr(rgb), L.ptr(depth), L.ptr(weights),
                                     L.stream_ptr(rs.device))
    L.check(rc)
    return rgb, depth, weights


# ----------------------------------------------------------------------------------------------- rays
def get_initial_rays_trig(n, num_steps, device, fov, resolution, ray_start, ray_end):
    """Sample points, z_vals and ray directions in camera space: ([n,R,S,3], [n,R,S,1], [n,R,3])."""
    device = torch.device(device)
    if device.type != 'cuda':
        raise RuntimeError('ide3d_b200.get_initial_rays_trig: device must be CUDA (no CPU path in this package)')
    W, H = resolution
    with torch.cuda.device(device):
        pts = torch.empty([n, W * H, num_steps, 3], device=device, dtype=torch.float32)
        zv = torch.empty([n, W * H, num_steps, 1], device=device, dtype=torch.float32)
        dirs = torch.empty([n, W * H, 3], device=device, dtype=torch.float32)
        rc = L.get_lib().ide3d_initial_rays(n, num_steps, float(fov), W, H, float(ray_start), float(ray_end),
                                            L.ptr(pts), L.ptr(zv), L.ptr(dirs), L.stream_ptr(device))
    L.check(rc)
    return pts, zv, dirs


_IDENTITY = {}


def _transform(points, z_vals, ray_directions, u, cam):
    _cuda_only(points, z_vals, ray_directions, cam)
    L.forbid_grad('transform_sampled_points / perturb_points', points, z_vals, ray_directions, cam)
    n, R, S, _ = points.shape
    p, z, d, c = _f32(points), _f32(z_vals), _f32(ray_directions), _f32(cam).reshape(n, 16)
    dev = p.device
    pw = torch.empty_like(p)
    zo = torch.empty_like(z)
    dw = torch.empty_like(d)
    ow = torch.empty_like(d)
    rc = L.get_lib().ide3d_transform_points(L.ptr(p), L.ptr(z), L.ptr(d), L.ptr(u), L.ptr(c), n, R, S, L.ptr(pw),
                                            L.ptr(zo), L.ptr(dw), L.ptr(ow), L.stream_ptr(dev))
    L.check(rc)
    return pw, zo, dw, ow


def perturb_points(points, z_vals, ray_directions, device):
    """Stratified jitter: offset = (U[0,1) - 0.5) * (z[1] - z[0]) along each ray."""
    u = torch.rand(z_vals.shape, device=z_vals.device)
    eye = torch.eye(4, device=points.device).unsqueeze(0).repeat(points.shape[0], 1, 1)
    pw, zo, _, _ = _transform(points, z_vals, ray_directions, u.contiguous(), eye)
    return pw, zo


def transform_sampled_points(points, z_vals, ray_directions, device, h_stddev=1, v_stddev=1, h_mean=math.pi * 0.5,
                             v_mean=math.pi * 0.5, radius=1, camera=None, mode='normal'):
    """Jitter the samples, pick a camera (sampled, or `camera` if given) and map camera space -> world space.
    Draw order matches the reference: jitter uniforms first, then the pose draws (:113-116)."""
    n = points.shape[0]
    u = torch.rand(z_vals.shape, device=z_vals.device)
    camera_origin, pitch, yaw = sample_camera_positions(n=n, r=radius, horizontal_stddev=h_stddev,
                                                        vertical_stddev=v_stddev, horizontal_mean=h_mean,
                                                        vertical_mean=v_mean, device=points.device, mode=mode)
    cam2world = create_cam2world_matrix(normalize_vecs(-camera_origin), camera_origin, device=points.device)
    if camera is not None:
        cam2world = camera
    pw, zo, dw, ow = _transform(points, z_vals, ray_directions, u.contiguous(), cam2world)
    return pw, zo, dw, ow, pitch, yaw


# ----------------------------------------------------------------------------------------------- camera poses
def truncated_normal_(tensor, mean=0, std=1):
    size = tensor.shape
    tmp = tensor.new_empty(size + (4,)).normal_()
    valid = (tmp < 2) & (tmp > -2)
    ind = valid.max(-1, keepdim=True)[1]
    tensor.data.copy_(tmp.gather(-1, ind).squeeze(-1))
    tensor.data.mul_(std).add_(mean)
    return tensor


def sample_camera_positions(device, n=1, r=1, horizontal_stddev=0.3, vertical_stddev=0.155,
                            horizontal_mean=math.pi * 0.5, vertical_mean=math.pi * 0.5, mode='normal', generator=None):
    """n camera origins on a sphere of radius r: theta = yaw, phi = pitch; returns (origins, phi, theta).  `generator` (a
    torch.Generator on `device`) feeds the uniform and gaussian draws instead of the global RNG."""
    def uni():
        return torch.rand((n, 1), device=device, generator=generator) - 0.5

    def gau():
        return torch.randn((n, 1), device=device, generator=generator)

    if mode == 'uniform':
        theta = uni() * 2 * horizontal_stddev + horizontal_mean
        phi = uni() * 2 * vertical_stddev + vertical_mean
    elif mode in ('normal', 'gaussian'):
        theta = gau() * horizontal_stddev + horizontal_mean
        phi = gau() * vertical_stddev + vertical_mean
    elif mode == 'hybrid':
        if random.random() < 0.5:
            theta = uni() * 2 * horizontal_stddev * 2 + horizontal_mean
            phi = uni() * 2 * vertical_stddev * 2 + vertical_mean
        else:
            theta = gau() * horizontal_stddev + horizontal_mean
            phi = gau() * vertical_stddev + vertical_mean
    elif mode == 'truncated_gaussian':
        theta = truncated_normal_(torch.zeros((n, 1), device=device)) * horizontal_stddev + horizontal_mean
        phi = truncated_normal_(torch.zeros((n, 1), device=device)) * vertical_stddev + vertical_mean
    elif mode == 'spherical_uniform':
        theta = uni() * 2 * horizontal_stddev + horizontal_mean
        v_std, v_mean = vertical_stddev / math.pi, vertical_mean / math.pi
        v = torch.clamp(uni() * 2 * v_std + v_mean, 1e-5, 1 - 1e-5)
        phi = torch.arccos(1 - 2 * v)
    else:   # any other value: use the means
        theta = torch.ones((n, 1), device=device, dtype=torch.float) * horizontal_mean
        phi = torch.ones((n, 1), device=device, dtype=torch.float) * vertical_mean
    phi = torch.clamp(phi, 1e-5, math.pi - 1e-5)
    out = torch.zeros((n, 3), device=device)
    out[:, 0:1] = r * torch.sin(phi) * torch.cos(theta)
    out[:, 2:3] = r * torch.sin(phi) * torch.sin(theta)
    out[:, 1:2] = r * torch.cos(phi)
    return out, phi, theta


def create_cam2world_matrix(forward_vector, origin, device=None):
    """cam2world = T(origin) @ R with R's columns (-left, up, -forward)."""
    fwd = normalize_vecs(forward_vector)
    up0 = torch.tensor([0, 1, 0], dtype=torch.float, device=device).expand_as(fwd)
    left = normalize_vecs(torch.cross(up0, fwd, dim=-1))
    up = normalize_vecs(torch.cross(fwd, left, dim=-1))
    n = fwd.shape[0]
    rot = torch.eye(4, device=device).unsqueeze(0).repeat(n, 1, 1)
    rot[:, :3, :3] = torch.stack((-left, up, -fwd), axis=-1)
    trans = torch.eye(4, device=device).unsqueeze(0).repeat(n, 1, 1)
    trans[:, :3, 3] = origin
    return trans @ rot


def create_world2cam_matrix(forward_vector, origin, device=None):
    return torch.inverse(create_cam2world_matrix(forward_vector, origin, device=device))


# ----------------------------------------------------------------------------------------------- importance pdf
def sample_pdf_u(bins, weights, u, eps=1e-5):
    """sample_pdf with the uniform draws u [R, N_importance] given (ide3d_sample_pdf: cumsum, searchsorted, gather, lerp in one kernel)."""
    _cuda_only(bins, weights, u)
    n_rays, n_s = weights.shape
    n_imp = u.shape[1]
    b, w, u = _f32(bins), _f32(weights), _f32(u)
    out = torch.empty([n_rays, n_imp], device=b.device, dtype=torch.float32)
    with torch.cuda.device(b.device):
        rc = L.get_lib().ide3d_sample_pdf(L.ptr(b), L.ptr(w), L.ptr(u), n_rays, n_s, n_imp, float(eps), L.ptr(out), L.stream_ptr(b.device))
    L.check(rc)
    return out


def sample_pdf(bins, weights, N_importance, det=False, eps=1e-5):
    """Inverse-CDF importance sampling: bins [R, S+1], weights [R, S] -> samples [R, N_importance]."""
    _cuda_only(bins, weights)
    L.forbid_grad('sample_pdf', bins, weights)
    n_rays = weights.shape[0]
    if det:
        u = torch.linspace(0, 1, N_importance, device=bins.device).expand(n_rays, N_importance)
    else:
        u = torch.rand(n_rays, N_importance, device=bins.device)
    return sample_pdf_u(bins, weights, u.contiguous(), eps)


class LookAtPoseSampler:
    """Camera on a sphere looking at `lookat_position` (phi = arccos(1 - 2 v / pi))."""

    @staticmethod
    def sample(horizontal_mean, vertical_mean, lookat_position, horizontal_stddev=0, vertical_stddev=0, radius=1,
               batch_size=1, device='cpu'):
        h = torch.randn((batch_size, 1), device=device) * horizontal_stddev + horizontal_mean
        v = torch.randn((batch_size, 1), device=device) * vertical_stddev + vertical_mean
        v = torch.clamp(v, 1e-5, math.pi - 1e-5)
        phi = torch.arccos(1 - 2 * (v / math.pi))
        origins = torch.zeros((batch_size, 3), device=device)
        origins[:, 0:1] = radius * torch.sin(phi) * torch.cos(h)
        origins[:, 2:3] = radius * torch.sin(phi) * torch.sin(h)
        origins[:, 1:2] = radius * torch.cos(phi)
        forward = normalize_vecs(lookat_position - origins)
        return create_cam2world_matrix(forward, origins, device=device)
