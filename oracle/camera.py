"""Oracle (test infrastructure): camera pose helpers restated from the reference.

Follows the reference's training/volumetric_rendering.py
  * sample_camera_positions   :147-193
  * create_cam2world_matrix   :195-213
  * LookAtPoseSampler.sample  :268-295
Deterministic restatement: the random modes take the standard-normal / uniform draws as explicit
arguments (``eps_h``, ``eps_v``) instead of consuming a global RNG, so tests can inject them.
"""

import math

import numpy as np


def _unit(v):
    v = np.asarray(v, dtype=np.float32)
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def camera_origin(theta, phi, r):
    """Spherical -> cartesian, reference :187-191 (theta = yaw, phi = pitch, phi clamped :185)."""
    theta = np.asarray(theta, dtype=np.float32).reshape(-1, 1)
    phi = np.clip(np.asarray(phi, dtype=np.float32).reshape(-1, 1), 1e-5, math.pi - 1e-5).astype(np.float32)
    out = np.zeros((theta.shape[0], 3), dtype=np.float32)
    out[:, 0:1] = r * np.sin(phi) * np.cos(theta)
    out[:, 2:3] = r * np.sin(phi) * np.sin(theta)
    out[:, 1:2] = r * np.cos(phi)
    return out, phi, theta


def sample_camera_positions(n=1, r=1.0, horizontal_stddev=0.3, vertical_stddev=0.155,
                            horizontal_mean=math.pi * 0.5, vertical_mean=math.pi * 0.5,
                            mode='normal', eps_h=None, eps_v=None):
    """Reference :147-193.  ``eps_h/eps_v`` are the raw draws ([n,1]): N(0,1) for the gaussian modes,
    U[0,1) for the uniform modes.  ``mode`` not in the known set means "use the mean" (:180-183)."""
    eps_h = np.zeros((n, 1), np.float32) if eps_h is None else np.asarray(eps_h, np.float32).reshape(n, 1)
    eps_v = np.zeros((n, 1), np.float32) if eps_v is None else np.asarray(eps_v, np.float32).reshape(n, 1)
    if mode == 'uniform':
        theta = (eps_h - 0.5) * 2 * horizontal_stddev + horizontal_mean
        phi = (eps_v - 0.5) * 2 * vertical_stddev + vertical_mean
    elif mode in ('normal', 'gaussian'):
        theta = eps_h * horizontal_stddev + horizontal_mean
        phi = eps_v * vertical_stddev + vertical_mean
    elif mode == 'spherical_uniform':
        theta = (eps_h - 0.5) * 2 * horizontal_stddev + horizontal_mean
        v_std, v_mean = vertical_stddev / math.pi, vertical_mean / math.pi
        v = np.clip((eps_v - 0.5) * 2 * v_std + v_mean, 1e-5, 1 - 1e-5)
        phi = np.arccos(1 - 2 * v)
    else:
        theta = np.full((n, 1), horizontal_mean, np.float32)
        phi = np.full((n, 1), vertical_mean, np.float32)
    return camera_origin(theta.astype(np.float32), phi.astype(np.float32), r)


def create_cam2world_matrix(forward, origin):
    """Reference :195-213.  cam2world = T(origin) @ R, R columns = (-left, up, -forward)."""
    fwd = _unit(forward)
    up0 = np.broadcast_to(np.array([0, 1, 0], np.float32), fwd.shape)
    left = _unit(np.cross(up0, fwd))
    up = _unit(np.cross(fwd, left))
    n = fwd.shape[0]
    rot = np.tile(np.eye(4, dtype=np.float32), (n, 1, 1))
    rot[:, :3, :3] = np.stack((-left, up, -fwd), axis=-1)
    trans = np.tile(np.eye(4, dtype=np.float32), (n, 1, 1))
    trans[:, :3, 3] = np.asarray(origin, np.float32)
    return (trans @ rot).astype(np.float32)


def look_at_pose(horizontal_mean, vertical_mean, lookat, radius=1.0, batch_size=1,
                 horizontal_stddev=0.0, vertical_stddev=0.0, eps_h=None, eps_v=None):
    """Reference LookAtPoseSampler.sample :278-295 (phi = arccos(1 - 2 v / pi))."""
    eps_h = np.zeros((batch_size, 1), np.float32) if eps_h is None else np.asarray(eps_h, np.float32)
    eps_v = np.zeros((batch_size, 1), np.float32) if eps_v is None else np.asarray(eps_v, np.float32)
    h = (eps_h * horizontal_stddev + horizontal_mean).astype(np.float32)
    v = (eps_v * vertical_stddev + vertical_mean).astype(np.float32)
    v = np.clip(v, 1e-5, math.pi - 1e-5)
    phi = np.arccos(1 - 2 * (v / math.pi)).astype(np.float32)
    origins = np.zeros((batch_size, 3), np.float32)
    origins[:, 0:1] = radius * np.sin(phi) * np.cos(h)
    origins[:, 2:3] = radius * np.sin(phi) * np.sin(h)
    origins[:, 1:2] = radius * np.cos(phi)
    fwd = _unit(np.asarray(lookat, np.float32).reshape(1, 3) - origins)
    return create_cam2world_matrix(fwd, origins)
