#!/usr/bin/env python
"""Generate tests/golden/mesh_turntable.npz: the 240 camera poses of the reference's render_mesh.py (:44-55), computed by the
REFERENCE's own sample_camera_positions / create_cam2world_matrix (imported read-only from the IDE-3D tree named by IDE3D_REFERENCE)
exactly as the script does -- float32 torch on the CPU, then P[:3, 3] += 0.5 in numpy -- and checked on the spot against oracle/camera.py.

    IDE3D_REFERENCE=/path/to/IDE-3D PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_mesh_golden.py

tests/test_mesh_render.py replays the fixture against ide3d_b200.mesh.turntable_poses.
"""

import math
import os
import sys

import numpy as np
import torch

REF = os.environ.get('IDE3D_REFERENCE', '')
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.dont_write_bytecode = True
sys.path.insert(0, REF)
sys.path.insert(1, ROOT)

from training import volumetric_rendering as ref_vr            # noqa: E402  (reference)

from oracle import camera as ocam                                # noqa: E402


def turntable(num=240, radius=2.7):
    poses = []
    for i in range(num):
        yaw = math.pi * (0.5 + 0.15 * math.cos(2 * math.pi * i / num))
        pitch = math.pi * (0.5 - 0.05 * math.sin(2 * math.pi * i / num))
        p, _, _ = ref_vr.sample_camera_positions(device=None, n=1, r=radius, horizontal_mean=yaw, vertical_mean=pitch, mode=None)
        c = ref_vr.create_cam2world_matrix(-p, p, device=None)
        P = c.reshape(-1, 4, 4).numpy()[0]
        P[:3, 3] += 0.5
        oo, _, _ = ocam.sample_camera_positions(n=1, r=radius, horizontal_mean=yaw, vertical_mean=pitch, mode=None)
        Po = np.array(ocam.create_cam2world_matrix(-oo, oo), np.float32).reshape(4, 4)
        Po[:3, 3] += 0.5
        err = np.abs(P - Po).max()
        assert err <= 2e-6, f'turntable pose {i}: oracle differs by {err:g}'
        poses.append(P)
    return np.stack(poses)


if __name__ == '__main__':
    path = os.path.join(HERE, 'mesh_turntable.npz')
    np.savez_compressed(path, w_frames=240, radius=2.7, poses=turntable(240, 2.7))
    print(f'mesh_turntable {os.path.getsize(path) / 1024:8.1f} KB')
