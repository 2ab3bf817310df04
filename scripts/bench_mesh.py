#!/usr/bin/env python
"""render_mesh.py on the GPU: density grid -> marching cubes -> vertex normals -> 240 turntable frames at 512^2 (ide3d_b200.mesh).
Two workloads: (a) an analytic 256^3 sphere grid, (b) the random-init generator's 256^3 sigma grid (seed 0, cube_size 1) at
threshold 10 -- or, when that mesh is empty, at the grid's 90th-percentile sigma (reported).  Prints one JSON line per workload:
triangle count, CUDA-event times of marching cubes, normals and raster + shade per 8-frame batch, the wall-clock time of all 240
frames to host uint8, frames/s, and the numpy oracle's time for one frame on the host cores; with the card and its power limit."""
import json, os, subprocess, sys, time
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ide3d_b200 import mesh
from oracle import rasterizer as ora

FRAMES, RES, BATCH = 240, 512, 8


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                       capture_output=True, text=True)
    name, _, limit = q.stdout.strip().partition(', ')
    return name or torch.cuda.get_device_name(), limit or 'unknown'


def event_ms(fn, reps=10):
    fn(); torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize(); ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def run(name, sigma, threshold, note=None):
    v, t = mesh.mesh_from_sigma_grid(sigma, size=256, sigma_threshold=threshold)
    poses = mesh.turntable_poses(FRAMES)
    nrm = mesh.vertex_normals(v, t)
    res = {'workload': name, 'sigma_threshold': round(float(threshold), 4), 'triangles': int(t.shape[0]), 'vertices': int(v.shape[0])}
    if note:
        res['note'] = note
    res['marching_cubes_ms'] = round(event_ms(lambda: mesh.mesh_from_sigma_grid(sigma, size=256, sigma_threshold=threshold)), 3)
    res['normals_ms'] = round(event_ms(lambda: mesh.vertex_normals(v, t)), 3)
    res['raster_shade_ms_per_8_frames'] = round(event_ms(lambda: mesh.rasterize(v, t, poses[:BATCH], resolution=RES, normals=nrm)), 3)
    walls = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        host = mesh.render_turntable(sigma, size=256, sigma_threshold=threshold, w_frames=FRAMES, resolution=RES, batch=BATCH).cpu()
        walls.append(time.perf_counter() - t0)
    wall = float(np.median(walls))
    res['all_240_frames_to_host_s'] = round(wall, 3)
    res['frames_per_s'] = round(FRAMES / wall, 1)
    res['foreground_fraction_frame0'] = round(float((host[0, ..., 0] != 255).float().mean()), 4)
    vn, tn, pn = v.cpu().numpy(), t.cpu().numpy(), poses[:1].numpy()
    t0 = time.perf_counter()
    rgb_o = ora.rasterize(vn, tn, pn, resolution=RES, normals=nrm.cpu().numpy())
    res['oracle_one_frame_host_s'] = round(time.perf_counter() - t0, 3)
    res['frame0_max_abs_diff_vs_oracle'] = int(np.abs(rgb_o[0].astype(np.int16) - host[0].numpy()).max())
    res['card'], res['power_limit'] = card()
    print(json.dumps(res), flush=True)
    return host


def main():
    torch.backends.cuda.matmul.allow_tf32 = False
    n = 256
    g = torch.arange(n, dtype=torch.float32, device='cuda')
    x, y, z = torch.meshgrid(g, g, g, indexing='ij')
    sphere = 10.0 + 4.0 * (0.3 * n - torch.sqrt((x - n / 2) ** 2 + (y - n / 2) ** 2 + (z - n / 2) ** 2))
    del x, y, z
    run('analytic sphere 256^3 (r = 0.3)', sphere, 10.0)
    del sphere

    from ide3d_b200.torch_utils import custom_ops
    custom_ops.verbosity = 'none'
    from ide3d_b200.compat import random_init_generator
    G = random_init_generator('cuda', seed=0)
    with torch.no_grad():
        zz = torch.from_numpy(np.random.RandomState(0).randn(1, G.z_dim)).float().cuda()
        c = torch.tensor([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 2.7, 0, 0, 0, 1, 4.2647, 0, 0.5, 0, 4.2647, 0.5, 0, 0, 1.]).cuda()[None]
        ws = G.mapping(zz, c)
        vws, _ = G.synthesis.split_ws(ws)
        img_v, seg_v = G.synthesis.backbone(vws, noise_mode='const')
        R = G.synthesis.renderer
        sg = R.sigma_grid(R.as_planes(img_v), R.as_planes(seg_v), grid_n=n, cube_length=1.0).reshape(n, n, n)
    thr, note = 10.0, None
    if mesh.mesh_from_sigma_grid(sg, size=n, sigma_threshold=thr)[1].shape[0] == 0:
        thr = float(np.percentile(sg.cpu().numpy(), 90))
        note = f'no surface at sigma 10 (max sigma {float(sg.max()):.4g}); threshold = the grid\'s 90th-percentile sigma'
    run('random-init generator sigma grid 256^3 (seed 0, cube_size 1)', sg, thr, note)


if __name__ == '__main__':
    main()
