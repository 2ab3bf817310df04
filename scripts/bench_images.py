#!/usr/bin/env python
"""Benchmark of the multi-view image path (gen_images.py:84-116) on the random-init ide3d-ffhq-64-512 generator (64^2 x 96 render ->
512^2), 3 yaws per seed.  CUDA events around device-synchronised regions, median of --reps after --warmup.  PNG encoding is not timed.
Prints one JSON line per case with the card name and power limit:

  (a) loop     gen_images.py's loop through this package at batch 1: per seed one mapping call, three G.synthesis calls, torch mask2color
               on the 512^2 logits, the make_grid + save_image conversion on the device (oracle.images.grid_bytes)
  (b) driver   images.render_multiview (views=3: one backbone pass per seed), strips downloaded to the host
  (c) no_share the driver's batches with views=1 and ws repeated per view (the backbone runs once per view): isolates backbone sharing
  (d) strips   ide3d_image_strips against the torch composition (oracle.images.compose_strips on the device), 8 seeds x 3 views
  (e) march    the ray-march for 24 frames: 8 plane sets x 3 views against 24 plane sets

    python scripts/bench_images.py [--seeds 16] [--reps 5] [--warmup 2]
"""
import argparse, json, os, subprocess, sys
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True, text=True)
    return r.stdout.strip() or 'unknown'


def timeit(fn, reps, warm):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(min(ts)), float(max(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--seeds', type=int, default=16)
    ap.add_argument('--batch-seeds', type=int, default=8)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_images needs a CUDA device'
    from ide3d_b200 import images, render
    from ide3d_b200.compat import random_init_generator
    from ide3d_b200.dnnlib.seg_tools import mask2color
    from oracle.images import compose_strips as torch_strips, grid_bytes
    torch.backends.cudnn.benchmark = True
    dev = torch.device('cuda')
    G = random_init_generator(device=dev, seed=0)
    gpu = card()
    seeds = list(range(args.seeds))
    V = len(images.YAWS)
    out = lambda **kw: print(json.dumps(dict(kw, **{'gpu (name, power limit)': gpu})), flush=True)

    cams = images.view_cameras(images.YAWS, dev)
    cs = torch.tensor(images.FRONTAL).float().to(dev).reshape(1, -1)

    @torch.no_grad()
    def loop():
        for seed in seeds:
            torch.manual_seed(seed)
            z = torch.from_numpy(np.random.RandomState(seed).randn(1, G.z_dim)).to(dev)
            ws = G.mapping(z=z, c=cs, truncation_psi=0.7)
            imgs, segs = [], []
            for k, yaw in enumerate(images.YAWS):
                img, seg = G.synthesis(ws, c=cams[k:k + 1], render_params=images.render_params(yaw), noise_mode='const', return_seg=True)
                imgs.append(img)
                segs.append((mask2color(seg) / 255. - 0.5) / 0.5)
            grid_bytes(torch.cat(imgs)).cpu()
            grid_bytes(torch.cat(segs)).cpu()

    def driver():
        images.render_multiview(G, seeds, psi=0.7, batch_seeds=args.batch_seeds)

    # (c): the driver's batches, but every view runs its own backbone (views=1, ws and jitter seeds repeated per view)
    z_all = torch.from_numpy(np.concatenate([np.random.RandomState(s).randn(1, G.z_dim) for s in seeds])).to(dev)
    with torch.no_grad():
        ws_all = G.mapping(z=z_all, c=cs.repeat(len(seeds), 1), truncation_psi=0.7)
    jit = torch.tensor([images.view_seeds(s, V) for s in seeds], dtype=torch.int64)
    rp = images.render_params(images.YAWS[0])

    @torch.no_grad()
    def batches(views):
        B = args.batch_seeds
        for b0 in range(0, len(seeds), B):
            w = ws_all[b0:b0 + B]
            k = w.shape[0]
            if views == 1:
                w = w.repeat_interleave(V, 0)
            img, seg_raw = G.synthesis(w, c=cams.repeat(k, 1), render_params=rp, noise_mode='const', return_seg='raw', views=views,
                                       seed=jit[b0:b0 + B].reshape(-1))
            a, b = images.compose_strips(img, seg_raw, V)
            torch.stack((a, b), 1).cpu()

    n_frames = len(seeds) * V
    for name, fn in (('loop', loop), ('driver', driver), ('no_share', lambda: batches(1)), ('share', lambda: batches(V))):
        med, lo, hi = timeit(fn, args.reps, args.warmup)
        out(case=name, seeds=len(seeds), views=V, batch_seeds=args.batch_seeds if name != 'loop' else 1, ms_median=med, ms_min=lo, ms_max=hi,
            seeds_per_s=1e3 * len(seeds) / med, frames_per_s=1e3 * n_frames / med)

    # (d) strips: 8 seeds x 3 views, 512^2 images (channels-last, as the SR blocks hand them out) and the strided 64^2 logits view
    n, H, R = 8 * V, G.img_resolution, G.neural_rendering_resolution
    g = torch.Generator(device=dev).manual_seed(0)
    img = torch.randn(n, 3, H, H, device=dev, generator=g).contiguous(memory_format=torch.channels_last)
    seg = torch.randn(n, R * R, 51, device=dev, generator=g).permute(0, 2, 1).reshape(n, 51, R, R)[:, 32:]
    t_k = timeit(lambda: images.compose_strips(img, seg, V), 50, 5)
    t_t = timeit(lambda: torch_strips(img, seg, V), 20, 3)
    same = bool(torch.equal(images.compose_strips(img, seg, V)[0], torch_strips(img, seg, V)[0]))
    out(case='strips', seeds=8, views=V, image=f'3x{H}^2', logits=f'19x{R}^2 strided view', kernel_ms=t_k[0], torch_composition_ms=t_t[0],
        speedup=t_t[0] / t_k[0], image_strip_equal=same)

    # (e) ray-march: 24 frames from 8 plane sets x 3 views against 24 plane sets (planes of the generator's backbone shape)
    P = G.synthesis.plane_resolution
    planes = lambda k: torch.randn(k, 96, P, P, device=dev, generator=g).contiguous(memory_format=torch.channels_last)
    tex8, seg8 = planes(8), planes(8)
    tex24, seg24 = tex8.repeat_interleave(V, 0), seg8.repeat_interleave(V, 0)
    dec = G.synthesis.renderer.packed()
    cam = cams.repeat(8, 1)[:, :16]
    kw = dict(resolution=(R, R), num_steps=96, jitter_seed=jit[:8].reshape(-1), box_scale=G.synthesis.renderer.box_scale)
    t_v = timeit(lambda: render.raymarch(tex8, seg8, dec, cam, views=V, **kw), 20, 3)
    t_m = timeit(lambda: render.raymarch(tex24, seg24, dec, cam, **kw), 20, 3)
    out(case='raymarch', frames=24, render=f'{R}^2 x 96', planes=f'{P}^2', shared_views_ms=t_v[0], separate_sets_ms=t_m[0],
        ratio=t_m[0] / t_v[0])


if __name__ == '__main__':
    main()
