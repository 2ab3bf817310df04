#!/usr/bin/env python
"""Benchmark of mask-driven editing (ide3d_b200.edit) on the bench generator (random-init ide3d-ffhq-64-512) with a random-init
HybridEncoder(512, num_ws - 8, 8).  Prints one JSON line per case, with the card name and power limit read in the same run.  Every
timed case alternates its arms over --rounds rounds after a warm-up of every arm; the median is reported.

  (a) geometry  the geometry branch for 1 and 8 masks at 512^2, from host uint8 masks: the reference structure (host float64 one-hot,
                upload, *2-1, full composition) vs the device one-hot composition vs the ide3d_seg_stem path; wall clock to a sync
  (b) stem      ide3d_seg_stem alone (tables + stem launches), CUDA events over --reps calls; GB/s over the algorithmic bytes
                N*H*W*(1 + 4*C0) + N*(H/2)*(W/2)*4*C1 against the 3.35 TB/s of the H100 SXM data sheet
  (c) painter   one Painter edit with a pivot, wall clock including the mask upload: the reference structure through this package
                (pivot render, E(render, float one-hot), splice, render) vs edit()
  (d) reenact   4 latents x 32 (mask, camera) frames: frames/s of reenact() vs the per-frame loop of infer_face_animation.py:144-148

    python scripts/bench_edit.py [--rounds 3] [--reps 20]
"""
import argparse, json, os, subprocess, sys, time
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True, text=True)
    return r.stdout.strip() or 'unknown'


def wall_ms(fn, reps):
    out = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t) * 1e3)
    return float(np.median(out))


def host_one_hot(mask_np):
    """mask2label_np (dnnlib/seg_tools.py:67-72) per mask, float64 on the host."""
    labels = np.zeros((mask_np.shape[0], 19) + mask_np.shape[1:])
    for n in range(mask_np.shape[0]):
        for i in range(19):
            labels[n, i][mask_np[n] == i] = 1.0
    return labels


def alternate(arms, rounds, reps):
    for fn in arms.values():                                   # warm-up: modules, cuDNN algorithms, allocator
        wall_ms(fn, 2)
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            res[k].append(wall_ms(fn, reps))
    return {k: float(np.median(v)) for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--frames', type=int, default=32)
    args = ap.parse_args()
    from ide3d_b200 import edit
    from ide3d_b200.compat import random_init_generator
    from ide3d_b200.encoder import HybridEncoder, one_hot_input
    from ide3d_b200.torch_utils.ops import seg_stem
    dev = torch.device('cuda')
    gpu = card()
    G = random_init_generator(device=dev, seed=0)
    torch.manual_seed(1)
    E = HybridEncoder(512, G.num_ws - 8, 8, w_dim=G.w_dim).eval().requires_grad_(False).to(dev)
    rs = np.random.RandomState(0)
    masks_np = np.kron(rs.randint(0, 19, (8, 32, 32)), np.ones((1, 16, 16), np.int64)).astype(np.uint8)
    emit = lambda d: print(json.dumps(dict(d, gpu=gpu)), flush=True)

    with torch.no_grad():
        # (a) geometry branch
        for n in (1, 8):
            m = torch.from_numpy(masks_np[:n])
            arms = {'reference': lambda: E.geometry(torch.from_numpy(host_one_hot(m.numpy())).float().to(dev) * 2 - 1),
                    'device_one_hot': lambda: E.geometry(one_hot_input(m.to(dev), 19)),
                    'kernel': lambda: E.geometry(m.to(dev))}
            r = alternate(arms, args.rounds, args.reps if n == 1 else max(3, args.reps // 4))
            emit(dict(case='geometry', masks=n, ms=r, speedup_vs_reference=r['reference'] / r['kernel'],
                      speedup_vs_device_one_hot=r['device_one_hot'] / r['kernel']))

        # (b) the stem kernel alone
        stem, block = E.convs_seg[0], E.convs_seg[1]
        for n in (1, 8):
            m = torch.from_numpy(masks_np[:n]).to(dev)
            c0, c1 = stem.weight.shape[0], block.skip.weight.shape[0]
            nbytes = n * 512 * 512 * (1 + 4 * c0) + n * 256 * 256 * 4 * c1
            times = []
            for _ in range(args.rounds):
                seg_stem.seg_stem(m, stem, block.conv1, block.skip)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(args.reps):
                    seg_stem.seg_stem(m, stem, block.conv1, block.skip)
                b.record()
                torch.cuda.synchronize()
                times.append(a.elapsed_time(b) / args.reps)
            ms = float(np.median(times))
            emit(dict(case='seg_stem', masks=n, ms=ms, algorithmic_bytes=nbytes, gbps=nbytes / ms / 1e6,
                      share_of_3350_gbps=nbytes / ms / 1e6 / 3350))

        # (c) one Painter edit with a pivot
        z = torch.from_numpy(rs.randn(4, G.z_dim)).float().to(dev)
        c_front = torch.tensor(edit.FRONTAL, device=dev).reshape(1, -1)
        ws = G.mapping(z, c_front.repeat(4, 1))
        pivot, label = ws[:1], c_front
        m1 = torch.from_numpy(masks_np[:1])
        w_avg = G.mapping.w_avg[None, None, :]

        def painter_reference():
            seg = torch.from_numpy(host_one_hot(m1.numpy())).view(1, 19, 512, 512).float().to(dev) * 2 - 1
            gen = G.synthesis(pivot, c=label, render_params={'num_steps': 96}, noise_mode='const')
            rec = w_avg + E(gen, seg)
            rec[:, 8:] = pivot[:, 8:]
            return G.synthesis(rec, c=label, noise_mode='const')
        r = alternate({'reference': painter_reference, 'edit': lambda: edit.edit(G, E, pivot, label, m1)}, args.rounds, args.reps)
        emit(dict(case='painter_edit', ms=r, speedup=r['reference'] / r['edit']))

        # (d) reenactment: 4 latents x F frames
        from ide3d_b200.images import view_cameras
        F_ = args.frames
        labels = view_cameras(tuple(np.linspace(-0.4, 0.4, F_)), device=dev)
        drive = torch.from_numpy(np.kron(rs.randint(0, 19, (F_, 32, 32)), np.ones((1, 16, 16), np.int64)).astype(np.uint8))
        rp = edit.REENACT_RENDER_PARAMS

        def reenact_loop():
            for f in range(F_):
                c = labels[f:f + 1].repeat(4, 1)
                seg = torch.from_numpy(host_one_hot(drive[f:f + 1].numpy())).float().to(dev) * 2 - 1
                cond = G.synthesis(ws, c, noise_mode='const', render_params=rp)
                rec = E(cond, seg.repeat(4, 1, 1, 1)) + w_avg
                G.synthesis(rec, c, noise_mode='const', render_params=rp)
        r = alternate({'loop': reenact_loop, 'reenact': lambda: edit.reenact(G, E, ws, labels, drive)}, args.rounds, 1)
        emit(dict(case='reenact', latents=4, frames=F_, ms=r, frames_per_s={k: 4 * F_ / v * 1e3 for k, v in r.items()},
                  speedup=r['loop'] / r['reenact']))


if __name__ == '__main__':
    main()
