#!/usr/bin/env python
"""Benchmark of pivotal tuning (ide3d_b200.pti) on the bench generator (random-init ide3d-ffhq-64-512: 256^2 planes, 64^2 x 48
render -> 512^2) with a random-init AlexNet LPIPS.  Prints one JSON line per case, with the card name and power limit read in the
same run.

  (a) step      ms per tuning step (median over --rounds rounds, each visiting every case and arm in turn, of the median per-step
                interval after --warmup steps; CUDA events at the same point of every step) for plain and mirror, each against the same
                step with the reference's structure through this package (single_id_coach.py:60-89): the mirrored view as a second
                G.synthesis call, the LPIPS head as torch ops, the target's trunk recomputed every step
  (b) lpips     the LPIPS head alone, forward + backward, 1 sample at the AlexNet-on-512^2 layer shapes: kernels against
                lpips_head_torch autograd, ms (CUDA events, median of --reps) and kernel launches (torch.profiler, a separate pass)
  (c) freeview  free_view_frames (chunks of 24 cameras, one backbone pass each) against the 240-call batch-1 loop of
                run_pti.py:154-182, both to host uint8

    python scripts/bench_pti.py [--steps 12] [--warmup 3] [--reps 20] [--rounds 3] [--frames 240]
"""
import argparse, copy, json, os, subprocess, sys
import numpy as np
import torch
import torch.nn.functional as F
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True, text=True)
    return r.stdout.strip() or 'unknown'


def median_interval_ms(events, warmup):
    torch.cuda.synchronize()
    return float(np.median([a.elapsed_time(b) for a, b in zip(events[warmup:], events[warmup + 1:])]))


def ours_step(G, ws, c, target, lpips, mirror, steps, warmup):
    from ide3d_b200 import pti
    evs = []

    def mark(*_):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        evs.append(e)
    pti.tune(G, ws, c, target, lpips=lpips, steps=steps, mirror=mirror, lpips_threshold=-1.0, on_step=mark)
    return median_interval_ms(evs, warmup)


def reference_step(G, ws, c, target, lpips, mirror, steps, warmup):
    """single_id_coach.py:60-89 through this package: one synthesis call per view, trunk of the target every step, torch head."""
    from ide3d_b200 import projector
    from ide3d_b200.torch_utils.ops.lpips import lpips_head_torch
    R = copy.deepcopy(G).eval().requires_grad_(True)
    opt = torch.optim.Adam(R.parameters(), lr=3e-4)
    views = [(c, target[None])] + ([(projector.mirror_label(c), torch.flip(target[None], (3,)))] if mirror else [])
    evs = []
    for _ in range(steps):
        loss = 0.0
        for cam, real in views:
            img = R.synthesis(ws, c=cam, noise_mode='const', force_fp32=True)
            lp = lpips_head_torch(lpips.trunk(img), lpips.trunk(real), lpips.lin)[0]
            loss = loss + (F.mse_loss(img, real) + lp)
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        evs.append(e)
        opt.zero_grad()
        loss.backward()
        opt.step()
    return median_interval_ms(evs, warmup)


def launches(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type.name == 'CUDA' and 'Memcpy' not in e.name and 'Memset' not in e.name)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=12)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--frames', type=int, default=240)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_pti needs a CUDA device'
    from ide3d_b200 import pti
    from ide3d_b200.compat import random_init_generator
    from ide3d_b200.torch_utils.ops import lpips as LP
    from oracle import pti as opti
    dev = torch.device('cuda')
    name = card()
    G = random_init_generator(device=dev, seed=0)
    lpips = opti.standin_lpips().to(dev)
    torch.manual_seed(0)
    c = pti.free_view_cameras(1, dev)
    with torch.no_grad():
        ws = G.mapping(torch.randn(1, G.z_dim, device=dev), c, truncation_psi=0.7)
        target = G.synthesis(ws + 0.05 * torch.randn_like(ws), c=c, noise_mode='const')[0].clamp(-1, 1)

    # (a) tuning steps, alternating cases and arms
    results = {}
    for _ in range(args.rounds):
        for mirror in (False, True):
            for arm, fn in (('ours', ours_step), ('reference', reference_step)):
                results.setdefault((mirror, arm), []).append(fn(G, ws, c, target, lpips, mirror, args.steps, args.warmup))
    for mirror in (False, True):
        o, r = (float(np.median(results[(mirror, a)])) for a in ('ours', 'reference'))
        print(json.dumps(dict(case='step', mirror=mirror, ours_ms=round(o, 3), reference_ms=round(r, 3), speedup=round(r / o, 2),
                              ours_rounds=[round(v, 2) for v in results[(mirror, 'ours')]],
                              reference_rounds=[round(v, 2) for v in results[(mirror, 'reference')]], card=name)), flush=True)

    # (b) the head alone at the 512^2 AlexNet shapes
    g = torch.Generator(device=dev).manual_seed(1)
    shapes = [(64, 127, 127), (192, 63, 63), (384, 31, 31), (256, 31, 31), (256, 31, 31)]
    fx = [torch.relu(torch.randn(1, *s, device=dev, generator=g)).requires_grad_(True) for s in shapes]
    fy = [torch.relu(torch.randn(1, *s, device=dev, generator=g)) for s in shapes]
    lin = lpips.lin

    def run(head):
        for t in fx:
            t.grad = None
        head(fx, fy, lin).sum().backward()

    times = {}
    for _ in range(args.rounds):
        for arm, head in (('kernel', LP.lpips_head), ('torch', LP.lpips_head_torch)):
            for _ in range(3):
                run(head)
            ts = []
            for _ in range(args.reps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                run(head)
                b.record()
                torch.cuda.synchronize()
                ts.append(a.elapsed_time(b))
            times.setdefault(arm, []).append(float(np.median(ts)))
    k, t = float(np.median(times['kernel'])), float(np.median(times['torch']))
    print(json.dumps(dict(case='lpips_head', kernel_ms=round(k, 4), torch_ms=round(t, 4), speedup=round(t / k, 2),
                          kernel_launches=launches(lambda: run(LP.lpips_head)), torch_launches=launches(lambda: run(LP.lpips_head_torch)),
                          card=name)), flush=True)

    # (c) free-view frames
    rp = {'h_stddev': 0., 'v_stddev': 0., 'fov': 18, 'num_steps': 96}
    cams = pti.free_view_cameras(args.frames, dev)

    def loop():
        out = []
        with torch.no_grad():
            for f in range(args.frames):
                img = G.synthesis(ws, c=cams[f:f + 1], render_params=rp, noise_mode='const')
                out.append((img * 127.5 + 128).clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).cpu().numpy()[0])
        return np.stack(out)

    ft = {}
    pti.free_view_frames(G, ws, num_frames=24)
    loop_frames = None
    for _ in range(args.rounds):
        for arm, fn in (('free_view_frames', lambda: pti.free_view_frames(G, ws, num_frames=args.frames)), ('loop', loop)):
            torch.manual_seed(7)
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            out = fn()
            b.record()
            torch.cuda.synchronize()
            ft.setdefault(arm, []).append(a.elapsed_time(b))
            if arm == 'loop':
                loop_frames = out
            else:
                ours_frames = out
    diff = int(np.abs(ours_frames.astype(np.int16) - loop_frames.astype(np.int16)).max())
    o, r = float(np.median(ft['free_view_frames'])), float(np.median(ft['loop']))
    print(json.dumps(dict(case='freeview', frames=args.frames, ours_ms=round(o, 1), loop_ms=round(r, 1), speedup=round(r / o, 2),
                          max_uint8_diff=diff, card=name)), flush=True)


if __name__ == '__main__':
    main()
