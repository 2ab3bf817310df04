#!/usr/bin/env python
"""Benchmark of the projector (ide3d_b200.projector) on the bench generator (random-init ide3d-ffhq-64-512: 256^2 planes, 64^2 x 96
render -> 512^2).  Prints one JSON line per case, with the card name and power limit read in the same run.

  (a) step     ms per projection step (median over --rounds rounds, each visiting every case and arm in turn, of the median
               per-step interval after --warmup steps) for plain W, mirror,
               mirror + refine_camera and mirror + refine_camera + target_seg; each against the same step with the reference's
               structure through this package: the mirrored view as two G.synthesis calls, the noise regulariser, its backward and the
               renormalisation as the torch loop, the seg term as interpolate + F.cross_entropy
  (b) noise    regulariser forward + backward + renormalisation over the generator's noise buffers: kernels against the torch loop,
               ms (CUDA events) and kernel launches (torch.profiler, a separate run)
  (c) seg_xent seg_cross_entropy forward + backward, 2 frames, 64^2 -> 512^2, against interpolate + F.cross_entropy autograd

The feature network is torchvision's VGG16 architecture, random-init, behind the projectors' feature contract (five ReLU taps,
unit-normalised per channel and concatenated): the reference's vgg16.pt has the same convolutions, and nothing is downloaded.

    python scripts/bench_project.py [--steps 20] [--warmup 5] [--reps 20] [--rounds 3]
"""
import argparse, contextlib, json, os, subprocess, sys
import numpy as np
import torch
import torch.nn.functional as F
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True, text=True)
    return r.stdout.strip() or 'unknown'


class VGGFeatures(torch.nn.Module):
    TAPS = (3, 8, 15, 22, 29)

    def __init__(self):
        super().__init__()
        import torchvision
        self.body = torchvision.models.vgg16(weights=None).features[:30]

    def forward(self, img, resize_images=True, return_lpips=False):
        x = (img / 255 - 0.45) / 0.225
        fs = []
        for i, layer in enumerate(self.body):
            x = layer(x)
            if i in self.TAPS:
                fs.append((x / (x.square().sum(1, keepdim=True).sqrt() + 1e-10)).flatten(1) / (x.shape[2] * x.shape[3]) ** 0.5)
        return torch.cat(fs, 1)


def events_between(n):
    evs = []

    def on_step(step, dist, loss):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        evs.append(e)
    return evs, on_step


@contextlib.contextmanager
def reference_structure():
    """The reference's step structure through this package: two synthesis calls for the mirror, torch loops for the noise, torch
    cross-entropy."""
    from ide3d_b200.torch_utils.ops import projection as P
    from ide3d_b200.training import triplane
    from oracle import projector as op
    S = triplane.SynthesisNetwork
    fwd = S.forward

    def two_calls(self, ws, c=None, views=1, return_seg=False, **kw):
        if views == 1:
            return fwd(self, ws, c=c, return_seg=return_seg, **kw)
        outs = [fwd(self, ws, c=c[j::views], return_seg=return_seg, **kw) for j in range(views)]
        if return_seg:
            return torch.cat([o[0] for o in outs]), torch.cat([o[1] for o in outs])
        return torch.cat(outs)
    saved = (S.forward, P.noise_regularizer, P.noise_normalize_, P.seg_cross_entropy)
    S.forward, P.noise_regularizer, P.noise_normalize_, P.seg_cross_entropy = two_calls, op.noise_reg, op.noise_normalize_, op.seg_cross_entropy
    try:
        yield
    finally:
        S.forward, P.noise_regularizer, P.noise_normalize_, P.seg_cross_entropy = saved


def step_ms(G, label, target, feats, mask, opts, steps, warmup):
    from ide3d_b200 import projector
    evs, on_step = events_between(steps)
    torch.manual_seed(0)
    projector.project(G, label, target, features=feats, num_steps=steps + warmup + 1, w_avg_samples=1000, on_step=on_step,
                      target_seg=mask if opts.get('seg') else None, seg_weight=1.0 if opts.get('seg') else 0.0,
                      mirror=opts.get('mirror', False), refine_camera=opts.get('refine', False))
    torch.cuda.synchronize()
    t = [a.elapsed_time(b) for a, b in zip(evs[warmup:-1], evs[warmup + 1:])]
    return float(np.median(t))


def timeit(fn, reps, warm):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def kernel_launches(fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(e.count for e in prof.key_averages() if e.device_type == torch.autograd.DeviceType.CUDA and 'Memcpy' not in e.key
               and 'Memset' not in e.key)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_project.py measures on a CUDA device'
    from ide3d_b200.compat import random_init_generator
    from ide3d_b200.torch_utils.ops import projection
    from ide3d_b200.training.triplane import upsample_seg
    from oracle import projector as op
    dev = torch.device('cuda')
    gpu = card()
    G = random_init_generator(device=dev, seed=0)
    sys.path.insert(0, ROOT)
    from bench import make_labels
    label = make_labels(1).to(dev)
    feats = VGGFeatures().eval().requires_grad_(False).to(dev)
    with torch.no_grad():
        ws = G.mapping(torch.randn(1, G.z_dim, device=dev), label)
        img, seg_raw = G.synthesis(ws, c=label, noise_mode='const', return_seg='raw')
    target = ((img[0] + 1) * 127.5).clamp(0, 255)
    mask = upsample_seg(seg_raw, (512, 512)).argmax(1)[0].to(torch.uint8)

    cases = {'plain': {}, 'mirror': dict(mirror=True), 'mirror_refine': dict(mirror=True, refine=True),
             'mirror_refine_seg': dict(mirror=True, refine=True, seg=True)}
    times = {(name, arm): [] for name in cases for arm in ('ours', 'ref')}
    for _ in range(args.rounds):                     # every round visits every case and both arms in turn: drift spreads over all of them
        for name, opts in cases.items():
            times[name, 'ours'].append(step_ms(G, label, target, feats, mask, opts, args.steps, args.warmup))
            with reference_structure():
                times[name, 'ref'].append(step_ms(G, label, target, feats, mask, opts, args.steps, args.warmup))
    for name in cases:
        ours, ref = times[name, 'ours'], times[name, 'ref']
        print(json.dumps({'case': f'step/{name}', 'ms_per_step': float(np.median(ours)), 'reference_structure_ms_per_step': float(np.median(ref)),
                          'speedup': float(np.median(ref) / np.median(ours)), 'ms_per_step_rounds': ours,
                          'reference_structure_rounds': ref, 'gpu': gpu}), flush=True)

    torch.manual_seed(0)
    bufs = [b.detach().clone().normal_() for n, b in G.synthesis.named_buffers() if 'noise_const' in n]

    def noise_step(reg, norm):
        def run():
            live = [b.requires_grad_(True) for b in bufs]
            reg(live).mul(1e5).backward()
            for b in live:
                b.grad = None
                b.requires_grad_(False)
            norm(live)
        return run
    fused, loop = noise_step(projection.noise_regularizer, projection.noise_normalize_), noise_step(op.noise_reg, op.noise_normalize_)
    print(json.dumps({'case': 'noise', 'buffers': len(bufs), 'sides': sorted({b.shape[0] for b in bufs}),
                      'kernel_ms': timeit(fused, args.reps, 3), 'torch_loop_ms': timeit(loop, args.reps, 3),
                      'kernel_launches': kernel_launches(fused), 'torch_loop_launches': kernel_launches(loop), 'gpu': gpu}), flush=True)

    g = torch.Generator(device=dev).manual_seed(0)
    feat = torch.randn(2, 64 * 64, 51, generator=g, device=dev, requires_grad=True)
    m2 = torch.randint(0, 19, (2, 512, 512), generator=g, device=dev, dtype=torch.uint8)
    view = lambda: feat.permute(0, 2, 1).reshape(2, 51, 64, 64)[:, 32:]
    ker = lambda: projection.seg_cross_entropy(view(), m2).backward()
    tor = lambda: F.cross_entropy(upsample_seg(view(), (512, 512)), m2.long()).backward()
    print(json.dumps({'case': 'seg_xent', 'frames': 2, 'render': 64, 'out': 512, 'kernel_ms': timeit(ker, args.reps, 3),
                      'torch_ms': timeit(tor, args.reps, 3), 'gpu': gpu}), flush=True)


if __name__ == '__main__':
    main()
