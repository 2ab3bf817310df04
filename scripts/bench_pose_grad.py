#!/usr/bin/env python
"""Pose refinement / PTI-style renderer steps at BASELINE configs[1] sizes (8 frames, 64^2 x 96, 256^2 planes, bench generator):
forward (fused kernel) + backward on the backward-kernel path (ide3d_raymarch_bwd_cam) and on the composed-chain path
(render_grad.composed_chain + autograd), alternating the two paths rep by rep in one process.  Workloads:
  a  planes + decoder heads + camera
  b  camera only (frozen planes and decoder)
  c  hierarchical 96 + 96 samples, planes + decoder heads
One JSON line with the card name and power limit, the median times and the largest gradient difference between the paths."""
import json, os, subprocess, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ide3d_b200 import render, render_grad
from ide3d_b200.torch_utils import custom_ops
custom_ops.verbosity = 'none'


def power_limit():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def main():
    from bench import make_labels, make_latents, build_generator, NUM_STEPS, RENDER
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 8
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    G = build_generator('cuda')
    with torch.no_grad():
        c = make_labels(8).cuda()[:n]
        ws = G.mapping(make_latents(n, G.z_dim).cuda(), c)
        vws, _ = G.synthesis.split_ws(ws)
        img_v, seg_v = G.synthesis.backbone(vws, noise_mode='const')
    cam = c[:, :16].reshape(-1, 4, 4)
    Rn = G.synthesis.renderer
    RR = RENDER * RENDER
    g = torch.Generator(device='cuda').manual_seed(0)
    gf = torch.randn(n, RR, 51, device='cuda', generator=g)
    gd = torch.randn(n, RR, 1, device='cuda', generator=g)
    importance_u = torch.rand(n * RR, NUM_STEPS, device='cuda', generator=g)
    kw = dict(resolution=(RENDER, RENDER), num_steps=NUM_STEPS, jitter_seed=5, box_scale=Rn.box_scale)

    def step(planes, heads_grad, camera, hierarchical):
        t, s = img_v.detach().clone().requires_grad_(planes), seg_v.detach().clone().requires_grad_(planes)
        heads = [tuple(h[:2]) + tuple(x.detach().clone().requires_grad_(heads_grad) for x in h[2:]) for h in Rn.heads()]
        cm = cam.detach().clone().requires_grad_(camera)
        if hierarchical:
            feat, d, _ = render.raymarch_hierarchical(t, s, heads, cm, n_importance=NUM_STEPS, importance_u=importance_u, **kw)
        else:
            feat, d, _ = render.raymarch(t, s, heads, cm, **kw)
        (feat * gf).sum().add((d * gd).sum()).backward()
        return {k: v for k, v in (('tex', t.grad), ('w1', heads[0][2].grad), ('cam', cm.grad)) if v is not None}

    def once(args, kernel):
        render_grad.USE_BACKWARD_KERNEL = kernel
        try:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); out = step(*args); b.record(); torch.cuda.synchronize()
            return a.elapsed_time(b), out
        finally:
            render_grad.USE_BACKWARD_KERNEL = True

    workloads = {'a_planes_heads_camera': (True, True, True, False), 'b_camera_only': (False, False, True, False),
                 'c_hierarchical_96_96_planes_heads': (True, True, False, True)}
    result = {'gpu': torch.cuda.get_device_name(), 'power_limit': power_limit(),
              'config': f'renderer forward + backward, {n} frames {RENDER}^2 x {NUM_STEPS}, {img_v.shape[-1]}^2 planes', 'reps': reps}
    for name, args in workloads.items():
        once(args, True); once(args, False)                                   # warm-up of both paths
        tk, tc = [], []
        for _ in range(reps):
            ms, gk = once(args, True); tk.append(ms)
            ms, gc = once(args, False); tc.append(ms)
        mk, mc = float(np.median(tk)), float(np.median(tc))
        result[name] = {'kernel_path_ms': mk, 'composed_chain_path_ms': mc, 'speedup': mc / mk,
                        'max_abs_grad_diff': {k: float((gk[k] - gc[k]).abs().max()) for k in gk},
                        'grad_scale': {k: float(gc[k].abs().max()) for k in gk}}
    print(json.dumps(result))


if __name__ == '__main__':
    main()
