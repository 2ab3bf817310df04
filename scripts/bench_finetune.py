#!/usr/bin/env python
"""Benchmark of encoder fine-tuning (ide3d_b200.finetune) on the bench generator (random-init ide3d-ffhq-64-512) with a random-init
HybridEncoder(512, num_ws - 8, 8) and a seeded BiSeNet(20).  Prints one JSON line per case, with the card name and power limit read in
the same run.  Every case alternates its arms over --rounds rounds after a warm-up of every arm; the median is reported.

  (a) step      one fine-tuning step (forward, backward, Adam) to a sync: finetune.run's step vs the reference's per-step structure
                through this package (oracle.finetune.reference_step: BiSeNet twice on the render and once on the image, full E twice,
                the composition stem under grad, torch upsample + cross-entropy + argmax)
  (b) stem      the stem, conv1 and skip forward + backward at 512^2, C0 = 32, N = 1 and 8: ide3d_seg_stem + ide3d_seg_stem_bwd vs the
                device one-hot composition; CUDA events over --reps calls.  For the backward kernels alone, GB/s over the bytes they
                must move (mask, grad_y1, grad_skip: N*H*W*(1 + 4*C0) + N*(H/2)*(W/2)*4*C1) against the 3.35 TB/s of the H100 SXM
                data sheet
  (c) tail      the cross-entropy and parse of BiSeNet's 64^2 logits at 512^2, forward + backward: the _ac kernels vs torch's
                align_corners=True upsample, cross_entropy and argmax

    python scripts/bench_finetune.py [--rounds 3] [--reps 20]
"""
import argparse, copy, json, os, subprocess, sys, time
import numpy as np
import torch
import torch.nn.functional as F
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


def event_ms(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def alternate(arms, rounds, reps, timer=wall_ms):
    for fn in arms.values():
        timer(fn, 2)
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            res[k].append(timer(fn, reps))
    return {k: float(np.median(v)) for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--reps', type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_finetune needs a CUDA device'
    from ide3d_b200 import _lib, edit
    from ide3d_b200.compat import random_init_generator
    from ide3d_b200.encoder import HybridEncoder, one_hot_input
    from ide3d_b200.parsing import BiSeNet, remap_ids
    from ide3d_b200.torch_utils.ops import projection, seg_stem
    from oracle import finetune as of
    dev = torch.device('cuda')
    name = card()

    G = random_init_generator(device=dev, seed=0)
    G.rendering_kwargs['perturb'] = None
    G = copy.deepcopy(G).eval().requires_grad_(False)
    torch.manual_seed(1)
    E = HybridEncoder(512, G.num_ws - 8, 8, w_dim=G.w_dim)
    for p in E.parameters():
        if p.ndim == 1:
            p.data.normal_(0, 0.2)
    E = E.to(dev)
    net = BiSeNet(20)
    net.load_state_dict(of.bisenet_state(net))
    net = net.eval().requires_grad_(False).to(dev)
    label = torch.tensor(edit.FRONTAL, device=dev).reshape(1, -1)
    z = torch.from_numpy(np.random.RandomState(0).randn(1, G.z_dim)).float().to(dev)
    with torch.no_grad():
        code = G.mapping(z, label)
        image = G.synthesis(code, label, noise_mode='const').clamp(-1, 1)
        target_labels = seg_stem.seg_labels(net.logits(image), (512, 512), align_corners=True)
        target_seg = remap_ids(target_labels)
        app = E.appearance(image)
    w_avg = G.mapping.w_avg[None, None, :]
    params = list(E.convs_seg.parameters()) + list(E.projector_seg.parameters())
    for p in E.parameters():
        p.requires_grad_(False)
    for p in params:
        p.requires_grad_(True)
    opt = torch.optim.Adam(params, lr=1e-5, betas=(0.9, 0.99))

    def product_step():                                   # the body of finetune.run's loop
        opt.zero_grad()
        geo = E.geometry(target_seg) + w_avg
        rec = torch.cat((geo, code[:, 8:]), 1)
        img = G.synthesis(rec, c=label, noise_mode='const')
        logits = net.logits(img)
        with torch.no_grad():
            cyc = remap_ids(seg_stem.seg_labels(logits, (512, 512), align_corners=True))
        cycle = torch.cat((E.geometry(cyc, signed=False), app), 1)
        loss = (F.smooth_l1_loss(rec, code) * 10 + F.mse_loss(img, image)
                + projection.seg_cross_entropy(logits, target_labels, align_corners=True) + F.smooth_l1_loss(rec, cycle))
        loss.backward()
        opt.step()

    seg_float = one_hot_input(target_seg, 19)
    E_ref = copy.deepcopy(E)
    params_ref = list(E_ref.convs_seg.parameters()) + list(E_ref.projector_seg.parameters())
    for p in E_ref.parameters():
        p.requires_grad_(True)                           # requires_grad(E, True): the reference back-propagates into the image branch
    opt_ref = torch.optim.Adam(params_ref, lr=1e-5, betas=(0.9, 0.99))

    def reference_step():
        opt_ref.zero_grad()
        sum(of.reference_step(G, E_ref, image, seg_float, code, label, net, w_avg).values()).backward()
        opt_ref.step()

    t = alternate({'reference': reference_step, 'finetune': product_step}, args.rounds, 3)
    print(json.dumps({'case': 'step', 'card': name, 'reference_ms': round(t['reference'], 2), 'finetune_ms': round(t['finetune'], 2),
                      'speedup': round(t['reference'] / t['finetune'], 2)}), flush=True)

    # (b) stem forward + backward
    stem, block = E.convs_seg[0], E.convs_seg[1]
    for n in (1, 8):
        g = torch.Generator(device=dev).manual_seed(n)
        mask = torch.randint(0, 19, (n, 32, 32), device=dev, dtype=torch.uint8, generator=g)
        mask = mask.repeat_interleave(16, 1).repeat_interleave(16, 2).contiguous()
        gy = torch.randn(n, 32, 512, 512, device=dev, generator=g).contiguous(memory_format=torch.channels_last)
        gs = torch.randn(n, 64, 256, 256, device=dev, generator=g).contiguous(memory_format=torch.channels_last)
        ps = [stem.weight, stem.bias, block.conv1.weight, block.conv1.bias, block.skip.weight]

        def kernel():
            y1, sk = seg_stem.seg_stem(mask, stem, block.conv1, block.skip)
            torch.autograd.grad((y1, sk), ps, (gy, gs))

        def composition():
            x = stem(one_hot_input(mask, 19).contiguous(memory_format=torch.channels_last))
            torch.autograd.grad((block.conv1(x), block.skip(x)), ps, (gy, gs))

        t = alternate({'composition': composition, 'kernel': kernel}, args.rounds, args.reps, event_ms)
        y1, sk = seg_stem.seg_stem(mask, stem, block.conv1, block.skip)
        bwd_only = event_ms(lambda: torch.autograd.grad((y1, sk), ps, (gy, gs), retain_graph=True), args.reps)
        n0 = _lib.launch_count()
        torch.autograd.grad((y1, sk), ps, (gy, gs), retain_graph=True)
        launches = _lib.launch_count() - n0
        nbytes = n * 512 * 512 * (1 + 4 * 32) + n * 256 * 256 * 4 * 64
        print(json.dumps({'case': 'stem', 'card': name, 'n': n, 'composition_ms': round(t['composition'], 3),
                          'kernel_ms': round(t['kernel'], 3), 'speedup': round(t['composition'] / t['kernel'], 2),
                          'bwd_ms': round(bwd_only, 3), 'bwd_launches': launches, 'bwd_MB': round(nbytes / 1e6, 1),
                          'bwd_TBps': round(nbytes / bwd_only / 1e9, 3), 'share_of_3.35TBps': round(nbytes / bwd_only / 1e9 / 3.35, 3)}),
              flush=True)
        del gy, gs, y1, sk

    # (c) the cross-entropy + parse tail of BiSeNet's logits
    logits = torch.randn(1, 20, 64, 64, device=dev, generator=torch.Generator(device=dev).manual_seed(3)).requires_grad_(True)

    def tail_kernels():
        loss = projection.seg_cross_entropy(logits, target_labels, align_corners=True)
        torch.autograd.grad(loss, logits)
        seg_stem.seg_labels(logits.detach(), (512, 512), align_corners=True)

    def tail_torch():
        up = F.interpolate(logits, (512, 512), mode='bilinear', align_corners=True)
        loss = F.cross_entropy(up, target_labels.long())
        torch.autograd.grad(loss, logits)
        F.interpolate(logits.detach(), (512, 512), mode='bilinear', align_corners=True).argmax(1)

    t = alternate({'torch': tail_torch, 'kernels': tail_kernels}, args.rounds, args.reps, event_ms)
    print(json.dumps({'case': 'tail', 'card': name, 'torch_ms': round(t['torch'], 3), 'kernels_ms': round(t['kernels'], 3),
                      'speedup': round(t['torch'] / t['kernels'], 2)}), flush=True)


if __name__ == '__main__':
    main()
