#!/usr/bin/env python
"""Benchmark of hybrid-encoder training (ide3d_b200.train_encoder) on the bench generator (random-init ide3d-ffhq-64-512) with a random
HybridEncoder(512, num_ws - 8, 8), a seeded BiSeNet(20), torchvision's VGG19 and AlexNet with random weights and a seeded IR-SE50.
Prints one JSON line per case, with the card name and power limit read in the same run; every case alternates its arms over --rounds
rounds after a warm-up of every arm, and reports the median.

  (a) step   one training step at batch 8 (forward, backward, Adam) to a sync, synthetic only and synthetic + real (every lambda
             non-zero): train_encoder.step_losses vs the script's per-step structure through this package
             (oracle.train_encoder.reference_step), with the peak memory of each
  (b) head   the VGG L1 head forward + backward over the five VGG19 taps of a batch of 8 at 512^2 (31.98 M elements per image):
             ide3d_feat_l1_fwd + _bwd vs torch's five F.l1_loss calls; CUDA events over --reps calls, and GB/s over the counted bytes
             (kernel 20 B per element: x and y read forward, x and y read and grad_x written backward) against the 3.35 TB/s of the
             H100 SXM data sheet

    python scripts/bench_train_encoder.py [--rounds 3] [--reps 10]
"""
import argparse, copy, json, os, subprocess, sys, tempfile, time
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LAMBDAS = dict(vgg=1.0, l2=1.0, lpips=0.8, id=0.1, entropy=0.1, cycle=1.0)
TAPS = ((64, 512, 512), (128, 256, 256), (256, 128, 128), (512, 64, 64), (512, 32, 32))


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
    peak = {}
    for k, fn in arms.items():
        torch.cuda.reset_peak_memory_stats()
        timer(fn, 2)
        peak[k] = torch.cuda.max_memory_allocated() / 2 ** 30
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            res[k].append(timer(fn, reps))
    return {k: float(np.median(v)) for k, v in res.items()}, peak


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--batch', type=int, default=8)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_train_encoder needs a CUDA device'
    import torchvision
    from ide3d_b200.arcface import Backbone, IDLoss
    from ide3d_b200.compat import random_init_generator
    from ide3d_b200.encoder import HybridEncoder
    from ide3d_b200.parsing import BiSeNet
    from ide3d_b200.torch_utils.ops.lpips import LPIPS
    from ide3d_b200.torch_utils.ops.vgg_loss import VGGLoss, feat_l1
    from ide3d_b200.train_encoder import PortraitDataset, _Encode, cam_sampler, step_losses
    from oracle import finetune as of, pti as opti, train_encoder as ot
    dev = torch.device('cuda')
    name = card()
    B = args.batch

    # (b) the head first: its buffers are freed before the steps
    g = torch.Generator(device=dev).manual_seed(0)
    fx = [torch.relu(torch.randn(B, c, h, w, device=dev, generator=g)).requires_grad_(True) for c, h, w in TAPS]
    fy = [torch.relu(torch.randn(B, c, h, w, device=dev, generator=g)) for c, h, w in TAPS]
    elems = sum(B * c * h * w for c, h, w in TAPS)

    def head_kernel():
        total, _ = feat_l1(fx, fy, (1.0,) * 5)
        torch.autograd.grad(total, fx)

    def head_torch():
        total = sum(torch.nn.functional.l1_loss(x, y) for x, y in zip(fx, fy))
        torch.autograd.grad(total, fx)

    t, _ = alternate({'kernel': head_kernel, 'torch': head_torch}, args.rounds, args.reps, event_ms)
    gb = 20 * elems / 1e9
    print(json.dumps({'case': 'head', 'card': name, 'batch': B, 'elements_M': round(elems / 1e6, 2), 'counted_GB': round(gb, 2),
                      'kernel_ms': round(t['kernel'], 3), 'torch_ms': round(t['torch'], 3),
                      'kernel_GBps': round(gb / t['kernel'] * 1e3, 1), 'share_of_3.35TBps': round(gb / t['kernel'] * 1e3 / 3350, 3)}))
    del fx, fy
    torch.cuda.empty_cache()

    # (a) one step
    G = random_init_generator(device=dev, seed=0)
    G.rendering_kwargs['perturb'] = None
    G = copy.deepcopy(G).eval().requires_grad_(False)
    torch.manual_seed(1)
    E = HybridEncoder(512, G.num_ws - 8, 8, w_dim=G.w_dim).to(dev).requires_grad_(True)
    net = BiSeNet(20)
    net.load_state_dict(of.bisenet_state(net))
    net = net.eval().requires_grad_(False).to(dev)
    torch.manual_seed(2)
    vgg = VGGLoss(torchvision.models.vgg19(weights=None).features).to(dev)
    lpips = LPIPS(opti.standin_alexnet().features, opti.standin_lin()).to(dev)
    irse = Backbone(112, 50, mode='ir_se', drop_ratio=0.6)
    irse.load_state_dict(ot.irse50_state(irse))
    id_net = IDLoss(irse).to(dev)
    mods = dict(vgg=vgg, lpips=lpips, id_net=id_net)
    w_avg = G.mapping.w_avg[None, None, :]
    opt = torch.optim.Adam(E.parameters(), lr=1e-4, betas=(0.9, 0.99))
    z = torch.from_numpy(np.random.RandomState(0).randn(B, G.w_dim)).float().to(dev)
    cam = cam_sampler(B, dev, torch.Generator(dev).manual_seed(0))
    with tempfile.TemporaryDirectory() as d:
        img_dir, seg_dir, _ = ot.write_portraits(d, n=B)
        ds = PortraitDataset(img_dir, seg_dir, 512)
        real = tuple(torch.stack([ds[i][k] for i in range(B)]).to(dev) for k in range(3))
    for tag, r in (('gen', None), ('gen+real', real)):
        def product():
            opt.zero_grad()
            loss = step_losses(G, _Encode(E), parser=net, lambdas=LAMBDAS, z=z, cam=cam, real=r, start_from_latent_avg=True, **mods)
            sum(loss.values()).backward()
            opt.step()

        def reference():
            opt.zero_grad()
            loss = ot.reference_step(G, E, net, lambdas=LAMBDAS, w_avg=w_avg, z=z, cam=cam, real=r, start_from_latent_avg=True,
                                     **(mods if r is not None else {}))
            sum(loss.values()).backward()
            opt.step()

        t, peak = alternate({'package': product, 'script_structure': reference}, args.rounds, 3)
        print(json.dumps({'case': 'step', 'branches': tag, 'card': name, 'batch': B, 'package_ms': round(t['package'], 1),
                          'script_structure_ms': round(t['script_structure'], 1), 'package_peak_GiB': round(peak['package'], 2),
                          'script_structure_peak_GiB': round(peak['script_structure'], 2)}))


if __name__ == '__main__':
    main()
