"""Visualizer frames: ide3d_b200.viz.renderer.Renderer against the reference's structure run through this package.

    python scripts/bench_viz.py [--rounds 3] [--frames 20]

Generator: compat.random_init_generator (the bench generator, 512^2).  Per-call latency of Renderer.render (its render_time, CUDA events
around the call, plus the host copy of the image) at 512^2, seeds [[0, 1]], noise 'const'.  Cases:
  cold      a new latent every frame (random_seed and the w0 seed change), no backbone caching
  drag      one latent, the yaw changes every frame, do_backbone_caching=True (the first frame of the run is not timed)
  depth     render_type 'image_depth', camera drag with caching
  layer     capture of synthesis.vb64.conv1 (a 64^2 x 512 layer) with the FFT view, yaw changing
Arms, alternated per round: `pkg` = Renderer as shipped; `ref` = the reference's structure through this package: the backbone every
call and the display tail in torch (torch.fft.fftn, embedding for the colormap).  Medians over the frames of every round.  Also timed:
the display tail alone (CUDA events over 50 calls) and its launch count, ours against the torch tail, for a 512^2 RGB image and for the
64^2 x 512 layer with the FFT view.  Prints one JSON line per case and per tail measurement."""

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                           # noqa: BLE001 -- the card's name is informational
        return f'unknown ({e})'


def torch_display(out, render_type='image', sel_channels=3, base_channel=0, img_normalize=False, img_scale_db=0, fft_show=False,
                  fft_all=True, fft_range_db=50, fft_beta=8, cmap=None):
    """viz/renderer.py:362-406 in torch on the device (the reference arm's tail)."""
    out = out.to(torch.float32).clone()
    if sel_channels > out.shape[0]:
        sel_channels = 1
    base_channel = max(min(base_channel, out.shape[0] - sel_channels), 0)
    sel = out[base_channel:base_channel + sel_channels]
    stats = torch.stack([out.mean(), sel.mean(), out.std(), sel.std(), out.norm(float('inf')), sel.norm(float('inf'))])
    if render_type == 'image_depth':
        out -= out.min()
        out /= out.max()
        out -= .5
        out *= -2
    img = sel
    if img_normalize:
        img = img / img.norm(float('inf'), dim=[1, 2], keepdim=True).clip(1e-8, 1e8)
    img = img * (10 ** (img_scale_db / 20))
    img = (img * 127.5 + 128).clamp(0, 255).to(torch.uint8).permute(1, 2, 0)
    if fft_show:
        sig = out if fft_all else sel
        sig = sig - sig.mean(dim=[1, 2], keepdim=True)
        sig = sig * torch.kaiser_window(sig.shape[1], periodic=False, beta=fft_beta, device=out.device)[None, :, None]
        sig = sig * torch.kaiser_window(sig.shape[2], periodic=False, beta=fft_beta, device=out.device)[None, None, :]
        fft = torch.fft.fftn(sig, dim=[1, 2]).abs().square().sum(dim=0)
        fft = fft.roll(shifts=[fft.shape[0] // 2, fft.shape[1] // 2], dims=[0, 1])
        fft = (fft / fft.mean()).log10() * 10
        hi = cmap.shape[0] - 1
        x = ((fft / fft_range_db + 1) / 2 * hi + 0.5).clamp(0, hi).to(torch.int64)
        img = torch.cat([img.expand(-1, -1, 3), torch.nn.functional.embedding(x, cmap)], dim=1)
    return img, stats


CASES = {
    'cold': dict(),
    'drag': dict(do_backbone_caching=True),
    'depth': dict(do_backbone_caching=True, render_type='image_depth'),
    'layer': dict(layer_name='synthesis.vb64.conv1', fft_show=True, sel_channels=3, img_normalize=True),
}


def frames(r, G, case, n):
    """Per-frame seconds of n frames of a case (one untimed frame first)."""
    kw = CASES[case]
    times = []
    for i in range(n + 1):
        args = dict(pkl=G, yaw=0.4 * np.sin(i / 3), **kw)
        if case == 'cold':
            args.update(w0_seeds=[[i, 1]], random_seed=i)
        res = r.render(**args)
        assert 'error' not in res, res.error
        if i:
            times.append(res.render_time)
    return times


def time_tail(fn, reps=50):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps * 1e-3


def torch_kernel_count(fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type.name == 'CUDA')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--frames', type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_viz needs a CUDA device'
    from ide3d_b200 import _lib as L
    from ide3d_b200.compat import random_init_generator
    from ide3d_b200.torch_utils.ops import viz as viz_ops
    from ide3d_b200.viz import renderer as R
    info = gpu_info()
    G = random_init_generator(device='cuda', seed=0)
    k = torch.arange(1024)
    lut = torch.stack([k // 4, k // 8, 255 - k // 4], 1).to(torch.uint8).cuda()

    class Reference(R.Renderer):
        """The reference's structure: no backbone cache, the torch tail."""
        def _render_impl(self, res, **kw):
            kw['do_backbone_caching'] = False
            saved = viz_ops.display
            R.viz_ops.display = torch_display
            try:
                super()._render_impl(res, **kw)
            finally:
                R.viz_ops.display = saved

    arms = {'pkg': R.Renderer(cmap=lut), 'ref': Reference(cmap=lut)}
    for r in arms.values():                          # warm every case and shape
        for case in CASES:
            frames(r, G, case, 2)
    results = {case: {arm: [] for arm in arms} for case in CASES}
    for _ in range(args.rounds):
        for case in CASES:
            for arm, r in arms.items():
                results[case][arm] += frames(r, G, case, args.frames)
    for case in CASES:
        pkg, ref = (float(np.median(results[case][a])) for a in ('pkg', 'ref'))
        print(json.dumps(dict(case=case, gpu=info, pkg_ms=round(pkg * 1e3, 3), ref_ms=round(ref * 1e3, 3), speedup=round(ref / pkg, 2),
                              frames=len(results[case]['pkg']), rounds=args.rounds)))

    g = torch.Generator().manual_seed(0)
    maps = {'rgb512': (torch.randn(3, 512, 512, generator=g).cuda(), {}),
            'layer64x512_fft': (torch.randn(512, 64, 64, generator=g).cuda(), dict(fft_show=True, cmap=lut))}
    for name, (x, kw) in maps.items():
        ours = lambda: viz_ops.display(x, **kw)
        theirs = lambda: torch_display(x, **kw)
        n0 = L.launch_count()
        ours()
        launches = L.launch_count() - n0
        t_ours, t_torch = time_tail(ours), time_tail(theirs)
        print(json.dumps(dict(tail=name, gpu=info, ours_us=round(t_ours * 1e6, 1), torch_us=round(t_torch * 1e6, 1),
                              ours_launches=launches, torch_kernels=torch_kernel_count(theirs))))


if __name__ == '__main__':
    main()
