#!/usr/bin/env python
"""Tail micro-benchmark of the video frame composition (gen_videos.py:129-139 + layout_grid's uint8 conversion): the fused
ide3d_video_frames kernel against the reference's torch composition (oracle.frames on the device: interpolate to 512^2, mask2color,
the float passes, cat, uint8) for one 8-frame batch, 64^2 logits -> 512^2 frames.  CUDA events, median of --reps.  Prints one JSON line
per case with the card name and power limit.

    python scripts/bench_frames.py [--reps 50]

Achieved bytes/s use the bytes the fused pass needs, computed from the shapes: image_seg reads the image (3.1 MB per frame) and the
64^2 logits (0.3 MB) and writes the uint8 cell (1.6 MB); image_depth reads the image twice (min/max pass, then the map) and writes 0.8 MB.
"""
import argparse, json, os, subprocess, sys
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True, text=True)
    return r.stdout.strip() or 'unknown'


def timeit(fn, reps, warm=5):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--frames', type=int, default=8)
    args = ap.parse_args()
    from ide3d_b200 import video
    from ide3d_b200.training import networks
    from oracle import frames as ofr
    assert torch.cuda.is_available(), 'bench_frames needs a CUDA device'
    dev = torch.device('cuda')
    n, H, R, C = args.frames, 512, 64, 19
    g = torch.Generator(device=dev).manual_seed(0)
    img = torch.randn(n, 3, H, H, device=dev, generator=g)
    if networks.CHANNELS_LAST:                                    # the layout the super-resolution blocks hand out
        img = img.contiguous(memory_format=torch.channels_last)
    feat = torch.randn(n, R * R, 51, device=dev, generator=g)    # ray-march output; the logits are its strided channel view
    seg = feat.permute(0, 2, 1).reshape(n, 51, R, R)[:, 32:]
    img_b, seg_b = n * 3 * H * H * 4, n * C * R * R * 4
    cases = {
        'image_seg': (img_b + seg_b + n * 3 * H * 2 * H, lambda: video.compose_frames(img, seg, 'image_seg'),
                      lambda: ofr.compose_frames(img, seg, 'image_seg')),
        'image_depth': (2 * img_b + n * 3 * H * H, lambda: video.compose_frames(img, None, 'image_depth'),
                        lambda: ofr.compose_frames(img, None, 'image_depth')),
    }
    gpu = card()
    for mode, (nbytes, fused, composed) in cases.items():
        t_f = timeit(fused, args.reps)
        t_c = timeit(composed, args.reps)
        same = bool(torch.equal(fused()[..., :H], composed()[..., :H]))
        print(json.dumps({'op': f'video frames {mode}', 'frames': n, 'logits': f'{C}x{R}^2 strided view' if mode == 'image_seg' else None,
                          'image': f'3x{H}^2 {"channels_last" if networks.CHANNELS_LAST else "NCHW"}', 'fused_ms': t_f, 'torch_composition_ms': t_c,
                          'speedup': t_c / t_f, 'fused_bytes': nbytes, 'fused_GBps': nbytes / t_f / 1e6, 'image_part_equal': same,
                          'gpu (name, power limit)': gpu}))


if __name__ == '__main__':
    main()
