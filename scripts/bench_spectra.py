"""Time avg_spectra's paths and print one JSON line (also written to --out when given).

    python scripts/bench_spectra.py [--runs 3] [--images 256] [--zip-images 256] [--gen-images 64] [--out FILE]

accum   Accumulating --images uint8 images of 512^2 x 3 at interp 4 (P = 2048): ide3d_spectrum_accum in calls of 16 images against the
        reference's per-image torch structure on the same GPU (float64 whitening and window, zero pad to 2048^2, fftn, |X|^2, channel
        mean; avg_spectra.py:163-166).  The two arms alternate, --runs times each.  Also reports the two results' difference.
zip     `calc`'s whole stream from a zip of --zip-images 512^2 PNGs (DataLoader with 3 workers, batches of 32, pinned non-blocking copies,
        then the kernel) against the reference's batch-1 loader: images / s.  Host PNG decoding is expected to bound both.
gen     Generator-source images / s (oracle.spectra.StandInSpectrumGenerator, 512^2, on the device), batches of 32 against the batch-1
        loop, rendering and the spectrum included.
Algorithmic FLOPs of the kernel arm count 5 N log2 N per complex length-N FFT (radix-2: N/2 log2 N butterflies of 10 flops).
"""

import argparse
import json
import math
import os
import subprocess
import sys
import tempfile
import time
import zipfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in q.stdout.strip().splitlines()[0].split(',')]
        return {'gpu': name, 'power_limit': power}
    except Exception as e:                                     # report, do not guess
        return {'gpu': torch.cuda.get_device_name(), 'power_limit': f'not read ({type(e).__name__})'}


def event_time(fn):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3, out


def wall_time(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, out


def reference_spectrum(images, N, interp, mean, std, beta, dev):
    """avg_spectra.py:153-167 on the device, one image at a time."""
    P = N * interp
    window = torch.kaiser_window(N, periodic=False, beta=beta, device=dev)
    window *= window.square().sum().rsqrt()
    window = window.ger(window).unsqueeze(0).unsqueeze(1)
    spectrum = torch.zeros([P, P], dtype=torch.float64, device=dev)
    for image in images.split(1):
        image = (image.to(torch.float64) - mean) / std
        image = torch.nn.functional.pad(image * window, [0, P - N, 0, P - N])
        spectrum += torch.fft.fftn(image, dim=[2, 3]).abs().square().mean(dim=[0, 1])
    return spectrum / images.shape[0]


def kernel_spectrum(images, N, interp, mean, std, beta, dev, per_call=16):
    from ide3d_b200.torch_utils.ops import spectra as ops
    acc = ops.Spectrum(N, images.shape[1], mean, std, beta=beta, interp=interp, device=dev)
    for i in range(0, images.shape[0], per_call):
        acc.add(images[i:i + per_call])
    return acc.result()


def kernel_flops_bytes(B, C, N, interp):
    P, H = N * interp, N * interp // 2 + 1
    fft = 5 * N * math.log2(N)
    flops = B * C * (N * interp + H * interp) * fft                                   # row FFTs + column FFTs
    nbytes = B * C * (N * N + 2 * H * N * 16) + 2 * H * P * 8                          # images, Y written and read, accumulator
    return flops, nbytes


def bench_accum(args, dev, out):
    N, interp, mean, std, beta = 512, 4, 112.684, 69.509, 8.0
    g = torch.Generator(device=dev).manual_seed(0)
    images = torch.randint(0, 256, (args.images, 3, N, N), dtype=torch.uint8, device=dev, generator=g)
    kernel_spectrum(images[:16], N, interp, mean, std, beta, dev)
    reference_spectrum(images[:2], N, interp, mean, std, beta, dev)
    tk, tr = [], []
    for _ in range(args.runs):                                                              # alternate the arms
        t, k = event_time(lambda: kernel_spectrum(images, N, interp, mean, std, beta, dev))
        tk.append(t)
        t, r = event_time(lambda: reference_spectrum(images, N, interp, mean, std, beta, dev))
        tr.append(t)
    flops, nbytes = kernel_flops_bytes(args.images, 3, N, interp)
    out['accum'] = dict(images=args.images, size=N, interp=interp, runs=args.runs,
                        kernel_s=[round(t, 5) for t in tk], reference_s=[round(t, 5) for t in tr],
                        kernel_us_per_image=round(min(tk) / args.images * 1e6, 2), reference_us_per_image=round(min(tr) / args.images * 1e6, 2),
                        speedup=round(min(tr) / min(tk), 2), kernel_gflop=round(flops / 1e9, 2), kernel_gb=round(nbytes / 1e9, 3),
                        kernel_tflops=round(flops / min(tk) / 1e12, 3),
                        rel_diff=float(((k - r).abs().max() / r.abs().max()).item()))


def write_zip(path, n, res=512):
    import PIL.Image
    rs = np.random.RandomState(0)
    with zipfile.ZipFile(path, 'w') as z:
        for i in range(n):
            base = rs.randint(0, 256, size=(8, 8, 3)).astype(np.uint8)
            img = PIL.Image.fromarray(base).resize((res, res), PIL.Image.BILINEAR)
            name = os.path.join(tempfile.gettempdir(), f'bench_spectra_{i}.png')
            img.save(name)
            z.write(name, f'{i // 1000:05d}/img{i:08d}.png')
            os.remove(name)


def bench_zip(args, dev, out):
    from ide3d_b200 import avg_spectra
    tmp = tempfile.mkdtemp()
    zpath = os.path.join(tmp, 'ds.zip')
    write_zip(zpath, args.zip_images)

    def run(batch):
        n, size, it = avg_spectra.stream_source_images(zpath, None, 0, dev, batch=batch)
        return avg_spectra.compute_spectrum(it, size, 112.684, 69.509, 8.0, 4, dev)

    run(32)
    tb, t1 = [], []
    for _ in range(args.runs):
        tb.append(wall_time(lambda: run(32))[0])
        t1.append(wall_time(lambda: run(1))[0])
    out['zip'] = dict(images=args.zip_images, size=512, interp=4, runs=args.runs, batch32_images_per_s=round(args.zip_images / min(tb), 1),
                      batch1_images_per_s=round(args.zip_images / min(t1), 1), batch32_s=[round(t, 3) for t in tb],
                      batch1_s=[round(t, 3) for t in t1], host_cpus=os.cpu_count())


def bench_gen(args, dev, out):
    from ide3d_b200 import avg_spectra
    from oracle import spectra as osp
    G = osp.StandInSpectrumGenerator().to(dev).eval()

    def run(batch):
        n, size, it = avg_spectra.stream_source_images(G, args.gen_images, 0, dev, batch=batch)
        return avg_spectra.compute_spectrum(it, size, 112.684, 69.509, 8.0, 4, dev)

    run(32)
    tb, t1 = [], []
    for _ in range(args.runs):
        t, a = wall_time(lambda: run(32))
        tb.append(t)
        t, b = wall_time(lambda: run(1))
        t1.append(t)
    out['gen'] = dict(images=args.gen_images, size=512, interp=4, runs=args.runs, batch32_images_per_s=round(args.gen_images / min(tb), 1),
                      batch1_images_per_s=round(args.gen_images / min(t1), 1), rel_diff=float(((a - b).abs().max() / b.abs().max()).item()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--images', type=int, default=256)
    ap.add_argument('--zip-images', type=int, default=256)
    ap.add_argument('--gen-images', type=int, default=64)
    ap.add_argument('--skip', default='')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_spectra needs a CUDA device'
    dev = torch.device('cuda')
    out = card()
    skip = set(args.skip.split(','))
    for name, fn in (('accum', bench_accum), ('zip', bench_zip), ('gen', bench_gen)):
        if name not in skip:
            fn(args, dev, out)
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
