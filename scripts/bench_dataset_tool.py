"""Measure dataset_tool: (a) ide3d_resample_u8 against PIL.Image.resize(LANCZOS) on one host core, (b) images/s end to end.

    python scripts/bench_dataset_tool.py [--images N] [--workers W ...] [--out DIR]

(a) kernel time per 1024^2 -> 512^2 RGB image at batch 8 (CUDA events over 50 warmed calls), and the bytes it moves (the input read,
    the uint8 intermediate written and read, the output written), against PIL's resize of the same images on one host core.
(b) N seeded 1024^2 RGB PNGs converted to a 512^2 zip with `--resolution 512x512`, at each worker count W, with and without --seg-dest
    (seeded BiSeNet weights), against a single-process loop that decodes with PIL, resizes with PIL and stores an uncompressed PNG into a
    ZIP_STORED archive: the reference's per-image loop, restated here.
GPU name, power limit and host CPU count are printed beside the numbers.  Prints one JSON line; with --out it is also written there.
"""

import argparse
import io
import json
import os
import subprocess
import sys
import tempfile
import time
import zipfile

import numpy as np
import PIL.Image
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from ide3d_b200 import dataset_tool, parsing  # noqa: E402
from ide3d_b200.torch_utils.ops import resample  # noqa: E402


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def seeded_image(rng, size=1024):
    yy, xx = np.mgrid[0:size, 0:size].astype(np.float32)
    base = np.stack([np.sin(xx / rng.uniform(5, 40) + rng.uniform(0, 6)) + np.cos(yy / rng.uniform(5, 40)) for _ in range(3)], -1)
    return np.clip(base * 60 + 128 + rng.normal(0, 10, size=base.shape), 0, 255).astype(np.uint8)


def bench_kernel(imgs):
    x = torch.from_numpy(np.stack(imgs)).cuda()
    out = torch.empty([len(imgs), 512, 512, 3], dtype=torch.uint8, device='cuda')
    for _ in range(5):
        resample.resample_u8(x, out)
    torch.cuda.synchronize()
    calls = 50
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(calls):
        resample.resample_u8(x, out)
    t1.record()
    torch.cuda.synchronize()
    per_image_us = t0.elapsed_time(t1) * 1e3 / calls / len(imgs)
    bytes_per_image = 1024 * 1024 * 3 + 2 * 1024 * 512 * 3 + 512 * 512 * 3
    pil_t = []
    for im in imgs:
        p = PIL.Image.fromarray(im)
        s = time.perf_counter()
        want = np.array(p.resize((512, 512), PIL.Image.LANCZOS))
        pil_t.append(time.perf_counter() - s)
    equal = all(np.array_equal(out[i].cpu().numpy(), np.array(PIL.Image.fromarray(im).resize((512, 512), PIL.Image.LANCZOS)))
                for i, im in enumerate(imgs))
    del want
    return dict(kernel_us_per_image=per_image_us, bytes_per_image=bytes_per_image,
                kernel_gbps=bytes_per_image / (per_image_us * 1e-6) / 1e9, pil_ms_per_image=1e3 * float(np.median(pil_t)),
                bit_identical=equal)


def reference_loop(src, dest):
    """decode, PIL resize, store uncompressed PNG: the reference's loop for this source, in one process."""
    files = sorted(os.listdir(src))
    with zipfile.ZipFile(dest, 'w', compression=zipfile.ZIP_STORED) as zf:
        for idx, f in enumerate(files):
            img = np.array(PIL.Image.open(os.path.join(src, f)))
            img = np.array(PIL.Image.fromarray(img).resize((512, 512), PIL.Image.LANCZOS))
            b = io.BytesIO()
            PIL.Image.fromarray(img, 'RGB').save(b, format='png', compress_level=0, optimize=False)
            s = f'{idx:08d}'
            zf.writestr(f'{s[:5]}/img{s}.png', b.getbuffer())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=96)
    ap.add_argument('--workers', type=int, nargs='+', default=None)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    cpus = os.cpu_count()
    workers = a.workers or sorted({1, min(8, cpus), cpus})
    rng = np.random.default_rng(0)
    res = dict(gpu=gpu_info(), host_cpus=cpus)
    res['kernel'] = bench_kernel([seeded_image(rng) for _ in range(8)])
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, 'src')
        os.makedirs(src)
        for i in range(a.images):
            PIL.Image.fromarray(seeded_image(rng)).save(os.path.join(src, f'{i:05d}.png'))
        net = parsing.BiSeNet()
        torch.manual_seed(0)
        torch.save(net.state_dict(), os.path.join(tmp, 'bisenet.pth'))
        s = time.perf_counter()
        reference_loop(src, os.path.join(tmp, 'ref.zip'))
        res['pil_loop_images_per_s'] = a.images / (time.perf_counter() - s)
        dataset_tool.convert(src, os.path.join(tmp, 'warm.zip'), resolution=(512, 512), workers=1, max_images=8)     # CUDA set-up
        runs = []
        for w in workers:
            for seg in (False, True):
                dest = os.path.join(tmp, f'o{w}{int(seg)}.zip')
                kw = dict(seg_dest=os.path.join(tmp, f's{w}.zip'), parser=os.path.join(tmp, 'bisenet.pth')) if seg else {}
                torch.cuda.synchronize()
                s = time.perf_counter()
                dataset_tool.convert(src, dest, resolution=(512, 512), workers=w, **kw)
                runs.append(dict(workers=w, seg=seg, images_per_s=a.images / (time.perf_counter() - s)))
                with zipfile.ZipFile(dest) as z1, zipfile.ZipFile(os.path.join(tmp, 'ref.zip')) as z0:
                    runs[-1]['equal_to_pil_loop'] = all(z1.read(n) == z0.read(n) for n in z0.namelist())
        res['end_to_end'] = runs
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'bench_dataset_tool.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
