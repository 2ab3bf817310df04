"""Time the metric paths at FFHQ's pr50k3_full / fid50k_full shapes and print one JSON line.

    python scripts/bench_metrics.py [--runs 3] [--ref-rows 2000] [--skip kernels,stats,gen]

kernels  The precision / recall stage on 70,000 real and 50,000 generated fp16 features of D = 4096 (VGG16): kth_dist over both
         manifolds (nhood_size 3, so kth 4) and within for both directions -- against the reference's structure
         (metrics/precision_recall.py): torch.cdist in 10k-column blocks, each copied to the host, host kthvalue in fp32, host
         (dist <= kth).any(1) in fp16.  The reference arm runs --ref-rows rows of each of the four passes and is scaled to the
         full row counts (its cost is linear in rows: every row block sees all columns).
stats    FeatureStats on 50,000 x 2048 Inception features in batches of 64: float64 sums on the device against the reference's
         per-batch copy to the host and x64.T @ x64 in numpy (--ref-batches batches of it, scaled).
gen      The generator-feature loop of compute_feature_stats_for_generator with a zero-cost detector: images / s of a random-init
         ide3d-ffhq-64-512 generator, quantised to uint8 as the metrics do.  Real Inception / VGG16 time is not measured.
The card's name and power limit are read in the same run and printed with the numbers.
"""

import argparse
import json
import os
import subprocess
import sys
import time

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


def timed(fn, runs):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(runs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) / 1e3)
    return ts


def feats(n, d, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    base = torch.rand(1, d, generator=g, device=dev)
    return ((base + 0.5 * torch.rand(n, d, generator=g, device=dev)) * torch.rand(n, 1, generator=g, device=dev).add(0.5)).half()


def bench_kernels(args, dev):
    from ide3d_b200.torch_utils.ops import knn
    real, gen = feats(70000, 4096, 1, dev), feats(50000, 4096, 2, dev)

    def pr():
        kr, kg = knn.kth_dist(real, real, 4), knn.kth_dist(gen, gen, 4)
        return knn.within(gen, real, kr.half().float()).float().mean(), knn.within(real, gen, kg.half().float()).float().mean()

    ts = timed(pr, args.runs)
    parts = {}
    for name, fn in (('kth_real', lambda: knn.kth_dist(real, real, 4)), ('kth_gen', lambda: knn.kth_dist(gen, gen, 4))):
        parts[name] = min(timed(fn, args.runs))
    kr = knn.kth_dist(real, real, 4).half().float()
    kg = knn.kth_dist(gen, gen, 4).half().float()
    parts['within_precision'] = min(timed(lambda: knn.within(gen, real, kr), args.runs))
    parts['within_recall'] = min(timed(lambda: knn.within(real, gen, kg), args.runs))
    flop = 2 * 4096 * (70000 ** 2 + 50000 ** 2 + 2 * 70000 * 50000)          # upper bound: within may stop early

    # the reference's structure on --ref-rows rows of each pass (precision_recall.py:17-60, num_gpus = 1)
    def compute_distances(rows, cols, col_batch_size=10000):
        nb = (cols.shape[0] - 1) // col_batch_size + 1
        batches = torch.nn.functional.pad(cols, [0, 0, 0, -cols.shape[0] % nb]).chunk(nb)
        return torch.cat([torch.cdist(rows.unsqueeze(0), b.unsqueeze(0))[0].cpu() for b in batches], dim=1)[:, :cols.shape[0]]

    n = args.ref_rows
    ref = {}
    for name, rows, cols in (('kth_real', real, real), ('kth_gen', gen, gen)):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        kth = compute_distances(rows[:n], cols).to(torch.float32).kthvalue(4).values.to(torch.float16)
        ref[name] = (time.perf_counter() - t0) * rows.shape[0] / n
    kth_real = kr.half().cpu()
    kth_gen = kg.half().cpu()
    for name, rows, cols, kth in (('within_precision', gen, real, kth_real), ('within_recall', real, gen, kth_gen)):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        (compute_distances(rows[:n], cols) <= kth).any(dim=1)
        ref[name] = (time.perf_counter() - t0) * rows.shape[0] / n
    return {'pr_stage_s': ts, 'pr_stage_tflops_upper': flop / min(ts) / 1e12, 'parts_s': parts,
            'reference_structure_s': ref, 'reference_structure_total_s': sum(ref.values()), 'reference_rows_run': n,
            'cpu_threads': torch.get_num_threads()}


def bench_stats(args, dev):
    from ide3d_b200.metrics.metric_utils import FeatureStats
    g = torch.Generator(device=dev).manual_seed(3)
    batches = [torch.rand(64, 2048, generator=g, device=dev) for _ in range(50000 // 64)]

    def device_stats():
        s = FeatureStats(capture_mean_cov=True, max_items=50000)
        for b in batches:
            s.append_torch(b)
        return s.get_mean_cov()

    ts = timed(device_stats, args.runs)
    nb = args.ref_batches
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    mean, cov = np.zeros(2048), np.zeros((2048, 2048))
    for b in batches[:nb]:
        x64 = b.cpu().numpy().astype(np.float64)
        mean += x64.sum(0)
        cov += x64.T @ x64
    ref = (time.perf_counter() - t0) * len(batches) / nb
    return {'device_s': ts, 'numpy_per_batch_s': ref, 'numpy_batches_run': nb, 'batches': len(batches)}


def bench_gen(args, dev):
    import ide3d_b200.compat as compat
    from ide3d_b200.metrics import metric_utils
    G = compat.random_init_generator(device=dev)

    class Zero(torch.nn.Module):
        def forward(self, x, **kw):
            return torch.zeros(x.shape[0], 8, device=x.device)

    import tempfile
    from oracle.metrics import write_dataset
    ds, _ = write_dataset(os.path.join(tempfile.mkdtemp(), 'labels'))          # camera labels for G's c (c_dim 25)
    metric_utils._feature_detector_cache[('zero', dev)] = Zero()
    opts = metric_utils.MetricOptions(G=G, G_kwargs={}, num_gpus=1, rank=0, device=dev, cache=False,
                                      dataset_kwargs=dict(class_name='ide3d_b200.training.dataset.ImageFolderDataset', path=ds, use_labels=True))
    n = args.gen_items
    run = lambda: metric_utils.compute_feature_stats_for_generator(opts=opts, detector_url='zero', detector_kwargs={}, capture_mean_cov=True,
                                                                   max_items=n)
    ts = timed(run, args.runs)
    return {'items': n, 's': ts, 'images_per_s': n / min(ts), 'generator': 'random-init ide3d-ffhq-64-512', 'batch_gen': 4}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--ref-rows', type=int, default=2000)
    ap.add_argument('--ref-batches', type=int, default=100)
    ap.add_argument('--gen-items', type=int, default=512)
    ap.add_argument('--skip', default='')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_metrics.py needs a CUDA device')
    dev = torch.device('cuda', 0)
    skip = set(filter(None, args.skip.split(',')))
    out = {'card': card(), 'runs': args.runs}
    for name, fn in (('kernels', bench_kernels), ('stats', bench_stats), ('gen', bench_gen)):
        if name not in skip:
            out[name] = fn(args, dev)
            torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
