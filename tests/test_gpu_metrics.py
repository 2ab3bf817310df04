"""H100: the k-NN kernels of the precision / recall metric (ide3d_knn_kth_dist, ide3d_knn_within) against float64, and the metrics
end to end on the device with the stand-in detectors and generator against the CPU golden of the reference's metric modules.

Distances are compared squared.  The kernel's squared distance |x|^2 + |y|^2 - 2 x.y accumulates in fp32 over D terms, so each
entry is within DELTA * (|x|^2 + |y|^2) of the float64 value; a kth order statistic moves by no more than its entries do.  The
largest error measured on an H100 80GB HBM3 (700 W) is 2.55e-5 at D = 4096 (1.3e-7 to 2.1e-7 at D = 40): the tensor cores' fp32
accumulation of the dot products loses about one bit per 16-deep step, and those losses do not cancel.  torch.cdist on fp16, which
the reference uses, rounds each distance to 11 bits (4.9e-4).  DELTA is 3.9x the measured error.
"""

import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, load_golden

pytestmark = pytest.mark.gpu

DELTA = 1e-4


def _feats(n, d, seed, dev):
    """VGG-like features: non-negative, a shared mean direction plus per-row spread, fp16."""
    g = torch.Generator(device='cpu').manual_seed(seed)
    base = torch.rand(1, d, generator=g)
    x = (base + 0.5 * torch.rand(n, d, generator=g)) * torch.rand(n, 1, generator=g).add(0.5)
    return x.to(torch.float16).to(dev)


def _d2_f64(a, b):
    a, b = a.double(), b.double()
    return ((a * a).sum(1)[:, None] + (b * b).sum(1)[None, :] - 2 * a @ b.t()).clamp_min(0)


def _check_kth(rows, cols, kth):
    from ide3d_b200.torch_utils.ops import knn
    out = knn.kth_dist(rows, cols, kth)
    torch.cuda.synchronize()
    ref = torch.cat([_d2_f64(r, cols).kthvalue(kth, dim=1).values for r in rows.split(1024)])
    nr, nc = rows.double().pow(2).sum(1), cols.double().pow(2).sum(1)
    scale = nr + nc.max()
    err = ((out.double() ** 2 - ref).abs() / scale).max().item()
    print(f'kth_dist R={rows.shape[0]} C={cols.shape[0]} D={rows.shape[1]} kth={kth}: max |d^2 - ref| / (|x|^2 + max|y|^2) = {err:.2e}')
    assert err <= DELTA
    return out


@pytest.mark.parametrize('kth', [1, 3, 4, 9, 16])       # 3 and 9 select inside a longer list (lists of 4 and 16)
@pytest.mark.parametrize('d', [40, 4096])
def test_kth_dist_ragged_with_duplicates(kth, d):
    dev = torch.device('cuda')
    cols = _feats(1000, d, seed=d + kth, dev=dev)
    cols[500:520] = cols[0:20]                       # duplicate rows: zero distances and ties
    cols[700:705] = cols[3]
    rows = torch.cat([cols[:200], _feats(100, d, seed=7, dev=dev)])    # R = 300: a slice of cols (self-distance counts) + others
    out = _check_kth(rows, cols, kth)
    if kth == 1:
        assert (out[:200] ** 2 <= DELTA * 2 * rows[:200].double().pow(2).sum(1)).all()


def test_kth_dist_production_manifold():
    """2048 rows of a 70,000 x 4096 manifold against all of it (pr50k3_full's real-feature pass, one row batch)."""
    dev = torch.device('cuda')
    cols = _feats(70000, 4096, seed=11, dev=dev)
    _check_kth(cols[:2048], cols, 4)


def test_kth_dist_one_column_tile_per_split():
    dev = torch.device('cuda')
    cols = _feats(130, 64, seed=3, dev=dev)          # two column tiles, the second with 2 columns
    _check_kth(_feats(5, 64, seed=4, dev=dev), cols, 16)


@pytest.mark.parametrize('d', [40, 4096])
def test_within_against_float64(d):
    from ide3d_b200.torch_utils.ops import knn
    dev = torch.device('cuda')
    manifold = _feats(3000, d, seed=21, dev=dev)
    radius = knn.kth_dist(manifold, manifold, 4)
    # the first 1280 probes are manifold rows (each hits at its own column), the rest are new points near and far; with several
    # column splits no CTA here gets a hit for every row inside its split, so the early stop is covered by test_within_stops_early
    probes = torch.cat([manifold[torch.randperm(3000, generator=torch.Generator().manual_seed(0))[:1280].to(dev)],
                        _feats(1717, d, seed=22, dev=dev), _feats(300, d, seed=23, dev=dev) * 3])
    flags = knn.within(probes, manifold, radius)
    torch.cuda.synchronize()
    d2 = _d2_f64(probes, manifold)
    r2 = radius.double() ** 2
    want = (d2 <= r2[None]).any(1)
    scale = probes.double().pow(2).sum(1)[:, None] + manifold.double().pow(2).sum(1)[None] + r2[None]
    near = ((d2 - r2[None]).abs() <= DELTA * scale).any(1)
    bad = (flags != want) & ~near
    print(f'within D={d}: {int(want.sum())} / {probes.shape[0]} hits, {int(near.sum())} probes inside the fp32 margin, '
          f'{int((flags != want).sum())} flags differ')
    assert not bad.any()
    assert flags[:1280].all()


def test_refusals_on_device():
    from ide3d_b200.torch_utils.ops import knn
    dev = torch.device('cuda')
    x = _feats(10, 16, seed=0, dev=dev)
    with pytest.raises(RuntimeError, match='kth'):
        knn.kth_dist(x, x, 17)
    with pytest.raises(RuntimeError, match='exceeds'):
        knn.kth_dist(x, x[:3], 4)
    with pytest.raises(RuntimeError, match='multiple of 8'):
        knn.kth_dist(x[:, :12].contiguous(), x[:, :12].contiguous(), 1)


def _margin(probes, manifold, r2, d2):
    """Probes with some j where the fp32 kernel could decide |d^2 - r^2| either way."""
    scale = probes.double().pow(2).sum(1)[:, None] + manifold.double().pow(2).sum(1)[None] + r2[None]
    return ((d2 - r2[None]).abs() <= DELTA * scale).any(1), DELTA * scale


@pytest.mark.parametrize('d', [40, 4096])
def test_within_stops_early(d):
    """CTAs that stop early, by construction.  With one more row tile than SMs there is one column split, so CTA t walks the column
    tiles 0, 1, ... in order.  The 128 probes of row tile t < 96 are copies of the manifold rows of column tile t % 4: each has a hit
    (its own distance, 0) in that tile at the latest, so the CTA stops at tile t % 4 or before, with later tiles left.  The other row
    tiles hold far points and walk every tile.  The float64 decisions give, per CTA, the tile by which it must have stopped and the
    earliest it can stop; the test asserts that stops at tiles 0 to 3 all occur (a stop at tile >= 2 takes the producer's vote wait,
    at D = 4096 the drained tile is 64 chunks deep, more than the 4-stage ring), and checks every flag against float64."""
    from ide3d_b200.torch_utils.ops import knn
    dev = torch.device('cuda')
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    tiles, col_tiles = sms + 1, 8
    manifold = _feats(col_tiles * 128, d, seed=31, dev=dev)
    radius = knn.kth_dist(manifold, manifold, 4)
    g = torch.Generator().manual_seed(1)
    copies = [manifold[(t % 4) * 128 + torch.randperm(128, generator=g).to(dev)] for t in range(96)]
    far = _feats((tiles - 96) * 128 - 37, d, seed=32, dev=dev) * 3                    # ragged last tile
    probes = torch.cat(copies + [far])
    flags = knn.within(probes, manifold, radius)
    torch.cuda.synchronize()
    d2 = _d2_f64(probes, manifold)
    r2 = radius.double() ** 2
    want = (d2 <= r2[None]).any(1)
    near, tol = _margin(probes, manifold, r2, d2)
    bad = (flags != want) & ~near
    assert not bad.any() and flags[:96 * 128].all()

    sure = d2 <= r2[None] - tol                                                         # hits the kernel must see
    maybe = d2 <= r2[None] + tol                                                        # hits it may see
    def stop_tile(hit):                                                                  # first tile by which every row of the CTA has a hit
        per_tile = hit[:96 * 128].reshape(96, 128, col_tiles, 128).any(3)               # [cta, row, column tile]
        done = per_tile.cumsum(2).clamp(max=1).all(1)                                    # [cta, column tile]
        return torch.where(done.any(1), done.float().argmax(1), torch.full((96,), col_tiles, device=hit.device))
    latest, earliest = stop_tile(sure), stop_tile(maybe)
    print(f'within D={d}: {tiles} row tiles x {col_tiles} column tiles, CTAs stopping by tile 0..3: '
          f'{[int((latest == j).sum()) for j in range(4)]}, earliest possible {[int((earliest == j).sum()) for j in range(4)]}, '
          f'{int(near.sum())} probes inside the margin')
    assert (latest <= torch.arange(96, device=dev) % 4).all()
    for j in range(4):                                                                   # stops at every one of tiles 0..3 happen
        assert ((latest == j) & (earliest == j)).any(), j


def test_metrics_end_to_end_against_cpu_golden(tmp_path, monkeypatch):
    """fid / kid / is / pr on the device (stand-in generator and detectors on cuda, FeatureStats in float64 on the device, PR through
    both kernels) against the reference's values on the CPU (tests/golden/metrics.npz).  Measured on an H100 80GB HBM3 (700 W), TF32
    off: FID 2.7e-7 and KID 2.1e-5 relative, IS mean equal, IS std 6.4e-8, features within 7.6e-6; the bounds below are 4x to 10x
    those.  PR: the kernels may differ from the float64 decision on the same device features only for probes inside the fp32 margin
    (5 of 48 for precision, 0 for recall), and the float64 decision equals the golden; measured, both equal the golden exactly."""
    sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
    import make_metrics_golden as mg
    from ide3d_b200.dnnlib import util as dutil
    from ide3d_b200.metrics import (frechet_inception_distance, inception_score, kernel_inception_distance, metric_utils,
                                    precision_recall)
    from oracle import metrics as om
    golden = load_golden('metrics')
    ds, _ = mg.setup(str(tmp_path))
    monkeypatch.setattr(dutil, '_dnnlib_cache_dir', os.path.join(str(tmp_path), 'cache'))
    monkeypatch.setattr(torch.backends.cudnn, 'allow_tf32', False)
    monkeypatch.setattr(torch.backends.cuda.matmul, 'allow_tf32', False)
    metric_utils._feature_detector_cache.clear()
    dev = torch.device('cuda')
    opts = lambda: metric_utils.MetricOptions(G=om.StandInMetricGenerator(), G_kwargs={}, device=dev, cache=False,
                                              dataset_kwargs=dict(class_name='ide3d_b200.training.dataset.ImageFolderDataset', path=ds,
                                                                  use_labels=True, max_size=None, xflip=False))
    n = mg.SIZES['num_gen']
    fid = frechet_inception_distance.compute_fid(opts(), max_real=None, num_gen=n)
    kid = kernel_inception_distance.compute_kid(opts(), max_real=1000000, num_gen=n, num_subsets=mg.SIZES['kid_subsets'], max_subset_size=1000)
    is_mean, is_std = inception_score.compute_is(opts(), num_gen=n, num_splits=mg.SIZES['is_splits'])
    p, r = precision_recall.compute_pr(opts(), max_real=200000, num_gen=n, nhood_size=3, row_batch_size=10000, col_batch_size=10000)
    errs = dict(fid=abs(fid / golden['fid'] - 1), kid=abs(kid / golden['kid'] - 1), is_mean=abs(is_mean / golden['is_mean'] - 1),
                is_std=abs(is_std - golden['is_std']))
    feats = {}
    for url, tag in ((mg.INCEPTION_URL, 'inception'), (mg.VGG16_URL, 'vgg')):
        kw = dict(return_features=True)
        feats[f'gen_{tag}'] = metric_utils.compute_feature_stats_for_generator(opts(), url, kw, capture_all=True, max_items=n).get_all_torch()
        feats[f'real_{tag}'] = metric_utils.compute_feature_stats_for_dataset(opts(), url, kw, capture_all=True).get_all_torch()
        for k in (f'gen_{tag}', f'real_{tag}'):
            errs[k] = (feats[k].cpu().numpy() - golden[k]).__abs__().max()
    # PR: float64 decisions on the device features (fp16, as compute_pr takes them), and the probes inside the margin
    real, gen = feats['real_vgg'].half(), feats['gen_vgg'].half()
    counts = {}
    for name, manifold, probes, got in (('precision', real, gen, p), ('recall', gen, real, r)):
        r64 = _d2_f64(manifold, manifold).kthvalue(4, dim=1).values.sqrt().half().double()
        d2 = _d2_f64(probes, manifold)
        r2 = r64 ** 2
        near, tol = _margin(probes, manifold, r2, d2)
        ulp = (2 * r64 * r64.abs().clamp(min=2 ** -14) * 2 ** -10)[None]                # fp16 rounding of the kernel's radius
        near |= ((d2 - r2[None]).abs() <= tol + ulp).any(1)
        p64 = (d2 <= r2[None]).any(1).float().mean().item()
        counts[name] = (got, p64, int(near.sum()))
        assert abs(got - p64) <= near.sum().item() / probes.shape[0] + 1e-7, name
        assert p64 == pytest.approx(float(golden[f'pr_{name}']), abs=near.sum().item() / probes.shape[0] + 1e-7), name
    print(f'end to end on the device vs the CPU golden: {errs}; PR (kernel, float64, probes in margin): {counts}')
    assert errs['fid'] <= 3e-6 and errs['kid'] <= 1e-4 and errs['is_mean'] <= 1e-6 and errs['is_std'] <= 5e-7
    assert max(errs[k] for k in ('gen_inception', 'real_inception', 'gen_vgg', 'real_vgg')) <= 5e-5

