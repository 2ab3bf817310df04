"""Precision / recall (metrics/precision_recall.py) with the neighbour search on sm_90a.

The reference builds every distance block with torch.cdist, copies it to the host and runs kthvalue and the comparison there.  Here
each rank takes a contiguous share of the manifold's rows, computes their (nhood_size + 1)th neighbour distance against the whole
gathered manifold with knn.kth_dist, and the shares are summed into the full radius vector; then each rank flags its share of the
probes with knn.within.  As in the reference the features are fp16 and the radius is rounded to fp16 before the comparison.
row_batch_size and col_batch_size are accepted for the reference's signature; the kernels need no batching.
"""

import torch

from ..torch_utils.ops import knn
from . import metric_utils

VGG16_URL = 'https://api.ngc.nvidia.com/v2/models/nvidia/research/stylegan3/versions/1/files/metrics/vgg16.pkl'


def _share(n, num_gpus, rank):
    return n * rank // num_gpus, n * (rank + 1) // num_gpus


def _all_reduce(t, num_gpus):
    if num_gpus > 1:
        torch.distributed.all_reduce(t)
    return t


def compute_pr(opts, max_real, num_gen, nhood_size, row_batch_size, col_batch_size):
    del row_batch_size, col_batch_size
    detector_url = VGG16_URL
    detector_kwargs = dict(return_features=True)

    real_features = metric_utils.compute_feature_stats_for_dataset(
        opts=opts, detector_url=detector_url, detector_kwargs=detector_kwargs,
        rel_lo=0, rel_hi=0, capture_all=True, max_items=max_real).get_all_torch().to(torch.float16).to(opts.device)

    gen_features = metric_utils.compute_feature_stats_for_generator(
        opts=opts, detector_url=detector_url, detector_kwargs=detector_kwargs,
        rel_lo=0, rel_hi=1, capture_all=True, max_items=num_gen).get_all_torch().to(torch.float16).to(opts.device)

    results = dict()
    for name, manifold, probes in [('precision', real_features, gen_features), ('recall', gen_features, real_features)]:
        lo, hi = _share(manifold.shape[0], opts.num_gpus, opts.rank)
        radius = torch.zeros(manifold.shape[0], dtype=torch.float32, device=opts.device)
        radius[lo:hi] = knn.kth_dist(manifold[lo:hi], manifold, nhood_size + 1)
        radius = _all_reduce(radius, opts.num_gpus).to(torch.float16).to(torch.float32)
        lo, hi = _share(probes.shape[0], opts.num_gpus, opts.rank)
        hits = knn.within(probes[lo:hi], manifold, radius).sum().to(torch.float64)
        results[name] = float(_all_reduce(hits, opts.num_gpus).to(torch.float32) / probes.shape[0])   # the reference's fp32 mean
    return results['precision'], results['recall']
