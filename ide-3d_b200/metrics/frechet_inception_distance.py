"""Frechet Inception Distance (metrics/frechet_inception_distance.py).  The statistics are summed on the device in float64; the
matrix square root stays scipy.linalg.sqrtm on the host, so the value follows the reference's."""

import numpy as np
import scipy.linalg

from . import metric_utils

INCEPTION_URL = 'https://api.ngc.nvidia.com/v2/models/nvidia/research/stylegan3/versions/1/files/metrics/inception-2015-12-05.pkl'


def compute_fid(opts, max_real, num_gen):
    detector_url = INCEPTION_URL
    detector_kwargs = dict(return_features=True)  # Return raw features before the softmax layer.

    mu_real, sigma_real = metric_utils.compute_feature_stats_for_dataset(
        opts=opts, detector_url=detector_url, detector_kwargs=detector_kwargs,
        rel_lo=0, rel_hi=0, capture_mean_cov=True, max_items=max_real).get_mean_cov()

    mu_gen, sigma_gen = metric_utils.compute_feature_stats_for_generator(
        opts=opts, detector_url=detector_url, detector_kwargs=detector_kwargs,
        rel_lo=0, rel_hi=1, capture_mean_cov=True, max_items=num_gen).get_mean_cov()

    if opts.rank != 0:
        return float('nan')

    m = np.square(mu_gen - mu_real).sum()
    s = scipy.linalg.sqrtm(np.dot(sigma_gen, sigma_real))       # the reference's disp=False is gone from scipy >= 1.14
    fid = np.real(m + np.trace(sigma_gen + sigma_real - s * 2))
    return float(fid)
