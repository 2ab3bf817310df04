"""Golden data of the metrics: the reference's own metric modules (metrics/metric_utils.py, frechet_inception_distance.py,
kernel_inception_distance.py, inception_score.py, precision_recall.py) and training/dataset.py run on the CPU with the stand-in
detectors and generator of oracle/metrics.py.

    python tests/golden/make_metrics_golden.py [/path/to/reference]   -> tests/golden/metrics.npz

The reference draws z with torch.randn and label indices with np.random.randint; both are patched to the package's rule, item i
drawing from np.random.RandomState([seed, i]) (metric_utils.item_draws), so the two implementations evaluate the same items.  KID's
subsets come from np.random.seed(0).  Sizes are small (20 real images, 48 generated, 8 / 16 features), see SIZES.
"""

import hashlib
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

INCEPTION_URL = 'https://api.ngc.nvidia.com/v2/models/nvidia/research/stylegan3/versions/1/files/metrics/inception-2015-12-05.pkl'
VGG16_URL = 'https://api.ngc.nvidia.com/v2/models/nvidia/research/stylegan3/versions/1/files/metrics/vgg16.pkl'
SIZES = dict(num_gen=48, kid_subsets=10, is_splits=4, nhood=3)
DETECTORS = {INCEPTION_URL: dict(features=8, classes=10, seed=0), VGG16_URL: dict(features=16, classes=10, seed=1, normalize=True)}


def detector_file(cache_dir, url):
    return os.path.join(cache_dir, 'downloads', hashlib.md5(url.encode('utf-8')).hexdigest() + '_' + url.split('/')[-1])


class _Unpinned(torch.Tensor):
    """pin_memory() needs CUDA; on the CPU the labels stay where they are."""

    def pin_memory(self):
        return self.as_subclass(torch.Tensor)


def setup(tmp):
    """The dataset (dir and zip) and both detectors in the download cache under `tmp`."""
    from oracle import metrics as om
    ds_dir, ds_zip = om.write_dataset(os.path.join(tmp, 'ffhq-mini'))
    for url, kw in DETECTORS.items():
        om.save_detector(detector_file(os.path.join(tmp, 'cache'), url), **kw)
    return ds_dir, ds_zip


def main(ref=None):
    ref = ref or os.environ.get('IDE3D_REFERENCE', '/root/reference')
    sys.path.insert(0, ref)
    import dnnlib as ref_dnnlib                                       # the reference's
    from metrics import metric_utils as rmu, frechet_inception_distance as rfid, kernel_inception_distance as rkid
    from metrics import inception_score as ris, precision_recall as rpr
    from training import dataset as rds
    from oracle import metrics as om
    from ide3d_b200.metrics.metric_utils import item_draws

    torch.set_num_threads(1)
    tmp = tempfile.mkdtemp()
    ds_dir, ds_zip = setup(tmp)
    ref_dnnlib.util.set_cache_dir(os.path.join(tmp, 'cache'))
    G = om.StandInMetricGenerator()
    out = {}

    # dataset restatement: images and labels, dir and zip, plain and with max_size + xflip
    for kind, path in (('dir', ds_dir), ('zip', ds_zip)):
        for tag, kw in (('plain', {}), ('sub', dict(max_size=7, xflip=True, random_seed=3))):
            d = rds.ImageFolderDataset(path=path, use_labels=True, **kw)
            items = [d[i] for i in range(len(d))]
            out[f'ds_{kind}_{tag}_images'] = np.stack([x for x, _ in items])
            out[f'ds_{kind}_{tag}_labels'] = np.stack([c for _, c in items])
            out[f'ds_{kind}_{tag}_name'] = np.array(d.name)

    # the (seed, i) draw rule in the reference's loop
    num_labels = len(rds.ImageFolderDataset(path=ds_dir, use_labels=True))
    counters = dict(z=0, c=0)

    def randn(shape, device=None, **_kw):
        n, zd = shape
        z = np.stack([item_draws(0, counters['z'] + k, zd, num_labels)[0] for k in range(n)])
        counters['z'] += n
        return torch.from_numpy(z).to(device)

    def randint(_n):
        i = counters['c']
        counters['c'] += 1
        return item_draws(0, i, G.z_dim, num_labels)[1]

    rmu.torch = types.SimpleNamespace(**{k: getattr(torch, k) for k in dir(torch) if not k.startswith('__')})
    rmu.torch.randn = randn
    rmu.torch.from_numpy = lambda a: torch.from_numpy(a).as_subclass(_Unpinned)
    rmu.np = types.SimpleNamespace(**{k: getattr(np, k) for k in dir(np) if not k.startswith('__')})
    rmu.np.random = types.SimpleNamespace(randint=randint)

    def opts(cache=False):
        counters.update(z=0, c=0)
        return rmu.MetricOptions(G=G, G_kwargs=dict(cond_render=False), num_gpus=1, rank=0, device=torch.device('cpu'), cache=cache,
                                 dataset_kwargs=dict(class_name='training.dataset.ImageFolderDataset', path=ds_dir, use_labels=True,
                                                     max_size=None, xflip=False))

    import scipy.linalg                                               # scipy >= 1.14 dropped sqrtm's disp argument: same matrix
    rfid.scipy = types.SimpleNamespace(linalg=types.SimpleNamespace(sqrtm=lambda a, disp=True: (scipy.linalg.sqrtm(a), None)))
    # torch has no fp16 cdist on the CPU: compute in fp32 and round the distances to fp16, as the CUDA kernel's output is
    rpr.torch = types.SimpleNamespace(**{k: getattr(torch, k) for k in dir(torch) if not k.startswith('__')})
    rpr.torch.cdist = lambda a, b: torch.cdist(a.float(), b.float()).half()
    G.forward = (lambda f: (lambda z, c, cond_render=False, **kw: f(z, c, **kw)))(G.forward)   # the reference passes G_kwargs on
    n = SIZES['num_gen']
    out['fid'] = np.float64(rfid.compute_fid(opts(), max_real=None, num_gen=n))
    np.random.seed(0)
    out['kid'] = np.float64(rkid.compute_kid(opts(), max_real=1000000, num_gen=n, num_subsets=SIZES['kid_subsets'], max_subset_size=1000))
    out['is_mean'], out['is_std'] = map(np.float64, ris.compute_is(opts(), num_gen=n, num_splits=SIZES['is_splits']))
    out['pr_precision'], out['pr_recall'] = map(np.float64, rpr.compute_pr(opts(), max_real=200000, num_gen=n, nhood_size=SIZES['nhood'],
                                                                           row_batch_size=10000, col_batch_size=10000))
    for url, tag in ((INCEPTION_URL, 'inception'), (VGG16_URL, 'vgg')):
        kw = dict(return_features=True)
        out[f'gen_{tag}'] = rmu.compute_feature_stats_for_generator(opts(), url, kw, capture_all=True, max_items=n).get_all()
        out[f'real_{tag}'] = rmu.compute_feature_stats_for_dataset(opts(), url, kw, capture_all=True).get_all()
    out['gen_probs'] = rmu.compute_feature_stats_for_generator(opts(), INCEPTION_URL, dict(no_output_bias=True), capture_all=True,
                                                               max_items=n).get_all()
    out['gen_z'] = np.stack([item_draws(0, i, G.z_dim, num_labels)[0] for i in range(n)])

    # a FeatureStats cache the reference writes
    o = opts(cache=True)
    rmu.compute_feature_stats_for_dataset(o, INCEPTION_URL, dict(return_features=True), capture_mean_cov=True)
    cache = os.path.join(tmp, 'cache', 'gan-metrics')
    (name,) = os.listdir(cache)
    out['cache_name'] = np.array(name)
    out['cache_bytes'] = np.frombuffer(open(os.path.join(cache, name), 'rb').read(), np.uint8)
    np.savez_compressed(os.path.join(HERE, 'metrics.npz'), **out)
    print({k: (v.shape if v.ndim else v) for k, v in out.items() if k != 'cache_bytes'})


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else None)
