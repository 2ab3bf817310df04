"""CPU: the metrics package against the reference's own metric modules (tests/golden/make_metrics_golden.py, stand-in detectors and
generator of oracle/metrics.py): dataset restatement, FeatureStats caches both ways, FID / KID / IS values, PR with the float64
k-NN in place of the kernels, the (seed, i) draw rule across world sizes, the jsonl record, and the refusals."""

import hashlib
import json
import os
import pickle
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, load_golden

sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
import make_metrics_golden as mg  # noqa: E402

from ide3d_b200 import _lib  # noqa: E402
from ide3d_b200.dnnlib import util as dutil  # noqa: E402
from ide3d_b200.metrics import (frechet_inception_distance, inception_score, kernel_inception_distance, metric_main,  # noqa: E402
                                metric_utils, precision_recall)
from ide3d_b200.training.dataset import ImageFolderDataset  # noqa: E402
from oracle import metrics as om  # noqa: E402

CPU = torch.device('cpu')


@pytest.fixture(scope='module')
def golden():
    return load_golden('metrics')


@pytest.fixture()
def env(tmp_path, monkeypatch):
    ds_dir, ds_zip = mg.setup(str(tmp_path))
    monkeypatch.setattr(dutil, '_dnnlib_cache_dir', os.path.join(str(tmp_path), 'cache'))
    metric_utils._feature_detector_cache.clear()
    return ds_dir, ds_zip


def _opts(ds, cache=False, **kw):
    return metric_utils.MetricOptions(G=om.StandInMetricGenerator(), G_kwargs={}, device=CPU, cache=cache,
                                      dataset_kwargs=dict(class_name='ide3d_b200.training.dataset.ImageFolderDataset', path=ds,
                                                          use_labels=True, max_size=None, xflip=False), **kw)


@pytest.mark.parametrize('kind', ['dir', 'zip'])
def test_dataset_matches_reference(env, golden, kind):
    path = env[0] if kind == 'dir' else env[1]
    for tag, kw in (('plain', {}), ('sub', dict(max_size=7, xflip=True, random_seed=3))):
        d = ImageFolderDataset(path=path, use_labels=True, **kw)
        items = [d[i] for i in range(len(d))]
        assert np.array_equal(np.stack([x for x, _ in items]), golden[f'ds_{kind}_{tag}_images'])
        assert np.array_equal(np.stack([c for _, c in items]), golden[f'ds_{kind}_{tag}_labels'])
        assert d.name == str(golden[f'ds_{kind}_{tag}_name'])
    assert d.label_shape == [25] and d.resolution == 32


def test_features_and_draws_match_reference(env, golden):
    n = mg.SIZES['num_gen']
    for url, tag in ((mg.INCEPTION_URL, 'inception'), (mg.VGG16_URL, 'vgg')):
        kw = dict(return_features=True)
        gen = metric_utils.compute_feature_stats_for_generator(_opts(env[0]), url, kw, capture_all=True, max_items=n).get_all()
        real = metric_utils.compute_feature_stats_for_dataset(_opts(env[0]), url, kw, capture_all=True).get_all()
        np.testing.assert_allclose(gen, golden[f'gen_{tag}'], rtol=0, atol=1e-5)
        assert np.array_equal(real, golden[f'real_{tag}'])


def test_fid_kid_is_match_reference(env, golden):
    """Measured on the CPU against the golden: FID 3.7e-9 relative, KID 3.2e-5 relative (the generated features differ in the
    last fp32 bits and KID's cubic kernel sums cancel), IS mean equal and IS std 3.2e-8 absolute."""
    n = mg.SIZES['num_gen']
    fid = frechet_inception_distance.compute_fid(_opts(env[0]), max_real=None, num_gen=n)
    kid = kernel_inception_distance.compute_kid(_opts(env[0]), max_real=1000000, num_gen=n, num_subsets=mg.SIZES['kid_subsets'],
                                                max_subset_size=1000)
    is_mean, is_std = inception_score.compute_is(_opts(env[0]), num_gen=n, num_splits=mg.SIZES['is_splits'])
    assert fid == pytest.approx(float(golden['fid']), rel=1e-7)
    assert kid == pytest.approx(float(golden['kid']), rel=1e-4)
    assert is_mean == pytest.approx(float(golden['is_mean']), rel=1e-5)
    assert is_std == pytest.approx(float(golden['is_std']), rel=1e-3, abs=1e-6)


def test_pr_with_float64_knn_matches_reference(env, golden, monkeypatch):
    monkeypatch.setattr(precision_recall.knn, 'kth_dist', om.knn_kth_dist)
    monkeypatch.setattr(precision_recall.knn, 'within', om.knn_within)
    p, r = precision_recall.compute_pr(_opts(env[0]), max_real=200000, num_gen=mg.SIZES['num_gen'], nhood_size=3,
                                       row_batch_size=10000, col_batch_size=10000)
    assert (p, r) == (float(golden['pr_precision']), float(golden['pr_recall']))


def test_feature_stats_cache_both_ways(env, golden, tmp_path):
    # the cache name is the reference's: <dataset name>-<detector name>-md5(repr(sorted(args))); the golden's tag hashes its own
    # temporary dataset path, so only its prefix is compared
    opts = _opts(env[0], cache=True)
    kw = dict(return_features=True)
    args = dict(dataset_kwargs=opts.dataset_kwargs, detector_url=mg.INCEPTION_URL, detector_kwargs=kw, stats_kwargs=dict(capture_mean_cov=True))
    name = f'ffhq-mini-inception-2015-12-05-{hashlib.md5(repr(sorted(args.items())).encode("utf-8")).hexdigest()}.pkl'
    assert str(golden['cache_name']).rsplit('-', 1)[0] == name.rsplit('-', 1)[0]
    cache_dir = dutil.make_cache_dir_path('gan-metrics')
    os.makedirs(cache_dir)
    with open(os.path.join(cache_dir, name), 'wb') as f:                    # the reference's file, loaded here
        f.write(golden['cache_bytes'].tobytes())
    theirs = metric_utils.compute_feature_stats_for_dataset(opts, mg.INCEPTION_URL, kw, capture_mean_cov=True)
    os.remove(os.path.join(cache_dir, name))
    mine = metric_utils.compute_feature_stats_for_dataset(opts, mg.INCEPTION_URL, kw, capture_mean_cov=True)
    assert os.listdir(cache_dir) == [name]
    for a, b in zip(theirs.get_mean_cov(), mine.get_mean_cov()):
        np.testing.assert_allclose(a, b, rtol=0, atol=1e-12)
    # and this package's file has the reference's __dict__ keys and types
    ref = pickle.loads(golden['cache_bytes'].tobytes())
    with open(os.path.join(cache_dir, name), 'rb') as f:
        ours = pickle.load(f)
    assert sorted(ours) == sorted(ref)
    assert all(type(ours[k]) is type(ref[k]) for k in ref)


@pytest.mark.parametrize('world, n', [(2, 10), (3, 2)])
def test_draws_independent_of_world_and_batch(env, world, n):
    """World 2 (two gloo processes, batch 8 of 2) evaluates the same items (z and labels) as world 1 (batch 4 of 4).  The features
    differ only by the stand-in generator's batch-composition rounding in fp32 (measured 6e-8), the sums by that and float64 order.
    World 3 with 2 items leaves rank 2 without an item: it still joins the gather and the sums."""
    one = metric_utils.compute_feature_stats_for_generator(_opts(env[0]), mg.INCEPTION_URL, dict(return_features=True), batch_size=4,
                                                           capture_all=True, capture_mean_cov=True, max_items=n)
    if not torch.distributed.is_gloo_available():
        pytest.skip('gloo unavailable')
    import subprocess
    import tempfile
    init = os.path.join(tempfile.mkdtemp(), 'init')
    code = f'''
import os, sys, numpy as np, torch
sys.path.insert(0, {ROOT!r}); sys.path.insert(0, {os.path.join(ROOT, 'tests', 'golden')!r})
rank = int(sys.argv[1])
torch.distributed.init_process_group('gloo', init_method='file://{init}', rank=rank, world_size={world})
from ide3d_b200.dnnlib import util as dutil
dutil.set_cache_dir({dutil.make_cache_dir_path()!r})
from ide3d_b200.metrics import metric_utils
from oracle import metrics as om
import make_metrics_golden as mg
o = metric_utils.MetricOptions(G=om.StandInMetricGenerator(), G_kwargs={{}}, device=torch.device('cpu'), cache=False, num_gpus={world},
    rank=rank, dataset_kwargs=dict(class_name='ide3d_b200.training.dataset.ImageFolderDataset', path={env[0]!r}, use_labels=True))
s = metric_utils.compute_feature_stats_for_generator(o, mg.INCEPTION_URL, dict(return_features=True), batch_size=8, batch_gen=2,
    capture_all=True, capture_mean_cov=True, max_items={n})
m, c = s.get_mean_cov()
np.savez({os.path.dirname(init)!r} + f'/out{{rank}}.npz', all=s.get_all(), m=m, c=c)
torch.distributed.destroy_process_group()
'''
    procs = [subprocess.Popen([sys.executable, '-c', code, str(r)]) for r in range(world)]
    assert all(p.wait(timeout=300) == 0 for p in procs)
    m1, c1 = one.get_mean_cov()
    for r in range(world):
        res = np.load(os.path.join(os.path.dirname(init), f'out{r}.npz'))
        np.testing.assert_allclose(res['all'], one.get_all(), rtol=0, atol=1e-6)
        np.testing.assert_allclose(res['m'], m1, rtol=0, atol=1e-6)
        np.testing.assert_allclose(res['c'], c1, rtol=0, atol=1e-6)


def test_report_metric_jsonl(tmp_path, capsys):
    rd = dict(results={'fid50k_full': 1.5}, metric='fid50k_full', total_time=2.0, total_time_str='2s', num_gpus=1)
    metric_main.report_metric(rd, run_dir=str(tmp_path), snapshot_pkl=str(tmp_path / 'network-snapshot.pkl'))
    line = json.loads(open(tmp_path / 'metric-fid50k_full.jsonl').read().strip())
    assert line['results'] == {'fid50k_full': 1.5} and line['snapshot_pkl'] == 'network-snapshot.pkl' and 'timestamp' in line


def test_registered_metrics_and_refusals(env):
    assert sorted(metric_main.list_valid_metrics()) == sorted(['fid50k_full', 'kid50k_full', 'pr50k3_full', 'is50k', 'fid50k', 'kid50k', 'pr50k3'])
    for name in ('ppl2_wend', 'eqt50k_int', 'eqt50k_frac', 'eqr50k', 'nope'):
        assert not metric_main.is_valid_metric(name)
        with pytest.raises(AssertionError, match='invalid metric'):
            metric_main.calc_metric(metric=name, G=None, dataset_kwargs={}, num_gpus=1, rank=0, device=CPU)
    o = _opts(env[0])
    o.G_kwargs['cond_render'] = True
    with pytest.raises(NotImplementedError):
        metric_utils.compute_feature_stats_for_generator(o, mg.INCEPTION_URL, {}, capture_all=True, max_items=2)
    url = 'https://example.invalid/metrics/missing.pkl'
    want = os.path.join(dutil.make_cache_dir_path('downloads'), hashlib.md5(url.encode()).hexdigest() + '_missing.pkl')
    with pytest.raises(FileNotFoundError, match=want.replace('.', r'\.')):
        metric_utils.get_feature_detector(url)
    from ide3d_b200.torch_utils.ops import knn
    x = torch.zeros(4, 8, dtype=torch.float16)
    with pytest.raises(RuntimeError, match='CUDA'):
        knn.kth_dist(x, x, 1)
    with pytest.raises(RuntimeError, match='CUDA'):
        knn.within(x, x, torch.zeros(4))


def test_entry_points_validate_arguments(lib):
    assert lib.ide3d_knn_kth_dist(None, 4, None, 4, 8, 1, None, None, 0, None) == _lib.INVALID
    assert b'null' in lib.ide3d_last_error()
    p = 1 << 20                                                  # a 16-byte aligned dummy address: never dereferenced
    for kth, msg in ((0, b'kth'), (17, b'kth'), (5, b'exceeds')):
        assert lib.ide3d_knn_kth_dist(p, 4, p, 4, 8, kth, p, p, 1 << 30, None) == _lib.INVALID
        assert msg in lib.ide3d_last_error()
    assert lib.ide3d_knn_kth_dist(p, 4, p, 4, 12, 1, p, p, 1 << 30, None) == _lib.INVALID and b'multiple of 8' in lib.ide3d_last_error()
    assert lib.ide3d_knn_kth_dist(p, 4, p, 4, 8, 1, p, p, 0, None) == _lib.INVALID and b'scratch' in lib.ide3d_last_error()
    assert lib.ide3d_knn_within(p, 4, p, 4, 8, None, p, p, 1 << 30, None) == _lib.INVALID and b'null' in lib.ide3d_last_error()
    assert lib.ide3d_knn_within(p, 4, p, 4, 20, p, p, p, 1 << 30, None) == _lib.INVALID and b'multiple of 8' in lib.ide3d_last_error()
    assert lib.ide3d_knn_within(p + 8, 4, p, 4, 8, p, p, p, 1 << 30, None) == _lib.INVALID and b'aligned' in lib.ide3d_last_error()
    assert lib.ide3d_knn_kth_dist_scratch_bytes(4, 4, 17) < 0 and lib.ide3d_knn_within_scratch_bytes(4, 0) < 0
