"""Utilities of the quality metrics, with the reference's names and calls (metrics/metric_utils.py).

Where this differs from the reference:
  - Detectors are read from local files only (get_feature_detector): a path, or the reference's URL resolved to the file its
    download cache would hold.  Nothing is fetched from the network.
  - FeatureStats sums the mean and covariance in float64 on the device and keeps captured features on the device in item order.
    Its save / load format is the reference's (the same __dict__ keys, numpy arrays), so cache files go both ways.
  - Generated item i draws its z and its label index from np.random.RandomState([seed, i]) (item_draws); rank r of W takes the
    items i = r (mod W).  Features are gathered in item order and the mean / covariance sums are all-reduced once, so every
    world size and batch size evaluates the same images.  The reference draws unseeded, per rank.
  - G_kwargs without cond_render means cond_render=False (the reference raises AttributeError for the G_kwargs={} its
    calc_metrics.py passes); cond_render=True raises NotImplementedError, since no dataset here renders conditioning images.
"""

import copy
import glob
import hashlib
import os
import pickle
import re
import time
import urllib.parse
import uuid

import numpy as np
import torch

from .. import dnnlib


class MetricOptions:
    def __init__(self, G=None, G_kwargs={}, dataset_kwargs={}, num_gpus=1, rank=0, device=None, progress=None, cache=True, seed=0):
        assert 0 <= rank < num_gpus
        self.G = G
        self.G_kwargs = dnnlib.EasyDict(G_kwargs)
        self.dataset_kwargs = dnnlib.EasyDict(dataset_kwargs)
        self.num_gpus = num_gpus
        self.rank = rank
        self.device = device if device is not None else torch.device('cuda', rank)
        self.progress = progress.sub() if progress is not None and rank == 0 else ProgressMonitor()
        self.cache = cache
        self.seed = seed


# ---------------------------------------------------------------------------------------------------------------- detectors

_feature_detector_cache = dict()


def get_feature_detector_name(url):
    return os.path.splitext(url.split('/')[-1])[0]


def detector_path(url):
    """The local file behind `url`: a path as given, a file:// URL's path, or for any other URL the file dnnlib.util.open_url of the
    reference leaves in its download cache, make_cache_dir_path('downloads')/<md5(url)>_<name>."""
    if not re.match('^[a-z]+://', url):
        return url
    if url.startswith('file://'):
        path = urllib.parse.urlparse(url).path
        return path[1:] if re.match(r'^/[a-zA-Z]:', path) else path
    cache_dir = dnnlib.util.make_cache_dir_path('downloads')
    url_md5 = hashlib.md5(url.encode('utf-8')).hexdigest()
    found = glob.glob(os.path.join(cache_dir, url_md5 + '_*'))
    if len(found) == 1:
        return found[0]
    return os.path.join(cache_dir, url_md5 + '_' + re.sub(r'[^0-9a-zA-Z-._]', '_', url.split('/')[-1]))


def get_feature_detector(url, device=torch.device('cpu'), num_gpus=1, rank=0, verbose=False):
    assert 0 <= rank < num_gpus
    key = (url, device)
    if key not in _feature_detector_cache:
        path = detector_path(url)
        if not os.path.isfile(path):
            raise FileNotFoundError(f'feature detector {url} not found: expected the file {path} (this package never downloads; '
                                    f'copy the reference\'s detector pickle there, or pass a local path)')
        with open(path, 'rb') as f:
            _feature_detector_cache[key] = pickle.load(f).to(device)
    return _feature_detector_cache[key]


# ---------------------------------------------------------------------------------------------------------------- draws

def item_draws(seed, i, z_dim, num_labels):
    """z [z_dim] float32 and the label index (None without labels) of generated item i: functions of (seed, i) only."""
    rs = np.random.RandomState([seed, i])
    z = rs.standard_normal(z_dim).astype(np.float32)
    return z, (int(rs.randint(num_labels)) if num_labels else None)


def _items(n, num_gpus, rank):
    return list(range(rank, n, num_gpus))


# ---------------------------------------------------------------------------------------------------------------- FeatureStats

class FeatureStats:
    def __init__(self, capture_all=False, capture_mean_cov=False, max_items=None):
        self.capture_all = capture_all
        self.capture_mean_cov = capture_mean_cov
        self.max_items = max_items
        self.num_items = 0
        self.num_features = None
        self.all_features = None       # list of [n, F] float32 tensors, in item order
        self.raw_mean = None           # [F] float64 tensor: sum of x
        self.raw_cov = None            # [F, F] float64 tensor: sum of x x^T

    def set_num_features(self, num_features, device=None):
        if self.num_features is not None:
            assert num_features == self.num_features
        else:
            self.num_features = num_features
            self.all_features = []
            self.raw_mean = torch.zeros([num_features], dtype=torch.float64, device=device)
            self.raw_cov = torch.zeros([num_features, num_features], dtype=torch.float64, device=device)

    def is_full(self):
        return (self.max_items is not None) and (self.num_items >= self.max_items)

    def append(self, x):
        self.append_torch(torch.as_tensor(np.asarray(x, dtype=np.float32)))

    def append_torch(self, x, num_gpus=1, rank=0):
        """Local batch of features.  Multi-rank runs gather once at the end (gather()), not per batch."""
        assert isinstance(x, torch.Tensor) and x.ndim == 2
        assert 0 <= rank < num_gpus
        x = x.to(torch.float32)
        if (self.max_items is not None) and (self.num_items + x.shape[0] > self.max_items):
            if self.num_items >= self.max_items:
                return
            x = x[:self.max_items - self.num_items]
        self.set_num_features(x.shape[1], x.device)
        self.num_items += x.shape[0]
        if self.capture_all:
            self.all_features.append(x)
        if self.capture_mean_cov:
            x64 = x.to(torch.float64)
            self.raw_mean += x64.sum(0)
            self.raw_cov.addmm_(x64.t(), x64)

    def gather(self, num_gpus, num_items, device):
        """Combine the ranks' stats of items i = rank (mod num_gpus): features interleaved back into item order, sums all-reduced.
        A rank that received no item (num_items < num_gpus) takes the feature count from the others and contributes zeros."""
        if num_gpus == 1:
            return self
        dev = torch.device(device)
        nf = torch.tensor([self.num_features or 0], dtype=torch.int64, device=dev)
        torch.distributed.all_reduce(nf, op=torch.distributed.ReduceOp.MAX)
        self.set_num_features(int(nf), dev)
        if self.capture_all:
            mine = torch.cat(self.all_features) if self.all_features else torch.zeros(0, self.num_features, device=dev)
            per = (num_items - 1) // num_gpus + 1
            pad = torch.zeros(per, self.num_features, dtype=torch.float32, device=dev)
            pad[:mine.shape[0]] = mine
            parts = [torch.empty_like(pad) for _ in range(num_gpus)]
            torch.distributed.all_gather(parts, pad)
            self.all_features = [torch.stack(parts, 1).flatten(0, 1)[:num_items]]
        if self.capture_mean_cov:
            torch.distributed.all_reduce(self.raw_mean)
            torch.distributed.all_reduce(self.raw_cov)
        self.num_items = num_items
        return self

    def get_all(self):
        return self.get_all_torch().cpu().numpy()

    def get_all_torch(self):
        assert self.capture_all
        return torch.cat(self.all_features, dim=0)

    def get_mean_cov(self):
        assert self.capture_mean_cov
        mean = self.raw_mean / self.num_items
        cov = self.raw_cov / self.num_items
        cov = cov - torch.outer(mean, mean)
        return mean.cpu().numpy(), cov.cpu().numpy()

    def save(self, pkl_file):
        """The reference's pickle: its FeatureStats.__dict__ with numpy arrays."""
        d = dict(capture_all=self.capture_all, capture_mean_cov=self.capture_mean_cov, max_items=self.max_items, num_items=self.num_items,
                 num_features=self.num_features,
                 all_features=None if self.all_features is None else [t.cpu().numpy() for t in self.all_features],
                 raw_mean=None if self.raw_mean is None else self.raw_mean.cpu().numpy(),
                 raw_cov=None if self.raw_cov is None else self.raw_cov.cpu().numpy())
        with open(pkl_file, 'wb') as f:
            pickle.dump(d, f)

    @staticmethod
    def load(pkl_file, device=None):
        with open(pkl_file, 'rb') as f:
            s = dnnlib.EasyDict(pickle.load(f))
        obj = FeatureStats(capture_all=s.capture_all, capture_mean_cov=s.capture_mean_cov, max_items=s.max_items)
        obj.num_items, obj.num_features = s.num_items, s.num_features
        if s.all_features is not None:
            obj.all_features = [torch.as_tensor(np.asarray(a, dtype=np.float32), device=device) for a in s.all_features]
        if s.raw_mean is not None:
            obj.raw_mean = torch.as_tensor(s.raw_mean, dtype=torch.float64, device=device)
            obj.raw_cov = torch.as_tensor(s.raw_cov, dtype=torch.float64, device=device)
        return obj


# ---------------------------------------------------------------------------------------------------------------- progress

class ProgressMonitor:
    def __init__(self, tag=None, num_items=None, flush_interval=1000, verbose=False, progress_fn=None, pfn_lo=0, pfn_hi=1000, pfn_total=1000):
        self.tag = tag
        self.num_items = num_items
        self.verbose = verbose
        self.flush_interval = flush_interval
        self.progress_fn = progress_fn
        self.pfn_lo = pfn_lo
        self.pfn_hi = pfn_hi
        self.pfn_total = pfn_total
        self.start_time = time.time()
        self.batch_time = self.start_time
        self.batch_items = 0
        if self.progress_fn is not None:
            self.progress_fn(self.pfn_lo, self.pfn_total)

    def update(self, cur_items):
        assert (self.num_items is None) or (cur_items <= self.num_items)
        if (cur_items < self.batch_items + self.flush_interval) and (self.num_items is None or cur_items < self.num_items):
            return
        cur_time = time.time()
        total_time = cur_time - self.start_time
        time_per_item = (cur_time - self.batch_time) / max(cur_items - self.batch_items, 1)
        if (self.verbose) and (self.tag is not None):
            print(f'{self.tag:<19s} items {cur_items:<7d} time {dnnlib.util.format_time(total_time):<12s} ms/item {time_per_item * 1e3:.2f}')
        self.batch_time = cur_time
        self.batch_items = cur_items

        if (self.progress_fn is not None) and (self.num_items is not None):
            self.progress_fn(self.pfn_lo + (self.pfn_hi - self.pfn_lo) * (cur_items / self.num_items), self.pfn_total)

    def sub(self, tag=None, num_items=None, flush_interval=1000, rel_lo=0, rel_hi=1):
        return ProgressMonitor(
            tag=tag,
            num_items=num_items,
            flush_interval=flush_interval,
            verbose=self.verbose,
            progress_fn=self.progress_fn,
            pfn_lo=self.pfn_lo + (self.pfn_hi - self.pfn_lo) * rel_lo,
            pfn_hi=self.pfn_lo + (self.pfn_hi - self.pfn_lo) * rel_hi,
            pfn_total=self.pfn_total,
        )


# ---------------------------------------------------------------------------------------------------------------- feature loops

def _broadcast_flag(flag, opts):
    if opts.num_gpus > 1:
        flag = torch.as_tensor(flag, dtype=torch.float32, device=opts.device)
        torch.distributed.broadcast(tensor=flag, src=0)
        flag = (float(flag.cpu()) != 0)
    return flag


def compute_feature_stats_for_dataset(opts, detector_url, detector_kwargs, rel_lo=0, rel_hi=1, batch_size=64, data_loader_kwargs=None, max_items=None, **stats_kwargs):
    dataset = dnnlib.util.construct_class_by_name(**opts.dataset_kwargs)
    if data_loader_kwargs is None:
        data_loader_kwargs = dict(pin_memory=opts.device.type == 'cuda', num_workers=3, prefetch_factor=2)

    # Cache file: the reference's name (its md5 tag over the same arguments) and format.
    cache_file = None
    if opts.cache:
        args = dict(dataset_kwargs=opts.dataset_kwargs, detector_url=detector_url, detector_kwargs=detector_kwargs, stats_kwargs=stats_kwargs)
        md5 = hashlib.md5(repr(sorted(args.items())).encode('utf-8'))
        cache_tag = f'{dataset.name}-{get_feature_detector_name(detector_url)}-{md5.hexdigest()}'
        cache_file = dnnlib.make_cache_dir_path('gan-metrics', cache_tag + '.pkl')
        if _broadcast_flag(os.path.isfile(cache_file) if opts.rank == 0 else False, opts):
            return FeatureStats.load(cache_file, device=opts.device)

    num_items = len(dataset)
    if max_items is not None:
        num_items = min(num_items, max_items)
    stats = FeatureStats(**stats_kwargs)
    progress = opts.progress.sub(tag='dataset features', num_items=num_items, rel_lo=rel_lo, rel_hi=rel_hi)
    detector = get_feature_detector(url=detector_url, device=opts.device, num_gpus=opts.num_gpus, rank=opts.rank, verbose=progress.verbose)

    item_subset = _items(num_items, opts.num_gpus, opts.rank)
    for images, _labels in torch.utils.data.DataLoader(dataset=dataset, sampler=item_subset, batch_size=batch_size, **data_loader_kwargs):
        if images.shape[1] == 1:
            images = images.repeat([1, 3, 1, 1])
        stats.append_torch(detector(images.to(opts.device), **detector_kwargs))
        progress.update(min(stats.num_items * opts.num_gpus, num_items))
    stats.gather(opts.num_gpus, num_items, opts.device)
    stats.max_items = num_items

    if cache_file is not None and opts.rank == 0:
        os.makedirs(os.path.dirname(cache_file), exist_ok=True)
        temp_file = cache_file + '.' + uuid.uuid4().hex
        stats.save(temp_file)
        os.replace(temp_file, cache_file)  # atomic
    return stats


def compute_feature_stats_for_generator(opts, detector_url, detector_kwargs, rel_lo=0, rel_hi=1, batch_size=64, batch_gen=None, **stats_kwargs):
    if batch_gen is None:
        batch_gen = min(batch_size, 4)
    assert batch_size % batch_gen == 0
    G_kwargs = dnnlib.EasyDict(opts.G_kwargs)
    if G_kwargs.pop('cond_render', False):
        raise NotImplementedError('cond_render=True needs dataset renders (get_render), which no dataset here provides')

    G = copy.deepcopy(opts.G).eval().requires_grad_(False).to(opts.device)
    dataset = dnnlib.util.construct_class_by_name(**opts.dataset_kwargs) if G.c_dim != 0 else None
    num_labels = len(dataset) if dataset is not None else 0

    num_items = stats_kwargs.get('max_items')
    assert num_items is not None
    stats = FeatureStats(**dict(stats_kwargs, max_items=None))
    progress = opts.progress.sub(tag='generator features', num_items=num_items, rel_lo=rel_lo, rel_hi=rel_hi)
    detector = get_feature_detector(url=detector_url, device=opts.device, num_gpus=opts.num_gpus, rank=opts.rank, verbose=progress.verbose)

    items = _items(num_items, opts.num_gpus, opts.rank)
    for b0 in range(0, len(items), batch_size):
        images = []
        for g0 in range(b0, min(b0 + batch_size, len(items)), batch_gen):
            draws = [item_draws(opts.seed, i, G.z_dim, num_labels) for i in items[g0:g0 + batch_gen]]
            z = torch.from_numpy(np.stack([d[0] for d in draws])).to(opts.device)
            if dataset is not None:
                c = torch.from_numpy(np.stack([dataset.get_label(d[1]) for d in draws])).to(opts.device)
            else:
                c = torch.zeros([len(draws), G.c_dim], device=opts.device)
            img = G(z=z, c=c, **G_kwargs)
            img = (img * 127.5 + 128).clamp(0, 255).to(torch.uint8)
            images.append(img)
        images = torch.cat(images)
        if images.shape[1] == 1:
            images = images.repeat([1, 3, 1, 1])
        stats.append_torch(detector(images, **detector_kwargs))
        progress.update(min(stats.num_items * opts.num_gpus, num_items))
    stats.gather(opts.num_gpus, num_items, opts.device)
    stats.max_items = num_items
    return stats
