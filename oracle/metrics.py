"""Test infrastructure of the metrics: stand-in detectors, a float64 k-NN and a small FFHQ-layout dataset.

StandInDetector has the call contract of the reference's TorchScript detectors (uint8 NCHW images in; return_features -> features,
no_output_bias -> softmax probabilities): an average pool to 8 x 8 (optionally contrast-normalised) and fixed random projections.
save_detector pickles one so the loading path (pickle.load(f).to(device)) is exercised.  knn_kth_dist / knn_within are the float64 neighbour search of
precision_recall.py.  write_dataset writes PNGs, dataset_eric_orig.json and names on both sides of 140000.
"""

import json
import os
import pickle
import zipfile

import numpy as np
import PIL.Image
import torch
import torch.nn.functional as F

from . import edit as oedit


class StandInDetector(torch.nn.Module):
    def __init__(self, features=8, classes=10, seed=0, normalize=False):
        super().__init__()
        self.normalize = normalize
        rs = np.random.RandomState(seed)
        self.register_buffer('w', torch.from_numpy(rs.randn(3 * 64, features).astype(np.float32) / 64))
        self.register_buffer('w_out', torch.from_numpy(rs.randn(features, classes).astype(np.float32)))
        self.register_buffer('b_out', torch.from_numpy(rs.randn(classes).astype(np.float32)))

    def forward(self, img, return_features=False, no_output_bias=False):
        x = F.adaptive_avg_pool2d(img.to(torch.float32) / 255, 8).flatten(1)
        if self.normalize:                    # per-image contrast normalisation: real and generated features overlap, PR is not 0 / 1
            x = (x - x.mean(1, keepdim=True)) / (x.std(1, keepdim=True) + 1e-3)
        f = torch.tanh(x @ self.w.to(x.device)) * 4
        if return_features:
            return f
        logits = f @ self.w_out.to(x.device) + (0 if no_output_bias else self.b_out.to(x.device))
        return torch.softmax(logits, 1)


def save_detector(path, **kwargs):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, 'wb') as f:
        pickle.dump(StandInDetector(**kwargs), f)
    return path


class StandInMetricGenerator(torch.nn.Module):
    """oracle.edit.standin_generator() behind the G(z, c) call of the metric loops."""

    def __init__(self):
        super().__init__()
        self.g = oedit.standin_generator()
        self.z_dim, self.c_dim = self.g.z_dim, self.g.c_dim

    def forward(self, z, c, **kw):
        return self.g.synthesis(self.g.mapping(z, c), c=c)


def knn_kth_dist(rows, cols, kth):
    d = torch.cdist(rows.double().cpu(), cols.double().cpu())
    return d.kthvalue(kth, dim=1).values.float()


def knn_within(probes, manifold, radius):
    d = torch.cdist(probes.double().cpu(), manifold.double().cpu())
    return (d <= radius.double().cpu()[None]).any(1)


def write_dataset(root, n=20, extra=3, res=32, seed=0):
    """FFHQ layout: n images named 0000xxxx.png below 140000 (kept) and `extra` at 14xxxx (skipped by non_rebalance), in two
    sub-folders, with dataset_eric_orig.json camera labels (25 floats).  Returns (dir, zip)."""
    rs = np.random.RandomState(seed)
    os.makedirs(root, exist_ok=True)
    names = [f'{i // 10:05d}/img{i * 7:08d}.png' for i in range(n)] + [f'00099/img{140000 + i:08d}.png' for i in range(extra)]
    labels = []
    for name in names:
        os.makedirs(os.path.join(root, os.path.dirname(name)), exist_ok=True)
        base = rs.randint(0, 256, size=(4, 4, 3)).astype(np.uint8)
        img = PIL.Image.fromarray(base).resize((res, res), PIL.Image.BILINEAR)
        img.save(os.path.join(root, name))
        labels.append([name, [round(float(v), 6) for v in rs.randn(25)]])
    with open(os.path.join(root, 'dataset_eric_orig.json'), 'w') as f:
        json.dump({'labels': labels}, f)
    zpath = root.rstrip('/') + '.zip'
    with zipfile.ZipFile(zpath, 'w') as z:
        for name in names + ['dataset_eric_orig.json']:
            z.write(os.path.join(root, name), name)
    return root, zpath
