"""Helpers of the reference's dnnlib/util.py: EasyDict, the cache directory (:124-139), format_time (:145), construct_class_by_name
(:307) and the network helpers (:561-617) on the sm_90a gather kernel.

    sample_from_triplane(coordinates [N,P,3], grid [N,96,H,W]) -> [N*P, 32]   (:580-599)
    sample_from_2dgrid(coordinates [N,P,2], grid [N,C,H,W])    -> [N*P, C]     (:603-617)
The tri-plane version is one launch of ide3d_sample_triplane (bilinear / zeros / align_corners=False, planes
(x,y), (y,z), (x,z) summed); the 2-D helper keeps torch's grid_sample because nothing on the hot path calls it.
"""

import ctypes as C
import importlib
import os
import tempfile

import numpy as np
import torch

from .. import _lib as L


class EasyDict(dict):
    """dict with attribute access (dnnlib/util.py:41-57)."""

    def __getattr__(self, name):
        try:
            return self[name]
        except KeyError:
            raise AttributeError(name)

    def __setattr__(self, name, value):
        self[name] = value

    def __delattr__(self, name):
        del self[name]


_dnnlib_cache_dir = None


def set_cache_dir(path):
    global _dnnlib_cache_dir
    _dnnlib_cache_dir = path


def make_cache_dir_path(*paths):
    """set_cache_dir's path, else $DNNLIB_CACHE_DIR, else ~/.cache/dnnlib (HOME, then USERPROFILE), else <tmp>/.cache/dnnlib."""
    if _dnnlib_cache_dir is not None:
        return os.path.join(_dnnlib_cache_dir, *paths)
    if 'DNNLIB_CACHE_DIR' in os.environ:
        return os.path.join(os.environ['DNNLIB_CACHE_DIR'], *paths)
    if 'HOME' in os.environ:
        return os.path.join(os.environ['HOME'], '.cache', 'dnnlib', *paths)
    if 'USERPROFILE' in os.environ:
        return os.path.join(os.environ['USERPROFILE'], '.cache', 'dnnlib', *paths)
    return os.path.join(tempfile.gettempdir(), '.cache', 'dnnlib', *paths)


def format_time(seconds):
    s = int(np.rint(seconds))
    if s < 60:
        return '{0}s'.format(s)
    elif s < 60 * 60:
        return '{0}m {1:02}s'.format(s // 60, s % 60)
    elif s < 24 * 60 * 60:
        return '{0}h {1:02}m {2:02}s'.format(s // (60 * 60), (s // 60) % 60, s % 60)
    return '{0}d {1:02}h {2:02}m'.format(s // (24 * 60 * 60), (s // (60 * 60)) % 24, (s // 60) % 60)


def construct_class_by_name(*args, class_name=None, **kwargs):
    """Import `module.Class` from its dotted name and construct it (the reference's names resolve after compat.install())."""
    module, name = class_name.rsplit('.', 1)
    return getattr(importlib.import_module(module), name)(*args, **kwargs)


def sample_from_triplane(coordinates, grid):
    L.require_cuda(coordinates, grid)
    L.forbid_grad('sample_from_triplane', coordinates, grid)
    n, p, _ = coordinates.shape
    if grid.shape[0] != n:
        grid = grid.expand(n, -1, -1, -1)
    g = grid if grid.dtype == torch.float32 else grid.float()
    if g.stride(1) != 1:             # the gather wants texel-contiguous channels; convert once
        from ..training.triplane import TriPlaneRenderer
        g = TriPlaneRenderer.as_planes(g.contiguous())
    co = coordinates.to(torch.float32).contiguous()
    out = torch.empty([n * p, 32], dtype=torch.float32, device=g.device)
    view = L.triplane_view(g)
    L.check(L.get_lib().ide3d_sample_triplane(C.byref(view), L.ptr(co), p, L.ptr(out), L.stream_ptr(g.device)))
    return out


def sample_from_2dgrid(coordinates, grid):
    batch_size = grid.shape[0]
    s = torch.nn.functional.grid_sample(grid, coordinates.reshape(batch_size, -1, 1, 2), mode='bilinear',
                                        padding_mode='zeros', align_corners=False)
    n, c, h, w = s.shape
    return s.permute(0, 3, 2, 1).reshape(n * h * w, c)
