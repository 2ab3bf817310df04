"""The slice of the reference's `dnnlib` the hot path uses: EasyDict, the cache directory and the network helpers of dnnlib/util.py."""

from . import util
from .util import EasyDict, make_cache_dir_path

__all__ = ['util', 'EasyDict', 'make_cache_dir_path']
