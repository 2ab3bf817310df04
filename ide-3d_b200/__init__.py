"""ide3d_b200 -- H100-native implementation of IDE-3D's volumetric-rendering hot path.

Layout (mirrors the reference's module names so its tools can import this package instead):
    csrc/                     hand-written sm_90a CUDA + the C-ABI (include/ide3d_b200.h)
    _lib.py, _plugins.py      ctypes binding, plugin-level functions (the pybind11 surface of the reference)
    torch_utils/ops/*         bias_act, upfirdn2d, filtered_lrelu, conv2d_gradfix, conv2d_resample, fma, grid_sample_gradfix
    torch_utils/custom_ops.py get_plugin()
    training/volumetric_rendering.py   the renderer free functions
    training/networks.py, training/triplane.py   backbone blocks and the TriPlaneGenerator
    dnnlib/util.py            sample_from_triplane
    dist.py                   one-process-per-GPU frame / voxel-slab sharding
    compat.py                 sys.modules aliases for the reference's scripts
The compute path is CUDA only; a missing library or a CPU tensor raises.
"""

__version__ = '0.1.0'

from . import _lib  # noqa: F401


def build(force=False, verbose=False):
    from .build import build as _build
    return _build(force=force, verbose=verbose)
