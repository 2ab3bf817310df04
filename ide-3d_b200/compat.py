"""Make the reference's own scripts import this package under the reference's module names.

    import ide3d_b200.compat as compat; compat.install()

After install(), `from training.volumetric_rendering import sample_camera_positions`, `from training.triplane
import TriPlaneGenerator`, `from torch_utils.ops import upfirdn2d`, `import dnnlib` ... resolve to the sm_90a
implementations, so gen_images.py / gen_videos.py / extract_shapes.py / viz/renderer.py run unchanged against a
generator built by `random_init_generator()`, and calc_metrics.py's subprocess_fn computes its metrics with
`metrics.metric_main` (the reference checkpoints embed their own class source and are not
available offline; see INTEGRATION.md).
"""

import importlib
import sys

_ALIASES = [
    'training', 'training.volumetric_rendering', 'training.networks', 'training.triplane',
    'torch_utils', 'torch_utils.custom_ops', 'torch_utils.misc', 'torch_utils.persistence', 'torch_utils.ops',
    'torch_utils.ops.bias_act', 'torch_utils.ops.upfirdn2d', 'torch_utils.ops.filtered_lrelu',
    'torch_utils.ops.conv2d_gradfix', 'torch_utils.ops.conv2d_resample', 'torch_utils.ops.fma',
    'torch_utils.ops.grid_sample_gradfix', 'training.dataset', 'torch_utils.training_stats',
    'metrics', 'metrics.metric_utils', 'metrics.frechet_inception_distance', 'metrics.kernel_inception_distance',
    'metrics.precision_recall', 'metrics.inception_score', 'metrics.metric_main',
]


def install(include_dnnlib=False):
    """Register sys.modules aliases.  dnnlib is aliased only on request: the reference's dnnlib has many helpers
    (open_url, seg_tools ...) the CLIs also use, so normally the real one stays importable and only
    `dnnlib.util.sample_from_triplane` is patched (patch_dnnlib())."""
    pkg = __name__.rsplit('.', 1)[0]
    names = list(_ALIASES) + (['dnnlib', 'dnnlib.util'] if include_dnnlib else [])
    for name in names:
        sys.modules[name] = importlib.import_module(f'{pkg}.{name}')
    try:                                   # extract_shapes.py:8 imports mrcfile only to write the sigma grid (:191-192)
        import mrcfile  # noqa: F401
    except ImportError:
        sys.modules['mrcfile'] = importlib.import_module(f'{pkg}.mrc')
        names.append('mrcfile')
    return names


def patch_dnnlib():
    """Swap the gather helper inside an already importable reference `dnnlib` for the CUDA one."""
    import dnnlib.util as ref_util
    from .dnnlib import util as ours
    ref_util.sample_from_triplane = ours.sample_from_triplane
    return ref_util


def random_init_generator(device='cuda', seed=0, **kwargs):
    """A TriPlaneGenerator with StyleGAN random initialisation (weights ~ N(0,1), zero biases, affine bias 1,
    zero noise strength) -- the 'random-init ide3d-ffhq-64-512' of BASELINE.json."""
    import torch
    from .training.triplane import TriPlaneGenerator
    state = torch.random.get_rng_state()
    torch.manual_seed(seed)
    try:
        g = TriPlaneGenerator(**kwargs).eval().requires_grad_(False)
    finally:
        torch.random.set_rng_state(state)
    return g.to(device)
