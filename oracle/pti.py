"""Oracle (test infrastructure): the stand-in LPIPS network of pivotal tuning and the CPU route of ide3d_b200.pti.

    standin_alexnet()       torchvision alexnet(weights=None) under a fixed torch seed: the trunk (on the stand-in generator's 32^2
                            images its feature maps are 7^2, 3^2, 1^2, 1^2, 1^2)
    standin_lin()           five seeded non-negative weight vectors in the shape of the lpips package's alex.pth lin layers
    standin_lpips()         ide3d_b200.torch_utils.ops.lpips.LPIPS over the two
    cpu_pti_ops()           inside the context, lpips_head (the sm_90a kernels) is lpips_head_torch, and the projector's kernels are
                            the torch restatements of oracle.projector, so pti.run / pti.tune run on the CPU

tests/golden/make_pti_golden.py runs the reference's coach with these weights inside its vendored LPIPS class; tests/test_pti.py
replays the trace through ide3d_b200.pti.
"""

import contextlib

import numpy as np
import torch

from . import projector as oproj

TRUNK_SEED = 21
LIN_SEED = 22
CHANNELS = (64, 192, 384, 256, 256)


def standin_alexnet():
    """torchvision's AlexNet with its default random initialisation drawn under torch.manual_seed(TRUNK_SEED); the caller's RNG state
    is restored."""
    import torchvision
    state = torch.random.get_rng_state()
    torch.manual_seed(TRUNK_SEED)
    try:
        return torchvision.models.alexnet(weights=None).eval()
    finally:
        torch.random.set_rng_state(state)


def standin_lin():
    rs = np.random.RandomState(LIN_SEED)
    return [torch.from_numpy(rs.rand(c).astype(np.float32) / c * 8) for c in CHANNELS]


def lin_state_dict():
    """standin_lin() under the keys of the lpips package's weights/v0.1/alex.pth."""
    return {f'lin{k}.model.1.weight': w.reshape(1, -1, 1, 1).clone() for k, w in enumerate(standin_lin())}


def standin_lpips():
    from ide3d_b200.torch_utils.ops.lpips import LPIPS
    return LPIPS(standin_alexnet().features, standin_lin()).eval()


@contextlib.contextmanager
def cpu_pti_ops():
    from ide3d_b200.torch_utils.ops import lpips as LP
    saved = LP.lpips_head
    LP.lpips_head = LP.lpips_head_torch
    try:
        with oproj.cpu_projector_ops():
            yield
    finally:
        LP.lpips_head = saved


def golden_inputs():
    """(label [1, 25] in the OpenGL convention, target [1, 3, 32, 32] in [-1, 1]) of the trace: the projector trace's camera and image,
    the image mapped to the data loader's range."""
    label, target = oproj.golden_inputs()
    return label, (target / 127.5 - 1)[None]
