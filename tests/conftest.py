import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100; run with -m gpu)')


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason='no CUDA device')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


def load_golden(name):
    with np.load(os.path.join(GOLDEN, name + '.npz')) as z:
        return {k: z[k] for k in z.files}


def T(a, device='cpu'):
    return torch.from_numpy(np.ascontiguousarray(a)).to(device)


@pytest.fixture(scope='session')
def lib():
    from ide3d_b200 import _lib
    return _lib.get_lib()


def assert_close(a, b, atol, rtol=0.0, what=''):
    a = torch.as_tensor(a).detach().double().cpu()
    b = torch.as_tensor(b).detach().double().cpu()
    assert a.shape == b.shape, f'{what}: shape {tuple(a.shape)} vs {tuple(b.shape)}'
    err = (a - b).abs()
    bound = atol + rtol * b.abs()
    bad = err > bound
    assert not bad.any(), f'{what}: max abs err {err.max().item():.3e} (atol {atol}, rtol {rtol}), {int(bad.sum())} / {bad.numel()} out of tolerance'
