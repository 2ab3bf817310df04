#!/usr/bin/env python
"""Generate tests/golden/projector_trace.npz by running the REFERENCE's three projectors, imported unmodified, on the CPU with the
stand-in generator and feature network of oracle/projector.py.

    IDE3D_REFERENCE=/path/to/IDE-3D PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_projector_golden.py

    inversion/training/projectors/w_projector_ide3d.py             'w'
    inversion/training/projectors/w_plus_projector_ide3d.py        'w_plus'
    inversion/training/projectors/w_projector_ide3d_join_view.py   'join_view'

The modules they import for logging and configuration are stubbed: wandb, configs (global_config on the CPU, hyperparameters),
utils.log_utils, and dnnlib, whose util.open_url returns the scripted stand-in feature network instead of reaching the network.
Recorded per projector: the returned ws and the per-step dist / loss, captured where the projector's logprint (verbose=True) formats
them (Tensor.__format__ for dist, Tensor.__float__ for loss), at full precision.  Inputs: oracle.projector.golden_inputs(), the
stand-in generator's seed, torch.manual_seed(TORCH_SEED) before each run, and the projector keyword arguments below.
tests/test_projector.py replays the trace against ide3d_b200.projector.project.
"""

import contextlib
import importlib.util
import io
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

KW = dict(num_steps=15, w_avg_samples=64, initial_learning_rate=0.01, initial_noise_factor=0.05, lr_rampdown_length=0.25,
          lr_rampup_length=0.05, noise_ramp_length=0.75, regularize_noise_weight=1e5)
TORCH_SEED = 1234
PROJECTORS = {'w': 'w_projector_ide3d.py', 'w_plus': 'w_plus_projector_ide3d.py', 'join_view': 'w_projector_ide3d_join_view.py'}


def _stub_modules(features_bytes):
    wandb = types.ModuleType('wandb')
    wandb.log = lambda *a, **k: None
    configs = types.ModuleType('configs')
    configs.global_config = types.SimpleNamespace(device='cpu', training_step=1, image_rec_result_log_snapshot=100)
    configs.hyperparameters = types.SimpleNamespace(first_inv_lr=5e-3)
    utils = types.ModuleType('utils')
    log_utils = types.ModuleType('utils.log_utils')
    log_utils.log_image_from_w = lambda *a, **k: None
    utils.log_utils = log_utils
    dnnlib = types.ModuleType('dnnlib')
    dnnlib.util = types.SimpleNamespace(open_url=lambda url, *a, **k: contextlib.nullcontext(io.BytesIO(features_bytes)))
    return {'wandb': wandb, 'configs': configs, 'configs.global_config': configs.global_config,
            'configs.hyperparameters': configs.hyperparameters, 'utils': utils, 'utils.log_utils': log_utils, 'dnnlib': dnnlib}


def _load(path, name):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def run_reference(ref_root):
    from oracle import projector as op
    label, target = op.golden_inputs()
    stubs = _stub_modules(op.standin_features_bytes())
    saved = {k: sys.modules.get(k) for k in stubs}
    sys.modules.update(stubs)
    out = dict(label=label.numpy(), target=target.numpy(), torch_seed=np.int64(TORCH_SEED), generator_seed=np.int64(5),
               w_avg_seed=np.int64(123), kwargs=np.array(repr(KW)))
    try:
        for key, fname in PROJECTORS.items():
            mod = _load(os.path.join(ref_root, 'inversion', 'training', 'projectors', fname), f'_ref_projector_{key}')
            G = op.StandInGenerator()
            record = []
            fmt, flt = torch.Tensor.__format__, torch.Tensor.__float__

            def rec_format(self, spec):
                record.append(('dist', self.item()))
                return fmt(self, spec)

            def rec_float(self):
                record.append(('loss', flt(self)))
                return flt(self)

            torch.manual_seed(TORCH_SEED)
            torch.Tensor.__format__, torch.Tensor.__float__ = rec_format, rec_float
            try:
                with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
                    ws = mod.project(G, label, target, device=torch.device('cpu'), verbose=True, w_name='golden', **KW)
            finally:
                torch.Tensor.__format__, torch.Tensor.__float__ = fmt, flt
            dist = [v for k, v in record if k == 'dist']
            loss = [v for k, v in record if k == 'loss']
            assert len(dist) == len(loss) == KW['num_steps'], (len(dist), len(loss))
            out[f'{key}_ws'] = ws.detach().numpy()
            out[f'{key}_dist'] = np.array(dist, np.float64)
            out[f'{key}_loss'] = np.array(loss, np.float64)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    return out


if __name__ == '__main__':
    ref = os.environ.get('IDE3D_REFERENCE')
    if not ref:
        sys.exit('set IDE3D_REFERENCE to the reference checkout')
    out = run_reference(ref)
    np.savez_compressed(os.path.join(HERE, 'projector_trace.npz'), **out)
    for k in PROJECTORS:
        print(k, out[f'{k}_ws'].shape, 'dist', out[f'{k}_dist'][[0, -1]], 'loss', out[f'{k}_loss'][[0, -1]])
