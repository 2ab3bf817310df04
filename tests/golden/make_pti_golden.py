#!/usr/bin/env python
"""Generate tests/golden/pti_trace.npz by running the REFERENCE's pivotal-tuning coach, imported unmodified, on the CPU with the
stand-in generator, VGG16 features and LPIPS weights of oracle/projector.py and oracle/pti.py.

    IDE3D_REFERENCE=/path/to/IDE-3D PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_pti_golden.py

    inversion/training/coaches/single_id_coach.py   SingleIDCoach.train: projection, then the tuning loop
    inversion/training/coaches/base_coach.py        calc_inversions, calc_loss, forward, configure_optimizers, get_label
    inversion/training/projectors/*.py              the three ide3d projectors
    inversion/criteria/l2_loss.py                   the l2 term
    inversion/criteria/lpips/                       the LPIPS class (what `from lpips import LPIPS` resolves to here)

Stubbed: wandb; configs (global_config on the CPU, paths under a temporary directory, hyperparameters with small first_inv_steps and
max_pti_steps); models.e4e.psp; utils.log_utils; utils.models_utils (load_old_G -> oracle.projector.StandInGenerator); dnnlib
(open_url -> the scripted stand-in VGG16); and lpips.LPIPS -> the vendored inversion/criteria/lpips class, whose torchvision AlexNet is
oracle.pti.standin_alexnet(), whose `.to("cuda")` stays on the CPU, and whose get_state_dict reads the stand-in lin weights from
pretrained_models/alex.pth in the working directory (written there in the lpips package's key format).

Runs: the coach's 'ide3d', 'ide3d_plus' and 'ide3d_join_view' projector types, and 'ide3d' again with an LPIPS threshold the first
run's trace crosses.  Recorded per run: the pivot, the label after the coach's OpenCV -> OpenGL flip, per evaluated step the l2 / lpips
/ loss of every BaseCoach.calc_loss call (one per view), the number of optimiser steps, and the tuned generator's state_dict.
tests/test_pti.py replays the trace through ide3d_b200.pti.run.
"""

import contextlib
import importlib
import io
import json
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

FIRST_INV_STEPS = 8
MAX_PTI_STEPS = 10
TORCH_SEED = 4321
IMAGE_NAME = 'img00000'
RUNS = {'w': ('ide3d', None), 'w_plus': ('ide3d_plus', None), 'join_view': ('ide3d_join_view', None), 'early_stop': ('ide3d', 'cross')}
OPENCV_FLIP = [1, 2, 5, 6, 9, 10]                      # base_coach.py:221


def _stubs(work, features_bytes, threshold):
    from oracle import projector as op
    wandb = types.ModuleType('wandb')
    wandb.log = lambda *a, **k: None
    configs = types.ModuleType('configs')
    configs.global_config = types.SimpleNamespace(device='cpu', training_step=1, image_rec_result_log_snapshot=100, run_name='golden',
                                                  pivotal_training_steps=0)
    configs.paths_config = types.SimpleNamespace(embedding_base_dir=os.path.join(work, 'embeddings'), input_data_id='golden',
                                                 pti_results_keyword='PTI', e4e_results_keyword='e4e',
                                                 checkpoints_dir=os.path.join(work, 'checkpoints'), e4e='')
    configs.hyperparameters = types.SimpleNamespace(
        lpips_type='alex', first_inv_type='w', optim_type='adam', latent_ball_num_of_samples=1, locality_regularization_interval=1,
        use_locality_regularization=False, regulizer_l2_lambda=0.1, regulizer_lpips_lambda=0.1, regulizer_alpha=30, pt_l2_lambda=1,
        pt_lpips_lambda=1, LPIPS_value_threshold=threshold, max_pti_steps=MAX_PTI_STEPS, first_inv_steps=FIRST_INV_STEPS,
        max_images_to_invert=30000, pti_learning_rate=3e-4, first_inv_lr=5e-3, train_batch_size=1, use_last_w_pivots=False)
    utils = types.ModuleType('utils')
    log_utils = types.ModuleType('utils.log_utils')
    log_utils.log_image_from_w = log_utils.log_images_from_w = lambda *a, **k: None
    models_utils = types.ModuleType('utils.models_utils')

    def toogle_grad(model, flag=True):
        for p in model.parameters():
            p.requires_grad = flag
    models_utils.toogle_grad = toogle_grad
    models_utils.load_old_G = lambda: op.StandInGenerator().eval().float()
    utils.log_utils, utils.models_utils = log_utils, models_utils
    models = types.ModuleType('models')
    e4e = types.ModuleType('models.e4e')
    psp = types.ModuleType('models.e4e.psp')
    psp.pSp = None
    dnnlib = types.ModuleType('dnnlib')
    dnnlib.util = types.SimpleNamespace(open_url=lambda url, *a, **k: contextlib.nullcontext(io.BytesIO(features_bytes)))
    lpips = types.ModuleType('lpips')
    lpips.LPIPS = _vendored_lpips
    return {'wandb': wandb, 'configs': configs, 'configs.global_config': configs.global_config,
            'configs.paths_config': configs.paths_config, 'configs.hyperparameters': configs.hyperparameters, 'utils': utils,
            'utils.log_utils': log_utils, 'utils.models_utils': models_utils, 'models': models, 'models.e4e': e4e,
            'models.e4e.psp': psp, 'dnnlib': dnnlib, 'lpips': lpips}


def _vendored_lpips(net='alex', **kw):
    """`LPIPS(net=...)` of the pip package, answered by the reference's vendored class with the stand-in weights."""
    from oracle import pti as opti
    networks = importlib.import_module('inversion.criteria.lpips.networks')
    vendored = importlib.import_module('inversion.criteria.lpips.lpips')
    networks.models = types.SimpleNamespace(alexnet=lambda *a, **k: opti.standin_alexnet())
    to = torch.nn.Module.to
    torch.nn.Module.to = lambda self, *a, **k: self if a and a[0] == 'cuda' else to(self, *a, **k)
    try:
        return vendored.LPIPS(net_type=net)
    finally:
        torch.nn.Module.to = to


def run_reference(ref_root):
    from oracle import projector as op
    from oracle import pti as opti
    label, target = opti.golden_inputs()
    opencv = label.clone()
    opencv[:, OPENCV_FLIP] *= -1
    out = dict(label=label.numpy(), target=target.numpy(), torch_seed=np.int64(TORCH_SEED), generator_seed=np.int64(5),
               first_inv_steps=np.int64(FIRST_INV_STEPS), max_pti_steps=np.int64(MAX_PTI_STEPS), w_avg_samples=np.int64(600))
    sys.path[:0] = [os.path.join(ref_root, 'inversion'), ref_root]
    cwd = os.getcwd()
    threshold_cross = None
    with tempfile.TemporaryDirectory() as work:
        os.makedirs(os.path.join(work, 'pretrained_models'))
        torch.save(opti.lin_state_dict(), os.path.join(work, 'pretrained_models', 'alex.pth'))
        labels_path = os.path.join(work, 'labels.json')
        with open(labels_path, 'w') as f:
            json.dump({'labels': [[f'{IMAGE_NAME[3:8]}/{IMAGE_NAME}.png', opencv[0].tolist()]]}, f)
        os.chdir(work)
        try:
            for key, (ptype, thr) in RUNS.items():
                threshold = 0.0 if thr is None else threshold_cross
                stubs = _stubs(work, op.standin_features_bytes(), threshold)
                saved = {k: sys.modules.get(k) for k in stubs}
                sys.modules.update(stubs)
                try:
                    for name in [m for m in sys.modules if m == 'training' or m.startswith(('training.', 'criteria'))]:
                        del sys.modules[name]
                    base = importlib.import_module('training.coaches.base_coach')
                    single = importlib.import_module('training.coaches.single_id_coach')
                    record, steps = [], [0]
                    calc_loss, configure = base.BaseCoach.calc_loss, base.BaseCoach.configure_optimizers

                    def rec_calc_loss(self, *a, **k):
                        loss, l2, lp = calc_loss(self, *a, **k)
                        record.append((l2.item(), lp.item(), loss.item()))
                        return loss, l2, lp

                    def counted_optimizer(self):
                        opt = configure(self)
                        step = opt.step
                        opt.step = lambda *a, **k: (steps.__setitem__(0, steps[0] + 1), step(*a, **k))[1]
                        return opt

                    base.BaseCoach.calc_loss, base.BaseCoach.configure_optimizers = rec_calc_loss, counted_optimizer
                    coach = single.SingleIDCoach([([IMAGE_NAME], target)], use_wandb=False, image_name=IMAGE_NAME,
                                                 label_path=labels_path, projector_type=ptype)
                    steps[0] = 0
                    torch.manual_seed(TORCH_SEED)
                    with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
                        coach.train()
                    base.BaseCoach.calc_loss, base.BaseCoach.configure_optimizers = calc_loss, configure
                    emb = os.path.join(work, 'embeddings', 'golden', 'PTI', IMAGE_NAME)
                    views = 2 if ptype == 'ide3d_join_view' else 1
                    rec = np.array(record, np.float64).reshape(-1, views, 3)
                    out[f'{key}_pivot'] = torch.load(os.path.join(emb, '0.pt')).detach().numpy()
                    out[f'{key}_label'] = torch.load(os.path.join(emb, '0_label.pt')).numpy()
                    out[f'{key}_l2'], out[f'{key}_lpips'], out[f'{key}_loss'] = rec[..., 0], rec[..., 1], rec[..., 2]
                    out[f'{key}_updates'] = np.int64(steps[0])
                    out[f'{key}_threshold'] = np.float64(threshold)
                    for name, v in coach.G.state_dict().items():
                        out[f'{key}_state.{name}'] = v.detach().numpy()
                    if key == 'w':                     # a threshold between the lpips of steps 3 and 4 of this run
                        lp = rec[:, 0, 1]
                        assert lp[4] < lp[3], lp
                        threshold_cross = float((lp[3] + lp[4]) / 2)
                finally:
                    for k, v in saved.items():
                        if v is None:
                            sys.modules.pop(k, None)
                        else:
                            sys.modules[k] = v
        finally:
            os.chdir(cwd)
    return out


if __name__ == '__main__':
    ref = os.environ.get('IDE3D_REFERENCE')
    if not ref:
        sys.exit('set IDE3D_REFERENCE to the reference checkout')
    out = run_reference(ref)
    np.savez_compressed(os.path.join(HERE, 'pti_trace.npz'), **out)
    for k in RUNS:
        print(k, 'pivot', out[f'{k}_pivot'].shape, 'updates', out[f'{k}_updates'], 'lpips', out[f'{k}_lpips'][[0, -1]].ravel(),
              'loss', out[f'{k}_loss'][[0, -1]].ravel())
