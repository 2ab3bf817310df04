#!/usr/bin/env python
"""Generate tests/golden/finetune_trace.npz by running the REFERENCE's encoder fine-tuning, imported read-only, on the CPU with seeded
weights and the stand-in generator.

    IDE3D_REFERENCE=/path/to/IDE-3D PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_finetune_golden.py

    apps/finetune_hybrid_encoder.py:69-213   finetune(), executed from its AST (decorators stripped; the module imports tensorboardX,
                                             the ID loss and a D:/ path at the top), 3 steps, with --target_seg and without
    inversion/BiSeNet.py, resnet.py          BiSeNet(20) with oracle.finetune.bisenet_state (weights and BatchNorm statistics)
    inversion/networks.py:1604-1665          HybridEncoder(512, 2, 8, w_dim=16) with oracle.edit.encoder_state

Stubs for what the script touches outside the computation: initFaceParsing returns the seeded BiSeNet (its weights are never loaded,
nothing is downloaded); legacy / dnnlib.util.open_url return the stand-in generator and the encoder; the code and label go through
torch.save / torch.load of temporary files and the image and mask through PNGs; pickle.dump is captured; tqdm passes through; `sum`
records the step's four loss terms; torch.device('cuda') is the CPU.  Recorded: the per-step losses, what the tuning changed in the
weights (tuned - initial) -- the stem and block 0 whole, projector_seg's first PROJ_ROWS output channels, and a per-tensor sum of the
change for all of convs_seg and projector_seg (the whole projector is 4 MB a run) --, the saved mask.png, and BiSeNet's logits
(average-pooled 16x16) for the image.  The image (oracle.edit.golden_images(1, seed=44)) and the mask (oracle.edit.golden_masks()[1])
are regenerated, not stored.
"""

import ast
import builtins
import contextlib
import io
import os
import sys
import tempfile
import types

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

STEPS = 3
WHOLE = ('convs_seg.0.', 'convs_seg.1.')
PROJ_ROWS = 16
IMAGE_SEED = 44


def _function(path, name):
    tree = ast.parse(open(path).read())
    for node in ast.walk(tree):
        if isinstance(node, ast.FunctionDef) and node.name == name:
            node.decorator_list = []
            return ast.Module([node], [])
    raise KeyError(name)


def run_reference(ref):
    from oracle import edit as oe, finetune as of
    sys.path[:0] = [ref]
    for name, attr in (('numpy.lib.arraysetops', 'isin'), ('numpy.lib.function_base', 'angle')):
        m = types.ModuleType(name)
        setattr(m, attr, getattr(np, attr))
        sys.modules.setdefault(name, m)
    import inversion.networks as rn
    from inversion.BiSeNet import BiSeNet
    from dnnlib import seg_tools
    from PIL import Image

    torch.manual_seed(0)
    net = BiSeNet(20).eval()
    net.load_state_dict(of.bisenet_state(net))
    net.requires_grad_(False)
    G = oe.standin_generator()
    image_u8 = oe.to_uint8(oe.golden_images(1, seed=IMAGE_SEED))
    image = image_u8.float() / 127.5 - 1
    rs = np.random.RandomState(45)
    code = torch.from_numpy((rs.randn(1, G.num_ws, G.w_dim) * 0.5).astype(np.float32)) + G.mapping.w_avg
    label = torch.from_numpy(np.concatenate([np.eye(4).reshape(-1) + np.r_[np.zeros(11), 2.7, np.zeros(4)],
                                             [4.2647, 0, 0.5, 0, 4.2647, 0.5, 0, 0, 1]]).astype(np.float32))[None]
    mask = oe.golden_masks()[1]
    with torch.no_grad():
        logits = net(image)[0]
    out = dict(code=code.numpy(), label=label.numpy(), bisenet_names=np.array(list(net.state_dict())),
               bisenet_logits=F.avg_pool2d(logits, 16).numpy())

    tdev = types.ModuleType('torch_cpu')
    tdev.__dict__.update(torch.__dict__)
    tdev.device = lambda *a, **k: torch.device('cpu')

    class _Bar:
        def __init__(self, it, **kw):
            self.it = it

        def __iter__(self):
            return iter(self.it)

        def set_description(self, *a, **k):
            pass

    for tag, use_seg in (('seg', True), ('parse', False)):
        torch.manual_seed(0)
        E = rn.HybridEncoder(**oe.ENCODER_ARGS)
        initial = oe.encoder_state(E)
        E.load_state_dict(initial)
        steps, dumped = [], {}

        def record_sum(terms, start=0):
            if len(terms) == 4 and all(isinstance(t, torch.Tensor) for t in terms):
                steps.append([float(t.detach()) for t in terms])
            return builtins.sum(terms, start)

        with tempfile.TemporaryDirectory() as work:
            img_path, seg_path = os.path.join(work, 'img00000001.png'), os.path.join(work, 'seg.png')
            code_path, label_path = os.path.join(work, 'code.pt'), os.path.join(work, 'label.pt')
            Image.fromarray(image_u8[0].permute(1, 2, 0).numpy()).save(img_path)
            Image.fromarray(mask.numpy()).save(seg_path)
            torch.save(code, code_path)
            torch.save(label, label_path)
            ns = dict(np=np, torch=tdev, os=os, copy=__import__('copy'), F=F, optim=torch.optim, Image=Image, glob=__import__('glob'),
                      json=__import__('json'), sum=record_sum, tqdm=_Bar,
                      conv2d_gradfix=types.SimpleNamespace(enabled=False),
                      dnnlib=types.SimpleNamespace(util=types.SimpleNamespace(open_url=lambda *a, **k: contextlib.nullcontext(None))),
                      legacy=types.SimpleNamespace(load_network_pkl=lambda f: {'G_ema': G}, load_encoder_pkl=lambda f: {'E': E}),
                      initFaceParsing=lambda **k: (net, None), face_parsing=seg_tools.face_parsing, parsing_img=seg_tools.parsing_img,
                      mask2label_np=seg_tools.mask2label_np,
                      requires_grad=lambda model, flag=True: [p.requires_grad_(flag) for p in model.parameters()],
                      pickle=types.SimpleNamespace(dump=lambda obj, f: dumped.update(obj)))
            exec(compile(_function(os.path.join(ref, 'apps', 'finetune_hybrid_encoder.py'), 'finetune'), 'finetune_hybrid_encoder.py',
                         'exec'), ns)
            with contextlib.redirect_stdout(io.StringIO()):
                ns['finetune'](target_img=img_path, target_seg=seg_path if use_seg else None, target_code=code_path,
                               target_label=label_path, outdir=work, g_ckpt='G.pkl', e_ckpt='E.pkl', local_rank=0,
                               start_from_latent_avg=True, max_steps=STEPS)
            saved_mask = np.array(Image.open(os.path.join(work, 'img00000001', 'mask.png')))
        assert len(steps) == STEPS and dumped['E'] is E
        out[f'{tag}_losses'] = np.array(steps, np.float64)                        # [steps, 4]: ws, gen_l2, entropy, cycle
        state = E.state_dict()
        names = [n for n in state if n.startswith('convs_seg.') or n.startswith('projector_seg.')]
        out[f'{tag}_names'] = np.array(names)
        delta = {n: state[n].detach().double() - initial[n].double() for n in names}
        for n in names:
            if n.startswith(WHOLE):
                out[f'{tag}_d_{n}'] = delta[n].float().numpy()
        out[f'{tag}_d_projector_rows'] = delta['projector_seg.weight'][:PROJ_ROWS].float().numpy()
        out[f'{tag}_d_sums'] = np.array([delta[n].sum().item() for n in names])
        out[f'{tag}_mask'] = saved_mask
    return out


if __name__ == '__main__':
    ref = os.environ.get('IDE3D_REFERENCE')
    if not ref:
        sys.exit('set IDE3D_REFERENCE to the reference checkout')
    out = run_reference(ref)
    np.savez_compressed(os.path.join(HERE, 'finetune_trace.npz'), **out)
    for k, v in out.items():
        if not k.startswith(('seg_d_convs', 'parse_d_convs')):
            print(f'{k:24s} {v.dtype} {v.shape}')
    print(f'{os.path.getsize(os.path.join(HERE, "finetune_trace.npz")) / 1024:.1f} KB')
