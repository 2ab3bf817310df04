#!/usr/bin/env python
"""Generate tests/golden/edit_trace.npz by running the REFERENCE's hybrid encoder and its three editing drivers, imported read-only, on
the CPU with the seeded weights and the stand-in generator of oracle/edit.py.

    IDE3D_REFERENCE=/path/to/IDE-3D PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_edit_golden.py

    inversion/networks.py:1604-1665         HybridEncoder(512, 2, 8, w_dim=16) with oracle.edit.encoder_state: E(img, mask2label_np*2-1)
    apps/infer_hybrid_encoder.py:43-100     test(): PNG image + PNG mask -> E + w_avg, --target_code splice, render
    Painter/run_UI.py:167-203, 290-295, 532-537   run_deep_model (inversion=True) with mask_labels / id_remap, per mask
    apps/infer_face_animation.py:91-151     run_video_animation: 2 seeds driven by 3 (image, mask, camera) frames

Painter/run_UI.py's methods and the two scripts' functions are executed from their AST (the modules import PyQt5, BiSeNet weights and a
video writer at the top) with stubs for what they touch outside the computation: a `self` holding the stand-in generator and the
reference encoder, QImage / QPixmap / cv2.resize (display only), legacy / dnnlib.util.open_url (return the stand-ins), imageio's
writer and layout_grid (record the frames instead of encoding them), face_parsing (returns the recorded mask as one_hot, the way BiSeNet's
parse arrives), utils.save_image and torch.device('cuda') (CPU).  Images are stored average-pooled 16x16 (32^2) to keep the file small;
ws are stored whole.  The encoder's weights and the images are not stored: oracle.edit.encoder_state and golden_images regenerate
them (the PNG inputs are their uint8 rounding, oracle.edit.to_uint8).
"""

import ast
import contextlib
import io
import json
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

SEEDS = [0, 1]
FRAMES = 3


def _functions(path, names):
    tree = ast.parse(open(path).read())
    out = []
    for node in ast.walk(tree):
        if isinstance(node, ast.FunctionDef) and node.name in names:
            node.decorator_list = []
            out.append(node)
    assert len(out) == len(names), (path, names, [n.name for n in out])
    return ast.Module(out, [])


def _pool(img):
    return F.avg_pool2d(img.detach().float(), 16).numpy()


def _camera(yaw, pitch):
    fwd = np.array([np.sin(yaw) * np.cos(pitch), np.sin(pitch), np.cos(yaw) * np.cos(pitch)])
    z = -fwd
    x = np.cross([0, 1, 0], z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    m = np.eye(4)
    m[:3, 0], m[:3, 1], m[:3, 2], m[:3, 3] = x, y, -z, 2.7 * fwd
    return np.concatenate([m.reshape(-1), [4.2647, 0, 0.5, 0, 4.2647, 0.5, 0, 0, 1]]).astype(np.float32)


def run_reference(ref):
    from oracle import edit as oe
    sys.path[:0] = [ref]
    for name, attr in (('numpy.lib.arraysetops', 'isin'), ('numpy.lib.function_base', 'angle')):
        m = types.ModuleType(name)
        setattr(m, attr, getattr(np, attr))
        sys.modules.setdefault(name, m)
    sys.modules['inversion.BiSeNet'] = types.SimpleNamespace(BiSeNet=None)         # dnnlib/seg_tools.py imports it at the top
    import inversion.networks as rn
    from dnnlib.seg_tools import mask2label_np
    torch.manual_seed(0)
    E = rn.HybridEncoder(**oe.ENCODER_ARGS).eval()
    E.load_state_dict(oe.encoder_state(E))
    E.requires_grad_(False)
    G = oe.standin_generator()
    masks, images = oe.golden_masks(), oe.golden_images(3)
    labels = np.stack([_camera(0.3, 0.1), _camera(-0.2, 0.0), _camera(0.1, -0.15)])
    state = E.state_dict()
    out = dict(masks=masks.numpy(), labels=labels, state_names=np.array(list(state)),
               state_shapes=np.array([','.join(map(str, v.shape)) for v in state.values()]))

    # ---- the encoder on the reference's input: mask2label_np(mask) * 2 - 1
    with torch.no_grad():
        seg = torch.from_numpy(np.stack([mask2label_np(m) for m in masks.numpy()])).float() * 2 - 1
        out['encoder_ws'] = E(images, seg).numpy()

    ws_avg = G.mapping.w_avg[None, None, :]
    rs = np.random.RandomState(43)
    pivot = torch.from_numpy((rs.randn(1, G.num_ws, G.w_dim) * 0.5).astype(np.float32)) + ws_avg
    out['pivot'] = pivot.numpy()

    with tempfile.TemporaryDirectory() as work:
        from PIL import Image
        # ---- infer_hybrid_encoder.test: image 0 with mask 1, spliced with the pivot
        img_path, seg_path, code_path = (os.path.join(work, n) for n in ('img00000001.png', 'seg.png', 'code.pt'))
        img_u8 = oe.to_uint8(images[:1])[0].permute(1, 2, 0).numpy()
        Image.fromarray(img_u8).save(img_path)
        Image.fromarray(masks[1].numpy()).save(seg_path)
        torch.save(pivot, code_path)
        saved = {}
        ns = dict(np=np, torch=torch, os=os, Image=Image, mask2label_np=mask2label_np,
                  conv2d_gradfix=types.SimpleNamespace(enabled=False),
                  utils=types.SimpleNamespace(save_image=lambda t, *a, **k: saved.__setitem__('rec_img', t.detach().clone())))
        exec(compile(_functions(os.path.join(ref, 'apps', 'infer_hybrid_encoder.py'), ['test']), 'infer_hybrid_encoder.py', 'exec'), ns)
        with torch.no_grad():
            ns['test'](target_img=img_path, target_seg=seg_path, target_code=code_path, target_label=torch.from_numpy(labels[:1]),
                       outdir=work, G=G, E=E, new_G=None, bisNet=None, start_from_latent_avg=True, device='cpu')
        out['encode_ws'] = torch.load(os.path.join(work, 'img00000001', 'rec_ws.pt')).numpy()
        out['encode_img'] = _pool(saved['rec_img'])

        # ---- Painter: run_deep_model with inversion=True for masks 1 and 2, each from the pivot
        ns = dict(np=np, torch=torch, cv2=types.SimpleNamespace(resize=lambda a, size: a),
                  QPixmap=types.SimpleNamespace(fromImage=lambda *a: None), QImage=lambda *a: None)
        ns['QImage'].Format_RGB888 = 0
        exec(compile(_functions(os.path.join(ref, 'Painter', 'run_UI.py'), ['run_deep_model', 'mask_labels', 'id_remap']), 'run_UI.py',
                     'exec'), ns)
        from dnnlib.seg_tools import COLOR_MAP
        rec_ws, fake = [], []
        for k in (1, 2):
            self = types.SimpleNamespace(generator=G, encoder=E, ws_avg=ws_avg, w=pivot.clone(), inversion=True, color_map=COLOR_MAP,
                                         mat_img=masks[k].numpy(), GT_scene_image_pts=types.SimpleNamespace(setPixmap=lambda *a: None))
            for name in ('mask_labels', 'id_remap'):
                setattr(self, name, ns[name].__get__(self))
            torch.Tensor.cuda = lambda t, *a, **kw: t
            try:
                with contextlib.redirect_stdout(io.StringIO()):
                    ns['run_deep_model'](self, label=torch.from_numpy(labels[:1]))
            finally:
                del torch.Tensor.cuda
            rec_ws.append(self.w.numpy())
            fake.append(_pool(self.fake_img))
        out['painter_ws'], out['painter_img'] = np.concatenate(rec_ws), np.concatenate(fake)

        # ---- face animation: seeds 0, 1 driven by the three (image, mask, camera) frames
        drive = os.path.join(work, 'drive')
        os.makedirs(drive)
        names = [f'frame{f:03d}.png' for f in range(FRAMES)]
        opencv = labels.copy()
        opencv[:, [1, 2, 5, 6, 9, 10]] *= -1                                          # the script flips them back on read
        with open(os.path.join(drive, 'dataset.json'), 'w') as fh:
            json.dump({'labels': [[n, opencv[f].tolist()] for f, n in enumerate(names)]}, fh)
        drive_u8 = oe.to_uint8(images).permute(0, 2, 3, 1).numpy()
        for f, n in enumerate(names):
            Image.fromarray(drive_u8[f]).save(os.path.join(drive, n))
        parse = iter(masks)
        frames, rec = [], []
        E_rec = lambda img, seg: (lambda r: (rec.append(r.numpy()), r)[1])(E(img, seg))
        tdev = types.ModuleType('torch_cpu')
        tdev.__dict__.update(torch.__dict__)
        tdev.device = lambda *a, **k: torch.device('cpu')
        from tqdm import tqdm
        import glob
        ns = dict(torch=tdev, np=np, os=os, glob=glob, json=json, tqdm=tqdm, Image=Image, F=F,
                  dnnlib=types.SimpleNamespace(util=types.SimpleNamespace(open_url=lambda *a, **k: contextlib.nullcontext(None))),
                  legacy=types.SimpleNamespace(load_network_pkl=lambda f: {'G_ema': G}, load_encoder_pkl=lambda f: {'E': E_rec}),
                  imageio=types.SimpleNamespace(get_writer=lambda *a, **k: types.SimpleNamespace(append_data=lambda a: None,
                                                                                                   close=lambda: None)),
                  initFaceParsing=lambda **k: (None, None),
                  face_parsing=lambda img, bisNet=None: torch.from_numpy(mask2label_np(next(parse).numpy())).float()[None],
                  layout_grid=lambda result, grid_w=None, grid_h=1: frames.append(_pool(result[1:])))
        E_rec.to = lambda *a, **k: E_rec
        exec(compile(_functions(os.path.join(ref, 'apps', 'infer_face_animation.py'), ['run_video_animation']), 'infer_face_animation.py',
                     'exec'), ns)
        with torch.no_grad(), contextlib.redirect_stderr(io.StringIO()), contextlib.redirect_stdout(io.StringIO()):
            ns['run_video_animation'](drive_root=drive, network_pkl='G', encoder_pkl='E', grid_dims=(len(SEEDS) + 1, 1), seeds=SEEDS,
                                      outdir=os.path.join(work, 'out'), truncation_psi=1, truncation_cutoff=14)
        out['anim_seeds'] = np.array(SEEDS)
        out['anim_ws'] = np.stack(rec)                     # [F, B, num_ws, w_dim]: E(...) + w_avg is added after the recorded call
        out['anim_img'] = np.stack(frames)                 # [F, B, 3, 32, 32]
    return out


if __name__ == '__main__':
    ref = os.environ.get('IDE3D_REFERENCE')
    if not ref:
        sys.exit('set IDE3D_REFERENCE to the reference checkout')
    out = run_reference(ref)
    np.savez_compressed(os.path.join(HERE, 'edit_trace.npz'), **out)
    for k, v in out.items():
        print(f'{k:16s} {v.dtype} {v.shape}')
    print(f'{os.path.getsize(os.path.join(HERE, "edit_trace.npz")) / 1024:.1f} KB')
