#!/usr/bin/env python
"""Generate tests/golden/encoder_train_trace.npz by running the REFERENCE's hybrid-encoder training, imported read-only, on the CPU at
world 1 with seeded weights and the stand-in generator.

    IDE3D_REFERENCE=/path/to/IDE-3D PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_encoder_train_golden.py

    apps/train_hybrid_encoder.py:155-392   train() and VGGLoss, executed from the AST (the module imports tensorboardX and a D:/ path
                                           at the top), 3 steps at batch 2: --train_gen alone (l2, entropy, cycle non-zero), and
                                           --train_gen --train_real with every lambda but adv non-zero, both --start_from_latent_avg
    training/dataset_seg.py                CameraLabeledDataset over oracle.train_encoder.write_portraits (6 portraits)
    inversion/networks.py                  HybridEncoder(512, 2, 8, w_dim=16) under torch.manual_seed(0) (recorded), then loaded with
                                           oracle.edit.encoder_state
    inversion/BiSeNet.py                   BiSeNet(20) with oracle.finetune.bisenet_state
    inversion/criteria/lpips               the reference's LPIPS with oracle.pti's seeded AlexNet and lin weights
    inversion/criteria/id_loss.py          the reference's IDLoss with oracle.train_encoder.irse50_state
torchvision's vgg19(pretrained=True) answers oracle.train_encoder.standin_vgg19(); the modules are built before the script's
torch.manual_seed(rank), so its camera draws are the first of that seed, as on the GPU, where they do not share the CPU's generator.
Stubs for what the script touches outside the computation: the stand-in synthesis answers return_raw=True with the image twice, DDP is the module itself, setup / tensorboard / the sample PNGs do nothing,
the DataLoader is a worker-less loop (torch 2 refuses its prefetch_factor without workers, and its base seed would shift the CPU
camera draws) and Sampler.__init__ ignores its argument (torch 2 refuses it) and records the sampler's indices, the pickled snapshot is
captured, and `sum` records the step's loss terms.  Recorded: the initial E's per-tensor sums, the z and camera draws, the data order,
the per-step losses, E's gradients at each step before Adam's update (step 0's whole for the stem and block 0 of both branches,
per-tensor max |g| and sums for all), and the weight change (trained - initial: the same tensors whole, per-tensor sums for all).
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
sys.path.insert(0, HERE)

STEPS = 3
BATCH = 2
WHOLE = ('convs_seg.0.', 'convs_seg.1.', 'convs_img.0.', 'convs_img.1.')
RUNS = {'gen': dict(train_gen=True, train_real=False, vgg=0.0, l2=1.0, lpips=0.0, id=0.0, entropy=0.5, cycle=2.0),
        'both': dict(train_gen=True, train_real=True, vgg=0.8, l2=1.0, lpips=0.6, id=0.4, entropy=0.5, cycle=2.0)}


def _nodes(path, names):
    tree = ast.parse(open(path).read())
    out = []
    for node in tree.body:
        if isinstance(node, (ast.FunctionDef, ast.ClassDef)) and node.name in names:
            node.decorator_list = []
            out.append(node)
    return ast.Module(out, [])


def run_reference(ref):
    from oracle import edit as oe, finetune as of, pti as opti, train_encoder as ot
    from make_pti_golden import _vendored_lpips
    sys.path[:0] = [ref, os.path.join(ref, 'inversion')]
    for name, attr in (('numpy.lib.arraysetops', 'isin'), ('numpy.lib.function_base', 'angle')):
        m = types.ModuleType(name)
        setattr(m, attr, getattr(np, attr))
        sys.modules.setdefault(name, m)
    import inversion.networks as rn
    from inversion.BiSeNet import BiSeNet
    from inversion.psp.encoders.model_irse import Backbone
    from dnnlib import seg_tools
    from training import dataset_seg
    from training.volumetric_rendering import sample_camera_positions, create_cam2world_matrix
    from torch_utils import misc as ref_misc
    torch.utils.data.Sampler.__init__ = lambda self, *a, **k: None     # the reference passes the dataset, which torch 2 refuses

    torch.manual_seed(0)
    net = BiSeNet(20).eval()
    net.load_state_dict(of.bisenet_state(net))
    net.requires_grad_(False)
    G = oe.standin_generator()
    synthesis_forward = type(G.synthesis).forward

    def with_raw(self, ws, c=None, return_raw=False, **kw):                  # the script's return_raw=True: (image, raw image)
        img = synthesis_forward(self, ws, c=c, **kw)
        return (img, img) if return_raw else img
    type(G.synthesis).forward = with_raw
    out = {}
    with tempfile.TemporaryDirectory() as work:
        img_dir, seg_dir, labels = ot.write_portraits(work)
        ds = dataset_seg.CameraLabeledDataset(path=img_dir, seg_path=seg_dir, load_seg=True, use_labels=True, xflip=False,
                                              resolution=512)
        out['dataset_labels'] = np.stack([ds[i][2] for i in range(len(ds))])
        out['dataset_seg_argmax'] = np.stack([np.where(ds[i][1].max(0) > 0, ds[i][1].argmax(0), 255) for i in range(len(ds))]).astype(np.uint8)
        out['dataset_image_sums'] = np.array([ds[i][0].astype(np.int64).sum() for i in range(len(ds))])
        sampler = ref_misc.InfiniteSampler(ds, rank=0, num_replicas=1, seed=0)
        it = iter(sampler)
        out['sampler_order'] = np.array([next(it) for _ in range(20)])
        it = iter(ref_misc.InfiniteSampler(ds, rank=1, num_replicas=2, seed=3))
        out['sampler_order_r1w2'] = np.array([next(it) for _ in range(20)])
        irse = Backbone(input_size=112, num_layers=50, drop_ratio=0.6, mode='ir_se')
        out['irse_names'] = np.array(list(irse.state_dict()))
        irse_state = ot.irse50_state(irse)

        os.makedirs(os.path.join(work, 'pretrained_models'))
        torch.save(opti.lin_state_dict(), os.path.join(work, 'pretrained_models', 'alex.pth'))
        torch.save(irse_state, os.path.join(work, 'pretrained_models', 'model_ir_se50.pth'))
        cwd = os.getcwd()
        os.chdir(work)
        try:
            lpips_mod = _vendored_lpips('alex')
            from inversion.criteria import id_loss as ref_id
            id_mod = ref_id.IDLoss()
        finally:
            os.chdir(cwd)
        vgg_net = ot.standin_vgg19()

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

        for tag, opts in RUNS.items():
            torch.manual_seed(0)
            E0 = rn.HybridEncoder(**oe.ENCODER_ARGS)
            out[f'{tag}_initial_sums'] = np.array([v.double().sum().item() for v in E0.state_dict().values()])
            out['encoder_names'] = np.array(list(E0.state_dict()))
            E = rn.HybridEncoder(**oe.ENCODER_ARGS)
            initial = oe.encoder_state(E)
            E.load_state_dict(initial)
            steps, zs, cams, order, grads = [], [], [], [], []
            pname = {id(p): n for n, p in E.named_parameters()}

            class _Adam(torch.optim.Adam):
                def step(self, *a, **k):                    # E's gradients of the step, before the update
                    grads.append({pname[id(p)]: p.grad.detach().clone() for g in self.param_groups for p in g['params']})
                    return super().step(*a, **k)

            def record_sum(terms, start=0):
                if terms and all(isinstance(t, torch.Tensor) and t.ndim == 0 for t in terms):
                    steps.append([float(t.detach()) for t in terms])
                return builtins.sum(terms, start)

            def cam_sampler(batch, device):
                c = ns_cam(batch, device)
                cams.append(c.numpy().copy())
                return c

            class _Sampler:
                def __init__(self, inner):
                    self.inner = inner

                def __iter__(self):
                    for i in self.inner:
                        order.append(int(i))
                        yield i

            def loader(dataset, sampler, batch_size, **kw):
                def batches():                  # a DataLoader without workers, minus the base seed it draws from the torch RNG
                    it = iter(_Sampler(sampler))
                    while True:
                        yield torch.utils.data.default_collate([dataset[next(it)] for _ in range(batch_size)])
                return batches()

            class _NumpyRandom:
                def seed(self, s):
                    np.random.seed(s)

                def randn(self, *shape):
                    z = np.random.randn(*shape)
                    zs.append(z.copy())
                    return z

            tdev.utils = types.SimpleNamespace(data=types.SimpleNamespace(DataLoader=loader))
            np_ns = types.SimpleNamespace(**{k: getattr(np, k) for k in ('float32', 'array', 'zeros')}, random=_NumpyRandom())
            opt_ns = types.SimpleNamespace(
                data=img_dir, seg=seg_dir, outdir=os.path.join(work, tag), g_ckpt='G.pkl', e_ckpt='E.pkl', max_steps=STEPS, batch=BATCH,
                lr=1e-4, local_rank=0, adv=0.0, truncation=1.0, start_from_latent_avg=True, tensorboard=False, num_gpus=1, port='0',
                **opts)
            ns = dict(np=np_ns, torch=tdev, os=os, copy=__import__('copy'), F=F, optim=types.SimpleNamespace(Adam=_Adam), nn=torch.nn, glob=__import__('glob'),
                      math=__import__('math'), sum=record_sum, tqdm=_Bar, SummaryWriter=None, setup=lambda *a: None,
                      conv2d_gradfix=types.SimpleNamespace(enabled=False), misc=ref_misc, HybridEncoder=rn.HybridEncoder,
                      DDP=lambda module, **k: types.SimpleNamespace(module=module, __call__=None),
                      dnnlib=types.SimpleNamespace(util=types.SimpleNamespace(
                          open_url=lambda *a, **k: contextlib.nullcontext(None),
                          construct_class_by_name=lambda class_name, **k: dataset_seg.CameraLabeledDataset(**k))),
                      legacy=types.SimpleNamespace(load_network_pkl=lambda f: {'G_ema': G, 'D': torch.nn.Linear(1, 1)},
                                                   load_encoder_pkl=lambda f: {'E': E}),
                      initFaceParsing=lambda **k: (net, None), face_parsing=seg_tools.face_parsing, parsing_img=seg_tools.parsing_img,
                      mask2color=lambda masks, *a, **k: torch.zeros_like(masks[:, :3]),
                      requires_grad=lambda model, flag=True: [p.requires_grad_(flag) for p in model.parameters()], utils=types.SimpleNamespace(save_image=lambda *a, **k: None),
                      torchvision=types.SimpleNamespace(models=types.SimpleNamespace(vgg19=lambda *a, **k: vgg_net)),
                      LPIPS=lambda **k: lpips_mod, IDLoss=types.SimpleNamespace(IDLoss=lambda: id_mod),
                      pickle=types.SimpleNamespace(dump=lambda obj, f: None), sample_camera_positions=sample_camera_positions,
                      create_cam2world_matrix=create_cam2world_matrix)
            exec(compile(_nodes(os.path.join(ref, 'apps', 'train_hybrid_encoder.py'), {'VGGLoss', 'cam_sampler', 'train'}),
                         'train_hybrid_encoder.py', 'exec'), ns)
            ns_cam = ns['cam_sampler']
            ns['cam_sampler'] = cam_sampler

            class _DDP:
                def __init__(self, module, **k):
                    self.module = module

                def __call__(self, *a, **k):
                    return self.module(*a, **k)
            ns['DDP'] = _DDP
            with contextlib.redirect_stdout(io.StringIO()):
                ns['train'](0, 1, opt_ns)
            assert len(steps) == STEPS, len(steps)
            out[f'{tag}_losses'] = np.array(steps, np.float64)
            out[f'{tag}_z'] = np.stack(zs).astype(np.float32)
            out[f'{tag}_cams'] = np.stack(cams)
            out[f'{tag}_order'] = np.array(order[:STEPS * BATCH] if opts['train_real'] else [], np.int64)
            state = E.state_dict()
            names = list(state)
            delta = {n: state[n].detach().double() - initial[n].double() for n in names}
            for n in names:
                if n.startswith(WHOLE) and not n.endswith('resample_filter'):
                    out[f'{tag}_d_{n}'] = delta[n].float().numpy()
            out[f'{tag}_d_sums'] = np.array([delta[n].sum().item() for n in names])
            out[f'{tag}_d_absmax'] = np.array([delta[n].abs().max().item() for n in names])
            pnames = [n for n, _ in E.named_parameters()]
            out[f'{tag}_grad_names'] = np.array(pnames)
            out[f'{tag}_grad_absmax'] = np.array([[g[n].abs().max().item() for n in pnames] for g in grads])
            out[f'{tag}_grad_sums'] = np.array([[g[n].double().sum().item() for n in pnames] for g in grads])
            for n in pnames:
                if n.startswith(WHOLE):
                    out[f'{tag}_g0_{n}'] = grads[0][n].numpy()
    return out


if __name__ == '__main__':
    ref = os.environ.get('IDE3D_REFERENCE')
    if not ref:
        sys.exit('set IDE3D_REFERENCE to the reference checkout')
    out = run_reference(ref)
    np.savez_compressed(os.path.join(HERE, 'encoder_train_trace.npz'), **out)
    for k, v in out.items():
        if '_d_convs' not in k:
            print(f'{k:28s} {v.dtype} {v.shape}')
    print(f'{os.path.getsize(os.path.join(HERE, "encoder_train_trace.npz")) / 1024:.1f} KB')
