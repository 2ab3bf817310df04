"""CPU: ide3d_b200.train_encoder against the reference's apps/train_hybrid_encoder.py (tests/golden/encoder_train_trace.npz, recorded by
make_encoder_train_golden.py with the weights of oracle/train_encoder.py, oracle/finetune.py, oracle/pti.py and oracle/edit.py), the
dataset reader, InfiniteSampler, state_dict loading of the loss networks, argument validation, and the ABI of the new entry points."""

import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from conftest import ROOT, load_golden

GEN = ('loss_ws', 'loss_gen_l2', 'loss_gen_entropy', 'loss_cycle')
REAL = ('loss_vgg', 'loss_real_l2', 'loss_lpips', 'loss_id', 'loss_real_entropy', 'loss_real_cycle')
RUNS = {'gen': dict(train_gen=True, train_real=False, lambdas=dict(l2=1.0, entropy=0.5, cycle=2.0)),
        'both': dict(train_gen=True, train_real=True, lambdas=dict(vgg=0.8, l2=1.0, lpips=0.6, id=0.4, entropy=0.5, cycle=2.0))}


@pytest.fixture(scope='module')
def trace():
    return load_golden('encoder_train_trace')


@pytest.fixture(scope='module')
def portraits():
    from oracle import train_encoder as ot
    with tempfile.TemporaryDirectory() as d:
        yield ot.write_portraits(d)


def _parser():
    from ide3d_b200.parsing import BiSeNet
    from oracle import finetune as of
    torch.manual_seed(0)
    net = BiSeNet(20)
    net.load_state_dict(of.bisenet_state(net), strict=True)
    return net.eval().requires_grad_(False)


def _encoder():
    from ide3d_b200.encoder import HybridEncoder
    from oracle import edit as oe
    E = HybridEncoder(**oe.ENCODER_ARGS)
    E.load_state_dict(oe.encoder_state(E))
    return E


def _irse():
    from ide3d_b200.arcface import Backbone
    from oracle import train_encoder as ot
    net = Backbone(112, 50, mode='ir_se', drop_ratio=0.6)
    net.load_state_dict(ot.irse50_state(net), strict=True)
    return net.eval()


def _err(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


@pytest.mark.parametrize('tag', ['gen', 'both'])
def test_train_replays_reference(trace, portraits, tag):
    """Three steps at batch 2, world 1, seed 0, start_from_latent_avg: the latent and camera draws and the data order equal the
    script's; the per-step losses, E's gradients before each update (step 0's element by element for the stem and block 0 of both
    branches, every tensor's max |g| at every step), the trained weights and the per-tensor sums of their change match.  Measured
    (gen / both): losses 3.4e-7 of max|loss|; step-0 gradients 5.9e-5 / 5.0e-5 of max|g|; per-tensor max|g| 1.0e-4 / 3.3e-4;
    trained weights 4.2e-5 / 4.3e-5 of max|w|; sums of the change 1.3e-4 / 1.0e-4.  The change itself, element by element, is not
    bounded here: it differs by up to 0.65 of max|dw| on 13 % / 20 % of those elements, most of which have step-0 gradients well
    above the gradient error, so Adam amplifying near-zero gradients does not explain it alone."""
    from ide3d_b200 import train_encoder as T
    from ide3d_b200.arcface import IDLoss
    from ide3d_b200.torch_utils.ops.vgg_loss import VGGLoss
    from oracle import edit as oe, pti as opti, train_encoder as ot
    run = RUNS[tag]
    E = _encoder()
    initial = {k: v.clone() for k, v in E.state_dict().items()}
    ds = T.PortraitDataset(portraits[0], portraits[1], 512)
    draws = {'z': [], 'cams': [], 'order': []}
    step_losses = T.step_losses

    def spy(G, enc, **kw):
        if kw['z'] is not None:
            draws['z'].append(kw['z'].numpy().copy())
            draws['cams'].append(kw['cam'].numpy().copy())
        return step_losses(G, enc, **kw)

    grads = []
    adam = torch.optim.Adam

    class _Adam(adam):
        def step(self, *a, **k):                            # E's gradients of the step, before the update
            grads.append([p.grad.detach().clone() for g in self.param_groups for p in g['params']])
            return super().step(*a, **k)

    getitem = T.PortraitDataset.__getitem__
    torch.optim.Adam = _Adam
    T.step_losses = spy
    T.PortraitDataset.__getitem__ = lambda self, i: (draws['order'].append(int(i)), getitem(self, i))[1]
    try:
        with ot.cpu_train_ops():
            E_t, losses = T.train(oe.standin_generator(), E, parser=_parser(), steps=3, batch=2, start_from_latent_avg=True,
                                  dataset=ds, vgg=VGGLoss(ot.standin_vgg19().features), lpips=opti.standin_lpips(), id_net=IDLoss(_irse()),
                                  **run)
    finally:
        T.step_losses, T.PortraitDataset.__getitem__, torch.optim.Adam = step_losses, getitem, adam
    assert np.array_equal(np.stack(draws['z']), trace[f'{tag}_z'])
    assert np.abs(np.stack(draws['cams']) - trace[f'{tag}_cams']).max() <= 1e-6
    assert draws['order'] == list(trace[f'{tag}_order'])
    names = GEN + (REAL if run['train_real'] else ())
    assert list(losses) == list(names)
    got = np.stack([losses[n] for n in names], 1)
    e_loss = _err(got, trace[f'{tag}_losses'])
    state = E_t.state_dict()
    enames = [str(n) for n in trace['encoder_names']]
    delta = {n: state[n].double() - initial[n].double() for n in enames}
    whole = [n for n in enames if f'{tag}_d_{n}' in trace]
    dmax = max(np.abs(trace[f'{tag}_d_{n}']).max() for n in whole)
    diff = torch.cat([(delta[n] - torch.from_numpy(trace[f'{tag}_d_{n}']).double()).abs().reshape(-1) for n in whole]) / dmax
    off = (diff > 1e-5).double().mean().item()
    sums = np.array([delta[n].sum().item() for n in enames])
    e_sums = _err(sums, trace[f'{tag}_d_sums'])
    wmax = max(initial[n].abs().max().item() for n in whole)
    e_w = diff.max().item() * dmax / wmax
    pnames = [str(n) for n in trace[f'{tag}_grad_names']]
    assert pnames == [n for n, _ in E.named_parameters()]
    g0 = dict(zip(pnames, grads[0]))
    gwhole = [n for n in pnames if f'{tag}_g0_{n}' in trace]
    gmax = max(np.abs(trace[f'{tag}_g0_{n}']).max() for n in gwhole)
    e_g0 = max((g0[n].double() - torch.from_numpy(trace[f'{tag}_g0_{n}']).double()).abs().max().item() for n in gwhole) / gmax
    gabs = np.array([[g.abs().max().item() for g in step] for step in grads])
    e_gabs = _err(gabs, trace[f'{tag}_grad_absmax'])
    print(f'{tag}: step-0 gradients {e_g0:.2e} of max|g|, per-tensor max|g| over 3 steps {e_gabs:.2e}')
    print(f'{tag}: losses {e_loss:.2e}, trained weights {e_w:.2e} of max|w|, their change {diff.max():.2e} of max|dw| '
          f'({off:.2e} of the elements beyond 1e-5), sums of the change {e_sums:.2e}')
    assert e_loss <= 1e-6 and e_g0 <= 2e-4 and e_gabs <= 1e-3 and e_w <= 1e-4 and e_sums <= 1e-3
    assert not E_t.training and not any(p.requires_grad for p in E_t.parameters())
    assert all(torch.equal(v, initial[k]) for k, v in E.state_dict().items())


def test_initial_encoder_equals_reference_construction(trace):
    """E=None: HybridEncoder(G.img_resolution, G.num_ws - 8, 8, G.w_dim) under torch.manual_seed(0), the global RNG untouched."""
    from ide3d_b200 import train_encoder as T
    from oracle import edit as oe
    before = torch.random.get_rng_state()
    E, losses = T.train(oe.standin_generator(), parser=None, steps=0)
    assert torch.equal(torch.random.get_rng_state(), before)
    assert list(E.state_dict()) == [str(n) for n in trace['encoder_names']]
    sums = np.array([v.double().sum().item() for v in E.state_dict().values()])
    assert np.array_equal(sums, trace['gen_initial_sums'])
    assert (E.n_latents_app, E.n_latents_geo, E.w_dim) == (2, 8, 16) and all(len(v) == 0 for v in losses.values())


def test_portrait_dataset_matches_reference(trace, portraits):
    """ids equal the reference's one-hot argmax (an all-zero row, ids >= 19, as 255 here), labels equal (OpenCV -> OpenGL flip);
    image 1 is 448^2 on disk and resized."""
    from ide3d_b200.train_encoder import PortraitDataset
    ds = PortraitDataset(portraits[0], portraits[1], 512)
    assert len(ds) == 6
    for i in range(len(ds)):
        img, ids, label = ds[i]
        assert img.dtype == torch.uint8 and img.shape == (3, 512, 512) and ids.dtype == torch.uint8 and ids.shape == (512, 512)
        assert label.dtype == torch.float32 and label.shape == (25,)
        assert np.array_equal(np.where(ids.numpy() >= 19, 255, ids.numpy()), trace['dataset_seg_argmax'][i])
        assert np.array_equal(label.numpy(), trace['dataset_labels'][i])
        assert int(img.long().sum()) == int(trace['dataset_image_sums'][i])
    assert np.array_equal(trace['dataset_labels'], portraits[2])
    with pytest.raises(ValueError, match='dataset.json'):
        PortraitDataset(portraits[1], portraits[1], 512)


def test_infinite_sampler_order(trace):
    from ide3d_b200.torch_utils.misc import InfiniteSampler
    data = list(range(6))
    it = iter(InfiniteSampler(data, rank=0, num_replicas=1, seed=0))
    assert [next(it) for _ in range(20)] == list(trace['sampler_order'])
    it = iter(InfiniteSampler(data, rank=1, num_replicas=2, seed=3))
    assert [next(it) for _ in range(20)] == list(trace['sampler_order_r1w2'])


def test_loss_networks_load_reference_state_dicts(trace):
    """IR-SE50 under the reference's names (strict); torchvision VGG19's features through VGGLoss.vgg19 (strict); ID loss value."""
    import torchvision
    from ide3d_b200.arcface import Backbone, IDLoss
    from ide3d_b200.torch_utils.ops.vgg_loss import TAPS, VGGLoss
    net = _irse()
    assert list(net.state_dict()) == [str(n) for n in trace['irse_names']]
    with tempfile.TemporaryDirectory() as d:
        torch.save(net.state_dict(), os.path.join(d, 'model_ir_se50.pth'))
        loaded = Backbone.ir_se50(os.path.join(d, 'model_ir_se50.pth'))
        assert not loaded.training and all(torch.equal(a, b) for a, b in zip(loaded.state_dict().values(), net.state_dict().values()))
        torch.manual_seed(0)
        torch.save(torchvision.models.vgg19(weights=None).state_dict(), os.path.join(d, 'vgg19.pth'))
        vgg = VGGLoss.vgg19(os.path.join(d, 'vgg19.pth'))
        assert len(vgg.slices) == len(TAPS) and isinstance(vgg.slices[-1][-1], torch.nn.ReLU)
        with pytest.raises(FileNotFoundError):
            VGGLoss.vgg19(os.path.join(d, 'missing.pth'))
        with pytest.raises(FileNotFoundError):
            Backbone.ir_se50(os.path.join(d, 'missing.pth'))
    x = torch.rand(2, 3, 64, 64) * 2 - 1
    idl = IDLoss(net)
    with torch.no_grad():
        assert abs(float(idl(x, x))) <= 1e-6
        f1, f2 = idl.extract_feats(x), idl.extract_feats(x.flip(0))
        assert abs(float(idl(x, x.flip(0))) - float((1 - (f1 * f2).sum(1)).mean())) <= 1e-6


def test_argument_validation(portraits):
    from ide3d_b200 import train_encoder as T
    from oracle import edit as oe
    G = oe.standin_generator()
    with pytest.raises(ValueError, match='adv'):
        T.train(G, parser=None, steps=0, lambdas=dict(adv=1.0))
    with pytest.raises(ValueError, match='unknown lambdas'):
        T.train(G, parser=None, steps=0, lambdas=dict(perceptual=1.0))
    with pytest.raises(ValueError, match='train_gen or train_real'):
        T.train(G, parser=None, steps=0, train_gen=False)
    with pytest.raises(ValueError, match='dataset'):
        T.train(G, parser=None, steps=0, train_real=True)
    ds = T.PortraitDataset(portraits[0], portraits[1], 512)
    with pytest.raises(ValueError, match='vgg module'):
        T.train(G, parser=None, steps=0, train_real=True, dataset=ds, lambdas=dict(vgg=1.0))
    with pytest.raises(ValueError, match='steps'):
        T.train(G, parser=None, steps=-1)
    with pytest.raises(ValueError, match='world'):
        T.train(G, parser=None, steps=0, batch=1, world=2, rank=0)
    with pytest.raises(ValueError, match='process group'):
        T.train(G, parser=None, steps=0, batch=2, world=2, rank=1)
    with pytest.raises(ValueError, match='outdir'):
        T.train(G, parser=None, steps=0, snapshot_every=1)
    from ide3d_b200.encoder import HybridEncoder
    with pytest.raises(ValueError, match='rows'):
        T.train(G, HybridEncoder(512, 4, 8, 16), parser=None, steps=0)


def test_camera_positions_generator_is_additive():
    from ide3d_b200.training.volumetric_rendering import sample_camera_positions
    torch.manual_seed(5)
    a = sample_camera_positions('cpu', n=4, r=2.7, mode='gaussian')
    b = sample_camera_positions('cpu', n=4, r=2.7, mode='gaussian', generator=torch.Generator().manual_seed(5))
    torch.manual_seed(5)
    c = sample_camera_positions('cpu', n=4, r=2.7, mode='gaussian')
    assert all(torch.equal(x, y) for x, y in zip(a, b)) and all(torch.equal(x, y) for x, y in zip(a, c))


def _probe_size():
    probe = r'''
    #include <stdio.h>
    #include "ide3d_b200.h"
    int main(void) { printf("%zu %zu\n", sizeof(ide3d_feat_l1_params), sizeof(ide3d_feat_l1_layer)); return 0; }'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, 'p.c')
        open(c, 'w').write(probe)
        exe = os.path.join(d, 'p')
        subprocess.run(['gcc', '-I', os.path.join(ROOT, 'include'), c, '-o', exe], check=True)
        return [int(v) for v in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]


def test_new_symbols_struct_layout_and_status_codes(lib):
    """Malformed parameters return a status without touching the device (the pointers below are never dereferenced)."""
    from ide3d_b200 import _lib
    for name in ('ide3d_feat_l1_scratch_bytes', 'ide3d_feat_l1_fwd', 'ide3d_feat_l1_bwd'):
        assert name in _lib.exported_symbols() and hasattr(lib, name)
    assert [ctypes.sizeof(_lib.FeatL1Params), ctypes.sizeof(_lib.FeatL1Layer)] == _probe_size()
    for name in ('ide3d_feat_l1_fwd', 'ide3d_feat_l1_bwd'):
        assert getattr(lib, name)(None, None) == _lib.INVALID and b'null params' in lib.ide3d_last_error()
    fake = 0x10000
    p = _lib.FeatL1Params()
    p.n, p.num_layers, p.dtype = 2, 1, _lib.F32
    layer = p.layers[0]
    layer.c, layer.h, layer.w, layer.weight, layer.x, layer.y = 3, 5, 7, 1.0, fake, fake
    layer.x_stride = layer.y_stride = (ctypes.c_int64 * 4)(105, 35, 7, 1)
    assert lib.ide3d_feat_l1_scratch_bytes(ctypes.byref(p)) == 8                 # 210 elements: one CTA
    p.dtype = _lib.F16
    assert lib.ide3d_feat_l1_scratch_bytes(ctypes.byref(p)) == _lib.UNSUPPORTED
    assert lib.ide3d_feat_l1_fwd(ctypes.byref(p), None) == _lib.UNSUPPORTED and b'fp32' in lib.ide3d_last_error()
    p.dtype, p.num_layers = _lib.F32, 9
    assert lib.ide3d_feat_l1_fwd(ctypes.byref(p), None) == _lib.UNSUPPORTED
    p.num_layers = 1
    assert lib.ide3d_feat_l1_fwd(ctypes.byref(p), None) == _lib.INVALID and b'null value' in lib.ide3d_last_error()
    assert lib.ide3d_feat_l1_bwd(ctypes.byref(p), None) == _lib.INVALID and b'null grad_x' in lib.ide3d_last_error()
    layer.grad_x, layer.gx_stride = fake, (ctypes.c_int64 * 4)(105, 35, 7, 1)
    assert lib.ide3d_feat_l1_bwd(ctypes.byref(p), None) == _lib.INVALID and b'null grad_value' in lib.ide3d_last_error()
    layer.y_stride = (ctypes.c_int64 * 4)(105, 35, -7, 1)
    assert lib.ide3d_feat_l1_scratch_bytes(ctypes.byref(p)) == _lib.INVALID
    layer.y_stride, layer.c = (ctypes.c_int64 * 4)(105, 35, 7, 1), 0
    assert lib.ide3d_feat_l1_scratch_bytes(ctypes.byref(p)) == _lib.INVALID


def test_resume_equals_straight_run(portraits):
    """2 steps, a snapshot, 2 more from it: equal to 4 steps straight (the latent, camera and data streams and Adam's state resume)."""
    from ide3d_b200 import train_encoder as T
    from ide3d_b200.torch_utils.ops.vgg_loss import VGGLoss
    from oracle import edit as oe, train_encoder as ot
    G, E = oe.standin_generator(), _encoder()
    ds = T.PortraitDataset(portraits[0], portraits[1], 512)
    kw = dict(parser=_parser(), batch=2, lambdas=dict(vgg=0.8, l2=1.0, cycle=2.0), train_real=True, dataset=ds,
              vgg=VGGLoss(ot.standin_vgg19().features), start_from_latent_avg=True)
    with ot.cpu_train_ops(), tempfile.TemporaryDirectory() as d:
        E4, l4 = T.train(G, E, steps=4, **kw)
        _, l2 = T.train(G, E, steps=2, snapshot_every=2, outdir=d, **kw)
        path = os.path.join(d, 'encoder-snapshot-000002.pt')
        with pytest.raises(ValueError, match='E=None'):
            T.train(G, E, steps=1, resume=path, **kw)
        for change in (dict(seed=1), dict(batch=4), dict(train_real=False)):
            with pytest.raises(ValueError, match='would not continue'):
                T.train(G, None, steps=1, resume=path, **{**kw, **change})
        before = torch.random.get_rng_state()
        E22, l22 = T.train(G, None, steps=2, resume=path, **kw)
        assert torch.equal(torch.random.get_rng_state(), before)
    assert all(torch.equal(a, b) for a, b in zip(E4.state_dict().values(), E22.state_dict().values()))
    for k in l4:
        assert np.array_equal(l4[k], np.concatenate([l2[k], l22[k]])), k


def _gloo_worker(rank, world, port, outdir):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    torch.set_num_threads(max(1, (os.cpu_count() or 2) // world))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        from ide3d_b200 import train_encoder as T
        from oracle import edit as oe, train_encoder as ot
        zs = []
        step_losses = T.step_losses

        def spy(G, enc, **kw):
            zs.append(kw['z'].clone())
            return step_losses(G, enc, **kw)
        T.step_losses = spy
        kw = dict(parser=_parser(), batch=2, world=world, rank=rank, lambdas=dict(cycle=1.0), start_from_latent_avg=True)
        with ot.cpu_train_ops():
            E3, _ = T.train(oe.standin_generator(), _encoder(), steps=3, **kw)
            T.train(oe.standin_generator(), _encoder(), steps=2, snapshot_every=2, outdir=outdir, **kw)
            E21, _ = T.train(oe.standin_generator(), None, steps=1, resume=os.path.join(outdir, 'encoder-snapshot-000002.pt'), **kw)
        torch.save(dict(z=torch.stack(zs), E3=E3.state_dict(), E21=E21.state_dict()), os.path.join(outdir, f'rank{rank}.pt'))
    finally:
        dist.destroy_process_group()


def test_resume_at_world_2_keeps_each_rank_stream():
    """Two gloo processes, E under DistributedDataParallel (three forwards before one backward with the cycle term): 3 steps straight
    equal 2 steps, a snapshot and 1 resumed step on each rank; after the resume the two ranks still draw different latents, each its
    own continuation; DDP keeps the ranks' encoders equal."""
    import socket
    import torch.multiprocessing as mp
    with tempfile.TemporaryDirectory() as d:
        with socket.socket() as s:
            s.bind(('127.0.0.1', 0))
            port = s.getsockname()[1]
        mp.start_processes(_gloo_worker, args=(2, port, d), nprocs=2, join=True, start_method='spawn')
        runs = [torch.load(os.path.join(d, f'rank{r}.pt'), weights_only=True) for r in range(2)]
    for r in runs:
        assert r['z'].shape[0] == 6 and torch.equal(r['z'][5], r['z'][2]) and torch.equal(r['z'][3:5], r['z'][:2])
        assert all(torch.equal(r['E3'][k], r['E21'][k]) for k in r['E3'])
    assert not torch.equal(runs[0]['z'][5], runs[1]['z'][5])
    assert all(torch.equal(runs[0]['E3'][k], runs[1]['E3'][k]) for k in runs[0]['E3'])


def test_feat_l1_rejects_mismatched_layers():
    from ide3d_b200.torch_utils.ops.vgg_loss import feat_l1
    x = [torch.zeros(2, 3, 4, 4), torch.zeros(1, 3, 2, 2)]
    with pytest.raises(ValueError, match='samples'):
        feat_l1(x, [t.clone() for t in x], (1.0, 1.0))
    with pytest.raises(ValueError, match='equal 4-d shapes'):
        feat_l1(x[:1], [torch.zeros(2, 3, 4, 5)], (1.0,))
