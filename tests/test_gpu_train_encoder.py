"""GPU: the multi-tap L1 head (ide3d_feat_l1_fwd / _bwd) against float64 autograd at the VGG19 512^2 tap shapes, and
ide3d_b200.train_encoder's step, resume and streams against the script's structure (oracle/train_encoder.py)."""

import os
import tempfile

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
TAP_SHAPES = ((64, 512, 512), (128, 256, 256), (256, 128, 128), (512, 64, 64), (512, 32, 32))     # VGG19 (2, 7, 12, 21, 30) at 512^2
WEIGHTS = (1.0, 0.5, 2.0, 0.25, 1.5)


def _feats(n, channels_last, seed=0, ties=False):
    g = torch.Generator(device=DEV).manual_seed(seed)
    fx, fy = [], []
    for c, h, w in TAP_SHAPES:
        x = torch.relu(torch.randn(n, c, h, w, device=DEV, generator=g))
        y = torch.relu(torch.randn(n, c, h, w, device=DEV, generator=g))
        if ties:
            y = torch.where(torch.rand(x.shape, device=DEV, generator=g) < 0.3, x, y)
        if channels_last:
            x, y = x.contiguous(memory_format=torch.channels_last), y.contiguous(memory_format=torch.channels_last)
        fx.append(x.requires_grad_(True))
        fy.append(y)
    return fx, fy


def _reference(fx, fy, g=1.0):
    x64 = [x.detach().double().requires_grad_(True) for x in fx]
    total = sum(w * torch.nn.functional.l1_loss(x, y.double()) for x, y, w in zip(x64, fy, WEIGHTS))
    grads = torch.autograd.grad(total * g, x64)
    return total.item(), grads


@pytest.mark.parametrize('n', [1, 8])
@pytest.mark.parametrize('channels_last', [False, True])
def test_feat_l1_matches_float64_autograd(n, channels_last):
    from ide3d_b200 import _lib as L
    from ide3d_b200.torch_utils.ops.vgg_loss import feat_l1
    fx, fy = _feats(n, channels_last, seed=n, ties=True)
    c0 = L.launch_count()
    total, layers = feat_l1(fx, fy, WEIGHTS)
    c1 = L.launch_count()
    (total * 0.7).backward()
    c2 = L.launch_count()
    assert (c1 - c0, c2 - c1) == (2, 1)
    ref, ref_g = _reference(fx, fy, 0.7)
    assert abs(total.item() - ref) <= 1e-6 * abs(ref)
    for l, (x, y) in enumerate(zip(fx, fy)):
        assert abs(layers[l].item() - torch.nn.functional.l1_loss(x.detach().double(), y.double()).item()) <= 1e-6 * layers[l].item()
        assert x.grad.is_contiguous(memory_format=torch.channels_last if channels_last else torch.contiguous_format)
        assert torch.equal(x.grad.double(), ref_g[l].to(torch.float32).double()) or \
            (x.grad.double() - ref_g[l]).abs().max() <= 1e-6 * ref_g[l].abs().max()
        tie = x.detach() == y
        assert tie.any() and bool((x.grad[tie] == 0).all())


def test_feat_l1_rerun_bit_identical_and_mixed_layouts():
    from ide3d_b200.torch_utils.ops.vgg_loss import feat_l1
    fx, fy = _feats(2, False, seed=3)
    a = feat_l1(fx, fy, WEIGHTS)
    b = feat_l1(fx, fy, WEIGHTS)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    ga = torch.autograd.grad(a[0], fx)
    gb = torch.autograd.grad(b[0], fx)
    assert all(torch.equal(p, q) for p, q in zip(ga, gb))
    mixed_y = [y.contiguous(memory_format=torch.channels_last) for y in fy]          # the strided walk
    c = feat_l1(fx, mixed_y, WEIGHTS)
    gc = torch.autograd.grad(c[0], fx)
    ref, ref_g = _reference(fx, fy)
    assert abs(c[0].item() - ref) <= 1e-6 * abs(ref)
    assert all((p.double() - q).abs().max() <= 1e-6 * q.abs().max() for p, q in zip(gc, ref_g))


def _layer(shape, kind, g):
    """A [n, c, h, w] fp32 tensor laid out for one walk of the kernel: 'dense' (contiguous), 'misaligned' (dense, 4 bytes past a
    16-byte boundary: the scalar flat walk), 'view' (a slice of a wider tensor: the strided walk)."""
    n, c, h, w = shape
    if kind == 'dense':
        return torch.randn(shape, device=DEV, generator=g)
    if kind == 'misaligned':
        return torch.randn(n * c * h * w + 1, device=DEV, generator=g)[1:].view(shape)
    return torch.randn(n, c, h, w + 3, device=DEV, generator=g)[..., 2:w + 2]


@pytest.mark.parametrize('kind', ['dense', 'misaligned', 'view'])
def test_feat_l1_scalar_and_strided_walks_with_partial_ctas(kind):
    """Odd sizes (numel not a multiple of 4 or of the 4096-element tile) and a layer whose float4 walk ends in a partial CTA: the
    kernel pair against float64 autograd, with 0 on ties, in 2 + 1 launches."""
    from ide3d_b200 import _lib as L
    from ide3d_b200.torch_utils.ops.vgg_loss import feat_l1
    shapes = ((3, 3, 5, 7), (3, 2, 9, 11), (3, 64, 33, 33), (3, 1, 1, 1))
    weights = (1.0, 0.5, 2.0, 0.25)
    g = torch.Generator(device=DEV).manual_seed(11)
    fx = [_layer(s, kind, g).requires_grad_(True) for s in shapes]
    fy = []
    for x in fx:
        y = _layer(tuple(x.shape), kind, g)
        with torch.no_grad():
            y.copy_(torch.where(torch.rand(x.shape, device=DEV, generator=g) < 0.3, x, y))
        fy.append(y)
    c0 = L.launch_count()
    total, layers = feat_l1(fx, fy, weights)
    c1 = L.launch_count()
    total.backward()
    assert (c1 - c0, L.launch_count() - c1) == (2, 1)
    x64 = [x.detach().double().requires_grad_(True) for x in fx]
    ref = sum(w * torch.nn.functional.l1_loss(x, y.double()) for x, y, w in zip(x64, fy, weights))
    ref_g = torch.autograd.grad(ref, x64)
    assert abs(total.item() - ref.item()) <= 1e-6 * abs(ref.item())
    for l, (x, y) in enumerate(zip(fx, fy)):
        assert abs(layers[l].item() - torch.nn.functional.l1_loss(x.detach().double(), y.double()).item()) <= 1e-6 * layers[l].item()
        assert (x.grad.double() - ref_g[l]).abs().max() <= 1e-6 * ref_g[l].abs().max()
        assert bool((x.grad[x.detach() == y] == 0).all())


def test_feat_l1_refused_tables_fall_back_to_torch():
    from ide3d_b200 import _lib as L
    from ide3d_b200.torch_utils.ops.vgg_loss import feat_l1, feat_l1_torch
    g = torch.Generator(device=DEV).manual_seed(0)
    fx = [torch.randn(2, 4, 8, 8, device=DEV, generator=g).requires_grad_(True) for _ in range(9)]
    fy = [torch.randn(2, 4, 8, 8, device=DEV, generator=g) for _ in range(9)]
    c0 = L.launch_count()
    got = feat_l1(fx, fy, [1.0] * 9)
    assert L.launch_count() == c0
    assert torch.equal(got[0], feat_l1_torch(fx, fy, [1.0] * 9)[0])
    half = feat_l1([x.detach().half() for x in fx[:2]], [y.half() for y in fy[:2]], [1.0, 1.0])
    assert L.launch_count() == c0 and half[0].dtype == torch.float16


def _setup(lambdas_real=True):
    from ide3d_b200.arcface import Backbone, IDLoss
    from ide3d_b200.encoder import HybridEncoder
    from ide3d_b200.parsing import BiSeNet
    from ide3d_b200.torch_utils.ops.vgg_loss import VGGLoss
    from oracle import edit as oe, finetune as of, pti as opti, train_encoder as ot
    torch.manual_seed(0)
    parser = BiSeNet(20)
    parser.load_state_dict(of.bisenet_state(parser))
    parser = parser.eval().requires_grad_(False).to(DEV)
    E = HybridEncoder(**oe.ENCODER_ARGS)
    E.load_state_dict(oe.encoder_state(E))
    G = oe.standin_generator().to(DEV)
    irse = Backbone(112, 50, mode='ir_se', drop_ratio=0.6)
    irse.load_state_dict(ot.irse50_state(irse))
    mods = dict(vgg=VGGLoss(ot.standin_vgg19().features).to(DEV), lpips=opti.standin_lpips().to(DEV), id_net=IDLoss(irse).to(DEV))
    return G, E.to(DEV), parser, mods


LAMBDAS = dict(vgg=0.8, l2=1.0, lpips=0.6, id=0.4, entropy=0.5, cycle=2.0)


def _inputs(G, portraits, n=2):
    from ide3d_b200.train_encoder import PortraitDataset, cam_sampler
    rs = np.random.RandomState(0)
    z = torch.from_numpy(rs.randn(n, G.w_dim)).float().to(DEV)
    cam = cam_sampler(n, DEV, torch.Generator(DEV).manual_seed(0))
    ds = PortraitDataset(portraits[0], portraits[1], 512)
    items = [ds[i] for i in range(n)]
    real = tuple(torch.stack([it[k] for it in items]).to(DEV) for k in range(3))
    return z, cam, real


@pytest.fixture(scope='module')
def portraits():
    from oracle import train_encoder as ot
    with tempfile.TemporaryDirectory() as d:
        yield ot.write_portraits(d)


def test_first_step_matches_script_structure(portraits):
    """step_losses against oracle.train_encoder.reference_step (the full E twice per branch, BiSeNet twice per image, float one-hot
    masks, torch's heads) on the same latents, cameras and real batch, fp32 convolutions: losses and E's gradients."""
    import copy
    from ide3d_b200.train_encoder import _Encode, step_losses
    from oracle import train_encoder as ot
    G, E, parser, mods = _setup()
    z, cam, real = _inputs(G, portraits)
    w_avg = G.mapping.w_avg[None, None, :]
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        E1, E2 = copy.deepcopy(E).requires_grad_(True), copy.deepcopy(E).requires_grad_(True)
        got = step_losses(G, _Encode(E1), parser=parser, lambdas=LAMBDAS, z=z, cam=cam, real=real, start_from_latent_avg=True, **mods)
        sum(got.values()).backward()
        ref = ot.reference_step(G, E2, parser, lambdas=LAMBDAS, w_avg=w_avg, z=z, cam=cam, real=real, start_from_latent_avg=True, **mods)
        sum(ref.values()).backward()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    assert list(got) == list(ref)
    e_loss = max(abs(got[k].item() - ref[k].item()) for k in got) / max(abs(v.item()) for v in ref.values())
    g1 = torch.cat([p.grad.reshape(-1) for p in E1.parameters()])
    g2 = torch.cat([p.grad.reshape(-1) for p in E2.parameters()])
    e_grad = ((g1 - g2).abs().max() / g2.abs().max()).item()
    print(f'losses {e_loss:.2e} of max|loss|, E gradients {e_grad:.2e} of max|g|')
    assert e_loss <= 2e-6 and e_grad <= 1e-4                    # measured 3.4e-7 and 1.2e-5


def test_resume_equals_straight_run(portraits):
    from ide3d_b200.train_encoder import PortraitDataset, train
    G, E, parser, mods = _setup()
    ds = PortraitDataset(portraits[0], portraits[1], 512)
    lambdas = dict(vgg=0.8, l2=1.0, lpips=0.6, cycle=2.0)       # no BiSeNet or adaptive-pool backward: those use atomics
    kw = dict(parser=parser, batch=2, lambdas=lambdas, train_real=True, dataset=ds, start_from_latent_avg=True, **mods)
    det = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    try:
        with tempfile.TemporaryDirectory() as d:
            E4, l4 = train(G, E, steps=4, **kw)
            _, l2 = train(G, E, steps=2, snapshot_every=2, outdir=d, **kw)
            path = os.path.join(d, 'encoder-snapshot-000002.pt')
            assert os.path.isfile(path)
            E22, l22 = train(G, None, steps=2, resume=path, **kw)
    finally:
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = det
    # torch's pooling and interpolation backward kernels accumulate with atomics even under deterministic cuDNN, so the two runs
    # agree to rounding on the device (measured: weights 3.3e-5 of max|w|, losses 2.2e-4); tests/test_train_encoder.py checks the
    # resume bit for bit on the CPU
    wmax = max(v.abs().max().item() for v in E4.state_dict().values())
    e_w = max((a - b).abs().max().item() for a, b in zip(E4.state_dict().values(), E22.state_dict().values())) / wmax
    e_l = max(np.abs(l4[k] - np.concatenate([l2[k], l22[k]])).max() / max(np.abs(l4[k]).max(), 1e-30) for k in l4)
    print(f'resume: weights {e_w:.2e} of max|w|, losses {e_l:.2e}')
    assert e_w <= 1e-4 and e_l <= 1e-3


def test_camera_stream_equals_cam_sampler_in_sequence():
    from ide3d_b200 import train_encoder as T
    from oracle import edit as oe
    G = oe.standin_generator().to(DEV)
    seen = []
    step_losses = T.step_losses

    def spy(G, enc, **kw):
        seen.append(kw['cam'])
        zero = (enc('appearance', torch.zeros(1, 3, 512, 512, device=DEV)) * 0).sum()
        return {k: zero for k in T.GEN_LOSSES}
    T.step_losses = spy
    try:
        T.train(G, parser=None, steps=3, batch=2)
    finally:
        T.step_losses = step_losses
    g = torch.Generator(DEV).manual_seed(0)
    for c in seen:
        assert torch.equal(c, T.cam_sampler(2, DEV, g))


def _ddp_worker(rank, world, port, path, out):
    import torch.distributed as dist
    from ide3d_b200.train_encoder import _Encode, step_losses
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device('cuda', rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    try:
        from torch.nn.parallel import DistributedDataParallel
        data = torch.load(path, weights_only=False)
        G, E, parser = data['G'].to(dev), data['E'].to(dev).requires_grad_(True), data['parser'].to(dev)
        enc = DistributedDataParallel(_Encode(E), device_ids=[dev], broadcast_buffers=False)
        sl = slice(rank * data['n'], (rank + 1) * data['n'])
        loss = step_losses(G, enc, parser=parser, lambdas=dict(l2=1.0, entropy=0.5, cycle=2.0), z=data['z'][sl].to(dev),
                           cam=data['cam'][sl].to(dev), start_from_latent_avg=True)
        sum(loss.values()).backward()
        if rank == 0:
            torch.save([p.grad.cpu() for p in E.parameters()], out)
    finally:
        dist.destroy_process_group()


def test_ddp_world2_matches_world1():
    """One DDP step at world 2 on 2B samples gives world 1's gradient on the same 2B samples (every term is a batch mean)."""
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 visible GPUs')
    import socket
    import torch.multiprocessing as mp
    from ide3d_b200.train_encoder import _Encode, cam_sampler, step_losses
    G, E, parser, _ = _setup()
    n = 2
    z = torch.randn(2 * n, G.w_dim, device=DEV, generator=torch.Generator(DEV).manual_seed(1))
    cam = cam_sampler(2 * n, DEV, torch.Generator(DEV).manual_seed(2))
    with tempfile.TemporaryDirectory() as d:
        path, out = os.path.join(d, 'in.pt'), os.path.join(d, 'out.pt')
        torch.save(dict(G=G.cpu(), E=E.cpu(), parser=parser.cpu(), z=z.cpu(), cam=cam.cpu(), n=n), path)
        with socket.socket() as s:
            s.bind(('127.0.0.1', 0))
            port = s.getsockname()[1]
        mp.start_processes(_ddp_worker, args=(2, port, path, out), nprocs=2, join=True, start_method='spawn')
        g2 = torch.load(out)
    G, E, parser = G.to(DEV), E.to(DEV).requires_grad_(True), parser.to(DEV)
    loss = step_losses(G, _Encode(E), parser=parser, lambdas=dict(l2=1.0, entropy=0.5, cycle=2.0), z=z, cam=cam, start_from_latent_avg=True)
    sum(loss.values()).backward()
    g1 = torch.cat([p.grad.reshape(-1).cpu() for p in E.parameters()])
    g2 = torch.cat([g.reshape(-1) for g in g2])
    assert ((g1 - g2).abs().max() / g1.abs().max()).item() <= 1e-3
