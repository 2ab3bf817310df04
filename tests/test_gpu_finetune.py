"""GPU: encoder fine-tuning -- ide3d_seg_stem_bwd (csrc/seg_stem.cu), the align_corners=True cross-entropy and labels, BiSeNet and
ide3d_b200.finetune.run.

  * ide3d_seg_stem_bwd against float64 autograd through the composition at C0 = 32 and 64, N = 1 and 3, five mask kinds, for the
    one_hot * 2 - 1 input and the {0, 1} re-parameterisation; bit-identical reruns; three launches
  * E.geometry(uint8) under grad takes the kernel and matches the float one-hot composition's parameter gradients
  * ide3d_seg_xent_*_ac / ide3d_seg_labels_ac against F.interpolate(align_corners=True) then cross_entropy / argmax
  * BiSeNet on the device against the CPU module
  * finetune.run with the bench generator: its first step against the reference's structure, 20 steps lower the loss, the caller's
    models untouched, only the geometry branch tuned, no stale cache, and the returned mask"""

import copy

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')
KINDS = ['random', 'blocky', 'one_class', 'out_of_range', 'borders']


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


@pytest.fixture
def fp32_convolutions():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _layers(c0, seed):
    from ide3d_b200.encoder import Conv2dLayer, EncoderResBlock
    torch.manual_seed(seed)
    stem, block = Conv2dLayer(19, c0, 1), EncoderResBlock(c0, 2 * c0)
    for m in (stem, block):
        for p in m.parameters():
            if p.ndim == 1:
                p.data.normal_(0, 0.3)
    return stem.to(DEV), block.to(DEV)


def _masks(kind, n, size, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    if kind == 'random':
        return torch.randint(0, 19, (n, size, size), device=DEV, generator=g, dtype=torch.uint8)
    if kind == 'blocky':
        b = torch.randint(0, 19, (n, size // 16, size // 16), device=DEV, generator=g, dtype=torch.uint8)
        return b.repeat_interleave(16, 1).repeat_interleave(16, 2).contiguous()
    if kind == 'one_class':
        return torch.full((n, size, size), 13, device=DEV, dtype=torch.uint8)
    if kind == 'out_of_range':
        return torch.randint(0, 256, (n, size, size), device=DEV, generator=g, dtype=torch.uint8)
    m = torch.randint(0, 19, (n, size, size), device=DEV, generator=g, dtype=torch.uint8)
    m[:, :2, :], m[:, -2:, :], m[:, :, :2], m[:, :, -2:] = 18, 4, 200, 1
    return m


def _params(stem, block):
    return [stem.weight, stem.bias, block.conv1.weight, block.conv1.bias, block.skip.weight]


def _reference_grads(mask, stem, block, gy, gs, signed, y1):
    """float64 autograd through the composition.  conv1's lrelu derivative is taken where the kernel's y1 is positive (bias_act's own
    rule, y > 0): at a pre-activation within rounding of zero the fp32 and float64 forwards can fall on different sides, and for a
    random mask one such pixel moves gb1 by 2e-3 of its max."""
    from ide3d_b200.encoder import one_hot_input
    s64, b64 = copy.deepcopy(stem).double(), copy.deepcopy(block).double()
    for m in (s64, b64.conv1, b64.conv2, b64.skip):
        m.resample_filter = m.resample_filter.float()
    b64.conv1.activation, b64.conv1.act_gain = 'linear', 1.0
    x = one_hot_input(mask, 19, torch.float64)
    x = s64(x if signed else (x + 1) / 2)
    gz = gy.double() * 2 ** 0.5 * torch.where(y1 > 0, 1.0, 0.2).double()
    loss = (b64.conv1(x) * gz).sum() + (b64.skip(x) * gs.double()).sum()
    return torch.autograd.grad(loss, _params(s64, b64))


def _kernel_grads(mask, stem, block, gy, gs, signed):
    from ide3d_b200 import _lib
    from ide3d_b200.encoder import _UnsignedStem
    from ide3d_b200.torch_utils.ops import seg_stem
    y1, sk = seg_stem.seg_stem(mask, stem if signed else _UnsignedStem(stem), block.conv1, block.skip)
    loss = (y1 * gy).sum() + (sk * gs).sum()
    n0 = _lib.launch_count()
    grads = torch.autograd.grad(loss, _params(stem, block))
    return grads, _lib.launch_count() - n0, y1.detach()


@pytest.mark.parametrize('c0, size', [(32, 512), (64, 256)])
@pytest.mark.parametrize('n', [1, 3])
@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('signed', [True, False])
def test_seg_stem_bwd_matches_float64_composition(c0, size, n, kind, signed):
    stem, block = _layers(c0, c0 + n)
    mask = _masks(kind, n, size, seed=n + 7)
    if kind == 'random' and n == 3:
        mask = mask.transpose(1, 2)                                                       # any strides
    g = torch.Generator(device=DEV).manual_seed(c0 + n)
    gy = torch.randn(n, c0, size, size, device=DEV, generator=g)
    gs = torch.randn(n, 2 * c0, size // 2, size // 2, device=DEV, generator=g)
    got, launches, y1 = _kernel_grads(mask, stem, block, gy, gs, signed)
    again, _, _ = _kernel_grads(mask, stem, block, gy, gs, signed)
    ref = _reference_grads(mask, stem, block, gy, gs, signed, y1)
    errs = [rel(a, b) for a, b in zip(got, ref)]
    print(f'C0 {c0} n {n} {kind} signed={signed}: w0 {errs[0]:.1e} b0 {errs[1]:.1e} w1 {errs[2]:.1e} b1 {errs[3]:.1e} '
          f'ws {errs[4]:.1e} of max|g|')
    assert max(errs) <= 1e-5
    assert all(torch.equal(a, b) for a, b in zip(got, again))
    assert launches == 3


def test_geometry_under_grad_takes_the_kernel(fp32_convolutions, monkeypatch):
    from ide3d_b200.encoder import HybridEncoder, one_hot_input
    from ide3d_b200.torch_utils.ops import seg_stem
    torch.manual_seed(2)
    E = HybridEncoder(512, 2, 8, w_dim=16)
    for p in E.parameters():
        if p.ndim == 1:
            p.data.normal_(0, 0.2)
    E = E.to(DEV)
    calls = []
    real = seg_stem.seg_stem
    monkeypatch.setattr(seg_stem, 'seg_stem', lambda *a, **k: calls.append(1) or real(*a, **k))
    mask = torch.cat([_masks('blocky', 1, 512, 3), _masks('borders', 1, 512, 4)])
    r = torch.randn(2, 8, 16, device=DEV, generator=torch.Generator(device=DEV).manual_seed(5))
    params = list(E.convs_seg.parameters()) + list(E.projector_seg.parameters())
    got = torch.autograd.grad((E.geometry(mask) * r).sum(), params)
    assert calls == [1]
    ref = torch.autograd.grad((E.geometry(one_hot_input(mask, 19)) * r).sum(), params)
    errs = [rel(a, b) for a, b in zip(got, ref)]
    print(f'geometry under grad, kernel vs composition: worst {max(errs):.2e} of max|g| per tensor')
    assert max(errs) <= 3e-3                                                               # measured 2.7e-4


def _logits(n, c, h, w, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(n, c, h, w, device=DEV, generator=g) * 2


@pytest.mark.parametrize('shape', [(1, 20, 64, 64, 512, 512), (2, 20, 16, 24, 61, 90), (1, 7, 1, 5, 9, 1)])
def test_ac_cross_entropy_and_labels(shape):
    from ide3d_b200.torch_utils.ops import projection, seg_stem
    n, c, h, w, oh, ow = shape
    seg = _logits(n, c, h, w, 1).requires_grad_(True)
    mask = torch.randint(0, c, (n, oh, ow), device=DEV, dtype=torch.uint8, generator=torch.Generator(device=DEV).manual_seed(2))
    loss = projection.seg_cross_entropy(seg, mask, align_corners=True)
    (grad,) = torch.autograd.grad(loss, seg)
    (grad2,) = torch.autograd.grad(projection.seg_cross_entropy(seg, mask, align_corners=True), seg)
    s64 = seg.detach().double().requires_grad_(True)
    up = F.interpolate(s64, (oh, ow), mode='bilinear', align_corners=True)
    ref = F.cross_entropy(up, mask.long())
    (gref,) = torch.autograd.grad(ref, s64)
    print(f'{shape}: CE {rel(loss, ref):.1e}, grad {rel(grad, gref):.1e}')
    assert rel(loss, ref) <= 1e-6 and rel(grad, gref) <= 1e-5
    assert torch.equal(grad, grad2)
    ids = seg_stem.seg_labels(seg.detach(), (oh, ow), align_corners=True)
    up = F.interpolate(seg.detach(), (oh, ow), mode='bilinear', align_corners=True)
    top2 = up.topk(min(2, c), dim=1).values
    decided = (top2[:, 0] - top2[:, -1]) > 1e-5
    differ = int((ids != up.argmax(1).to(torch.uint8)).sum())
    print(f'{shape}: labels differ at {differ} pixels, {int((~decided).sum())} within 1e-5 of a tie')
    assert torch.equal(ids[decided], up.argmax(1).to(torch.uint8)[decided])
    assert int((~decided).sum()) <= max(4, ids.numel() // 10000)


@pytest.fixture(scope='module')
def parser():
    from ide3d_b200.parsing import BiSeNet
    from oracle import finetune as of
    net = BiSeNet(20)
    net.load_state_dict(of.bisenet_state(net))
    return net.eval().requires_grad_(False)


def test_bisenet_on_device_matches_cpu(parser, fp32_convolutions):
    x = torch.rand(2, 3, 512, 512, generator=torch.Generator().manual_seed(3)) * 2 - 1
    with torch.no_grad():
        ref = parser.logits(x)
        got = copy.deepcopy(parser).to(DEV).logits(x.to(DEV))
    print(f'BiSeNet logits, device vs CPU: {rel(got.cpu(), ref):.2e} of max|ref|')
    assert rel(got.cpu(), ref) <= 1e-4


@pytest.fixture(scope='module')
def setup(parser):
    from ide3d_b200 import edit
    from ide3d_b200.compat import random_init_generator
    from ide3d_b200.encoder import HybridEncoder
    G = random_init_generator(device=DEV, seed=0)
    G.rendering_kwargs['perturb'] = None
    torch.manual_seed(1)
    E = HybridEncoder(512, G.num_ws - 8, 8, w_dim=G.w_dim)
    for p in E.parameters():
        if p.ndim == 1:
            p.data.normal_(0, 0.2)
    E = E.eval().requires_grad_(False).to(DEV)
    z = torch.from_numpy(__import__('numpy').random.RandomState(0).randn(1, G.z_dim)).float().to(DEV)
    label = torch.tensor(edit.FRONTAL, device=DEV).reshape(1, -1)
    with torch.no_grad():
        code = G.mapping(z, label)
        image = G.synthesis(code, label, noise_mode='const').clamp(-1, 1)
    code = code + 0.05 * torch.randn(code.shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(6))
    return G, E, image, code, label, copy.deepcopy(parser).to(DEV)


def test_first_step_matches_the_reference_structure(setup, monkeypatch, fp32_convolutions):
    """One step of finetune.run (kernel stem and its backward, one BiSeNet call on the render, the _ac tail) against one step in the
    reference's structure (composition stem under grad, full E twice, BiSeNet twice on the render, torch upsample + CE + argmax).
    With fp32 convolutions, measured: losses within 1.8e-5, gradients 9.4e-4 of their max (the two renders differ in the last bits,
    table vs composition stem, and the cycle's target is an argmax of the render's logits).  With TF32 the same comparison gives
    2.7e-3 and 6.5e-2."""
    from ide3d_b200 import finetune
    from ide3d_b200.encoder import one_hot_input
    from oracle import finetune as of
    G, E, image, code, label, parser = setup
    mask = _masks('blocky', 1, 512, 9)[0]
    captured = []

    class Capture(torch.optim.Adam):
        def step(self, closure=None):
            captured.append([p.grad.clone() for g in self.param_groups for p in g['params']])
            return super().step(closure)

    monkeypatch.setattr(torch.optim, 'Adam', Capture)
    _, _, losses = finetune.run(G, E, image, code, label, parser=parser, mask=mask, steps=1)
    E_ref = copy.deepcopy(E)
    params = list(E_ref.convs_seg.parameters()) + list(E_ref.projector_seg.parameters())
    for p in params:
        p.requires_grad_(True)
    ref = of.reference_step(copy.deepcopy(G).requires_grad_(False), E_ref, image, one_hot_input(mask[None], 19), code, label, parser,
                            G.mapping.w_avg[None, None, :])
    ref_grads = torch.autograd.grad(sum(ref.values()), params)
    e_loss = {k: abs(float(losses[k][0]) - float(v.detach())) / abs(float(v.detach())) for k, v in ref.items()}
    e_grad = max(rel(a, b) for a, b in zip(captured[0], ref_grads))
    print('first step vs reference structure: ' + ', '.join(f'{k} {v:.1e}' for k, v in e_loss.items()) + f'; gradients {e_grad:.2e}')
    assert max(e_loss.values()) <= 2e-4
    assert e_grad <= 1e-2


def test_finetune_run(setup):
    from ide3d_b200 import finetune
    from ide3d_b200.encoder import HybridEncoder
    from ide3d_b200.parsing import parse
    G, E, image, code, label, parser = setup
    e0 = {k: v.clone() for k, v in E.state_dict().items()}
    g0 = {k: v.clone() for k, v in G.state_dict().items()}
    E_t, mask, losses = finetune.run(G, E, image, code, label, parser=parser, steps=20)
    total = sum(losses[k] for k in finetune.LAMBDAS)
    print('summed loss per step: ' + ' '.join(f'{v:.4f}' for v in total))
    assert total.shape == (20,) and total[-1] < total[0]
    assert all(torch.equal(v, e0[k]) for k, v in E.state_dict().items())
    assert all(torch.equal(v, g0[k]) for k, v in G.state_dict().items())
    changed = {k for k, v in E_t.state_dict().items() if not torch.equal(v, e0[k])}
    assert changed and all(k.startswith(('convs_seg.', 'projector_seg.')) for k in changed)
    assert not E_t.training and not any(p.requires_grad for p in E_t.parameters())
    fresh = HybridEncoder(512, G.num_ws - 8, 8, w_dim=G.w_dim).to(DEV).eval()
    fresh.load_state_dict(E_t.state_dict())
    with torch.no_grad():
        target = parse(parser, image)
        assert torch.equal(E_t.geometry(target), fresh.geometry(target))
        rec = torch.cat((E_t.geometry(target) + G.mapping.w_avg, code[:, 8:]), 1)
        render = G.synthesis(rec, c=label, render_params=dict(finetune.RENDER_PARAMS), noise_mode='const')
    assert mask.dtype == torch.uint8 and mask.shape == (512, 512)
    assert torch.equal(mask, parse(parser, render)[0])
