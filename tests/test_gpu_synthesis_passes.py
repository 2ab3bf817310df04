"""GPU: the ToRGB layer folded into the last epilogue of a block and the styles chained across blocks (networks.FUSED_TORGB,
ide3d_modconv_epilogue_rgb).  The kernel against the composition it replaces (epilogue -> x * s_rgb -> fp32 1x1 convolution ->
bias) at the shapes of the two super-resolution blocks; G.synthesis with the switch on and off; the standalone block contract;
the gradient path; the fall-back for shapes the kernel does not take."""

import math

import pytest
import torch

from conftest import assert_close

pytestmark = pytest.mark.gpu
DEV = 'cuda'
LABEL = [1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 2.7, 0, 0, 0, 1, 4.2647, 0, 0.5, 0, 4.2647, 0.5, 0, 0, 1]


def _operands(n, c, res, o=3, seed=0, noise='const'):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, c, res, res, generator=g).to(DEV).contiguous(memory_format=torch.channels_last)
    scale = (torch.rand(n, c, generator=g) + 0.5).to(DEV)
    b = (torch.randn(c, generator=g) * 0.1).to(DEV)
    nz = None if noise is None else (torch.randn(res, res, generator=g) * 0.1).to(DEV)
    s_next = torch.randn(n, c, generator=g).to(DEV)
    w = torch.randn(o, c, 1, 1, generator=g).to(DEV)
    s_rgb = (torch.randn(n, c, generator=g) / math.sqrt(c)).to(DEV)
    b_rgb = torch.randn(o, generator=g).to(DEV)
    return x, scale, nz, b, s_next, w, s_rgb, b_rgb


def _composed(x, scale, nz, b, s_next, w, s_rgb, b_rgb):
    from ide3d_b200.torch_utils.ops import bias_act
    t = bias_act.scaled_bias_act(x, scale=scale, noise=nz, b=b, act='lrelu')
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        rgb = torch.nn.functional.conv2d(t * s_rgb[:, :, None, None], w) + b_rgb[None, :, None, None]
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    return t, t * s_next[:, :, None, None], rgb.contiguous()


@pytest.mark.parametrize('c,res', [(128, 256), (64, 512), (64, 256), (128, 128)])
@pytest.mark.parametrize('noise', [None, 'const'])
@torch.no_grad()
def test_kernel_matches_epilogue_then_1x1_conv(c, res, noise):
    from ide3d_b200.torch_utils.ops import bias_act
    ops = _operands(3, c, res, noise=noise)                                  # odd batch
    x, scale, nz, b, s_next, w, s_rgb, b_rgb = ops
    t_ref, y2_ref, rgb_ref = _composed(*ops)
    y, y2, rgb = bias_act.scaled_bias_act(x, scale=scale, noise=nz, b=b, act='lrelu', next_scale=s_next, rgb=(w, s_rgb, b_rgb))
    assert rgb.shape == (3, 3, res, res) and rgb.is_contiguous()
    assert torch.equal(y, t_ref) and torch.equal(y2, y2_ref)                   # same per-element arithmetic as the epilogue
    assert_close(rgb, rgb_ref, atol=1e-5 * rgb_ref.abs().max().item(), what='rgb')
    # the other output subsets, and bit-identical reruns
    ys, rgb2 = bias_act.scaled_bias_act(x, scale=scale, noise=nz, b=b, act='lrelu', y_scale=s_next, rgb=(w, s_rgb, b_rgb))
    assert torch.equal(ys, y2_ref) and torch.equal(rgb2, rgb)
    (only,) = bias_act.scaled_bias_act(x, scale=scale, noise=nz, b=b, act='lrelu', emit_y=False, rgb=(w, s_rgb, b_rgb))
    assert torch.equal(only, rgb)


@pytest.mark.parametrize('c', [4, 96, 256, 512])
@torch.no_grad()
def test_kernel_other_widths(c):
    """C/4 not a power of two <= 32: the shared-memory reduction; still fixed-order (rerun bit-identical)."""
    from ide3d_b200.torch_utils.ops import bias_act
    ops = _operands(3, c, 40, o=4, seed=c)
    x, scale, nz, b, s_next, w, s_rgb, b_rgb = ops
    t_ref, _, rgb_ref = _composed(*ops)
    y, rgb = bias_act.scaled_bias_act(x, scale=scale, noise=nz, b=b, act='lrelu', rgb=(w, s_rgb, b_rgb))
    assert torch.equal(y, t_ref)
    assert_close(rgb, rgb_ref, atol=1e-5 * rgb_ref.abs().max().item(), what=f'rgb C={c}')
    _, again = bias_act.scaled_bias_act(x, scale=scale, noise=nz, b=b, act='lrelu', rgb=(w, s_rgb, b_rgb))
    assert torch.equal(again, rgb)


@pytest.mark.parametrize('case', ['odd_channels', 'nchw', 'fp16', 'five_outputs'])
@torch.no_grad()
def test_unsupported_shapes_fall_back(case):
    from ide3d_b200 import _plugins
    from ide3d_b200.torch_utils.ops import bias_act
    c, o = (6, 3) if case == 'odd_channels' else (8, 5 if case == 'five_outputs' else 3)
    ops = list(_operands(2, c, 16, o=o, seed=1))
    if case == 'nchw':
        ops[0] = ops[0].contiguous()
    if case == 'fp16':
        ops[0] = ops[0].half()
    x, scale, nz, b, s_next, w, s_rgb, b_rgb = ops
    assert _plugins.modconv_epilogue_rgb(x, scale, nz, b, 3, 0.2, math.sqrt(2), -1.0, rgb=(w, s_rgb, b_rgb)) is None
    t_ref, _, _ = _composed(*ops)
    # the composition's 1x1 convolution is cuDNN's: fp32 here, so that it can be held to the fp32 reference
    y, rgb = _switch(True, lambda: bias_act.scaled_bias_act(x, scale=scale, noise=nz, b=b, act='lrelu', rgb=(w, s_rgb, b_rgb)))
    assert torch.equal(y, t_ref) and rgb.shape == (2, o, 16, 16) and rgb.dtype == x.dtype
    _, _, rgb_ref = _composed(x.float(), scale, nz, b, s_next, w, s_rgb, b_rgb)
    assert_close(rgb.float(), rgb_ref, atol=(3e-3 if case == 'fp16' else 1e-5) * rgb_ref.abs().max().item(), what=case)


@pytest.fixture(scope='module')
def small_g():
    from ide3d_b200.training.triplane import TriPlaneGenerator
    torch.manual_seed(0)
    G = TriPlaneGenerator(z_dim=32, w_dim=32, img_resolution=128, plane_resolution=64, render_size=32, channel_base=2048, channel_max=64,
                          sr_channels=(32, 32), mapping_kwargs=dict(num_layers=2)).eval().requires_grad_(False)
    for name, p in G.named_parameters():
        if name.endswith('noise_strength'):
            p.data.fill_(0.1)
    G = G.to(DEV)
    z = torch.randn(3, G.z_dim, generator=torch.Generator().manual_seed(5)).to(DEV)
    c = torch.tensor(LABEL).repeat(3, 1).to(DEV)
    c[1, 3] = 0.15
    with torch.no_grad():
        ws = G.mapping(z, c, truncation_psi=0.7)
    return G, ws, c


def _switch(fused, fn):
    """fn() with the fold on / off, fp32 convolutions and deterministic cuDNN algorithms (at these small shapes cuDNN may otherwise
    pick algorithms whose sums change from call to call, which would hide what the fold itself does)."""
    from ide3d_b200.training import networks as nw
    saved = (nw.FUSED_TORGB, torch.backends.cudnn.allow_tf32, torch.backends.cudnn.deterministic)
    try:
        nw.FUSED_TORGB = fused
        torch.backends.cudnn.allow_tf32, torch.backends.cudnn.deterministic = False, True
        return fn()
    finally:
        nw.FUSED_TORGB, torch.backends.cudnn.allow_tf32, torch.backends.cudnn.deterministic = saved


@pytest.mark.parametrize('views,return_seg', [(1, False), (1, 'raw'), (3, False), (3, 'raw')])
@torch.no_grad()
def test_synthesis_switch_on_off(small_g, views, return_seg):
    G, ws, c = small_g
    cams = c.repeat_interleave(views, 0)
    if views > 1:
        cams[1::views, 3] += 0.1
    run = lambda: G.synthesis(ws, c=cams, noise_mode='const', num_steps=16, perturb=None, views=views, return_seg=return_seg)
    off, on = _switch(False, run), _switch(True, run)
    if return_seg:
        (off, seg_off), (on, seg_on) = off, on
        assert_close(seg_on, seg_off, atol=1e-6 * seg_off.abs().max().item(), what='seg_raw')   # same planes: x * s0 is the same product
    assert on.shape == (ws.shape[0] * views, 3, 128, 128)
    assert_close(on, off, atol=1e-5 * off.abs().max().item(), what='image')
    again = _switch(True, run)
    assert torch.equal(on, again[0] if return_seg else again)    # bit-identical reruns


@torch.no_grad()
def test_standalone_block_returns_plain_x(small_g):
    """`x, img = block(x, img, ws)` keeps its meaning: the plain x (same bits as the unfused path), and the same image."""
    G, ws, c = small_g
    blk = G.synthesis.b128
    g = torch.Generator().manual_seed(2)
    x = torch.randn(3, blk.in_channels, 64, 64, generator=g).to(DEV).contiguous(memory_format=torch.channels_last)
    img = torch.randn(3, 3, 64, 64, generator=g).to(DEV)
    w = ws[:, -3:]
    x_off, img_off = _switch(False, lambda: blk(x, img.clone(), w, noise_mode='const'))
    x_on, img_on = _switch(True, lambda: blk(x, img.clone(), w, noise_mode='const'))
    assert_close(x_on, x_off, atol=1e-6 * x_off.abs().max().item(), what='x')      # the same epilogue arithmetic
    assert_close(img_on, img_off, atol=1e-5 * img_off.abs().max().item(), what='img')


def test_gradients_unchanged(small_g):
    """With gradients enabled the blocks take the unfused composition whatever the switch says."""
    G, ws, c = small_g

    def grad():
        w = ws.detach().clone().requires_grad_(True)
        img = G.synthesis(w, c=c, noise_mode='const', num_steps=16, perturb=None)
        img.square().mean().backward()
        return img.detach(), w.grad

    (i_off, g_off), (i_on, g_on) = _switch(False, grad), _switch(True, grad)
    assert_close(i_on, i_off, atol=1e-6 * i_off.abs().max().item(), what='image')
    assert_close(g_on, g_off, atol=1e-6 * g_off.abs().max().item(), what='d image / d ws')     # cuDNN backward may reorder sums
