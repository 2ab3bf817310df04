"""CPU: when the tri-plane backbone's convolutions run on fp16 operands (networks.fp16_operands).  Exactly when cuDNN may use TF32,
force_fp32 and the grouped convolution are off and every block can fold its neighbours' passes (NHWC, IDE3D_FUSED_TORGB, no
conv_clamp, no use_fp16 block); a block refuses the fp16 operands off the chained inference path."""

import pytest
import torch


@pytest.fixture
def net():
    from ide3d_b200.training.triplane import SynthesisNetwork
    torch.manual_seed(0)
    return SynthesisNetwork(w_dim=16, img_resolution=32, plane_resolution=16, render_size=8, channel_base=256, channel_max=16,
                            sr_channels=(8, 8)).eval().requires_grad_(False)


@pytest.fixture
def tf32():
    prev = torch.backends.cudnn.allow_tf32
    yield lambda on: setattr(torch.backends.cudnn, 'allow_tf32', on)
    torch.backends.cudnn.allow_tf32 = prev


def test_selected_exactly_under_tf32_and_the_folded_chain(net, tf32, monkeypatch):
    from ide3d_b200.training import networks
    blocks = [getattr(net, f'vb{r}') for r in net.voxel_block_resolutions]
    tf32(True)
    assert networks.fp16_operands(blocks)
    assert networks.fp16_operands(blocks, force_fp32=False, fused_modconv=False)
    assert not networks.fp16_operands(blocks, force_fp32=True)
    assert not networks.fp16_operands(blocks, fused_modconv=True)
    tf32(False)
    assert not networks.fp16_operands(blocks)
    tf32(True)
    for name in ('CHANNELS_LAST', 'FUSED_TORGB', 'CHAIN_MODULATION'):
        with monkeypatch.context() as m:
            m.setattr(networks, name, False)
            assert not networks.fp16_operands(blocks), name
    blocks[1].use_fp16 = True
    assert not networks.fp16_operands(blocks)
    blocks[1].use_fp16 = False
    blocks[-1].conv1.conv_clamp = 256
    assert not networks.fp16_operands(blocks)
    blocks[-1].conv1.conv_clamp = None
    assert networks.fp16_operands(blocks)


def test_a_block_refuses_fp16_operands_off_the_chained_path(net, tf32):
    tf32(True)
    b = net.vb4
    ws = torch.randn(2, b.num_conv + b.num_torgb, 16)
    with pytest.raises(RuntimeError, match='fp16 operands'):
        b._features(None, ws, False, False, {'fp16_operands': True})                     # no style plan
    ws.requires_grad_(True)
    with torch.enable_grad(), pytest.raises(RuntimeError, match='fp16 operands'):       # gradients: not the inference path
        b._features(None, ws, False, False, {'fp16_operands': True, 'style_plan': {}})


def test_the_style_plan_and_so_the_fp16_path_needs_inference_on_cuda(net, tf32):
    """SynthesisNetwork.forward passes fp16_operands only together with a style plan, and there is none on the CPU or with gradients."""
    tf32(True)
    ws = torch.randn(2, net.num_ws, 16)
    assert net._style_plan(ws, fp16_blocks=net._blocks()) is None
    ws.requires_grad_(True)
    with torch.enable_grad():
        assert net._style_plan(ws, fp16_blocks=net._blocks()) is None


def test_fp16_exponent_keeps_the_convolution_output_at_the_input_scale(net):
    """e = round(log2(sqrt(fan_in) * rms(W))): for the N(0, 1) initialisation that is log2(sqrt(9 C))."""
    import math
    for layer in (net.vb8.conv0, net.vb8.conv1, net.b32.conv1):
        fan_in = layer.weight[0].numel()
        rms = float(layer.weight.square().mean().sqrt())
        assert layer.fp16_exponent() == round(math.log2(math.sqrt(fan_in) * rms))
    layer = net.vb8.conv1
    with torch.no_grad():
        layer.weight.mul_(8.0)
    assert layer.fp16_exponent() == round(math.log2(math.sqrt(layer.weight[0].numel()) * float(layer.weight.square().mean().sqrt())))
