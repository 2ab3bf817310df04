"""GPU: the fp16 operand path of the tri-plane backbone's convolutions (networks.fp16_operands, DESIGN.md §2).

- Each epilogue on fp16 input equals its float32 instantiation applied to the same values upcast: every fp16 output is that float32
  result rounded once, and the float32 outputs (ToRGB, the skip sums) are bit-equal.  Shapes of the benchmark (8 samples): the
  backbone's, and the super-resolution blocks' (which the kernels take, though the generator keeps those blocks in float32).
- cuDNN's fp16 convolution accumulates in float32: against a float64 convolution of the same fp16 operands its error stays within the
  float32 accumulation bound plus one fp16 rounding of the output.
- The per-layer 2^-e weight scaling is exact: a layer's output with and without it is bit-equal on data whose intermediate values stay
  normal fp16 numbers.
"""

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = 'cuda'
N = 8


def _cl(t):
    return t.contiguous(memory_format=torch.channels_last)


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _rand(shape, seed, scale=1.0, dtype=torch.float32):
    return (torch.randn(shape, generator=_gen(seed), device=DEV) * scale).to(dtype)


@pytest.fixture(autouse=True)
def _no_grad():
    with torch.no_grad():
        yield


# (C, R): conv1 of vb64, vb128, vb256 (plus the 192-channel ToRGB inputs they write), and the two SR blocks with their folded ToRGB
@pytest.mark.parametrize('c,r,rgb', [(512, 64, False), (256, 128, False), (128, 256, False), (128, 256, True), (64, 512, True)])
def test_epilogue_rgb_fp16_is_the_fp32_result_rounded_once(c, r, rgb):
    from ide3d_b200.torch_utils.ops import bias_act
    x16 = _cl(_rand([N, c, r, r], 1, 4.0, torch.float16))
    d, b = _rand([N, c], 2).abs() + 0.5, _rand([c], 3, 0.1)
    noise = _rand([r, r], 4, 0.2)
    ys, s2 = _rand([N, c], 5), _rand([N, c], 6)
    kw = dict(scale=d, noise=noise, b=b, act='lrelu')
    if rgb:
        kw.update(y_scale=ys, rgb=(_rand([3, c, 1, 1], 7), _rand([N, c], 8, 0.05), _rand([3], 9)))
    else:
        kw.update(y_scale=ys, next_scale=s2)
    out16 = bias_act.scaled_bias_act(x16, fp32_tail=True, **kw)
    out32 = bias_act.scaled_bias_act(_cl(x16.float()), **kw)
    assert len(out16) == len(out32) == 2
    for a, ref in zip(out16, out32):
        if ref.shape[1] == c:
            assert a.dtype == torch.float16 and a.is_contiguous(memory_format=torch.channels_last)
            assert torch.equal(a, ref.half())
        else:
            assert a.dtype == torch.float32 and torch.equal(a, ref)


@pytest.mark.parametrize('c,r', [(512, 64), (256, 128), (128, 256), (128, 256), (64, 512)])
def test_fir_epilogue_fp16_is_the_fp32_result_rounded_once(c, r):
    """conv0's tail: FIR of the transposed convolution's output [N, C, R+1, R+1] -> R x R, x * dcoefs + noise + b, lrelu, * s1."""
    from ide3d_b200.torch_utils.ops import upfirdn2d
    f = upfirdn2d.setup_filter([1, 3, 3, 1]).to(DEV)
    x16 = _cl(_rand([N, c, r + 1, r + 1], 11, 4.0, torch.float16))
    kw = dict(padding=[1, 1, 1, 1], gain=4, scale=_rand([N, c], 12).abs() + 0.5, noise=_rand([r, r], 13, 0.2), b=_rand([c], 14, 0.1),
              act='lrelu', act_gain=2 ** 0.5, next_scale=_rand([N, c], 15), only_next=True)
    y16 = upfirdn2d.upfirdn2d_epilogue(x16, f, fp32_tail=True, **kw)
    y32 = upfirdn2d.upfirdn2d_epilogue(_cl(x16.float()), f, **kw)
    assert y16.dtype == torch.float16 and y16.shape == (N, c, r, r) and y16.is_contiguous(memory_format=torch.channels_last)
    assert torch.equal(y16, y32.half())


@pytest.mark.parametrize('c,r', [(512, 4), (32, 128), (512, 64), (128, 256)])
def test_linear_modulation_fp16_is_the_fp32_result_rounded_once(c, r):
    """`x * s0` in front of the first convolution of a chain (vb4's constant, b256's feature image)."""
    from ide3d_b200.torch_utils.ops import bias_act
    x = _cl(_rand([N, c, r, r], 21, 3.0))
    s = _rand([N, c], 22)
    y16 = bias_act.scaled_bias_act(x, scale=s, out_dtype=torch.float16)
    y32 = bias_act.scaled_bias_act(x, scale=s)
    assert y16.dtype == torch.float16 and y16.is_contiguous(memory_format=torch.channels_last)
    assert torch.equal(y16, y32.half())


@pytest.mark.parametrize('r', [8, 64, 256])
def test_skip_add_of_an_fp16_contribution(r):
    """upsample2d(img) + y + b with y the fp16 [img | seg] output of the backbone's 1x1 ToRGB (a channel slice) onto float32 img."""
    from ide3d_b200.torch_utils.ops import upfirdn2d
    f = upfirdn2d.setup_filter([1, 3, 3, 1]).to(DEV)
    img = _cl(_rand([N, 96, r // 2, r // 2], 31))
    y16 = _cl(_rand([N, 192, r, r], 32, 2.0, torch.float16))
    b = _rand([192], 33)
    for sl in (slice(0, 96), slice(96, 192)):
        out = upfirdn2d.upsample2d_add(img, f, y16[:, sl], b[sl])
        ref = upfirdn2d.upsample2d_add(img, f, y16[:, sl].float(), b[sl])
        assert out.dtype == torch.float32 and torch.equal(out, ref)


@pytest.mark.parametrize('c,r', [(128, 256), (64, 512)])
def test_cudnn_fp16_convolution_accumulates_in_fp32(c, r):
    """vb256 conv1 and b512 conv1 (3x3, stride 1, NHWC) as the synthesis runs them.  Bound per output: one fp16 rounding of the result
    (2^-11 relative) plus K * 2^-24 * sum|x w| for a float32 sum of K = 9C products.  An fp16 accumulator would typically be off by
    sqrt(K) * 2^-11 of sum|x w|, over 200x the second term here (K = 576, 1152)."""
    n = 2
    x = _cl(_rand([n, c, r, r], 41, 1.0, torch.float16))
    w = _cl(_rand([c, c, 3, 3], 42, 1.0 / 16, torch.float16))
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    try:
        y = torch.nn.functional.conv2d(x, w, padding=1)
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    assert y.dtype == torch.float16
    ref = torch.nn.functional.conv2d(x.double(), w.double(), padding=1)
    mag = torch.nn.functional.conv2d(x.double().abs(), w.double().abs(), padding=1)
    k = 9 * c
    err = (y.double() - ref).abs()
    bound = ref.abs() * 2.0 ** -11 + k * 2.0 ** -24 * mag
    assert bool((err <= bound).all()), float((err - bound).max())


@pytest.mark.parametrize('up', [1, 2])
def test_power_of_two_weight_scaling_is_exact(up):
    """A SynthesisLayer on the fp16 path with its weight copy W * 2^-e and dcoefs * 2^e against the same layer with e = 0.  W, x and
    styles are positive fp16 numbers, so every convolution output is a normal fp16 number in both runs."""
    from ide3d_b200.training import networks
    c, r = 128, 64
    torch.manual_seed(0)
    layer = networks.SynthesisLayer(c, c, w_dim=16, resolution=r, up=up, channels_last=True).to(DEV).eval()
    layer.weight.copy_((torch.rand(layer.weight.shape, generator=_gen(51), device=DEV) + 0.5).half().float())
    e = layer.fp16_exponent()
    assert e != 0
    x = _cl((torch.rand([N, c, r // up, r // up], generator=_gen(52), device=DEV) + 0.5).half())
    s = torch.rand([N, c], generator=_gen(53), device=DEV) + 0.5
    d = torch.rand([N, c], generator=_gen(54), device=DEV) * 1e-3 + 1e-3
    kw = dict(noise_mode='const', fused_modconv=False, styles=s, premodulated=True, next_styles=s, only_next=True, fp16=True)
    if up == 1:
        kw = dict(noise_mode='const', fused_modconv=False, styles=s, premodulated=True, y_styles=s, emit_y=True, next_styles=s, fp16=True)
    scaled = layer(x, None, dcoefs=d * 2.0 ** e, **kw)
    layer.__dict__.pop('_const_cache')                        # drop the scaled weight copy
    orig = networks.SynthesisLayer.fp16_exponent
    try:
        networks.SynthesisLayer.fp16_exponent = lambda self: 0
        plain = layer(x, None, dcoefs=d, **kw)
    finally:
        networks.SynthesisLayer.fp16_exponent = orig
    scaled = scaled if isinstance(scaled, (list, tuple)) else [scaled]
    plain = plain if isinstance(plain, (list, tuple)) else [plain]
    for a, b in zip(scaled, plain):
        assert a.dtype == torch.float16 and torch.equal(a, b)
