"""StyleGAN2 building blocks of the tri-plane backbone and the super-resolution head.

The IDE-3D release does not contain its generator source (it travels inside the checkpoint pickle, SURVEY.md §0);
the nearest in-repo definitions are in inversion/networks.py (modulated_conv2d :55-130, FullyConnectedLayer
:136-165, MappingNetwork :243-325, SynthesisLayer :330-514, ToRGBLayer :670-713, SegSynthesisBlock :966-1139).
The classes below restate those layers for inference: same parameter names/shapes/initialisation and the same
arithmetic, with the StyleNeRF-only options (pixelshuffle / liif / 3-D modes, magnitude EMA, ...) left out.
Every convolution goes to cuDNN (conv2d_resample -> conv2d_gradfix); the surrounding ops are this package's
sm_90a kernels: upfirdn2d (FIR after the transposed conv, skip-image upsampling) and bias_act.
"""

import math
import os

import numpy as np
import torch

from ..torch_utils import misc, persistence
from ..torch_utils.ops import bias_act, conv2d_resample, fma, upfirdn2d


FUSED_MODCONV_MIN_RES = 1 << 30      # block resolutions >= this use the grouped (weight-modulated) convolution

# Layout choice: activations of every block are channels_last (NHWC) regardless of dtype.  The tf32 / fp16 tensor-core
# convolutions cuDNN picks are NHWC kernels -- with NCHW tensors it brackets every convolution with nchwToNhwc / nhwcToNchw
# passes -- and the renderer gathers NHWC tri-planes
# anyway.  The reference only does this for its fp16 layers (inversion/networks.py:746).  IDE3D_CHANNELS_LAST=0 restores
# the reference's NCHW fp32 layout (same values).
CHANNELS_LAST = os.environ.get('IDE3D_CHANNELS_LAST', '1') != '0'
STYLE_PLAN = os.environ.get('IDE3D_STYLE_PLAN', '1') != '0'      # styles + demodulation coefficients of a whole synthesis call in two launches (StylePlan)
CHAIN_MODULATION = True              # epilogues also write the next layer's `x * styles` (SynthesisBlock._features)
# fp32 NHWC inference without conv_clamp: the last epilogue of a block also computes its ToRGB output (<= 4 channels) and, inside a
# synthesis call, writes the next block's `x * styles` instead of x (nothing at all for the last block).  IDE3D_FUSED_TORGB=0 restores
# the separate passes (x * s_rgb, cuDNN 1x1 convolution, bias, x * s0 of the next block) for A/B runs.
FUSED_TORGB = os.environ.get('IDE3D_FUSED_TORGB', '1') != '0'
# 1x1 convolutions of NHWC activations as one [N*H*W, I] x [I, O] matrix product (cuBLASLt, tf32 exactly when the cuDNN convolution
# it replaces would use tf32) instead of cuDNN's conv3d_fprop kernels, which stream these shapes at ~40 % of the HBM peak.
# Off by default; kept as a switch for A/B runs.
CONV1X1_AS_MATMUL = os.environ.get('IDE3D_CONV1X1_MM', '0') != '0'


def fp16_operands(blocks, force_fp32=False, fused_modconv=None):
    """Do the convolutions of a chained synthesis call run on fp16 operands (DESIGN.md §2)?  Exactly when cuDNN may use TF32
    (torch.backends.cudnn.allow_tf32: every operand is then rounded to a 10-bit mantissa anyway, which is what fp16 keeps), the
    caller did not ask for fp32 (force_fp32) or the grouped convolution, and every block can fold its neighbours' passes into its
    epilogues (can_fold: NHWC, no conv_clamp) without a use_fp16 block.  The caller also needs the style plan, i.e. fp32 inference
    without gradients.  The convolution operands are then fp16 -- each tensor between two convolutions is written in fp16 by the
    epilogue that produces it -- and everything else (styles, demodulation, noise, bias, the epilogues' arithmetic, the ToRGB
    output and the skip images) stays float32."""
    return (bool(torch.backends.cudnn.allow_tf32) and not force_fp32 and not fused_modconv
            and all(b.can_fold() and not b.use_fp16 for b in blocks))


def _cached(module, name, tensors, make):
    """Derived constant of parameters / buffers, recomputed when any of them changes (data pointer, version, device)."""
    key = tuple((t.data_ptr(), t._version, str(t.device)) for t in tensors)
    store = module.__dict__.setdefault('_const_cache', {})
    hit = store.get(name)
    if hit is None or hit[0] != key:
        with torch.no_grad():
            hit = store[name] = (key, make())
    return hit[1]


def _fp16_copy(weight, e=0, transpose=False):
    """weight * 2^-e (exact) rounded to fp16, in the layout cuDNN's NHWC kernels want; transpose: the [I, O, k, k] operand of the
    transposed convolution."""
    fmt = torch.channels_last if CHANNELS_LAST else torch.contiguous_format
    w = weight.detach().to(torch.float32) * (2.0 ** -e)
    return (w.transpose(0, 1) if transpose else w).to(torch.float16).contiguous(memory_format=fmt)


def _conv1x1_nhwc(x, weight):
    """x [N,I,H,W] channels_last dense, weight [O,I,1,1] -> [N,O,H,W] channels_last (a view of the [N*H*W, O] product)."""
    n, c, h, w = x.shape
    o = weight.shape[0]
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = bool(torch.backends.cudnn.allow_tf32)
    try:
        y = x.permute(0, 2, 3, 1).reshape(n * h * w, c) @ weight.reshape(o, c).t()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    return y.reshape(n, h, w, o).permute(0, 3, 1, 2)


def normalize_2nd_moment(x, dim=1, eps=1e-8):
    return x * (x.square().mean(dim=dim, keepdim=True) + eps).rsqrt()


def modulated_conv2d(x, weight, styles, noise=None, up=1, down=1, padding=0, resample_filter=None, demodulate=True,
                     flip_weight=True, fused_modconv=True, epilogue=None, premodulated=False, dcoefs=None, w_transposed=None, w16=None):
    """Style-modulated convolution (inversion/networks.py:55-130).  x [N,I,H,W], weight [O,I,k,k], styles [N,I].
    epilogue (activation-scaled path only): dict(b, act, gain, clamp) -- the bias_act that always follows (:512, :707) is
    then applied here, fused with the demodulation / noise pass (`bias_act.scaled_bias_act`); optional keys next_scale /
    only_next make that pass also emit `y * next_styles`, the input of the next activation-scaled convolution.
    premodulated: x already carries `* styles` (written by the previous layer's epilogue).
    w16 (activation-scaled inference, see fp16_operands): the layer's fp16 weight W * 2^-e (for up > 1 with w_transposed its
    transposed fp16 copy); the convolution then runs on fp16 operands and dcoefs already carry the 2^e."""
    batch_size = x.shape[0]
    out_channels, in_channels, kh, kw = weight.shape
    if x.dtype == torch.float16 and demodulate and w16 is None:      # keep fp16 in range (:78-81)
        weight = weight * (1 / np.sqrt(in_channels * kh * kw) / weight.norm(float('inf'), dim=[1, 2, 3], keepdim=True))
        styles = styles / styles.norm(float('inf'), dim=1, keepdim=True)
    w = None
    if fused_modconv:
        dcoefs = None
        w = weight.unsqueeze(0) * styles.reshape(batch_size, 1, -1, 1, 1)            # [N,O,I,k,k]
    if demodulate and fused_modconv:
        dcoefs = (w.square().sum(dim=[2, 3, 4]) + 1e-8).rsqrt()                       # [N,O]
        w = w * dcoefs.reshape(batch_size, -1, 1, 1, 1)
    elif demodulate and dcoefs is not None:
        pass                                        # precomputed for the whole synthesis call (StylePlan below)
    elif demodulate:
        # sum_{i,k} (W[o,i,k] s[n,i])^2 = sum_i s[n,i]^2 sum_k W[o,i,k]^2 : a [N,I] x [I,O] product instead of
        # materialising the [N,O,I,k,k] modulated weight just to reduce it (same value up to fp32 summation order)
        dcoefs = (styles.square() @ weight.square().sum(dim=[2, 3]).t() + 1e-8).rsqrt()

    assert not (premodulated and (fused_modconv or (x.dtype == torch.float16 and demodulate and w16 is None)))
    assert w16 is None or not fused_modconv
    if not fused_modconv:                           # scale activations instead of weights (:97-111)
        if not premodulated:
            x = bias_act.scaled_bias_act(x, scale=styles, **({} if w16 is None else dict(out_dtype=torch.float16)))  # x * styles[:, :, None, None]
        wc = weight.to(x.dtype) if w16 is None else w16
        if epilogue is not None and w16 is not None:
            epilogue = dict(epilogue, fp32_tail=True)                      # fp16 convolution output, float32 tail operands
        if epilogue is not None and up > 1 and down == 1 and kh > 1:      # the FIR after the transposed conv applies the tail
            e = dict(epilogue)
            e['act_gain'] = e.pop('gain', None)
            e.update(scale=dcoefs if demodulate else None, noise=noise)
            return conv2d_resample.conv2d_resample(x=x, w=wc, f=resample_filter, up=up, down=down,
                                                   padding=padding, flip_weight=flip_weight, fir_epilogue=e, w_transposed=w_transposed)
        if (CONV1X1_AS_MATMUL and kh == 1 and kw == 1 and up == 1 and down == 1 and padding == 0 and x.dtype == torch.float32 and x.is_cuda
                and x.is_contiguous(memory_format=torch.channels_last) and not x.is_contiguous()
                and not (torch.is_grad_enabled() and (x.requires_grad or weight.requires_grad))):
            x = _conv1x1_nhwc(x, weight)
        else:
            x = conv2d_resample.conv2d_resample(x=x, w=wc, f=resample_filter, up=up, down=down, padding=padding, flip_weight=flip_weight)
        if epilogue is not None:
            return bias_act.scaled_bias_act(x, scale=dcoefs if demodulate else None, noise=noise, **epilogue)
        if demodulate and noise is not None:
            x = fma.fma(x, dcoefs.to(x.dtype).reshape(batch_size, -1, 1, 1), noise.to(x.dtype))
        elif demodulate:
            x = x * dcoefs.to(x.dtype).reshape(batch_size, -1, 1, 1)
        elif noise is not None:
            x = x.add_(noise.to(x.dtype))
        return x

    # one grouped convolution for the whole batch (:113-129)
    x = x.reshape(1, -1, *x.shape[2:])
    w = w.reshape(-1, in_channels, kh, kw)
    x = conv2d_resample.conv2d_resample(x=x, w=w.to(x.dtype), f=resample_filter, up=up, down=down, padding=padding,
                                        groups=batch_size, flip_weight=flip_weight)
    x = x.reshape(batch_size, -1, *x.shape[2:])
    if noise is not None:
        x = x.add_(noise)
    if epilogue is not None:
        b = epilogue['b']
        return bias_act.bias_act(x, None if b is None else b.to(x.dtype), act=epilogue.get('act', 'linear'), gain=epilogue.get('gain'),
                                 clamp=epilogue.get('clamp'))
    return x


@persistence.persistent_class
class FullyConnectedLayer(torch.nn.Module):
    """inversion/networks.py:136-165: weight ~ N(0,1)/lr_mult, runtime gain lr_mult/sqrt(in)."""

    def __init__(self, in_features, out_features, bias=True, activation='linear', lr_multiplier=1, bias_init=0):
        super().__init__()
        self.in_features, self.out_features, self.activation = in_features, out_features, activation
        self.weight = torch.nn.Parameter(torch.randn([out_features, in_features]) / lr_multiplier)
        self.bias = torch.nn.Parameter(torch.full([out_features], np.float32(bias_init))) if bias else None
        self.weight_gain = lr_multiplier / np.sqrt(in_features)
        self.bias_gain = lr_multiplier

    def effective(self):
        """(W, b) with the runtime gains folded in -- what the fused renderer kernel consumes."""
        w = self.weight.to(torch.float32) * self.weight_gain
        b = None if self.bias is None else self.bias.to(torch.float32) * self.bias_gain
        return w, b

    def forward(self, x):
        w = self.weight.to(x.dtype) * self.weight_gain
        b = self.bias
        if b is not None:
            b = b.to(x.dtype)
            if self.bias_gain != 1:
                b = b * self.bias_gain
        if self.activation == 'linear' and b is not None:
            return torch.addmm(b.unsqueeze(0), x, w.t())
        x = x.matmul(w.t())
        return bias_act.bias_act(x, b, act=self.activation)


@persistence.persistent_class
class MappingNetwork(torch.nn.Module):
    """z (+ camera label c) -> ws [N, num_ws, w_dim]; inversion/networks.py:243-325."""

    def __init__(self, z_dim, c_dim, w_dim, num_ws, num_layers=8, embed_features=None, layer_features=None,
                 activation='lrelu', lr_multiplier=0.01, w_avg_beta=0.995):
        super().__init__()
        self.z_dim, self.c_dim, self.w_dim, self.num_ws = z_dim, c_dim, w_dim, num_ws
        self.num_layers, self.w_avg_beta = num_layers, w_avg_beta
        if embed_features is None:
            embed_features = w_dim
        if c_dim == 0:
            embed_features = 0
        if layer_features is None:
            layer_features = w_dim
        feats = [z_dim + embed_features] + [layer_features] * (num_layers - 1) + [w_dim]
        if c_dim > 0:
            self.embed = FullyConnectedLayer(c_dim, embed_features)
        for idx in range(num_layers):
            setattr(self, f'fc{idx}', FullyConnectedLayer(feats[idx], feats[idx + 1], activation=activation,
                                                          lr_multiplier=lr_multiplier))
        if num_ws is not None and w_avg_beta is not None:
            self.register_buffer('w_avg', torch.zeros([w_dim]))

    def forward(self, z=None, c=None, truncation_psi=1, truncation_cutoff=None, skip_w_avg_update=False, **_unused):
        x = None
        if self.z_dim > 0:
            misc.assert_shape(z, [None, self.z_dim])
            x = normalize_2nd_moment(z.to(torch.float32))
        if self.c_dim > 0:
            misc.assert_shape(c, [None, self.c_dim])
            y = normalize_2nd_moment(self.embed(c.to(torch.float32)))
            x = torch.cat([x, y], dim=1) if x is not None else y
        for idx in range(self.num_layers):
            x = getattr(self, f'fc{idx}')(x)
        if self.w_avg_beta is not None and self.training and not skip_w_avg_update:
            self.w_avg.copy_(x.detach().mean(dim=0).lerp(self.w_avg, self.w_avg_beta))
        if self.num_ws is not None:
            x = x.unsqueeze(1).repeat([1, self.num_ws, 1])
        if truncation_psi != 1:
            if self.num_ws is None or truncation_cutoff is None:
                x = self.w_avg.lerp(x, truncation_psi)
            else:
                x[:, :truncation_cutoff] = self.w_avg.lerp(x[:, :truncation_cutoff], truncation_psi)
        return x


@persistence.persistent_class
class SynthesisLayer(torch.nn.Module):
    """Modulated 3x3 conv (+2x up), noise, bias_act; inversion/networks.py:330-514 ('default' upsampling)."""

    def __init__(self, in_channels, out_channels, w_dim, resolution, kernel_size=3, up=1, use_noise=True,
                 activation='lrelu', resample_filter=[1, 3, 3, 1], conv_clamp=None, channels_last=False):
        super().__init__()
        self.resolution, self.up, self.use_noise = resolution, up, use_noise
        self.activation, self.conv_clamp = activation, conv_clamp
        self.register_buffer('resample_filter', upfirdn2d.setup_filter(resample_filter))
        self.padding = kernel_size // 2
        self.act_gain = bias_act.activation_funcs[activation].def_gain
        self.affine = FullyConnectedLayer(w_dim, in_channels, bias_init=1)
        memory_format = torch.channels_last if channels_last else torch.contiguous_format
        self.weight = torch.nn.Parameter(torch.randn([out_channels, in_channels, kernel_size, kernel_size]).to(memory_format=memory_format))
        if use_noise:
            self.register_buffer('noise_const', torch.randn([resolution, resolution]))
            self.noise_strength = torch.nn.Parameter(torch.zeros([]))
        self.bias = torch.nn.Parameter(torch.zeros([out_channels]))

    def forward(self, x, w, noise_mode='random', fused_modconv=True, gain=1, styles=None, premodulated=False, next_styles=None,
                only_next=False, dcoefs=None, y_styles=None, emit_y=True, rgb=None, fp16=False):
        """styles / premodulated / next_styles / only_next: block-internal chaining of activation-scaled layers -- the
        epilogue of this layer can already write `y * next_styles` for the layer that follows (see SynthesisBlock._features).
        y_styles / emit_y / rgb (3x3 layers without upsampling): the epilogue returns `y * y_styles` in place of y, or no y,
        and the ToRGB output of rgb = (weight, styles, bias) -- `bias_act.scaled_bias_act`.
        fp16 (inference on the chained path, see fp16_operands): the convolution runs on fp16 operands with the weight copy
        W * 2^-fp16_exponent(); dcoefs must then carry the factor 2^fp16_exponent() (StylePlan.run(fp16_blocks=...) does)."""
        assert noise_mode in ['random', 'const', 'none']
        if styles is None:
            styles = self.affine(w)
        noise = None
        if self.use_noise and noise_mode == 'random':
            noise = torch.randn([x.shape[0], 1, self.up * x.shape[2], self.up * x.shape[3]], device=x.device) * self.noise_strength
        # a projector freezes the layer but optimises noise_const (inversion/training/projectors/w_projector_ide3d.py:79-85)
        inference = not (torch.is_grad_enabled() and (self.weight.requires_grad or (self.use_noise and (
            self.noise_strength.requires_grad or self.noise_const.requires_grad))))
        if self.use_noise and noise_mode == 'const':
            # constants of the weights, cached per parameter version for inference (one multiply / one 9 MB weight copy per layer and step otherwise)
            noise = self._cached('noise', (self.noise_const, self.noise_strength), lambda: self.noise_const * self.noise_strength) if inference \
                else self.noise_const * self.noise_strength
        act_gain = self.act_gain * gain
        act_clamp = self.conv_clamp * gain if self.conv_clamp is not None else None
        epilogue = dict(b=self.bias, act=self.activation, gain=act_gain, clamp=act_clamp)
        if next_styles is not None:
            epilogue.update(next_scale=next_styles, only_next=only_next)
        if y_styles is not None:
            epilogue['y_scale'] = y_styles
        if not emit_y:
            epilogue['emit_y'] = False
        if rgb is not None:
            epilogue['rgb'] = rgb
        w_t = w16 = None
        if fp16:
            assert inference and not fused_modconv and dcoefs is not None
            e = self.fp16_exponent()
            if self.up > 1:
                w_t = w16 = self._cached('w_t16', (self.weight,), lambda: _fp16_copy(self.weight, e, transpose=True))
            else:
                w16 = self._cached('w16', (self.weight,), lambda: _fp16_copy(self.weight, e))
        elif inference and self.up > 1 and not fused_modconv and x.dtype == self.weight.dtype:
            fmt = torch.channels_last if CHANNELS_LAST else torch.contiguous_format
            w_t = self._cached('w_t', (self.weight,), lambda: self.weight.detach().transpose(0, 1).contiguous(memory_format=fmt))
        return modulated_conv2d(x=x, weight=self.weight, styles=styles, noise=noise, up=self.up, padding=self.padding,
                                resample_filter=self.resample_filter, flip_weight=(self.up == 1), fused_modconv=fused_modconv,
                                epilogue=epilogue, premodulated=premodulated, dcoefs=None if fused_modconv else dcoefs, w_transposed=w_t,
                                w16=w16)

    def fp16_exponent(self):
        """e of the fp16 weight copy W * 2^-e: round(log2(sqrt(fan_in) * rms(W))), so that the convolution output before
        demodulation keeps the magnitude of its input `x * styles`, far from fp16's 65504.  Powers of two scale exactly: the
        demodulation coefficient takes 2^e back in float32 and no rounding changes."""
        def make():
            w = self.weight.detach().to(torch.float32)
            rms = float(w.square().mean().sqrt())
            return int(round(math.log2(math.sqrt(w[0].numel()) * rms))) if rms > 0 else 0
        return self._cached('fp16_e', (self.weight,), make)

    _cached = _cached


@persistence.persistent_class
class ToRGBLayer(torch.nn.Module):
    """Modulated 1x1 conv without demodulation + bias; inversion/networks.py:670-713 (w_dim > 0 branch)."""

    def __init__(self, in_channels, out_channels, w_dim, kernel_size=1, conv_clamp=None, channels_last=False):
        super().__init__()
        self.conv_clamp = conv_clamp
        self.affine = FullyConnectedLayer(w_dim, in_channels, bias_init=1)
        memory_format = torch.channels_last if channels_last else torch.contiguous_format
        self.weight = torch.nn.Parameter(torch.randn([out_channels, in_channels, kernel_size, kernel_size]).to(memory_format=memory_format))
        self.bias = torch.nn.Parameter(torch.zeros([out_channels]))
        self.weight_gain = 1 / np.sqrt(in_channels * (kernel_size ** 2))

    def styles(self, w):
        return self.affine(w) * self.weight_gain

    def forward(self, x, w, fused_modconv=True, styles=None, premodulated=False, raw=False):
        """raw: return the convolution output WITHOUT the bias (the caller folds `self.bias` into the skip-connection pass).
        An fp16 premodulated x (the fp16 operand path, see fp16_operands) is convolved with the layer's fp16 weight copy; the
        output is fp16, or float32 with the bias added.  The styles already carry 1/sqrt(fan_in) (weight_gain), so the output has
        the magnitude of x * rms(W) and the copy is not rescaled (e = 0)."""
        if styles is None:
            styles = self.styles(w)
        if premodulated and x.dtype == torch.float16 and self.weight.dtype == torch.float32:
            w16 = _cached(self, 'w16', (self.weight,), lambda: _fp16_copy(self.weight))
            y = modulated_conv2d(x=x, weight=self.weight, styles=styles, demodulate=False, fused_modconv=False, premodulated=True, w16=w16)
            return y if raw else bias_act.bias_act(y.to(torch.float32), self.bias, clamp=self.conv_clamp)
        return modulated_conv2d(x=x, weight=self.weight, styles=styles, demodulate=False, fused_modconv=fused_modconv,
                                epilogue=None if raw else dict(b=self.bias, clamp=self.conv_clamp), premodulated=premodulated)


@persistence.persistent_class
class SynthesisBlock(torch.nn.Module):
    """One resolution of a 'skip' StyleGAN2 synthesis network: [conv0(up 2)], conv1, torgb
    (inversion/networks.py:718-861).  Children order (conv0, conv1, torgb) matters to callers that index the
    flattened layer list (ide3d-nada/ZSSGAN/model/ZSSGAN_IDE3D.py:425-437)."""

    def __init__(self, in_channels, out_channels, w_dim, resolution, img_channels, is_last, resample_filter=[1, 3, 3, 1],
                 conv_clamp=None, use_fp16=False, fp16_channels_last=False, **layer_kwargs):
        super().__init__()
        self.in_channels, self.out_channels, self.w_dim = in_channels, out_channels, w_dim
        self.resolution, self.img_channels, self.is_last = resolution, img_channels, is_last
        self.architecture = 'skip'
        self.use_fp16 = use_fp16
        self.channels_last = use_fp16 and fp16_channels_last
        self.register_buffer('resample_filter', upfirdn2d.setup_filter(resample_filter))
        self.num_conv = 0
        self.num_torgb = 0
        if in_channels == 0:
            self.const = torch.nn.Parameter(torch.randn([out_channels, resolution, resolution]))
        if in_channels != 0:
            self.conv0 = SynthesisLayer(in_channels, out_channels, w_dim=w_dim, resolution=resolution, up=2,
                                        resample_filter=resample_filter, conv_clamp=conv_clamp,
                                        channels_last=self.channels_last or CHANNELS_LAST, **layer_kwargs)
            self.num_conv += 1
        self.conv1 = SynthesisLayer(out_channels, out_channels, w_dim=w_dim, resolution=resolution, conv_clamp=conv_clamp,
                                    channels_last=self.channels_last or CHANNELS_LAST, **layer_kwargs)
        self.num_conv += 1
        self.torgb = ToRGBLayer(out_channels, img_channels, w_dim=w_dim, conv_clamp=conv_clamp,
                                channels_last=self.channels_last or CHANNELS_LAST)
        self.num_torgb += 1

    def can_fold(self):
        """Can this block's epilogues take over its neighbours' passes (FUSED_TORGB)?  Only for the NHWC layout and without
        conv_clamp; the caller still needs the block on the chained path (fp32 inference, activation scaling)."""
        return FUSED_TORGB and CHAIN_MODULATION and CHANNELS_LAST and self.conv1.conv_clamp is None and self.torgb.conv_clamp is None

    def _features(self, x, ws, force_fp32, fused_modconv, layer_kwargs):
        """-> (x, w_rgb, fused_modconv, rgb_in, y_rgb).  Keys of layer_kwargs a synthesis network uses to chain its blocks (each
        needs the chained path below): premodulated_x -- x already carries conv0's styles (the previous block's epilogue wrote
        them); x_next_styles [N, C] -- return `x * x_next_styles` (the next block's conv0 styles) instead of x; drop_x -- return
        no x (nothing consumes it); fp16_operands -- run the convolutions on fp16 operands (fp16_operands(); needs the style plan's
        dcoefs for that path).  y_rgb is the ToRGB output (bias included) when conv1's epilogue computed it."""
        layer_kwargs = dict(layer_kwargs)
        premod_in = layer_kwargs.pop('premodulated_x', False)
        x_next_styles = layer_kwargs.pop('x_next_styles', None)
        drop_x = layer_kwargs.pop('drop_x', False)
        fp16 = layer_kwargs.pop('fp16_operands', False)
        misc.assert_shape(ws, [None, self.num_conv + self.num_torgb, self.w_dim])
        w_iter = iter(ws.unbind(dim=1))
        dtype = torch.float16 if self.use_fp16 and not force_fp32 else torch.float32
        memory_format = torch.channels_last if CHANNELS_LAST or (self.channels_last and not force_fp32) else torch.contiguous_format
        if fused_modconv is None:
            fused_modconv = (not self.training) and (dtype == torch.float32 or int(ws.shape[0]) == 1)
            # Scaling activations instead of weights keeps the convolution a plain batched one (the grouped per-sample
            # form is what the reference uses in eval, inversion/networks.py:802; both are the same arithmetic up to
            # rounding); the grouped form is used from FUSED_MODCONV_MIN_RES up.
            thr = int(os.environ.get('IDE3D_FUSED_MODCONV_MIN_RES', FUSED_MODCONV_MIN_RES))
            fused_modconv = fused_modconv and self.resolution >= thr
        # Inference in fp32 with activation scaling: every epilogue also writes the next layer's `x * styles`, so the
        # separate modulation passes of conv1 and ToRGB disappear (conv0 -> x*s1 only; conv1 -> x and x*s_rgb).
        chain = CHAIN_MODULATION and (not fused_modconv) and dtype == torch.float32 and not (torch.is_grad_enabled() and (
            ws.requires_grad or any(p.requires_grad for p in self.parameters())))
        if not chain and (premod_in or x_next_styles is not None or drop_x):
            raise RuntimeError('SynthesisBlock: cross-block chaining needs the chained fp32 inference path')
        if fp16 and not (chain and self.can_fold() and 'style_plan' in layer_kwargs):
            raise RuntimeError('SynthesisBlock: fp16 operands need the chained inference path with a style plan')
        rgb_in = y_rgb = None
        if self.in_channels == 0:
            x = self.const.to(dtype=dtype).unsqueeze(0).repeat([ws.shape[0], 1, 1, 1]).contiguous(memory_format=memory_format)
            w1 = next(w_iter)
        else:
            misc.assert_shape(x, [None, self.in_channels, self.resolution // 2, self.resolution // 2])
            x = x.to(memory_format=memory_format) if fp16 else x.to(dtype=dtype, memory_format=memory_format)   # fp16: x * s0 in fp16
            w0, w1 = next(w_iter), next(w_iter)
        w_rgb = next(w_iter)
        plan = layer_kwargs.pop('style_plan', None) if chain else None
        layer_kwargs.pop('style_plan', None)
        if chain:
            if plan is not None:                       # every style / demodulation coefficient of the call was computed up front
                (s1, d1), (s_rgb, _) = plan[self.conv1], plan[self.torgb]
                s0, d0 = plan[self.conv0] if self.in_channels != 0 else (None, None)
            else:
                s1, s_rgb, s0, d0, d1 = self.conv1.affine(w1), self.torgb.styles(w_rgb), None, None, None
            pre = False
            if self.in_channels != 0:
                x = self.conv0(x, w0, fused_modconv=False, styles=s0, dcoefs=d0, premodulated=premod_in, next_styles=s1, only_next=True,
                               fp16=fp16, **layer_kwargs)
                pre = True
            # ToRGB of <= 4 channels inside conv1's epilogue: a 3 x C dot product per pixel instead of x * s_rgb + a 1x1 convolution
            fold_rgb = x.is_cuda and self.torgb.weight.shape[0] <= 4 and self.can_fold()
            fold = {}
            if x_next_styles is not None:
                fold['y_styles'] = x_next_styles
            if drop_x:
                fold['emit_y'] = False
            if fold_rgb:
                fold['rgb'] = (self.torgb.weight, s_rgb, self.torgb.bias)
            outs = self.conv1(x, w1, fused_modconv=False, styles=s1, dcoefs=d1, premodulated=pre, next_styles=None if fold_rgb else s_rgb,
                              fp16=fp16, **fold, **layer_kwargs)          # (y | y * y_styles)?, (y * s_rgb | ToRGB output)
            x = None if drop_x else outs[0]
            if fold_rgb:
                y_rgb = outs[-1]
            else:
                rgb_in = (outs[-1], s_rgb)
        else:
            if self.in_channels != 0:
                x = self.conv0(x, w0, fused_modconv=fused_modconv, **layer_kwargs)
            x = self.conv1(x, w1, fused_modconv=fused_modconv, **layer_kwargs)
        return x, w_rgb, fused_modconv, rgb_in, y_rgb

    def _torgb(self, x, w_rgb, fused_modconv, rgb_in, raw=False):
        if rgb_in is not None:
            return self.torgb(rgb_in[0], w_rgb, fused_modconv=False, styles=rgb_in[1], premodulated=True, raw=raw)
        return self.torgb(x, w_rgb, fused_modconv=fused_modconv, raw=raw)

    def _fuse_skip(self, rgb_in, *imgs):
        """Can `upsample2d(img) + y + bias` run as one pass?  (chained fp32 inference, NHWC, no clamp, a running image at half
        the resolution for every output group.)"""
        return (rgb_in is not None and CHANNELS_LAST and self.torgb.conv_clamp is None and all(
            i is not None and i.dtype == torch.float32 and i.shape[-1] * 2 == self.resolution and i.shape[1] % 4 == 0 and
            i.stride(1) == 1 for i in imgs))

    def _accumulate(self, img, y):
        """Skip connection: upsample the running image with the FIR and add the new contribution."""
        if img is not None and img.shape[-1] * 2 == y.shape[-1]:
            img = upfirdn2d.upsample2d(img, self.resample_filter)
        if CHANNELS_LAST and y.stride(1) == 1 and y.shape[1] % 4 == 0:      # keep NHWC (y may be a channel slice of the ToRGB output)
            y = y.to(dtype=torch.float32)
            return img.add_(y) if img is not None else y.contiguous(memory_format=torch.channels_last)
        y = y.to(dtype=torch.float32, memory_format=torch.contiguous_format)
        return img.add_(y) if img is not None else y

    def forward(self, x, img, ws, force_fp32=False, fused_modconv=None, **layer_kwargs):
        x, w_rgb, fused_modconv, rgb_in, y_rgb = self._features(x, ws, force_fp32, fused_modconv, layer_kwargs)
        if y_rgb is not None:
            return x, self._accumulate(img, y_rgb)
        if self._fuse_skip(rgb_in, img):
            y = self._torgb(x, w_rgb, fused_modconv, rgb_in, raw=True)
            return x, upfirdn2d.upsample2d_add(img, self.resample_filter, y, self.torgb.bias)
        img = self._accumulate(img, self._torgb(x, w_rgb, fused_modconv, rgb_in))
        return x, img


@persistence.persistent_class
class SegSynthesisBlock(SynthesisBlock):
    """Dual-path block of the tri-plane backbone: one feature stream, two skip-accumulated outputs -- the texture
    tri-plane `img` and the shape/semantic tri-plane `seg` (the dual ToRGB/ToSEG path of
    inversion/networks.py:1093-1134).  Call contract from extract_shapes.py:127-129:
        x, img, seg = block(x, img, ws, condition_img=seg)
    Both heads share one style vector (`w_shared`, :1093) and are evaluated as ONE modulated 1x1 convolution whose
    output channels are [img_channels | seg_channels], so the child list stays (conv0, conv1, torgb)."""

    def __init__(self, in_channels, out_channels, w_dim, resolution, img_channels, seg_channels, is_last, **kwargs):
        super().__init__(in_channels, out_channels, w_dim, resolution, img_channels + seg_channels, is_last, **kwargs)
        self.img_channels, self.seg_channels = img_channels, seg_channels

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        """Checkpoints of the in-repo reference class (inversion/networks.py:1093-1134) carry two output layers, `torgb` and `toseg`,
        each with its own affine.  They are the same function as this block's single [img | seg] ToRGB exactly when the two affines
        coincide; then the weights / biases are concatenated along the output channels.  Anything else cannot be represented by the
        released 3-children-per-block structure this class follows, and fails loudly instead of loading half a block."""
        ts = prefix + 'toseg.'
        if any(k.startswith(ts) for k in state_dict):
            for name in ('affine.weight', 'affine.bias'):
                a, b = state_dict.get(prefix + 'torgb.' + name), state_dict.get(ts + name)
                if a is None or b is None or a.shape != b.shape or not torch.equal(a, b):
                    raise RuntimeError(f'SegSynthesisBlock: {ts}{name} differs from torgb.{name}; a block with independent torgb / toseg '
                                       'affines has no equivalent in this single-ToRGB structure')
            for name in ('weight', 'bias'):
                state_dict[prefix + 'torgb.' + name] = torch.cat([state_dict[prefix + 'torgb.' + name], state_dict[ts + name]], 0)
            for k in [k for k in state_dict if k.startswith(ts)]:
                del state_dict[k]
        return super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)

    def forward(self, x, img, ws, condition_img=None, force_fp32=False, fused_modconv=None, **layer_kwargs):
        x, w_shared, fused_modconv, rgb_in, y = self._features(x, ws, force_fp32, fused_modconv, layer_kwargs)
        if y is not None:
            return x, self._accumulate(img, y[:, :self.img_channels]), self._accumulate(condition_img, y[:, self.img_channels:])
        if self._fuse_skip(rgb_in, img, condition_img):
            y, b, ci = self._torgb(x, w_shared, fused_modconv, rgb_in, raw=True), self.torgb.bias, self.img_channels
            img = upfirdn2d.upsample2d_add(img, self.resample_filter, y[:, :ci], b[:ci])
            seg = upfirdn2d.upsample2d_add(condition_img, self.resample_filter, y[:, ci:], b[ci:])
            return x, img, seg
        y = self._torgb(x, w_shared, fused_modconv, rgb_in)
        img = self._accumulate(img, y[:, :self.img_channels])
        seg = self._accumulate(condition_img, y[:, self.img_channels:])
        return x, img, seg


class StylePlan:
    """Styles and demodulation coefficients of every modulated convolution of a synthesis network in two kernel launches
    (ide3d_style_plan) instead of ~8 library launches per layer.  Built once per network; holds fp32 device copies of the constants
    (sum_k W^2 per layer) keyed on the parameters' versions.  `run(ws)` -> {layer module: (styles [N, I], dcoefs [N, O] | None)}.
    Inference only, fp32, activation-scaled (not weight-modulated) convolutions -- SynthesisBlock._features decides."""

    def __init__(self, blocks_with_base):
        """blocks_with_base: [(SynthesisBlock, index of the block's first w in ws)] in ws order."""
        self.entries = []                       # (layer, w_index, demodulate, out_scale)
        for block, base in blocks_with_base:
            j = base
            if block.in_channels != 0:
                self.entries.append((block.conv0, j, True, 1.0)); j += 1
            self.entries.append((block.conv1, j, True, 1.0)); j += 1
            self.entries.append((block.torgb, j, False, float(block.torgb.weight_gain)))
        assert len(self.entries) <= 32
        self._key = None
        self._consts = None

    def _constants(self, device):
        params = [p for layer, *_ in self.entries for p in (layer.affine.weight, layer.affine.bias, layer.weight)]
        key = (str(device),) + tuple((p.data_ptr(), p._version) for p in params)
        if key == self._key:
            return self._consts
        from .. import _lib as L
        keep, structs = [], (L.StyleLayer * len(self.entries))()
        s_off = d_off = 0
        for k, (layer, w_index, demod, out_scale) in enumerate(self.entries):
            aw = layer.affine.weight.detach().to(device=device, dtype=torch.float32).contiguous()
            ab = layer.affine.bias.detach().to(device=device, dtype=torch.float32).contiguous()
            o, i = layer.weight.shape[0], layer.weight.shape[1]
            wsq = layer.weight.detach().to(device=device, dtype=torch.float32).square().sum(dim=[2, 3]).contiguous() if demod else None
            keep += [aw, ab, wsq]
            structs[k] = L.StyleLayer(aw.data_ptr(), ab.data_ptr(), wsq.data_ptr() if demod else None, float(layer.affine.weight_gain),
                                      float(layer.affine.bias_gain), float(out_scale), int(w_index), int(i), int(o), 0, 0)
            structs[k].style_off, structs[k].dcoef_off = s_off, d_off        # per-sample offsets; scaled by N in run()
            s_off += i
            d_off += o if demod else 0
        self._key, self._consts = key, (keep, structs, s_off, d_off)
        return self._consts

    def _dcoef_multipliers(self, n, device, fp16_blocks):
        """[n * d_tot] float32: over each demodulating layer's dcoefs, 2^e (SynthesisLayer.fp16_exponent) for the layers of
        fp16_blocks, 1 for the others."""
        sel = {m for b in fp16_blocks for m in b.modules()}
        ex = lambda layer: layer.fp16_exponent() if layer in sel else 0
        key = (n, str(device), tuple(ex(layer) for layer, _, demod, _ in self.entries if demod))
        if getattr(self, '_mult_key', None) != key:
            parts = [torch.full([n * layer.weight.shape[0]], 2.0 ** ex(layer), dtype=torch.float32)
                     for layer, _, demod, _ in self.entries if demod]
            self._mult_key, self._mult = key, torch.cat(parts).to(device)
        return self._mult

    @torch.no_grad()
    def run(self, ws, fp16_blocks=()):
        """fp16_blocks: blocks on fp16 operands (fp16_operands); their layers' dcoefs carry the 2^e of the fp16 weight copy."""
        import ctypes as C
        from .. import _lib as L
        ws = ws.detach().to(torch.float32).contiguous()
        n, num_ws, w_dim = ws.shape
        _, base, s_tot, d_tot = self._constants(ws.device)
        structs = (L.StyleLayer * len(self.entries))()
        for k in range(len(self.entries)):
            C.memmove(C.byref(structs[k]), C.byref(base[k]), C.sizeof(L.StyleLayer))
            structs[k].style_off, structs[k].dcoef_off = base[k].style_off * n, base[k].dcoef_off * n
        styles = torch.empty(n * s_tot, dtype=torch.float32, device=ws.device)
        dcoefs = torch.empty(max(1, n * d_tot), dtype=torch.float32, device=ws.device)
        with torch.cuda.device(ws.device):
            L.check(L.get_lib().ide3d_style_plan(L.ptr(ws), n, num_ws, w_dim, structs, len(self.entries), L.ptr(styles), L.ptr(dcoefs),
                                                 L.stream_ptr(ws.device)))
        if len(fp16_blocks) and d_tot > 0:
            dcoefs[:n * d_tot].mul_(self._dcoef_multipliers(n, ws.device, fp16_blocks))
        out = {}
        for k, (layer, _, demod, _) in enumerate(self.entries):
            i, o = structs[k].in_ch, structs[k].out_ch
            s = styles[structs[k].style_off:structs[k].style_off + n * i].view(n, i)
            d = dcoefs[structs[k].dcoef_off:structs[k].dcoef_off + n * o].view(n, o) if demod else None
            out[layer] = (s, d)
        return out
