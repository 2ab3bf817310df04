"""The hybrid encoder of IDE-3D's portrait editing: image + semantic mask -> ws (inversion/networks.py:1507-1665).

    Conv2dLayer       inversion/networks.py:169-226 (the '2d' mode): weight * 1/sqrt(fan_in), conv2d_resample, bias_act
    EncoderResBlock   :1507-1521  conv1 (3x3, lrelu), conv2 (3x3, down 2, lrelu), skip (1x1, down 2, linear, no bias),
                      out = (conv2(conv1(x)) + skip(x)) / sqrt(2)
    EqualConv2d       :1524-1556  F.conv2d with weight * 1/sqrt(fan_in)
    HybridEncoder     :1604-1665  two branches -- convs_img / projector_img on the image, convs_seg / projector_seg on the 19-channel
                      semantic map -- whose rows are concatenated geometry first

Same constructor arguments, parameter and buffer names and state_dict shapes as the reference, so a reference encoder's state_dict
loads unchanged.  Activations are fp32 channels_last on the GPU, like training/networks.py.

Extension: the semantic input may be a uint8 class-id mask [N, H, W] instead of the float map.  It stands for mask2label_np(mask)*2-1
(dnnlib/seg_tools.py:67-72, Painter/run_UI.py:290-295): a value >= input_seg_dim is an all-zero one-hot row, i.e. -1 in every channel.
The geometry branch then opens with ide3d_seg_stem (torch_utils/ops/seg_stem.py): the stem, block 0's conv1 and its skip computed from
one byte per pixel through per-class tables, without building the one-hot map; under autograd its backward is ide3d_seg_stem_bwd,
which gives those three layers' weight and bias gradients from the same tables.  Shapes the kernel does not take run the composition
(device one-hot, *2-1, the three layers) instead, with or without gradients.  geometry(mask, signed=False) reads the mask as the
{0, 1} one-hot instead (dnnlib/seg_tools.py:93-98 scatter, what encoder fine-tuning's cycle term feeds the encoder).
"""

import math

import numpy as np
import torch
import torch.nn.functional as F

from .torch_utils import persistence
from .torch_utils.ops import bias_act, conv2d_resample, seg_stem, upfirdn2d
from .training import networks

CHANNELS = {4: 512, 8: 512, 16: 512, 32: 512, 64: 256, 128: 128, 256: 64, 512: 32, 1024: 16}     # :1609-1619


@persistence.persistent_class
class Conv2dLayer(torch.nn.Module):
    def __init__(self, in_channels, out_channels, kernel_size, bias=True, activation='linear', up=1, down=1, resample_filter=(1, 3, 3, 1),
                 conv_clamp=None, channels_last=False, trainable=True, mode='2d', **unused):
        super().__init__()
        if mode != '2d':
            raise NotImplementedError(f"Conv2dLayer: only mode='2d' is implemented, got {mode!r}")
        self.activation, self.up, self.down, self.conv_clamp, self.mode = activation, up, down, conv_clamp, mode
        self.register_buffer('resample_filter', upfirdn2d.setup_filter(list(resample_filter)))
        self.padding = kernel_size // 2
        self.weight_gain = 1 / np.sqrt(in_channels * kernel_size ** 2)
        self.act_gain = bias_act.activation_funcs[activation].def_gain
        memory_format = torch.channels_last if channels_last else torch.contiguous_format
        weight = torch.randn([out_channels, in_channels, kernel_size, kernel_size]).to(memory_format=memory_format)
        bias = torch.zeros([out_channels]) if bias else None
        if trainable:
            self.weight = torch.nn.Parameter(weight)
            self.bias = torch.nn.Parameter(bias) if bias is not None else None
        else:
            self.register_buffer('weight', weight)
            if bias is not None:
                self.register_buffer('bias', bias)
            else:
                self.bias = None

    def forward(self, x, gain=1):
        w = self.weight * self.weight_gain
        b = self.bias.to(x.dtype) if self.bias is not None else None
        x = conv2d_resample.conv2d_resample(x=x, w=w.to(x.dtype), f=self.resample_filter, up=self.up, down=self.down,
                                            padding=self.padding, flip_weight=(self.up == 1))
        act_clamp = self.conv_clamp * gain if self.conv_clamp is not None else None
        return bias_act.bias_act(x, b, act=self.activation, gain=self.act_gain * gain, clamp=act_clamp)


@persistence.persistent_class
class EncoderResBlock(torch.nn.Module):
    def __init__(self, in_channel, out_channel, blur_kernel=(1, 3, 3, 1)):
        super().__init__()
        self.conv1 = Conv2dLayer(in_channel, in_channel, 3, activation='lrelu')
        self.conv2 = Conv2dLayer(in_channel, out_channel, 3, down=2, activation='lrelu')
        self.skip = Conv2dLayer(in_channel, out_channel, 1, down=2, activation='linear', bias=False)

    def tail(self, y1, skip):
        """The block after conv1 and the skip branch: (conv2(y1) + skip) / sqrt(2)."""
        return (self.conv2(y1) + skip) / math.sqrt(2)

    def forward(self, x):
        return self.tail(self.conv1(x), self.skip(x))


@persistence.persistent_class
class EqualConv2d(torch.nn.Module):
    def __init__(self, in_channel, out_channel, kernel_size, stride=1, padding=0, bias=True):
        super().__init__()
        self.weight = torch.nn.Parameter(torch.randn(out_channel, in_channel, kernel_size, kernel_size))
        self.scale = 1 / math.sqrt(in_channel * kernel_size ** 2)
        self.stride, self.padding = stride, padding
        self.bias = torch.nn.Parameter(torch.zeros(out_channel)) if bias else None

    def forward(self, x):
        return F.conv2d(x, self.weight * self.scale, bias=self.bias, stride=self.stride, padding=self.padding)

    def __repr__(self):
        return (f'{self.__class__.__name__}({self.weight.shape[1]}, {self.weight.shape[0]}, {self.weight.shape[2]}, '
                f'stride={self.stride}, padding={self.padding})')


def _branch(size, in_dim):
    convs = [Conv2dLayer(in_dim, CHANNELS[size], 1)]
    ch = CHANNELS[size]
    for i in range(int(math.log(size, 2)), 2, -1):
        convs.append(EncoderResBlock(ch, CHANNELS[2 ** (i - 1)]))
        ch = CHANNELS[2 ** (i - 1)]
    return torch.nn.Sequential(*convs), ch


def _layout(x):
    return x.contiguous(memory_format=torch.channels_last) if networks.CHANNELS_LAST and x.is_cuda else x


def one_hot_input(mask, classes, dtype=torch.float32):
    """uint8 [N, H, W] -> [N, classes, H, W] = mask2label_np(mask) * 2 - 1 on the mask's device (a value >= classes gives -1 everywhere)."""
    hot = F.one_hot(mask.long().clamp(max=classes), classes + 1)[..., :classes]
    return hot.permute(0, 3, 1, 2).to(dtype) * 2 - 1


class _UnsignedStem:
    """The stem's weight and bias re-parameterised for a {0, 1} one-hot input (see HybridEncoder._mask_stem); differentiable."""

    def __init__(self, stem):
        self.weight = stem.weight / 2
        self.bias = stem.bias + stem.weight_gain / 2 * stem.weight.sum((1, 2, 3))
        self.weight_gain = stem.weight_gain


@persistence.persistent_class
class HybridEncoder(torch.nn.Module):
    def __init__(self, size, n_latents_app, n_latents_geo, w_dim=512, add_dim=0, input_img_dim=3, input_seg_dim=19, **unused):
        super().__init__()
        self.size, self.w_dim, self.add_dim = size, w_dim, add_dim
        self.n_latents_app, self.n_latents_geo = n_latents_app, n_latents_geo
        self.input_seg_dim = input_seg_dim
        self.convs_img, ch = _branch(size, input_img_dim)
        self.projector_img = EqualConv2d(ch, n_latents_app * w_dim + add_dim, 4, padding=0, bias=False)
        self.convs_seg, ch = _branch(size, input_seg_dim)
        self.projector_seg = EqualConv2d(ch, n_latents_geo * w_dim, 4, padding=0, bias=False)

    def appearance(self, img):
        """img [N, 3, H, W] in [-1, 1] -> [N, n_latents_app, w_dim]; with add_dim > 0, (that, pcm [N, add_dim])."""
        out = self.projector_img(self.convs_img(_layout(img)))
        if self.add_dim == 0:
            return out.reshape(len(img), self.n_latents_app, self.w_dim)
        pws, pcm = out[:, :-self.add_dim], out[:, -self.add_dim:]
        return pws.reshape(len(img), self.n_latents_app, self.w_dim), pcm.reshape(len(img), self.add_dim)

    def geometry(self, seg, *, signed=True):
        """seg: the float semantic map [N, input_seg_dim, H, W] (one_hot * 2 - 1 or anything else), or a uint8 class-id mask [N, H, W]
        -> [N, n_latents_geo, w_dim].  A uint8 mask stands for one_hot * 2 - 1 (signed=True) or for the {0, 1} one_hot itself
        (signed=False); a float map is used as it is."""
        if seg.dtype == torch.uint8:
            if seg.ndim != 3:
                raise ValueError(f'HybridEncoder.geometry: a uint8 mask must be [N, H, W], got {tuple(seg.shape)}')
            x = self._mask_stem(seg, signed)
            rest = self.convs_seg[2:]
        else:
            x, rest = _layout(seg), self.convs_seg
        return self.projector_seg(rest(x)).reshape(len(seg), self.n_latents_geo, self.w_dim)

    def _mask_stem(self, mask, signed=True):
        """convs_seg[0:2] applied to one_hot_input(mask) (or its {0, 1} form): the table kernel, or the composition it replaces.
        The kernel always reads one_hot * 2 - 1; for {0, 1} the stem is re-parameterised in front of it: with w0' = w0 / 2 and
        b0' = b0 + wg0 / 2 * sum_j w0[:, j], wg0 w0' (2 h - 1) + b0' = wg0 w0 h + b0 (exact; the "no class" row gives b0)."""
        stem, block = self.convs_seg[0], self.convs_seg[1]
        table_stem = stem if signed else _UnsignedStem(stem)
        out = seg_stem.seg_stem(mask, table_stem, block.conv1, block.skip)
        if out is None:
            x = one_hot_input(mask, self.input_seg_dim, stem.weight.dtype)
            return block(stem(_layout(x if signed else (x + 1) / 2)))
        return block.tail(*out)

    def forward(self, img, seg):
        geo = self.geometry(seg)
        app = self.appearance(img)
        if self.add_dim == 0:
            return torch.cat([geo, app], 1)
        return torch.cat([geo, app[0]], 1), app[1]
