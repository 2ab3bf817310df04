"""ArcFace IR-SE50, the identity network of hybrid-encoder training's ID loss (inversion/psp/encoders/model_irse.py, helpers.py;
inversion/criteria/id_loss.py).

    Backbone(input_size, num_layers, mode='ir', drop_ratio=0.4, affine=True)   the reference's modules under its names, so
                                                   model_ir_se50.pth loads with strict=True; forward -> l2-normalised [N, 512]
    Backbone.ir_se50(path)                         Backbone(112, 50, 'ir_se', drop_ratio=0.6) from a local file, in eval mode
    IDLoss(backbone)                               __call__(y_hat, y) -> mean_n (1 - <f(y_hat_n), f(y_n)>), f = extract_feats
                                                   (pool to 256, crop [35:223, 32:220], pool to 112); y may be the features
                                                   IDLoss.target(y) returned, computed once

The reference's IDLoss(y_hat, y, x) also extracts x's features for its logs and returns them; the loss is its first output, which is
what this one returns.
"""

import os
from collections import namedtuple

import torch
from torch.nn import (AdaptiveAvgPool2d, BatchNorm1d, BatchNorm2d, Conv2d, Dropout, Linear, MaxPool2d, Module, PReLU, ReLU, Sequential,
                      Sigmoid)


class Flatten(Module):
    def forward(self, x):
        return x.reshape(x.size(0), -1)


def l2_norm(x, axis=1):
    return x / torch.norm(x, 2, axis, True)


class Bottleneck(namedtuple('Block', ['in_channel', 'depth', 'stride'])):
    """A ResNet block's description."""


def get_block(in_channel, depth, num_units, stride=2):
    return [Bottleneck(in_channel, depth, stride)] + [Bottleneck(depth, depth, 1) for _ in range(num_units - 1)]


UNITS = {50: (3, 4, 14, 3), 100: (3, 13, 30, 3), 152: (3, 8, 36, 3)}


def get_blocks(num_layers):
    if num_layers not in UNITS:
        raise ValueError(f'Invalid number of layers: {num_layers}. Must be one of {sorted(UNITS)}')
    u = UNITS[num_layers]
    return [get_block(64, 64, u[0]), get_block(64, 128, u[1]), get_block(128, 256, u[2]), get_block(256, 512, u[3])]


class SEModule(Module):
    def __init__(self, channels, reduction):
        super().__init__()
        self.avg_pool = AdaptiveAvgPool2d(1)
        self.fc1 = Conv2d(channels, channels // reduction, kernel_size=1, padding=0, bias=False)
        self.relu = ReLU(inplace=True)
        self.fc2 = Conv2d(channels // reduction, channels, kernel_size=1, padding=0, bias=False)
        self.sigmoid = Sigmoid()

    def forward(self, x):
        return x * self.sigmoid(self.fc2(self.relu(self.fc1(self.avg_pool(x)))))


class _Unit(Module):
    def __init__(self, in_channel, depth, stride, se):
        super().__init__()
        if in_channel == depth:
            self.shortcut_layer = MaxPool2d(1, stride)
        else:
            self.shortcut_layer = Sequential(Conv2d(in_channel, depth, (1, 1), stride, bias=False), BatchNorm2d(depth))
        layers = [BatchNorm2d(in_channel), Conv2d(in_channel, depth, (3, 3), (1, 1), 1, bias=False), PReLU(depth),
                  Conv2d(depth, depth, (3, 3), stride, 1, bias=False), BatchNorm2d(depth)]
        if se:
            layers.append(SEModule(depth, 16))
        self.res_layer = Sequential(*layers)

    def forward(self, x):
        return self.res_layer(x) + self.shortcut_layer(x)


class bottleneck_IR(_Unit):                                      # noqa: N801 (the reference's name)
    def __init__(self, in_channel, depth, stride):
        super().__init__(in_channel, depth, stride, se=False)


class bottleneck_IR_SE(_Unit):                                   # noqa: N801
    def __init__(self, in_channel, depth, stride):
        super().__init__(in_channel, depth, stride, se=True)


class Backbone(Module):
    def __init__(self, input_size, num_layers, mode='ir', drop_ratio=0.4, affine=True):
        super().__init__()
        if input_size not in (112, 224):
            raise ValueError(f'Backbone: input_size must be 112 or 224, got {input_size}')
        if mode not in ('ir', 'ir_se'):
            raise ValueError(f"Backbone: mode must be 'ir' or 'ir_se', got {mode!r}")
        unit = bottleneck_IR if mode == 'ir' else bottleneck_IR_SE
        self.input_layer = Sequential(Conv2d(3, 64, (3, 3), 1, 1, bias=False), BatchNorm2d(64), PReLU(64))
        side = 7 if input_size == 112 else 14
        self.output_layer = Sequential(BatchNorm2d(512), Dropout(drop_ratio), Flatten(), Linear(512 * side * side, 512),
                                       BatchNorm1d(512, affine=affine))
        self.body = Sequential(*[unit(b.in_channel, b.depth, b.stride) for block in get_blocks(num_layers) for b in block])

    def forward(self, x):
        return l2_norm(self.output_layer(self.body(self.input_layer(x))))

    @classmethod
    def ir_se50(cls, path, map_location='cpu'):
        """IDLoss's network (id_loss.py:12-13) from a local model_ir_se50.pth.  Nothing is downloaded."""
        path = os.fspath(path)
        if not os.path.isfile(path):
            raise FileNotFoundError(f'Backbone.ir_se50: no weights at {path!r} (nothing is downloaded)')
        net = cls(112, 50, mode='ir_se', drop_ratio=0.6)
        net.load_state_dict(torch.load(path, map_location=map_location, weights_only=True), strict=True)
        return net.eval().requires_grad_(False)


class IDLoss(Module):
    def __init__(self, backbone):
        super().__init__()
        self.facenet = backbone.eval().requires_grad_(False)
        self.pool = AdaptiveAvgPool2d((256, 256))
        self.face_pool = AdaptiveAvgPool2d((112, 112))

    def extract_feats(self, x):
        if x.shape[2] != 256:
            x = self.pool(x)
        return self.facenet(self.face_pool(x[:, :, 35:223, 32:220]))

    @torch.no_grad()
    def target(self, y):
        return self.extract_feats(y).detach()

    def forward(self, y_hat, y):
        y_feats = y if y.ndim == 2 else self.target(y)
        return (1 - (self.extract_feats(y_hat) * y_feats).sum(1)).mean()
