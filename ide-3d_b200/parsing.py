"""BiSeNet face parsing (inversion/BiSeNet.py and inversion/resnet.py): the 20-class parser encoder fine-tuning uses on its renders.

    ConvBNReLU, BiSeNetOutput, AttentionRefinementModule, ContextPath, FeatureFusionModule, BiSeNet   BiSeNet.py:13-252
    BasicBlock, Resnet18                                                                              resnet.py:19-79

Same attribute names, so a reference `segNet-20Class.pth` state_dict loads with strict=True.  SpatialPath is not restated: the
reference never builds it (the 1/8 ResNet feature stands in for it).  conv_out16 / conv_out32 are built and carry weights in the
state_dict, though forward does not use them.  Convolutions and BatchNorm (in eval mode) stay with cuDNN.

    BiSeNet.forward(x)          (logits at x's size, None, None), the reference's return: logits(x) upsampled bilinearly with
                                align_corners=True
    BiSeNet.logits(x)           the logits before that upsampling, [N, n_classes, H/8, W/8]
    BiSeNet.load(path)          a local state_dict file (torch.load(weights_only=True)) -> the model in eval mode without grad;
                                nothing is ever downloaded
    parse(net, img, remap=True) uint8 class ids [N, H, W]: the argmax of the upsampled logits (ide3d_seg_labels_ac, without building
                                them); with remap, id_remap's table (dnnlib/seg_tools.py:59-64) to COLOR_MAP's 19 classes
    remap_ids(ids)              that table applied to uint8 ids
"""

import os

import torch
import torch.nn as nn
import torch.nn.functional as F

from .torch_utils.ops import seg_stem as _seg_ops

REMAP = (0, 1, 6, 7, 4, 5, 2, 2, 10, 11, 12, 8, 9, 15, 3, 17, 16, 18, 13, 14)      # dnnlib/seg_tools.py:59


class ConvBNReLU(nn.Module):
    def __init__(self, in_chan, out_chan, ks=3, stride=1, padding=1):
        super().__init__()
        self.conv = nn.Conv2d(in_chan, out_chan, kernel_size=ks, stride=stride, padding=padding, bias=False)
        self.bn = nn.BatchNorm2d(out_chan)

    def forward(self, x):
        return F.relu(self.bn(self.conv(x)))


class BiSeNetOutput(nn.Module):
    def __init__(self, in_chan, mid_chan, n_classes):
        super().__init__()
        self.conv = ConvBNReLU(in_chan, mid_chan, ks=3, stride=1, padding=1)
        self.conv_out = nn.Conv2d(mid_chan, n_classes, kernel_size=1, bias=False)

    def forward(self, x):
        return self.conv_out(self.conv(x))


class AttentionRefinementModule(nn.Module):
    def __init__(self, in_chan, out_chan):
        super().__init__()
        self.conv = ConvBNReLU(in_chan, out_chan, ks=3, stride=1, padding=1)
        self.conv_atten = nn.Conv2d(out_chan, out_chan, kernel_size=1, bias=False)
        self.bn_atten = nn.BatchNorm2d(out_chan)
        self.sigmoid_atten = nn.Sigmoid()

    def forward(self, x):
        feat = self.conv(x)
        atten = F.avg_pool2d(feat, feat.size()[2:])
        atten = self.sigmoid_atten(self.bn_atten(self.conv_atten(atten)))
        return torch.mul(feat, atten)


class BasicBlock(nn.Module):
    def __init__(self, in_chan, out_chan, stride=1):
        super().__init__()
        self.conv1 = nn.Conv2d(in_chan, out_chan, kernel_size=3, stride=stride, padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(out_chan)
        self.conv2 = nn.Conv2d(out_chan, out_chan, kernel_size=3, stride=1, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(out_chan)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = None
        if in_chan != out_chan or stride != 1:
            self.downsample = nn.Sequential(nn.Conv2d(in_chan, out_chan, kernel_size=1, stride=stride, bias=False),
                                            nn.BatchNorm2d(out_chan))

    def forward(self, x):
        residual = self.bn2(self.conv2(F.relu(self.bn1(self.conv1(x)))))
        shortcut = x if self.downsample is None else self.downsample(x)
        return self.relu(shortcut + residual)


def _layer(in_chan, out_chan, bnum, stride=1):
    return nn.Sequential(BasicBlock(in_chan, out_chan, stride=stride), *[BasicBlock(out_chan, out_chan) for _ in range(bnum - 1)])


class Resnet18(nn.Module):
    def __init__(self, in_chan=3, out_chan=512):
        super().__init__()
        self.conv1 = nn.Conv2d(in_chan, 64, kernel_size=7, stride=2, padding=3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
        self.layer1 = _layer(64, 64, 2)
        self.layer2 = _layer(64, 128, 2, stride=2)
        self.layer3 = _layer(128, 256, 2, stride=2)
        self.layer4 = _layer(256, out_chan, 2, stride=2)

    def forward(self, x):
        x = self.maxpool(F.relu(self.bn1(self.conv1(x))))
        feat8 = self.layer2(self.layer1(x))
        feat16 = self.layer3(feat8)
        return feat8, feat16, self.layer4(feat16)


def _up(x, size):
    return F.interpolate(x, size, mode='bilinear', align_corners=True)


class ContextPath(nn.Module):
    def __init__(self):
        super().__init__()
        self.resnet = Resnet18()
        self.arm16 = AttentionRefinementModule(256, 128)
        self.arm32 = AttentionRefinementModule(512, 128)
        self.conv_head32 = ConvBNReLU(128, 128, ks=3, stride=1, padding=1)
        self.conv_head16 = ConvBNReLU(128, 128, ks=3, stride=1, padding=1)
        self.conv_avg = ConvBNReLU(512, 128, ks=1, stride=1, padding=0)

    def forward(self, x):
        feat8, feat16, feat32 = self.resnet(x)
        avg = self.conv_avg(F.avg_pool2d(feat32, feat32.size()[2:]))
        feat32_sum = self.arm32(feat32) + _up(avg, feat32.size()[2:])
        feat32_up = self.conv_head32(_up(feat32_sum, feat16.size()[2:]))
        feat16_sum = self.arm16(feat16) + feat32_up
        feat16_up = self.conv_head16(_up(feat16_sum, feat8.size()[2:]))
        return feat8, feat16_up, feat32_up


class FeatureFusionModule(nn.Module):
    def __init__(self, in_chan, out_chan):
        super().__init__()
        self.convblk = ConvBNReLU(in_chan, out_chan, ks=1, stride=1, padding=0)
        self.conv1 = nn.Conv2d(out_chan, out_chan // 4, kernel_size=1, stride=1, padding=0, bias=False)
        self.conv2 = nn.Conv2d(out_chan // 4, out_chan, kernel_size=1, stride=1, padding=0, bias=False)
        self.relu = nn.ReLU(inplace=True)
        self.sigmoid = nn.Sigmoid()

    def forward(self, fsp, fcp):
        feat = self.convblk(torch.cat([fsp, fcp], dim=1))
        atten = self.sigmoid(self.conv2(self.relu(self.conv1(F.avg_pool2d(feat, feat.size()[2:])))))
        return torch.mul(feat, atten) + feat


class BiSeNet(nn.Module):
    def __init__(self, n_classes=20):
        super().__init__()
        self.cp = ContextPath()
        self.ffm = FeatureFusionModule(256, 256)
        self.conv_out = BiSeNetOutput(256, 256, n_classes)
        self.conv_out16 = BiSeNetOutput(128, 64, n_classes)
        self.conv_out32 = BiSeNetOutput(128, 64, n_classes)

    def logits(self, x):
        feat_res8, feat_cp8, _ = self.cp(x)
        return self.conv_out(self.ffm(feat_res8, feat_cp8))

    def forward(self, x):
        return _up(self.logits(x), x.size()[2:]), None, None

    @classmethod
    def load(cls, path, n_classes=20, map_location='cpu'):
        """The reference's initFaceParsing (dnnlib/seg_tools.py:126-129) from a local state_dict file such as segNet-20Class.pth."""
        path = os.fspath(path)
        if not os.path.isfile(path):
            raise FileNotFoundError(f'BiSeNet.load: no weights at {path!r} (nothing is downloaded)')
        net = cls(n_classes)
        net.load_state_dict(torch.load(path, map_location=map_location, weights_only=True), strict=True)
        return net.eval().requires_grad_(False)


def remap_ids(ids):
    """id_remap (dnnlib/seg_tools.py:63-64) on uint8 ids: BiSeNet's 20 classes -> COLOR_MAP's 19."""
    return torch.tensor(REMAP, dtype=torch.uint8, device=ids.device)[ids.long()]


@torch.no_grad()
def parse(net, img, remap=True):
    """parsing_img(net, img, remap=remap, return_mask=False) as uint8 ids [N, H, W] (dnnlib/seg_tools.py:101-117)."""
    ids = _seg_ops.seg_labels(net.logits(img), tuple(img.shape[-2:]), align_corners=True)
    return remap_ids(ids) if remap else ids
