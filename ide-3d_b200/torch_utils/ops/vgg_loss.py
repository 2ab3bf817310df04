"""The VGG19 perceptual L1 loss of hybrid-encoder training (apps/train_hybrid_encoder.py:120-152) with its head on sm_90a.

    feat_l1(feats_x, feats_y, weights) -> (total, per-layer means [L])   sum_l w_l mean|x_l - y_l| in one call of ide3d_feat_l1_fwd
                                           (two launches) and, backward, ide3d_feat_l1_bwd (one launch); differentiable in feats_x
    feat_l1_torch(...)                     the reference's formula, sum_l w_l F.l1_loss(x_l, y_l), for tables the kernel refuses
                                           (more than IDE3D_FEAT_L1_MAX_LAYERS layers, features that are not fp32) and targets
                                           that require grad
    VGGLoss                                torchvision's vgg19().features sliced at TAPS, run on (x + 1) / 2 without ImageNet
                                           normalisation, and the head; VGGLoss.vgg19(path) loads torchvision's state_dict
"""

import ctypes as C
import os

import torch
import torch.nn.functional as F

from ... import _lib as L

TAPS = (2, 7, 12, 21, 30)                          # feature_layers of train_hybrid_encoder.py:124


def feat_l1_torch(feats_x, feats_y, weights):
    """The reference's formula: (sum_l w_l F.l1_loss(x_l, y_l), the per-layer means [L] without grad)."""
    layers = [F.l1_loss(x, y) for x, y in zip(feats_x, feats_y)]
    return sum(w * v for w, v in zip(weights, layers)), torch.stack([v.detach().float() for v in layers])


def _strides(t):
    return (C.c_int64 * 4)(*t.stride())


def _params(fx, fy, weights, dtype):
    p = L.FeatL1Params()
    p.n, p.num_layers, p.dtype = fx[0].shape[0], len(fx), dtype
    for i, (x, y, w) in enumerate(zip(fx[:L.FEAT_L1_MAX_LAYERS], fy, weights)):
        layer = p.layers[i]
        layer.c, layer.h, layer.w, layer.weight = x.shape[1], x.shape[2], x.shape[3], float(w)
        layer.x, layer.x_stride = x.data_ptr(), _strides(x)
        layer.y, layer.y_stride = y.data_ptr(), _strides(y)
    return p


class _Unsupported(Exception):
    pass


class _FeatL1(torch.autograd.Function):
    @staticmethod
    def forward(ctx, weights, dtype, *tensors):
        nl = len(weights)
        fx, fy = tensors[:nl], tensors[nl:]
        dev = fx[0].device
        p = _params(fx, fy, weights, dtype)
        lib = L.get_lib()
        need = lib.ide3d_feat_l1_scratch_bytes(C.byref(p))
        if need == L.UNSUPPORTED:
            raise _Unsupported()
        L.check(int(need) if need < 0 else L.OK)
        scratch = torch.empty(need // 8, dtype=torch.float64, device=dev)
        value = torch.empty(nl + 1, dtype=torch.float32, device=dev)
        p.value, p.scratch, p.scratch_bytes = value.data_ptr(), scratch.data_ptr(), need
        L.check(lib.ide3d_feat_l1_fwd(C.byref(p), L.stream_ptr(dev)))
        ctx.weights, ctx.dtype = weights, dtype
        ctx.save_for_backward(*tensors)
        layers = value[:nl].clone()
        ctx.mark_non_differentiable(layers)
        return value[nl].clone(), layers

    @staticmethod
    def backward(ctx, grad_total, grad_layers):
        tensors = ctx.saved_tensors
        nl = len(ctx.weights)
        fx, fy = tensors[:nl], tensors[nl:]
        p = _params(fx, fy, ctx.weights, ctx.dtype)
        g = grad_total.detach().to(torch.float32).reshape(1).contiguous()
        p.grad_value = g.data_ptr()
        gx = []
        for i in range(nl):
            gx.append(torch.empty_like(fx[i], memory_format=torch.preserve_format))
            p.layers[i].grad_x, p.layers[i].gx_stride = gx[i].data_ptr(), _strides(gx[i])
        L.check(L.get_lib().ide3d_feat_l1_bwd(C.byref(p), L.stream_ptr(fx[0].device)))
        return (None, None, *gx, *([None] * nl))


def feat_l1(feats_x, feats_y, weights):
    """sum_l w_l mean|x_l - y_l| -> (total (0-d), the per-layer means [L], not differentiable).  feats_x: per layer [N, C, H, W],
    any strides (NCHW or channels_last); feats_y: the same shapes, no grad (the targets); weights: floats.  Differentiable in feats_x.
    CUDA tensors only."""
    feats_x, feats_y, weights = list(feats_x), list(feats_y), [float(w) for w in weights]
    if not feats_x or not len(feats_x) == len(feats_y) == len(weights):
        raise ValueError(f'feat_l1: {len(feats_x)} / {len(feats_y)} / {len(weights)} layers of x / y / weights')
    n, dev = feats_x[0].shape[0], feats_x[0].device
    for i, (x, y) in enumerate(zip(feats_x, feats_y)):
        if x.ndim != 4 or y.shape != x.shape or y.dtype != x.dtype:
            raise ValueError(f'feat_l1: layer {i}: x {tuple(x.shape)} {x.dtype} and y {tuple(y.shape)} {y.dtype} must be equal 4-d shapes')
        if x.shape[0] != n or x.device != dev or y.device != dev:
            raise ValueError(f'feat_l1: layer {i} has {x.shape[0]} samples on {x.device} / {y.device}; every layer must have the '
                             f'{n} samples of layer 0 on {dev}')
    L.require_cuda(*feats_x, *feats_y)
    if not any(y.requires_grad for y in feats_y):
        dtype = L.F32 if feats_x[0].dtype == torch.float32 and all(t.dtype == torch.float32 for t in feats_x) else -1
        try:
            return _FeatL1.apply(weights, dtype, *feats_x, *feats_y)
        except _Unsupported:
            pass
    return feat_l1_torch(feats_x, feats_y, weights)


class VGGLoss(torch.nn.Module):
    """VGGLoss(features, weights=(1,) * 5): `features` an nn.Sequential with torchvision vgg19().features's layout.  __call__(x, y) ->
    sum_l w_l mean|f_l((x + 1) / 2) - f_l((y + 1) / 2)| for images in [-1, 1]; y is an image batch or the list VGGLoss.target(y)
    returned, the target's features computed once under no_grad."""

    def __init__(self, features, weights=(1.0,) * len(TAPS)):
        super().__init__()
        if len(weights) != len(TAPS):
            raise ValueError(f'VGGLoss: {len(weights)} weights for {len(TAPS)} taps')
        self.weights = tuple(float(w) for w in weights)
        self.slices = torch.nn.ModuleList()
        prev = 0
        for tap in TAPS:
            self.slices.append(torch.nn.Sequential(*[features[i] for i in range(prev, tap)]))
            prev = tap
        self.requires_grad_(False)

    def trunk(self, x):
        out = []
        x = (x + 1) / 2
        for s in self.slices:
            x = s(x)
            out.append(x)
        return out

    @torch.no_grad()
    def target(self, y):
        return [f.detach() for f in self.trunk(y)]

    def forward(self, x, y):
        fy = y if isinstance(y, (list, tuple)) else self.target(y)
        return feat_l1(self.trunk(x), fy, self.weights)[0]

    @classmethod
    def vgg19(cls, path, weights=(1.0,) * len(TAPS), map_location='cpu'):
        """torchvision's VGG19 from a local state_dict file (features.* keys; classifier.* ignored).  Nothing is downloaded."""
        import torchvision
        if not os.path.isfile(path):
            raise FileNotFoundError(f'VGGLoss: weight file {os.fspath(path)!r} not found (nothing is downloaded)')
        net = torchvision.models.vgg19(weights=None)
        state = torch.load(os.fspath(path), map_location=map_location, weights_only=True)
        net.features.load_state_dict({k[len('features.'):]: v for k, v in state.items() if k.startswith('features.')}, strict=True)
        return cls(net.features, weights).eval()
