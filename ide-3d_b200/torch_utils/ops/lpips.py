"""LPIPS v0.1 (the perceptual loss of pivotal tuning, inversion/training/coaches/base_coach.py:13,44) with its head on sm_90a.

    lpips_head(feats_x, feats_y, lin) -> [N]   sum_l mean_p sum_c lin_l[c] (u_c - v_c)^2, u / v the features normalised over the
                                               channels (inversion/criteria/lpips/utils.py:6-8); every layer in one call of
                                               ide3d_lpips_fwd (two launches) and, backward, ide3d_lpips_bwd (one launch)
    lpips_head_torch(...)                      the reference's formula in torch ops, for tables the kernel refuses (more than
                                               IDE3D_LPIPS_MAX_LAYERS layers, features that are not fp32)
    LPIPS                                      the AlexNet trunk (scaling layer, torchvision's alexnet().features up to the fifth
                                               ReLU, tapped after every ReLU) and the head; LPIPS.alexnet(trunk, lin) loads weights

Where the torch formula has a zero feature vector its gradient is NaN (the derivative of sqrt at 0); the kernel writes 0 there, so a
ReLU trunk's gradient stays finite, as torch's threshold_backward makes it when it runs through the trunk.
"""

import ctypes as C
import os

import torch
import torch.nn.functional as F

from ... import _lib as L

EPS = 1e-10
SHIFT = (-.030, -.088, -.188)                     # inversion/criteria/lpips/networks.py:40-43
SCALE = (.458, .448, .450)
ALEX_TAPS = (1, 4, 7, 9, 11)                      # the ReLUs of alexnet().features (networks.py:79: target_layers 2, 5, 8, 10, 12)
ALEX_CHANNELS = (64, 192, 384, 256, 256)


def lpips_head_torch(feats_x, feats_y, lin):
    """The reference's head (lpips.py:29-35): normalise, difference squared, 1x1 convolution with lin, spatial mean, summed over the
    layers.  -> [N]; feats_y may have one sample for every sample of feats_x."""
    res = []
    for fx, fy, w in zip(feats_x, feats_y, lin):
        u = fx / (torch.sqrt(torch.sum(fx ** 2, dim=1, keepdim=True)) + EPS)
        v = fy / (torch.sqrt(torch.sum(fy ** 2, dim=1, keepdim=True)) + EPS)
        res.append(F.conv2d((u - v) ** 2, w.reshape(1, -1, 1, 1)).mean((2, 3)))
    return torch.cat(res, 1).sum(1)


class _Unsupported(Exception):
    pass


def _strides(t):
    s = t.stride()
    return (C.c_int64 * 4)(*s) if t.shape[0] > 1 else (C.c_int64 * 4)(0, *s[1:])


def _params(fx, fy, lin, n):
    p = L.LpipsParams()
    p.n, p.num_layers = n, len(fx)
    for i, (x, y, w) in enumerate(zip(fx[:L.LPIPS_MAX_LAYERS], fy, lin)):
        layer = p.layers[i]
        layer.c, layer.h, layer.w = x.shape[1], x.shape[2], x.shape[3]
        layer.x, layer.x_stride = x.data_ptr(), _strides(x)
        layer.y, layer.y_stride = y.data_ptr(), _strides(y)
        layer.lin = w.data_ptr()
    return p


class _LpipsHead(torch.autograd.Function):
    @staticmethod
    def forward(ctx, nl, *tensors):
        fx, fy, lin = tensors[:nl], tensors[nl:2 * nl], tensors[2 * nl:]
        n, dev = fx[0].shape[0], fx[0].device
        p = _params(fx, fy, lin, n)
        lib = L.get_lib()
        need = lib.ide3d_lpips_scratch_bytes(C.byref(p))
        if need == L.UNSUPPORTED:
            raise _Unsupported()
        L.check(int(need) if need < 0 else L.OK)
        scratch = torch.empty(need // 8, dtype=torch.float64, device=dev)
        value = torch.empty(n, dtype=torch.float32, device=dev)
        p.value, p.scratch, p.scratch_bytes = value.data_ptr(), scratch.data_ptr(), need
        L.check(lib.ide3d_lpips_fwd(C.byref(p), L.stream_ptr(dev)))
        ctx.nl = nl
        ctx.save_for_backward(*tensors)
        return value

    @staticmethod
    def backward(ctx, grad_value):
        nl = ctx.nl
        tensors = ctx.saved_tensors
        fx, fy, lin = tensors[:nl], tensors[nl:2 * nl], tensors[2 * nl:]
        n, dev = fx[0].shape[0], fx[0].device
        want_x, want_y = any(ctx.needs_input_grad[1:1 + nl]), any(ctx.needs_input_grad[1 + nl:1 + 2 * nl])
        p = _params(fx, fy, lin, n)
        g = grad_value.detach().to(torch.float32).contiguous()
        p.grad_value = g.data_ptr()
        gx, gy = [None] * nl, [None] * nl
        for i in range(nl):
            if want_x:
                gx[i] = torch.empty_like(fx[i], memory_format=torch.preserve_format)
                p.layers[i].grad_x, p.layers[i].gx_stride = gx[i].data_ptr(), _strides(gx[i])
            if want_y:               # per sample; a broadcast target's gradient is the sum over the samples
                gy[i] = torch.empty_like(fx[i])
                p.layers[i].grad_y, p.layers[i].gy_stride = gy[i].data_ptr(), (C.c_int64 * 4)(*gy[i].stride())
        L.check(L.get_lib().ide3d_lpips_bwd(C.byref(p), L.stream_ptr(dev)))
        if want_y:
            gy = [t if fy[i].shape[0] == n else t.sum(0, keepdim=True) for i, t in enumerate(gy)]
        return (None, *gx, *gy, *([None] * nl))


def _kernel_table(feats_x, feats_y, lin):
    return (all(t.dtype == torch.float32 and t.ndim == 4 for t in (*feats_x, *feats_y))
            and all(w.dtype == torch.float32 and w.is_contiguous() for w in lin)
            and len(feats_x) <= L.LPIPS_MAX_LAYERS)


def lpips_head(feats_x, feats_y, lin):
    """sum over layers of mean_p sum_c lin[c] (u_c - v_c)^2 -> [N].  feats_x: per layer [N, C, H, W] fp32, any strides (NCHW or
    channels_last); feats_y: the same shapes with N or 1 samples (one target for all); lin: per layer [C] (or [1, C, 1, 1]) fp32.
    Differentiable in feats_x and feats_y.  CUDA tensors only."""
    feats_x, feats_y = list(feats_x), list(feats_y)
    lin = [w.reshape(-1) for w in lin]
    if not feats_x or not len(feats_x) == len(feats_y) == len(lin):
        raise ValueError(f'lpips_head: {len(feats_x)} / {len(feats_y)} / {len(lin)} layers of x / y / lin')
    n = feats_x[0].shape[0]
    for i, (x, y, w) in enumerate(zip(feats_x, feats_y, lin)):
        if x.ndim != 4 or x.shape[0] != n or y.ndim != 4 or y.shape[0] not in (1, n) or y.shape[1:] != x.shape[1:] or w.numel() != x.shape[1]:
            raise ValueError(f'lpips_head: layer {i}: x {tuple(x.shape)}, y {tuple(y.shape)}, lin {tuple(w.shape)} do not match '
                             f'(x [{n}, C, H, W], y [{n} or 1, C, H, W], lin [C])')
    L.require_cuda(*feats_x, *feats_y, *lin)
    if _kernel_table(feats_x, feats_y, lin):
        try:
            return _LpipsHead.apply(len(feats_x), *feats_x, *feats_y, *lin)
        except _Unsupported:
            pass
    return lpips_head_torch(feats_x, feats_y, lin)


class LPIPS(torch.nn.Module):
    """LPIPS v0.1 with the AlexNet trunk.  LPIPS(features, lin): `features` an nn.Sequential with torchvision alexnet().features's
    layout, `lin` the five per-layer weight vectors.  __call__(x, y) -> [N] for images in [-1, 1]; y is an image batch ([N or 1, 3,
    H, W]) or the list LPIPS.target(y) returned, the target's trunk features computed once."""

    def __init__(self, features, lin):
        super().__init__()
        self.features = features[:ALEX_TAPS[-1] + 1]
        self.register_buffer('shift', torch.tensor(SHIFT)[None, :, None, None])
        self.register_buffer('scale', torch.tensor(SCALE)[None, :, None, None])
        lin = [torch.as_tensor(w, dtype=torch.float32).reshape(-1) for w in lin]
        if [w.numel() for w in lin] != list(ALEX_CHANNELS):
            raise ValueError(f'LPIPS: lin must hold {len(ALEX_CHANNELS)} vectors of {ALEX_CHANNELS} weights, got {[w.numel() for w in lin]}')
        for k, w in enumerate(lin):
            self.register_buffer(f'lin{k}', w)
        self.requires_grad_(False)

    @property
    def lin(self):
        return [getattr(self, f'lin{k}') for k in range(len(ALEX_CHANNELS))]

    def trunk(self, x):
        """The ReLU outputs at ALEX_TAPS of the scaled input (networks.py:45-58, without the normalisation the head does)."""
        x = (x - self.shift) / self.scale
        out = []
        for i, layer in enumerate(self.features):
            x = layer(x)
            if i in ALEX_TAPS:
                out.append(x)
        return out

    @torch.no_grad()
    def target(self, y):
        return [f.detach() for f in self.trunk(y)]

    def forward(self, x, y):
        fy = y if isinstance(y, (list, tuple)) else self.trunk(y)
        return lpips_head(self.trunk(x), fy, self.lin)

    @classmethod
    def alexnet(cls, trunk_path, lin_path, map_location='cpu'):
        """Weights from files: trunk_path a torchvision AlexNet state dict (features.* keys, classifier.* ignored), lin_path the lpips
        package's weights/v0.1/alex.pth (lin{k}.model.1.weight [1, C, 1, 1]).  Nothing is downloaded."""
        import torchvision
        for path in (trunk_path, lin_path):
            if not os.path.isfile(path):
                raise FileNotFoundError(f'LPIPS: weight file {os.fspath(path)!r} not found (nothing is downloaded)')
        net = torchvision.models.alexnet(weights=None)
        state = torch.load(os.fspath(trunk_path), map_location=map_location, weights_only=True)
        net.features.load_state_dict({k[len('features.'):]: v for k, v in state.items() if k.startswith('features.')})
        lin_state = torch.load(os.fspath(lin_path), map_location=map_location, weights_only=True)
        lin = [lin_state[f'lin{k}.model.1.weight'] for k in range(len(ALEX_CHANNELS))]
        return cls(net.features, lin).eval()
