"""Oracle (test infrastructure): the projector's losses restated with stock torch ops, stand-ins for the generator and the VGG16
feature network, and the CPU route of ide3d_b200.projector.

    inversion/training/projectors/w_projector_ide3d.py:113-122   noise regulariser: per buffer, at every avg-pool pyramid level down
                                                                to the first whose side is <= 8, mean(n * roll(n, 1, W))^2 +
                                                                mean(n * roll(n, 1, H))^2, summed
    inversion/training/projectors/w_projector_ide3d.py:138-142   renormalisation after every step: buf -= mean; buf *= rsqrt(mean(buf^2))
    (extension, no reference line)                               semantic-mask loss: F.cross_entropy of the logits upsampled with
                                                                training.triplane.upsample_seg's rule (bilinear, align_corners=False)

`cpu_projector_ops` routes ide3d_b200.torch_utils.ops.projection's three functions here, so the projector runs on the CPU with the
stand-ins below (tests/test_projector.py replays tests/golden/projector_trace.npz, recorded from the reference's own projectors by
tests/golden/make_projector_golden.py, that way).
"""

import contextlib
import io

import numpy as np
import torch
import torch.nn.functional as F

NOISE_SIDES = (4, 8, 16, 32)


def noise_reg(buffers):
    reg = 0.0
    for v in buffers:
        noise = v[None, None, :, :]
        while True:
            reg += (noise * torch.roll(noise, shifts=1, dims=3)).mean() ** 2
            reg += (noise * torch.roll(noise, shifts=1, dims=2)).mean() ** 2
            if noise.shape[2] <= 8:
                break
            noise = F.avg_pool2d(noise, kernel_size=2)
    return reg


@torch.no_grad()
def noise_normalize_(buffers):
    for buf in buffers:
        buf -= buf.mean()
        buf *= buf.square().mean().rsqrt()


def seg_cross_entropy(seg_raw, mask):
    up = F.interpolate(seg_raw, size=tuple(mask.shape[-2:]), mode='bilinear', align_corners=False)
    return F.cross_entropy(up, mask.long())


@contextlib.contextmanager
def cpu_projector_ops():
    """Inside the context, ide3d_b200.projector's kernel calls (noise regulariser, renormalisation, semantic cross-entropy) are the
    torch restatements above."""
    from ide3d_b200.torch_utils.ops import projection as P
    saved = (P.noise_regularizer, P.noise_normalize_, P.seg_cross_entropy)
    P.noise_regularizer, P.noise_normalize_, P.seg_cross_entropy = noise_reg, noise_normalize_, seg_cross_entropy
    try:
        yield
    finally:
        P.noise_regularizer, P.noise_normalize_, P.seg_cross_entropy = saved


# ------------------------------------------------------------------------------------------------ stand-in generator
def _param(rs, *shape, scale=1.0):
    return torch.nn.Parameter(torch.from_numpy((rs.randn(*shape) * scale).astype(np.float32)))


class StandInMapping(torch.nn.Module):
    def __init__(self, z_dim, c_dim, w_dim, num_ws, rs):
        super().__init__()
        self.num_ws = num_ws
        self.wz = _param(rs, z_dim, w_dim, scale=z_dim ** -0.5)
        self.wc = _param(rs, c_dim, w_dim, scale=0.2)

    def forward(self, z, c, truncation_psi=1, truncation_cutoff=None):
        w = torch.tanh(z.to(torch.float32) @ self.wz + c.to(torch.float32) @ self.wc)
        return w[:, None, :].repeat(1, self.num_ws, 1)


class StandInLayer(torch.nn.Module):
    """w [N, w_dim] -> [N, 3, side, side]: a styled constant modulated by the layer's noise buffer."""

    def __init__(self, side, w_dim, rs):
        super().__init__()
        self.register_buffer('noise_const', torch.from_numpy(rs.randn(side, side).astype(np.float32)))
        self.noise_strength = torch.nn.Parameter(torch.tensor(0.3))
        self.affine = _param(rs, w_dim, 3, scale=w_dim ** -0.5)
        self.const = _param(rs, 3, side, side, scale=0.5)

    def forward(self, w):
        return torch.tanh(w @ self.affine)[:, :, None, None] * (self.const + self.noise_const * self.noise_strength)


class StandInSynthesis(torch.nn.Module):
    """Differentiable stand-in for G.synthesis: one layer per noise buffer (sides NOISE_SIDES, ws rows 0..3) summed at the image
    resolution, then a camera term from cam2world (c[:, :16]) and per-class logits at the render resolution.  Honours views (the
    layers run once per latent, the camera part per view) and return_seg='raw' (a strided [N, 19, R, R] view, as the real
    generator returns)."""

    def __init__(self, w_dim, num_ws, img_resolution, render_size, rs):
        super().__init__()
        self.num_ws, self.img_resolution, self.render_size = num_ws, img_resolution, render_size
        self.layers = torch.nn.ModuleList([StandInLayer(s, w_dim, rs) for s in NOISE_SIDES])
        self.cam = _param(rs, 16, 3, scale=0.5)
        self.ramp = _param(rs, 1, 3, img_resolution, img_resolution, scale=1.0)
        self.seg_w = _param(rs, 3, 19, scale=1.0)
        self.seg_b = _param(rs, 19, scale=0.5)

    def forward(self, ws, c=None, noise_mode='const', force_fp32=False, return_seg=False, views=1, **kw):
        res = (self.img_resolution, self.img_resolution)
        x = 0
        for i, layer in enumerate(self.layers):
            x = x + F.interpolate(layer(ws[:, i]), size=res, mode='bilinear', align_corners=False)
        if views > 1:
            x = x.repeat_interleave(views, 0)
        cam = (c[:, :16, None] * self.cam).sum(1)                                     # per row: no batch-size dependent kernels
        img = torch.tanh(x + cam[:, :, None, None] * self.ramp)
        if not return_seg:
            return img
        small = F.adaptive_avg_pool2d(img, self.render_size)                          # [N, 3, R, R]
        logits = (small.permute(0, 2, 3, 1)[..., None] * self.seg_w).sum(3) + self.seg_b   # [N, R, R, 19]
        return img, logits.permute(0, 3, 1, 2)


class StandInGenerator(torch.nn.Module):
    def __init__(self, z_dim=16, c_dim=25, w_dim=8, num_ws=6, img_resolution=32, render_size=8, seed=5):
        super().__init__()
        rs = np.random.RandomState(seed)
        self.z_dim, self.c_dim, self.w_dim = z_dim, c_dim, w_dim
        self.img_resolution, self.img_channels = img_resolution, 3
        self.mapping = StandInMapping(z_dim, c_dim, w_dim, num_ws, rs)
        self.synthesis = StandInSynthesis(w_dim, num_ws, img_resolution, render_size, rs)
        self.num_ws = num_ws


# ------------------------------------------------------------------------------------------------ stand-in feature network
class StandInFeatures(torch.nn.Module):
    """The VGG16 TorchScript contract of the projectors (f(images [N,3,h,w] in 0..255, resize_images, return_lpips) -> [N, F]) with
    two random-init convolutions; return_lpips unit-normalises the features, as the LPIPS head does."""

    def __init__(self, seed: int = 11):
        super().__init__()
        rs = np.random.RandomState(seed)
        self.w1 = torch.nn.Parameter(torch.from_numpy((rs.randn(8, 3, 3, 3) / 5).astype(np.float32)))
        self.w2 = torch.nn.Parameter(torch.from_numpy((rs.randn(8, 8, 3, 3) / 8).astype(np.float32)))

    def forward(self, img: torch.Tensor, resize_images: bool = True, return_lpips: bool = False) -> torch.Tensor:
        x = img / 127.5 - 1
        if resize_images:
            x = F.interpolate(x, size=(32, 32), mode='area')
        x = F.relu(F.conv2d(x, self.w1, stride=2, padding=1))
        x = F.relu(F.conv2d(x, self.w2, stride=2, padding=1))
        f = x.flatten(1)
        if return_lpips:
            f = f / (f.square().sum(1, keepdim=True).sqrt() + 1e-8)
        return f


def standin_features():
    """The scripted stand-in, as torch.jit.load returns the reference's vgg16.pt."""
    return torch.jit.script(StandInFeatures().eval().requires_grad_(False))


def standin_features_bytes():
    buf = io.BytesIO()
    torch.jit.save(standin_features(), buf)
    return buf.getvalue()


# ------------------------------------------------------------------------------------------------ inputs of the golden trace
def golden_inputs():
    """(label [1, 25], target [3, 32, 32] in 0..255) the projector trace is recorded with: a camera 0.3 rad off frontal in yaw and
    0.1 in pitch at radius 2.7, the gen_images intrinsics, and a smooth random target."""
    rs = np.random.RandomState(3)
    yaw, pitch = 0.3, 0.1
    fwd = np.array([np.sin(yaw) * np.cos(pitch), np.sin(pitch), np.cos(yaw) * np.cos(pitch)])
    origin = 2.7 * fwd
    z = -fwd
    x = np.cross([0, 1, 0], z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    m = np.eye(4)
    m[:3, 0], m[:3, 1], m[:3, 2], m[:3, 3] = x, y, -z, origin
    intr = [4.2647, 0, 0.5, 0, 4.2647, 0.5, 0, 0, 1]
    label = torch.from_numpy(np.concatenate([m.reshape(-1), intr]).astype(np.float32))[None]
    small = torch.from_numpy(rs.rand(1, 3, 8, 8).astype(np.float32))
    target = (F.interpolate(small, size=(32, 32), mode='bilinear', align_corners=False)[0] * 255).round()
    return label, target
