"""CPU restatements behind ide3d_b200.viz.renderer (test infrastructure only).

  * StandInMapping / StandInGenerator: a mapping of elementwise float32 products and sums (same bits on every CPU) with the
    reference's truncation rule, and a synthesis module that returns seeded image / image_depth / image_raw maps derived from its
    inputs; tests/golden/make_viz_golden.py runs the reference's renderer over them.
  * display: the display tail of viz/renderer.py:362-406 in torch, with the FFT in float64 (the contract of
    torch_utils.ops.viz.display).
  * index_lut: a seeded colormap whose entries name their index, so a panel can be decoded to colormap indices.
"""

import numpy as np
import torch


class StandInMapping(torch.nn.Module):
    """ws[n, i, j] = z[n, j] * a[i, j] + c[n, j % c_dim] * b[i, j] + d[i, j], then the truncation of the reference's mapping."""

    def __init__(self, z_dim=16, c_dim=25, w_dim=8, num_ws=18, seed=0):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.z_dim, self.c_dim, self.w_dim, self.num_ws = z_dim, c_dim, w_dim, num_ws
        self.a, self.b, self.d = (torch.randn(num_ws, w_dim, generator=g) for _ in range(3))
        self.register_buffer('w_avg', torch.randn(w_dim, generator=g))
        self.calls = []

    def forward(self, z, c, truncation_psi=1, truncation_cutoff=None):
        self.calls.append((z.clone(), c.clone()))
        z = z.to(torch.float32)[:, None, :self.w_dim]
        cols = torch.arange(self.w_dim) % self.c_dim
        x = z * self.a + c.to(torch.float32)[:, None, cols] * self.b + self.d
        if truncation_psi != 1:
            rows = slice(None) if truncation_cutoff is None else slice(0, truncation_cutoff)
            x[:, rows] = self.w_avg + (x[:, rows] - self.w_avg) * truncation_psi
        return x


class StandInSynthesis(torch.nn.Module):
    """Seeded maps from the call's inputs: image [1, 3, 32, 32], image_depth [1, 1, 16, 16] (positive, a depth-like range),
    image_raw [1, 3, 16, 16].  Returns the dict of return_dict=True; the calls' inputs and outputs are kept."""

    def __init__(self, num_ws=18):
        super().__init__()
        self.num_ws = num_ws
        self.register_buffer('noise_const', torch.zeros(4, 4))
        self.calls = []

    def forward(self, ws, c, noise_mode='const', force_fp32=False, **_):
        seed = int(abs(float(ws.double().sum()) * 1e3 + float(c.double().sum()) * 1e2)) % (2 ** 31)
        g = torch.Generator().manual_seed(seed)
        out = dict(image=torch.randn(1, 3, 32, 32, generator=g) * 0.8,
                   image_depth=2.5 + 0.1 * torch.rand(1, 1, 16, 16, generator=g),
                   image_raw=torch.randn(1, 3, 16, 16, generator=g) * 3)
        self.calls.append((ws.clone(), c.clone(), {k: v.clone() for k, v in out.items()}))
        return out


class StandInGenerator(torch.nn.Module):
    def __init__(self, seed=0):
        super().__init__()
        self.mapping = StandInMapping(seed=seed)
        self.synthesis = StandInSynthesis(self.mapping.num_ws)
        self.z_dim, self.c_dim, self.img_resolution = self.mapping.z_dim, self.mapping.c_dim, 32

    @property
    def backbone(self):
        return self.synthesis

    def to(self, *args, **kwargs):
        """A CPU stand-in: the reference's .to('cuda') keeps it where it is."""
        return self


def index_lut(K=1024, seed=0):
    """uint8 [K, 3]: (k mod 256, k div 256, a seeded byte) -- distinct rows that give their index back."""
    k = torch.arange(K)
    rnd = torch.randint(0, 256, (K,), generator=torch.Generator().manual_seed(seed))
    return torch.stack([k & 255, k >> 8, rnd], 1).to(torch.uint8)


def decode(panel):
    p = np.asarray(panel).astype(np.int64)
    return p[..., 0] + 256 * p[..., 1]


def display(out, render_type='image', sel_channels=3, base_channel=0, img_normalize=False, img_scale_db=0, fft_show=False, fft_all=True,
            fft_range_db=50, fft_beta=8, cmap=None):
    """-> (uint8 [H, W, S] or [H, 2W, 3], float32 stats [6]); the FFT in float64 (the kernel's contract)."""
    out = out.to(torch.float32).clone()
    if sel_channels > out.shape[0]:
        sel_channels = 1
    base_channel = max(min(base_channel, out.shape[0] - sel_channels), 0)
    sel = out[base_channel:base_channel + sel_channels]
    stats = torch.stack([out.mean(), sel.mean(), out.std(), sel.std(), out.norm(float('inf')), sel.norm(float('inf'))])
    raw = out.clone()
    if render_type == 'image_depth':
        out -= out.min()
        out /= out.max()
        out -= .5
        out *= -2
    img = sel
    if img_normalize:
        img = img / img.norm(float('inf'), dim=[1, 2], keepdim=True).clip(1e-8, 1e8)
    img = img * (10 ** (img_scale_db / 20))
    img = (img * 127.5 + 128).clamp(0, 255).to(torch.uint8).permute(1, 2, 0)
    if not fft_show:
        return img, stats
    sig = (raw if fft_all else raw[base_channel:base_channel + sel_channels]).double()
    sig = sig - sig.mean(dim=[1, 2], keepdim=True)
    sig = sig * torch.kaiser_window(sig.shape[1], periodic=False, beta=fft_beta).double()[None, :, None]
    sig = sig * torch.kaiser_window(sig.shape[2], periodic=False, beta=fft_beta).double()[None, None, :]
    p = torch.fft.fftn(sig, dim=[1, 2]).abs().square().sum(dim=0)
    p = p.roll(shifts=[p.shape[0] // 2, p.shape[1] // 2], dims=[0, 1])
    hi = cmap.shape[0] - 1
    mean = p.mean()
    t = torch.zeros_like(p) if not mean > 0 else ((10 * (p / mean).log10() / fft_range_db + 1) / 2 * hi + 0.5)
    idx = torch.nan_to_num(t, nan=0.0, neginf=0.0).clamp(0, hi).floor().to(torch.int64)
    return torch.cat([img.expand(-1, -1, 3), cmap[idx]], dim=1), stats
