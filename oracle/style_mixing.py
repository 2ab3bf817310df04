"""CPU restatements behind ide3d_b200.style_mixing (test infrastructure only).

  * StandInMapping: a mapping network of elementwise float32 products and sums (no reductions), so its ws are the same bits on every
    CPU; the golden of tests/golden/make_style_mixing_golden.py and the tests build it from the same seed.
  * to_uint8: style_mixing.py:101's conversion in torch.
  * paste_grid: the canvas loop of style_mixing.py:138-153 with numpy slice assignment in place of PIL's paste.
  * style_grid: the contract of ide3d_style_grid (include/ide3d_b200.h) in torch, for CPU runs of the driver.
"""

import types

import numpy as np
import torch


class StandInMapping(torch.nn.Module):
    """ws[n, i, j] = z[n, j] * a[i, j] + c[n, j % c_dim] * b[i, j] + d[i, j] in float32; w_avg is a fixed random vector."""

    def __init__(self, z_dim=16, c_dim=25, w_dim=8, num_ws=18, seed=0):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.z_dim, self.c_dim, self.w_dim, self.num_ws = z_dim, c_dim, w_dim, num_ws
        self.a, self.b, self.d = (torch.randn(num_ws, w_dim, generator=g) for _ in range(3))
        self.register_buffer('w_avg', torch.randn(w_dim, generator=g))

    def forward(self, z, c, truncation_psi=1, truncation_cutoff=None):
        assert truncation_psi == 1
        z = z.to(torch.float32)[:, None, :self.w_dim]
        cols = torch.arange(self.w_dim) % self.c_dim
        cc = torch.zeros(z.shape[0], 1, self.w_dim) if c is None else c.to(torch.float32)[:, None, cols]
        return z * self.a + cc * self.b + self.d


def stand_in_generator(seed=0):
    """An object with what style_mixing.mix_ws reads from a generator."""
    m = StandInMapping(seed=seed)
    return types.SimpleNamespace(z_dim=m.z_dim, c_dim=m.c_dim, num_ws=m.num_ws, mapping=m)


def to_uint8(img):
    """[N, 3, H, W] float -> [N, H, W, 3] uint8 (style_mixing.py:101)."""
    return (img.permute(0, 2, 3, 1) * 127.5 + 128).clamp(0, 255).to(torch.uint8)


def paste_grid(image_dict, row_seeds, col_seeds, height, width):
    """style_mixing.py:138-153: image_dict[(row seed, col seed)] uint8 [H, W, 3] or [H, W, 3, STEP] -> the STEP canvases
    [(R+1) H, (C+1) W, 3], black where nothing is pasted."""
    first = image_dict[(row_seeds[0], col_seeds[0])]
    steps = first.shape[-1] if first.ndim == 4 else 1
    out = []
    for step in range(steps):
        canvas = np.zeros([height * (len(row_seeds) + 1), width * (len(col_seeds) + 1), 3], dtype=np.uint8)
        for row_idx, row_seed in enumerate([0] + list(row_seeds)):
            for col_idx, col_seed in enumerate([0] + list(col_seeds)):
                if row_idx == 0 and col_idx == 0:
                    continue
                key = (row_seed, col_seed)
                if row_idx == 0:
                    key = (col_seed, col_seed)
                if col_idx == 0:
                    key = (row_seed, row_seed)
                img = image_dict[key]
                img = img if img.ndim == 3 else img[:, :, :, step]
                canvas[height * row_idx:height * (row_idx + 1), width * col_idx:width * (col_idx + 1)] = img
        out.append(canvas)
    return out


def style_grid(img, first_row, rows, cols, views, out, out_stride_row, out_stride_view):
    """ide3d_style_grid's contract: the canvas rows first_row .. first_row + rows - 1 of a (cols + 1)-column grid written through
    out's byte strides (see include/ide3d_b200.h)."""
    if rows == 0:
        return out
    h, w = img.shape[2:]
    wc = (cols + 1) * w
    first_cell = 0 if first_row == 0 else first_row * (cols + 1) - 1
    u8 = to_uint8(img).reshape(-1, views, h, w, 3)
    dst = torch.as_strided(out, (rows, views, h, wc, 3), (out_stride_row, out_stride_view, wc * 3, 3, 1), out.storage_offset())
    for gi in range(rows):
        g = first_row + gi
        for j in range(cols + 1):
            slot = g * (cols + 1) + j
            tile = dst[gi, :, :, j * w:(j + 1) * w]
            if slot == 0:
                tile.zero_()
            else:
                tile.copy_(u8[slot - 1 - first_cell])
    return out
