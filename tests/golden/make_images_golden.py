"""Records tests/golden/image_strips.npz: the two PNG strips gen_images.py writes per seed (gen_images.py:109-116), computed with
torchvision itself -- make_grid(normalize=True, value_range=(-1, 1)) (the reference passes the old name `range=`) followed by save_image's
conversion -- from seeded synthesis-like inputs.

    python tests/golden/make_images_golden.py

Cases (prefix `v{views}_`), each for 2 seeds:
  img  [2*views, 3, H, W] float32, N(0, 1.3^2): values beyond +-1 exercise the clamp; case v3 carries one NaN pixel
  seg  [2*views, 19, h, w] float32: render-resolution logits, upsampled as G.synthesis(return_seg=True) does
  out_img / out_seg  uint8 [2, Hs, Ws, 3]: the bytes save_image hands to PIL
"""

import os
import sys

import numpy as np
import torch
from torchvision.utils import make_grid

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

H = W = 64
R = 16


def save_image_bytes(x):
    """torchvision.utils.save_image(x, ..., normalize=True, value_range=(-1, 1)) up to the PIL call: uint8 HWC."""
    grid = make_grid(x, nrow=8, padding=2, pad_value=0, normalize=True, value_range=(-1, 1))
    return grid.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to('cpu', torch.uint8).numpy()


def main():
    from ide3d_b200.dnnlib.seg_tools import COLOR_MAP
    out = {}
    for views in (1, 3):
        g = torch.Generator().manual_seed(100 + views)
        n = 2 * views
        img = torch.randn(n, 3, H, W, generator=g) * 1.3
        if views == 3:
            img[4, 1, 10, 20] = float('nan')
        seg = torch.randn(n, 19, R, R, generator=g) * 3
        up = torch.nn.functional.interpolate(seg, size=(H, W), mode='bilinear', align_corners=False)
        lut = torch.tensor([COLOR_MAP.get(k, [0, 0, 0]) for k in range(19)], dtype=torch.float32)
        col = (lut[up.argmax(1)].permute(0, 3, 1, 2) / 255. - 0.5) / 0.5                     # mask2color, then gen_images.py:110
        out[f'v{views}_img'] = img.numpy()
        out[f'v{views}_seg'] = seg.numpy()
        out[f'v{views}_out_img'] = np.stack([save_image_bytes(img[s * views:(s + 1) * views]) for s in range(2)])
        out[f'v{views}_out_seg'] = np.stack([save_image_bytes(col[s * views:(s + 1) * views]) for s in range(2)])
    np.savez_compressed(os.path.join(HERE, 'image_strips.npz'), **out)


if __name__ == '__main__':
    main()
