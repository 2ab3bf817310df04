"""Oracle (test infrastructure): the multi-view image strips of gen_images.py, restated with stock torch ops, and the multi-view
renderer contract on the CPU.

    gen_images.py:109-116   per seed, G.synthesis(..., return_seg=True) at each yaw; seg -> (mask2color(seg) / 255 - 0.5) / 0.5; the views
                            concatenated and written by save_image(..., normalize=True, range=(-1, 1)) -- `range` being the old name of
                            torchvision's value_range
    torchvision make_grid   nrow=8, padding=2, pad_value=0, normalize: clamp_(-1, 1), sub_(-1), div_(2); a single image is returned bare
    torchvision save_image  mul(255).add_(0.5).clamp_(0, 255), HWC, uint8

`compose_strips` runs on whatever device its inputs live on: on CUDA tensors it is what the fused kernel (ide3d_image_strips) is
compared with.  `cpu_multiview_ops` extends oracle.backend.cpu_reference_ops to the multi-view renderer arguments (views, per-frame
jitter seeds) and routes ide3d_b200.images.compose_strips here, so the batched multi-view driver runs on the CPU.
"""

import contextlib

import numpy as np
import torch

from . import backend as obk
from . import renderer as orr
from .frames import mask2color


def grid_bytes(x):
    """make_grid(x, nrow=8, padding=2, pad_value=0, normalize=True, value_range=(-1, 1)) followed by save_image's conversion, for
    x [V, 3, H, W] with V <= 8.  -> uint8 [Hs, Ws, 3]."""
    t = x.clone()
    t.clamp_(min=-1, max=1)
    t.sub_(-1).div_(2)
    v, ch, h, w = t.shape
    if v == 1:
        grid = t[0]
    else:
        grid = torch.zeros((ch, h + 4, v * (w + 2) + 2), dtype=t.dtype, device=t.device)
        for j in range(v):
            grid[:, 2:2 + h, 2 + j * (w + 2):2 + j * (w + 2) + w] = t[j]
    return grid.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to(torch.uint8)


def compose_strips(img, seg_raw, views):
    """(image strips, seg strips), each uint8 [S, Hs, Ws, 3], for img [S*views, 3, H, W] and the render-resolution logits seg_raw
    [S*views, C, h, w] (row s*views + j is view j of seed s), as gen_images.py builds and saves them per seed."""
    from ide3d_b200.dnnlib.seg_tools import COLOR_MAP
    seg = torch.nn.functional.interpolate(seg_raw, size=tuple(img.shape[-2:]), mode='bilinear', align_corners=False)
    col = (mask2color(seg, COLOR_MAP) / 255. - 0.5) / 0.5
    n = img.shape[0] // views
    imgs = [grid_bytes(img[s * views:(s + 1) * views]) for s in range(n)]
    segs = [grid_bytes(col[s * views:(s + 1) * views]) for s in range(n)]
    if n == 0:
        return (torch.empty(0, dtype=torch.uint8, device=img.device),) * 2
    return torch.stack(imgs), torch.stack(segs)


def _multiview_renderer_forward(self, img_v, seg_v, cam2world, img_size=64, num_steps=48, perturb='hash', jitter_u=None, seed=None,
                                views=1, **kw):
    """TriPlaneRenderer.forward with views / per-frame seeds, on top of oracle.backend's one-plane-set-per-frame restatement: the plane
    sets are repeated per view, and per-frame seeds become explicit uniforms of the frame-local sample indices."""
    from ide3d_b200.render import frame_seeds
    if views > 1:
        img_v, seg_v = img_v.repeat_interleave(views, 0), seg_v.repeat_interleave(views, 0)
    seeds = frame_seeds(seed)
    if seeds is not None:
        n = img_v.shape[0]
        res = (img_size, img_size) if isinstance(img_size, int) else tuple(img_size)
        if len(seeds) != n:
            raise ValueError(f'oracle: {len(seeds)} per-frame seeds for {n} frames')
        if jitter_u is None and perturb in ('hash', True):
            idx = np.arange(res[0] * res[1] * num_steps, dtype=np.uint64)
            jitter_u = torch.from_numpy(np.stack([orr.hash_uniform(idx, s) for s in seeds])).reshape(n, res[0] * res[1], num_steps, 1)
        seed = None
    return obk._renderer_forward(self, img_v, seg_v, cam2world, img_size=img_size, num_steps=num_steps, perturb=perturb,
                                 jitter_u=jitter_u, seed=seed, **kw)


@contextlib.contextmanager
def cpu_multiview_ops():
    """oracle.backend.cpu_reference_ops, plus: the renderer accepts views / per-frame seeds, and ide3d_b200.images.compose_strips is
    the torch composition above."""
    from ide3d_b200 import images
    from ide3d_b200.training import triplane as p_tp
    R = p_tp.TriPlaneRenderer
    with obk.cpu_reference_ops():
        saved = (R.forward, images.compose_strips)
        R.forward, images.compose_strips = _multiview_renderer_forward, compose_strips
        try:
            yield
        finally:
            R.forward, images.compose_strips = saved
