"""Batched, sharded driver for the multi-view images of gen_images.py.

The reference renders, per seed, the same latent from three yaws with three batch-1 G.synthesis calls -- three tri-plane backbone
passes on identical ws -- then builds the semantic colours from 512^2 logits and writes two save_image strips (gen_images.py:84-116).
Here the seeds are batched: one mapping call, one synthesis call per batch of seeds with `views=len(yaws)` (one backbone pass per
seed, the renderer and the super-resolution blocks per view), and the two strips of every seed composed in one kernel
(ide3d_image_strips) straight from the render-resolution logits.  The per-view depth jitter reproduces the loop's draws.  Batches are
sharded over the ranks and reach rank 0's host memory through dist.stream_sharded.
"""

import ctypes as C
import math
import os

import numpy as np
import torch

from . import _lib as L

YAWS = (-0.5, 0, 0.5)                                                         # gen_images.py:93
INTRINSICS = [4.2647, 0, 0.5, 0, 4.2647, 0.5, 0, 0, 1]                        # gen_images.py:107
FRONTAL = [1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 2.7, 0, 0, 0, 1] + INTRINSICS      # gen_images.py:87, the mapping's label
MAX_VIEWS = 8                                                                 # one make_grid row (nrow=8)


def render_params(yaw):
    """The render_params gen_images.py:96-103 passes with view `yaw` (with a camera given, only fov and num_steps are read)."""
    return {'h_mean': yaw + math.pi * 0.5, 'v_mean': math.pi * 0.5, 'h_stddev': 0., 'v_stddev': 0., 'fov': 18, 'num_steps': 96}


def view_cameras(yaws=YAWS, device='cpu'):
    """c [len(yaws), 25] exactly as gen_images.py:104-107 builds it for each yaw."""
    from .training.volumetric_rendering import create_cam2world_matrix, sample_camera_positions
    rows = []
    for yaw in yaws:
        camera_points, _, _ = sample_camera_positions(device, n=1, r=2.7, horizontal_mean=yaw + math.pi * 0.5, vertical_mean=math.pi * 0.5,
                                                      mode=None)
        c = create_cam2world_matrix(-camera_points, camera_points, device=device).reshape(1, -1)
        rows.append(torch.cat((c, torch.tensor(INTRINSICS).reshape(1, -1).to(c)), -1))
    return torch.cat(rows)


def view_seeds(seed, num_views):
    """The depth-jitter seeds the reference loop draws for `seed`: torch.manual_seed(seed), then one torch.randint(0, 2**62, (1,)) per
    G.synthesis call (TriPlaneRenderer.forward), in yaw order.  Drawn from a private generator: the global RNG state is not touched."""
    g = torch.Generator().manual_seed(int(seed))
    return [int(torch.randint(0, 2 ** 62, (1,), generator=g).item()) for _ in range(num_views)]


def strip_shape(views, height, width):
    """(strip_h, strip_w) of make_grid(nrow=8, padding=2) for one row of `views` images; the bare image for views == 1."""
    return (height, width) if views == 1 else (height + 4, views * (width + 2) + 2)


def compose_strips(img, seg_raw, views):
    """The two strips gen_images.py saves per seed, in one fused pass (ide3d_image_strips).  img [S*views, 3, H, W] float32, any strides;
    seg_raw [S*views, C, h, w] float32, any strides -- the render-resolution logits of G.synthesis(..., return_seg='raw'), upsampled inside
    the kernel by the rule of training.triplane.upsample_seg.  Row s*views + j is view j of seed s.
    -> (image strips, seg strips), each uint8 [S, Hs, Ws, 3] (HWC, what save_image hands to PIL).  CUDA tensors only."""
    L.require_cuda(img, seg_raw)
    L.forbid_grad('images.compose_strips', img, seg_raw)
    for name, t in (('img', img), ('seg_raw', seg_raw)):
        if t.dtype != torch.float32 or t.ndim != 4:
            raise RuntimeError(f'ide3d_b200.images.compose_strips: {name} must be float32 [N, C, H, W], got {t.dtype} {tuple(t.shape)}')
    views = int(views)
    if not 1 <= views <= MAX_VIEWS:
        raise ValueError(f'ide3d_b200.images.compose_strips: 1 <= views <= {MAX_VIEWS}, got {views}')
    n, ch, h, w = img.shape
    if ch != 3 or n % views or seg_raw.shape[0] != n:
        raise RuntimeError(f'ide3d_b200.images.compose_strips: need img [S*{views}, 3, H, W] and as many logit maps, got '
                           f'{tuple(img.shape)} and {tuple(seg_raw.shape)}')
    seeds = n // views
    hs, ws = strip_shape(views, h, w)
    out_img = torch.empty([seeds, hs, ws, 3], dtype=torch.uint8, device=img.device)
    out_seg = torch.empty_like(out_img)
    from .dnnlib.seg_tools import _lut_for
    lut = _lut_for(seg_raw.device, seg_raw.shape[1])
    p = L.StripsParams()
    p.image, p.seeds, p.views, p.height, p.width = img.data_ptr(), seeds, views, h, w
    p.image_stride_n, p.image_stride_c, p.image_stride_h, p.image_stride_w = img.stride()
    p.seg, (p.seg_c, p.seg_h, p.seg_w) = seg_raw.data_ptr(), seg_raw.shape[1:]
    p.seg_stride_n, p.seg_stride_c, p.seg_stride_h, p.seg_stride_w = seg_raw.stride()
    p.lut, p.out_image, p.out_seg = lut.data_ptr(), out_img.data_ptr(), out_seg.data_ptr()
    L.check(L.get_lib().ide3d_image_strips(C.byref(p), L.stream_ptr(img.device)))
    return out_img, out_seg


@torch.no_grad()
def render_multiview(G, seeds, rank=0, world=1, psi=1, noise_mode='const', yaws=YAWS, batch_seeds=8, outdir=None):
    """gen_images.py:84-116 as one batched, sharded call.  -> (img_strips, seg_strips), uint8 numpy arrays [len(seeds), Hs, Ws, 3] (views of one host copy) on
    rank 0 (None on the other ranks), seed order; Hs x Ws = strip_shape(len(yaws), G.img_resolution, G.img_resolution).  With `outdir`,
    rank 0 also writes seed%04d.png / seed%04d_seg.png there, as the reference does.

    Per seed: z = RandomState(seed).randn(1, z_dim), mapped with the frontal label; every yaw's camera is gen_images.py's; the depth jitter
    of view j uses the j-th seed the reference loop draws after torch.manual_seed(seed) (view_seeds), so with noise_mode 'const' or 'none'
    a strip is what the loop writes up to the batch size's effect on the convolution algorithms.  noise_mode='random' draws the backbone
    and super-resolution noise per batch, so it is not loop-reproducible.  The seed list is padded to a multiple of world * batch with
    repeats of its last seed (rendered and dropped)."""
    from . import dist as idist
    seeds = [int(s) for s in seeds]
    V = len(yaws)
    if not 1 <= V <= MAX_VIEWS:
        raise ValueError(f'render_multiview: 1 <= len(yaws) <= {MAX_VIEWS}, got {V}')
    if not seeds:
        raise ValueError('render_multiview: no seeds')
    dev = next(G.parameters()).device
    batch = max(1, min(int(batch_seeds), -(-len(seeds) // world)))
    total = -(-len(seeds) // (world * batch)) * world * batch
    padded = seeds + [seeds[-1]] * (total - len(seeds))

    cams = view_cameras(yaws, dev)                                                     # [V, 25], shared by every seed
    z = torch.from_numpy(np.concatenate([np.random.RandomState(s).randn(1, G.z_dim) for s in padded])).to(dev)
    label = torch.tensor(FRONTAL).float().to(dev).reshape(1, -1).repeat(total, 1)
    ws = G.mapping(z=z, c=label, truncation_psi=psi)
    jitter = torch.tensor([view_seeds(s, V) for s in padded], dtype=torch.int64)      # [total, V]
    rp = render_params(yaws[0])
    hs, wd = strip_shape(V, G.img_resolution, G.img_resolution)

    def render(idx):
        w_b = ws[idx]
        k = w_b.shape[0]
        img, seg_raw = G.synthesis(w_b, c=cams.repeat(k, 1), render_params=rp, noise_mode=noise_mode, return_seg='raw', views=V,
                                   seed=jitter[idx].reshape(-1))
        s_img, s_seg = compose_strips(img, seg_raw, V)
        return torch.stack((s_img, s_seg), 1)

    host = idist.stream_sharded(render, total, (2, hs, wd, 3), dev, rank, world, batch=batch, tag='strips')
    if host is None:
        return None
    strips = host[:len(seeds)].numpy().copy()                       # the host buffer is reused by the next call
    img_strips, seg_strips = strips[:, 0], strips[:, 1]
    if outdir is not None:
        import PIL.Image
        os.makedirs(outdir, exist_ok=True)
        for s, a, b in zip(seeds, img_strips, seg_strips):
            PIL.Image.fromarray(a, 'RGB').save(os.path.join(outdir, f'seed{s:04d}.png'))
            PIL.Image.fromarray(b, 'RGB').save(os.path.join(outdir, f'seed{s:04d}_seg.png'))
    return img_strips, seg_strips
