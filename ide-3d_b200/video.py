"""Batched driver for the latent-interpolation video of gen_videos.py (BASELINE config 3; SURVEY.md §8f rank 2).

The reference renders one (grid cell, frame) per `G.synthesis` call and evaluates a scipy spline and a camera pose on the host
in between (gen_videos.py:118-129), i.e. batch 1 and a host round trip per frame.  Every (w, camera) pair of the video is a pure
function of (seeds, frame index), so here they are all computed up front -- `interp_video_inputs`, same arithmetic, same nested
order (frame, grid row, grid column) -- and the frames are rendered by `dist.stream_frames_sharded` in batches, sharded over the
ranks, with the host download overlapping the next batch.  Video encoding (imageio / ffmpeg) is not part of this package; the
result is the uint8 frame grid `layout_grid` (gen_videos.py:24-38) would hand to the writer.
"""

import ctypes as C
import math

import numpy as np
import torch

from . import _lib as L

INTRINSICS = [4.2647, 0, 0.5, 0, 4.2647, 0.5, 0, 0, 1]           # gen_videos.py:85


def interp_video_inputs(G, seeds, shuffle_seed=None, w_frames=60 * 4, kind='cubic', grid_dims=(1, 1), num_keyframes=None, wraps=2,
                        psi=1, truncation_cutoff=14, cfg='FFHQ', device=None):
    """-> ws [F * grid_h * grid_w, num_ws, w_dim] (float64, as scipy returns them), c [F * grid_h * grid_w, 25] float32, and
    (F, grid_h, grid_w); row index = (frame * grid_h + yi) * grid_w + xi, the order of gen_videos.py:112-129."""
    import scipy.interpolate
    from .training.volumetric_rendering import LookAtPoseSampler
    grid_w, grid_h = grid_dims
    if num_keyframes is None:
        if len(seeds) % (grid_w * grid_h) != 0:
            raise ValueError('Number of input seeds must be divisible by grid W*H')
        num_keyframes = len(seeds) // (grid_w * grid_h)
    all_seeds = np.zeros(num_keyframes * grid_h * grid_w, dtype=np.int64)
    for idx in range(num_keyframes * grid_h * grid_w):
        all_seeds[idx] = seeds[idx % len(seeds)]
    if shuffle_seed is not None:
        np.random.RandomState(seed=shuffle_seed).shuffle(all_seeds)
    device = device if device is not None else next(G.parameters()).device
    lookat = torch.tensor([0, 0, 0.2] if cfg == 'FFHQ' else [0, 0, 0], dtype=torch.float32, device=device)
    intrinsics = torch.tensor(INTRINSICS, dtype=torch.float32, device=device).reshape(1, 9)

    # keyframe latents (:80-88)
    zs = torch.from_numpy(np.stack([np.random.RandomState(seed).randn(G.z_dim) for seed in all_seeds])).to(device)
    pose0 = LookAtPoseSampler.sample(math.pi / 2, math.pi / 2, lookat, radius=2.7, device=device)
    c0 = torch.cat([pose0.reshape(-1, 16), intrinsics], 1).repeat(len(zs), 1)
    ws = G.mapping(z=zs, c=c0, truncation_psi=psi, truncation_cutoff=truncation_cutoff)
    ws = ws.reshape(grid_h, grid_w, num_keyframes, *ws.shape[1:])

    # all frames of every cell's spline at once (:93-101, :127-128)
    F = num_keyframes * w_frames
    t = np.arange(F) / w_frames
    x = np.arange(-num_keyframes * wraps, num_keyframes * (wraps + 1))
    w_all = np.empty((F, grid_h, grid_w) + tuple(ws.shape[3:]), dtype=np.float64)
    for yi in range(grid_h):
        for xi in range(grid_w):
            y = np.tile(ws[yi][xi].cpu().numpy(), [wraps * 2 + 1, 1, 1])
            w_all[:, yi, xi] = scipy.interpolate.interp1d(x, y, kind=kind, axis=0)(t)

    # camera sweep (:118-124): the pose depends on the frame only, every cell of a frame shares it
    fi = np.arange(F)
    yaw = math.pi / 2 - 0.5 * np.sin(2 * math.pi * fi / F)
    pitch = math.pi / 2 - 0.05 + 0.25 * np.cos(2 * math.pi * fi / F)
    h = torch.from_numpy(yaw).to(torch.float32).reshape(F, 1).to(device)
    v = torch.from_numpy(pitch).to(torch.float32).reshape(F, 1).to(device)
    poses = LookAtPoseSampler.sample(h, v, lookat, radius=2.7, batch_size=F, device=device)
    c = torch.cat([poses.reshape(F, 16), intrinsics.expand(F, 9)], 1)
    c = c.reshape(F, 1, 1, 25).expand(F, grid_h, grid_w, 25)
    return (torch.from_numpy(w_all).reshape(F * grid_h * grid_w, *ws.shape[3:]), c.reshape(F * grid_h * grid_w, 25).contiguous(),
            (F, grid_h, grid_w))


def layout_frames(frames, F, grid_h, grid_w):
    """uint8 [F*grid_h*grid_w, C, H, W] (row order of interp_video_inputs) -> [F, grid_h*H, grid_w*W, C]: layout_grid
    (gen_videos.py:24-38) applied to every frame."""
    n, ch, ih, iw = frames.shape
    assert n == F * grid_h * grid_w
    g = frames.reshape(F, grid_h, grid_w, ch, ih, iw).permute(0, 1, 4, 2, 5, 3)
    return g.reshape(F, grid_h * ih, grid_w * iw, ch)


FRAME_WIDTH = {'image': 1, 'image_seg': 2, 'image_depth': 1}      # cell width in image widths, per image_mode (gen_videos.py:130-135)
_FRAME_MODES = {'image_seg': L.FRAMES_IMAGE_SEG, 'image_depth': L.FRAMES_IMAGE_DEPTH}


def compose_frames(img, seg_raw, image_mode):
    """The uint8 cells gen_interp_video writes in the image_seg / image_depth modes (gen_videos.py:129-139, then layout_grid's
    conversion :29-30), in one fused pass (ide3d_video_frames).  img [N, 3, H, W] float32, any strides; seg_raw [N, C, h, w] float32,
    any strides -- the render-resolution logits of G.synthesis(..., return_seg='raw'), upsampled inside the kernel by the rule of
    training.triplane.upsample_seg -- for image_seg, ignored for image_depth.  Returns uint8 [N, 3, H, k*W] (k = FRAME_WIDTH[image_mode]).
    image_depth normalises every frame by its own min / max, as the reference's batch-1 calls do.  CUDA tensors only."""
    if image_mode not in _FRAME_MODES:
        raise ValueError(f"compose_frames: image_mode must be one of {sorted(_FRAME_MODES)}, got {image_mode!r} ('image' frames are "
                         f"the plain uint8 conversion of the image)")
    seg = seg_raw if image_mode == 'image_seg' else None
    L.require_cuda(img, seg)
    L.forbid_grad('video.compose_frames', img, seg)
    for name, t in (('img', img), ('seg_raw', seg)):
        if t is not None and (t.dtype != torch.float32 or t.ndim != 4):
            raise RuntimeError(f'ide3d_b200.video.compose_frames: {name} must be float32 [N, C, H, W], got {t.dtype} {tuple(t.shape)}')
    n, ch, h, w = img.shape
    if ch != 3:
        raise RuntimeError(f'ide3d_b200.video.compose_frames: img must have 3 channels, got {ch}')
    out = torch.empty([n, 3, h, FRAME_WIDTH[image_mode] * w], dtype=torch.uint8, device=img.device)
    p = L.FramesParams()
    p.image, p.n, p.height, p.width = img.data_ptr(), n, h, w
    p.image_stride_n, p.image_stride_c, p.image_stride_h, p.image_stride_w = img.stride()
    p.mode, p.out = _FRAME_MODES[image_mode], out.data_ptr()
    if seg is not None:
        if seg.shape[0] != n:
            raise RuntimeError(f'ide3d_b200.video.compose_frames: {n} images but {seg.shape[0]} logit maps')
        from .dnnlib.seg_tools import _lut_for
        p.seg, (p.seg_c, p.seg_h, p.seg_w) = seg.data_ptr(), seg.shape[1:]
        p.seg_stride_n, p.seg_stride_c, p.seg_stride_h, p.seg_stride_w = seg.stride()
        p.lut = _lut_for(seg.device, seg.shape[1]).data_ptr()
    else:
        scratch = torch.empty([max(n, 1) * L.FRAMES_PARTIALS * 2], dtype=torch.float32, device=img.device)
        p.scratch = scratch.data_ptr()
    L.check(L.get_lib().ide3d_video_frames(C.byref(p), L.stream_ptr(img.device)))
    return out


@torch.no_grad()
def render_interp_video(G, seeds, rank=0, world=1, batch=8, out=None, synthesis_kwargs=None, image_mode='image', **kwargs):
    """All frames of gen_interp_video as uint8 grids [F, grid_h*H, grid_w*k*W, 3] on the host of rank 0 (None on the other ranks);
    image_mode as in gen_videos.py:184 -- 'image' (k = 1), 'image_seg' (the image with its colourised semantic mask on the right,
    k = 2) or 'image_depth' (the negated image, min/max-normalised per cell, k = 1).  kwargs: the arguments of `interp_video_inputs`;
    synthesis_kwargs: extra arguments of G.synthesis (default noise_mode='const' like gen_videos.py:129; the depth jitter is drawn per
    batch as in the reference).  F * grid cells must be a multiple of world * batch (pad the seed list or pick the batch accordingly)."""
    from . import dist as idist
    ws, c, (F, gh, gw) = interp_video_inputs(G, seeds, **kwargs)
    pin = torch.cuda.is_available()
    ws32 = ws.to(torch.float32)
    c32 = c.cpu()
    if pin:
        ws32, c32 = ws32.pin_memory(), c32.pin_memory()
    skw = dict(noise_mode='const')
    skw.update(synthesis_kwargs or {})
    frames = idist.stream_frames_sharded(G, ws32, c32, rank, world, batch=batch, out=out, image_mode=image_mode, **skw)
    return None if frames is None else layout_frames(frames, F, gh, gw)
