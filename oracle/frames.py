"""Oracle (test infrastructure): the video frame composition of gen_videos.py's image_seg / image_depth modes, restated with
stock torch ops on whatever device the inputs live on.

    gen_videos.py:129-139   G.synthesis(..., return_seg=True); image_depth: img = -img, (img - min) / (max - min) * 2 - 1 per call
                            (batch 1, so per cell); image_seg: (mask2color(seg) / 255 - 0.5) / 0.5 concatenated on the right
    gen_videos.py:24-38     layout_grid: (img * 127.5 + 128).clamp(0, 255).to(torch.uint8)
    dnnlib/seg_tools.py:75-82  mask2color: argmax over the classes, zero image, one masked assignment per COLOR_MAP entry

The 512^2 logits come from the same bilinear rule G.synthesis(return_seg=True) applies (training/triplane.upsample_seg).  On CUDA
tensors this is the composition the fused kernel (ide3d_video_frames) is compared with; `cpu_frame_ops` routes the product's
video.compose_frames here so the batched driver runs on the CPU next to oracle.backend.cpu_reference_ops.
"""

import contextlib

import torch


def mask2color(masks, color_map):
    """dnnlib/seg_tools.py:75-82 on masks.device: float32 [N, 3, H, W], values 0..255."""
    idx = torch.argmax(masks, dim=1).float()
    out = torch.zeros((idx.shape[0], idx.shape[1], idx.shape[2], 3), dtype=torch.float, device=masks.device)
    for key, col in color_map.items():
        out[idx == key] = torch.tensor(col, dtype=torch.float, device=masks.device)
    return out.permute(0, 3, 1, 2)


def to_uint8(x):
    """layout_grid's float_to_uint8 step (gen_videos.py:29-30)."""
    return (x * 127.5 + 128).clamp(0, 255).to(torch.uint8)


def compose_frames(img, seg_raw, image_mode):
    """uint8 [N, 3, H, k*W] cells, each as the reference's batch-1 frame loop builds it.  img [N, 3, H, W]; seg_raw [N, C, h, w]
    render-resolution logits (image_seg only)."""
    from ide3d_b200.dnnlib.seg_tools import COLOR_MAP
    if image_mode == 'image_depth':
        cells = []
        for i in range(img.shape[0]):
            x = -img[i:i + 1]
            cells.append((x - x.min()) / (x.max() - x.min()) * 2 - 1)
        return to_uint8(torch.cat(cells))
    if image_mode == 'image_seg':
        seg = torch.nn.functional.interpolate(seg_raw, size=tuple(img.shape[-2:]), mode='bilinear', align_corners=False)
        col = (mask2color(seg, COLOR_MAP) / 255. - 0.5) / 0.5
        return to_uint8(torch.cat((img, col), -1))
    raise ValueError(f'oracle.frames.compose_frames: no composition for image_mode {image_mode!r}')


@contextlib.contextmanager
def cpu_frame_ops():
    """Inside the context ide3d_b200.video.compose_frames (and so dist.stream_frames_sharded's image_seg / image_depth modes) is
    the composition above.  Combine with oracle.backend.cpu_reference_ops for a CPU run of the driver."""
    from ide3d_b200 import video
    saved = video.compose_frames
    video.compose_frames = compose_frames
    try:
        yield
    finally:
        video.compose_frames = saved
