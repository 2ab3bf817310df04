"""Semantic-mask helpers of the reference's dnnlib/seg_tools.py that sit right after the renderer (SURVEY.md §8f rank 4):
`COLOR_MAP` (:13-32) and `mask2color` (:75-82) -- argmax over the 19 semantic logits + colour look-up -- as ONE sm_90a pass
(ide3d_mask2color) instead of an argmax, a zero-fill and 19 masked assignments.  CUDA tensors only, like every op here."""

import ctypes as C

import torch

from .. import _lib as L

COLOR_MAP = {
    0: [0, 0, 0], 1: [204, 0, 0], 2: [76, 153, 0], 3: [204, 204, 0], 4: [51, 51, 255], 5: [204, 0, 204], 6: [0, 255, 255],
    7: [255, 204, 204], 8: [102, 51, 0], 9: [255, 0, 0], 10: [102, 204, 0], 11: [255, 255, 0], 12: [0, 0, 153], 13: [0, 0, 204],
    14: [255, 51, 153], 15: [0, 204, 204], 16: [0, 51, 0], 17: [255, 153, 51], 18: [0, 204, 0]}

_lut = {}


def _lut_for(device, num_classes):
    key = (str(device), num_classes)
    if key not in _lut:
        rows = [COLOR_MAP.get(k, [0, 0, 0]) for k in range(num_classes)]      # classes without a colour stay black (zeros, :77)
        _lut[key] = torch.tensor(rows, dtype=torch.float32, device=device).contiguous()
    return _lut[key]


def mask2color(masks, to_uint8=False):
    """masks [N, C, H, W] logits / one-hot -> colour image [N, 3, H, W], float32 values 0..255 (seg_tools.py:75-82).
    to_uint8 (extension): write uint8 directly (the conversion gen_videos.py:24-38 applies next)."""
    L.require_cuda(masks)
    m = masks if masks.dtype == torch.float32 else masks.float()
    n, c, h, w = m.shape
    out = torch.empty([n, 3, h, w], dtype=torch.uint8 if to_uint8 else torch.float32, device=m.device)
    s = m.stride()
    L.check(L.get_lib().ide3d_mask2color(L.ptr(m), n, c, h, w, s[0], s[1], s[2], s[3], L.ptr(_lut_for(m.device, c)), L.ptr(out),
                                         int(bool(to_uint8)), L.stream_ptr(m.device)))
    return out
