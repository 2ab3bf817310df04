"""PIL.Image.resize(size, PIL.Image.LANCZOS) of 8-bit L and RGB images on sm_90a, bit for bit (ide3d_resample_u8).

    lanczos_tables(in_size, out_size)        -> (ksize, bounds int32 [out, 2], coeffs int32 [out, ksize]), Pillow's tables
    resample_u8(src, dst)                    dst uint8 [N, OH, OW, C] = each src uint8 [N, H, W, C] resized to OW x OH
    resize_u8(src, (width, height))          the same into a fresh tensor

The tables are Pillow's precompute_coeffs and normalize_coeffs_8bpc (libImaging/Resample.c) in Python floats, which are C doubles:
math.sin is the libm call Pillow makes, and every operation runs in Pillow's order, so the integer tables are Pillow's.  The kernel
runs Pillow's two integer passes on them.  src and dst may be views (a centre crop of a larger image, a window of a canvas): only the
channel dimension must be contiguous.
"""

import functools
import math

import numpy as np
import torch

from ... import _lib as L

PRECISION_BITS = 22
LANCZOS_SUPPORT = 3.0


def _sinc(x):
    if x == 0.0:
        return 1.0
    x = x * math.pi
    return math.sin(x) / x


def _lanczos(x):
    if -3.0 <= x < 3.0:
        return _sinc(x) * _sinc(x / 3.0)
    return 0.0


@functools.lru_cache(maxsize=64)
def lanczos_tables(in_size, out_size):
    """Pillow's precompute_coeffs(in_size, 0, in_size, out_size, lanczos) and normalize_coeffs_8bpc for one axis."""
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = LANCZOS_SUPPORT * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    ss = 1.0 / filterscale
    bounds = np.zeros([out_size, 2], dtype=np.int32)
    coeffs = np.zeros([out_size, ksize], dtype=np.int32)
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        k = [_lanczos((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for w in k:
            ww += w
        if ww != 0.0:
            k = [w / ww for w in k]
        coeffs[xx, :xmax] = [int(-0.5 + w * (1 << PRECISION_BITS)) if w < 0 else int(0.5 + w * (1 << PRECISION_BITS)) for w in k]
        bounds[xx] = xmin, xmax
    bounds.flags.writeable = coeffs.flags.writeable = False
    return ksize, bounds, coeffs


def _operand(t, what):
    L.require_cuda(t)
    if t.dtype != torch.uint8 or t.ndim != 4 or t.shape[3] not in (1, 3) or (t.shape[3] == 3 and t.stride(3) != 1):
        raise RuntimeError(f'ide3d_b200.resample: {what} must be uint8 [N, H, W, C] with C = 1 or 3 contiguous, got '
                           f'{tuple(t.shape)} {t.dtype} strides {t.stride()}')
    return t


def resample_u8(src, dst):
    """dst[i] = PIL.Image.fromarray(src[i]).resize((OW, OH), LANCZOS), bit for bit, for every image of the batch."""
    src, dst = _operand(src, 'src'), _operand(dst, 'dst')
    n, h, w, c = src.shape
    if dst.shape[0] != n or dst.shape[3] != c or dst.device != src.device:
        raise RuntimeError(f'ide3d_b200.resample: dst {tuple(dst.shape)} on {dst.device} does not match src {tuple(src.shape)} on '
                           f'{src.device}')
    oh, ow = dst.shape[1], dst.shape[2]
    if n == 0:
        return dst
    kx, bx, cx = lanczos_tables(w, ow)
    ky, by, cy = lanczos_tables(h, oh)
    lib = L.get_lib()
    need = lib.ide3d_resample_u8_scratch_bytes(n, c, h, oh, ow, kx, ky)
    L.check(need if need < 0 else L.OK)
    scratch = torch.empty(need, dtype=torch.uint8, device=src.device)
    ptr = lambda a: a.ctypes.data
    L.check(lib.ide3d_resample_u8(src.data_ptr(), n, c, h, w, src.stride(0), src.stride(1), src.stride(2), dst.data_ptr(), oh, ow,
                                  dst.stride(0), dst.stride(1), dst.stride(2), kx, ptr(bx), ptr(cx), ky, ptr(by), ptr(cy),
                                  scratch.data_ptr(), need, L.stream_ptr(src.device)))
    return dst


def resize_u8(src, size):
    """A fresh uint8 [N, height, width, C] tensor: resample_u8 of src to size = (width, height), PIL's order."""
    width, height = size
    dst = torch.empty([src.shape[0], height, width, src.shape[3]], dtype=torch.uint8, device=src.device)
    return resample_u8(src, dst)
