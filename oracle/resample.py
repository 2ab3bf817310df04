"""numpy int64 restatement of Pillow's 8-bit resampler (libImaging/Resample.c, ImagingResample for L and RGB) with the Lanczos filter.

    lanczos_tables(in_size, out_size)   Pillow's precompute_coeffs + normalize_coeffs_8bpc: (ksize, bounds [out, 2], coeffs [out, ksize])
    resize(img, (width, height))        PIL.Image.fromarray(img).resize((width, height), LANCZOS) as uint8 [H, W] or [H, W, C]

The passes are Pillow's: horizontal first, over the source rows the vertical pass reads (ybox_first .. ybox_last), into a uint8
intermediate; then vertical.  A pass is skipped when its axis keeps its size; with both skipped the result is a copy.
"""

import math

import numpy as np

PRECISION_BITS = 22


def _lanczos(x):
    def sinc(v):
        if v == 0.0:
            return 1.0
        v = v * math.pi
        return math.sin(v) / v
    return sinc(x) * sinc(x / 3.0) if -3.0 <= x < 3.0 else 0.0


def lanczos_tables(in_size, out_size):
    scale = in_size / out_size
    filterscale = scale if scale >= 1.0 else 1.0
    support = 3.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros([out_size, 2], dtype=np.int64)
    coeffs = np.zeros([out_size, ksize], dtype=np.int64)
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        ss = 1.0 / filterscale
        xmin = int(center - support + 0.5)
        xmin = max(xmin, 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        k = np.zeros(xmax)
        ww = 0.0
        for x in range(xmax):
            k[x] = _lanczos((x + xmin - center + 0.5) * ss)
            ww += k[x]
        for x in range(xmax):
            if ww != 0.0:
                k[x] /= ww
            v = k[x] * (1 << PRECISION_BITS)
            coeffs[xx, x] = int(-0.5 + v) if k[x] < 0 else int(0.5 + v)
        bounds[xx] = xmin, xmax
    return ksize, bounds, coeffs


def _clip8(ss):
    return np.where(ss >= (1 << PRECISION_BITS << 8), 255, np.where(ss <= 0, 0, ss >> PRECISION_BITS)).astype(np.uint8)


def _pass(img, bounds, coeffs, axis):
    """One 8-bit pass along `axis` (1 = columns of each row, 0 = rows of each column) of img int64 [H, W, C]."""
    out = []
    for (first, count), k in zip(bounds, coeffs):
        taps = np.take(img, np.arange(first, first + count), axis=axis).astype(np.int64)
        shape = [1, 1, 1]
        shape[axis] = count
        ss = (1 << (PRECISION_BITS - 1)) + (taps * k[:count].reshape(shape)).sum(axis=axis)
        out.append(_clip8(ss))
    return np.stack(out, axis=axis)


def resize(img, size):
    img = np.asarray(img)
    if img.dtype != np.uint8 or img.ndim not in (2, 3):
        raise ValueError(f'8-bit L or RGB image expected, got {img.shape} {img.dtype}')
    width, height = size
    x = img[:, :, None] if img.ndim == 2 else img
    h, w = x.shape[:2]
    need_h, need_v = width != w, height != h
    _, bx, cx = lanczos_tables(w, width)
    _, by, cy = lanczos_tables(h, height)
    if need_h:
        first, last = by[0, 0], by[-1, 0] + by[-1, 1]
        x = _pass(x[first:last], bx, cx, axis=1)
        by = by - [first, 0]
    if need_v:
        x = _pass(x, by, cy, axis=0)
    x = np.array(x, dtype=np.uint8)
    return x[:, :, 0] if img.ndim == 2 else x
