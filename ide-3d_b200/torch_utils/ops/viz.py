"""The display tail of viz/renderer.py:362-406 on sm_90a: statistics, uint8 image and FFT panel of one [C, H, W] map.

    display(out, render_type, sel_channels, base_channel, img_normalize, img_scale_db, fft_show, fft_all, fft_range_db, fft_beta, cmap)
        -> (image uint8 [H, W, S] or [H, 2W, 3] with the FFT panel, stats float32 [6])

The image comes from ide3d_viz_image (two launches) and the panel from ide3d_viz_fft (float64, fft.cuh's radix-2 transform), both
writing into one canvas, so the panel needs no torch.cat.  float32 and float16 maps are read as they are (float16 widened exactly, as
.to(torch.float32) does); any other dtype is converted to float32 once on the host.

The panel is taken of the map before the depth normalisation.  That normalisation is affine, and the panel is invariant to affine maps
of its input (the mean is removed per channel and the power divided by its mean), so this is the reference's panel up to rounding.
Maps the FFT kernel refuses (not square, a side that is not a power of two in [4, 1024]) run the reference's torch arithmetic instead.
"""

import torch

from ... import _lib as L

_windows = {}


def _window(n, beta, device):
    """torch.kaiser_window(n, periodic=False, beta) as the reference builds it (float32), widened to float64 on the device."""
    key = (n, float(beta), str(device))
    w = _windows.get(key)
    if w is None:
        w = _windows[key] = torch.kaiser_window(n, periodic=False, beta=beta).to(device=device, dtype=torch.float64)
    return w


def _map(x):
    L.require_cuda(x)
    if x.ndim != 3:
        raise RuntimeError(f'ide3d_b200.viz: the map must be [C, H, W], got {tuple(x.shape)}')
    return x if x.dtype in (torch.float32, torch.float16) else x.to(torch.float32)


def window_channels(C, sel_channels, base_channel):
    """viz/renderer.py:369-371: (sel_channels, base_channel) for a map of C channels."""
    sel = 1 if sel_channels > C else int(sel_channels)
    if sel < 1:
        raise ValueError(f'ide3d_b200.viz: sel_channels must be >= 1, got {sel_channels}')
    return sel, max(min(int(base_channel), C - sel), 0)


def fft_torch(sig, beta, range_db, lut, out):
    """The reference's FFT panel in torch (viz/renderer.py:397-405) for maps the kernel refuses, into out [H, W, 3]; a NaN dB value
    (a constant map) gets index 0, as in the kernel."""
    sig = sig.to(torch.float32)
    sig = sig - sig.mean(dim=[1, 2], keepdim=True)
    sig = sig * torch.kaiser_window(sig.shape[1], periodic=False, beta=beta, device=sig.device)[None, :, None]
    sig = sig * torch.kaiser_window(sig.shape[2], periodic=False, beta=beta, device=sig.device)[None, None, :]
    p = torch.fft.fftn(sig, dim=[1, 2]).abs().square().sum(dim=0)
    p = p.roll(shifts=[p.shape[0] // 2, p.shape[1] // 2], dims=[0, 1])
    db = (p / p.mean()).log10() * 10
    hi = lut.shape[0] - 1
    x = torch.nan_to_num((db / range_db + 1) / 2, nan=float('-inf'))
    idx = (x * hi + 0.5).clamp(0, hi).to(torch.int64)
    out.copy_(torch.nn.functional.embedding(idx, lut))
    return out


def fft_panel(sig, beta, range_db, lut, out):
    """Write the FFT panel of sig [C, H, W] into out [H, W, 3] uint8 (any byte strides).  lut uint8 [K, 3] on sig's device."""
    sig = _map(sig)
    L.require_cuda(lut, out)
    if lut.dtype != torch.uint8 or lut.ndim != 2 or lut.shape[1] != 3 or lut.shape[0] < 1:
        raise RuntimeError(f'ide3d_b200.viz: the colormap must be uint8 [K, 3], got {lut.dtype} {tuple(lut.shape)}')
    lut = lut.contiguous()
    C, H, W = sig.shape
    lib = L.get_lib()
    need = lib.ide3d_viz_fft_scratch_bytes(C, H, W)
    if need == L.UNSUPPORTED:
        return fft_torch(sig, beta, range_db, lut, out)
    if need < 0:
        L.check(need)
    scratch = torch.empty(int(need), dtype=torch.uint8, device=sig.device)
    s = sig.stride()
    L.check(lib.ide3d_viz_fft(sig.data_ptr(), L.dtype_code(sig), C, H, W, s[0], s[1], s[2], _window(H, beta, sig.device).data_ptr(),
                              float(range_db), lut.data_ptr(), lut.shape[0], out.data_ptr(), out.stride(0), out.stride(1), out.stride(2),
                              scratch.data_ptr(), int(need), L.stream_ptr(sig.device)))
    return out


@torch.no_grad()
def display(out, render_type='image', sel_channels=3, base_channel=0, img_normalize=False, img_scale_db=0, fft_show=False, fft_all=True,
            fft_range_db=50, fft_beta=8, cmap=None):
    """viz/renderer.py:369-406 for the map out [C, H, W] (the frame's render type, or a captured layer): -> (image, stats) on out's
    device.  image uint8 [H, W, S] with S the selected channel count, or [H, 2W, 3] with the FFT panel on the right (S must then be 1
    or 3, as expand_as requires); stats float32 [6].  cmap uint8 [K, 3] on the device, needed for fft_show."""
    out = _map(out)
    C, H, W = out.shape
    sel, base = window_channels(C, sel_channels, base_channel)
    if fft_show:
        if sel not in (1, 3):
            raise RuntimeError(f'ide3d_b200.viz: the FFT view shows the image as 3 channels; {sel} selected channels cannot be expanded')
        if cmap is None:
            raise RuntimeError('ide3d_b200.viz: the FFT view needs a colormap')
        canvas = torch.empty([H, 2 * W, 3], dtype=torch.uint8, device=out.device)
        oc = 3
    else:
        canvas = torch.empty([H, W, sel], dtype=torch.uint8, device=out.device)
        oc = sel
    stats = torch.empty(6, dtype=torch.float32, device=out.device)
    lib = L.get_lib()
    need = lib.ide3d_viz_image_scratch_bytes(C, H, W)
    if need < 0:
        L.check(need)
    scratch = torch.empty(max(int(need), 16), dtype=torch.uint8, device=out.device)
    s = out.stride()
    L.check(lib.ide3d_viz_image(out.data_ptr(), L.dtype_code(out), C, H, W, s[0], s[1], s[2], base, sel, int(render_type == 'image_depth'),
                                int(bool(img_normalize)), float(10 ** (img_scale_db / 20)), canvas.data_ptr(), oc, canvas.stride(0),
                                canvas.stride(1), canvas.stride(2), stats.data_ptr(), scratch.data_ptr(), scratch.numel(),
                                L.stream_ptr(out.device)))
    if fft_show:
        fft_panel(out if fft_all else out[base:base + sel], fft_beta, fft_range_db, cmap, canvas[:, W:])
    return canvas, stats
