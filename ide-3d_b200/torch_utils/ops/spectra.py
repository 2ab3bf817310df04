"""Average power spectrum and image moments of avg_spectra.py on sm_90a.

    Spectrum(image_size, channels, mean, std, beta, interp, device)   .add(images uint8 [B, C, N, N], NCHW or NHWC) ... .result()
    image_moments(images, moments)                                      moments uint64 [3] += (count, sum x, sum x^2)

Spectrum keeps a float64 half-plane accumulator on the device and adds batches with ide3d_spectrum_accum, a pruned float64 FFT of the
non-zero N x N block (no P x P plane, no cuFFT); result() divides by the image count and mirrors it into the reference's [P, P] order
(ide3d_spectrum_finalize).  Shapes the kernel does not cover (ide3d_spectrum_accum returns -1: N not a power of two in [16, 1024],
interp not 1/2/4/8, P > 4096, more than 4 channels) fall back to the reference's arithmetic: torch float64 fftn of the padded plane,
on the device.

The whitening is the reference's (x - mean) / std in float64, passed to the kernel as a 256-entry table.  The window is the reference's
torch.kaiser_window(N, periodic=False, beta) * rsqrt(sum w^2), built in float32 as the reference builds it; the reference then rounds
the 2-D outer product to float32 as well, where this module keeps w[n1] * w[n2] in float64 (a relative difference below 6e-8 per pixel).
"""

import numpy as np
import torch

from ... import _lib as L

# the per-call scratch (the row pass's half-plane spectra of every image in the call) is capped near this; batches are split to fit
SCRATCH_CAP_BYTES = 512 << 20


def kaiser_window(image_size, beta, device):
    """The reference's window vector (float32 arithmetic, avg_spectra.py:157-158), returned as float64.  Built on the CPU, so that every
    device gets the same bits."""
    w = torch.kaiser_window(image_size, periodic=False, beta=beta)
    w *= w.square().sum().rsqrt()
    return w.to(device=device, dtype=torch.float64)


def whitening_lut(mean, std, device):
    """lut[v] = (v - mean) / std in float64 for every uint8 value v: the reference's per-pixel arithmetic."""
    return (torch.arange(256, dtype=torch.float64, device=device) - mean) / std


def _images(x):
    L.require_cuda(x)
    if x.dtype != torch.uint8 or x.ndim != 4:
        raise RuntimeError(f'ide3d_b200.spectra: images must be a 4-D uint8 tensor [B, C, H, W], got {tuple(x.shape)} {x.dtype}')
    return x


class Spectrum:
    """Running average power spectrum of one image stream (the body of avg_spectra.py `calc`)."""

    def __init__(self, image_size, channels, mean, std, beta=8, interp=4, device='cuda'):
        self.device = torch.empty(0, device=device).device        # 'cuda' -> 'cuda:<current>'
        L.require_cuda(torch.empty(0, device=self.device))
        self.image_size, self.channels, self.interp = int(image_size), int(channels), int(interp)
        self.spectrum_size = self.image_size * self.interp
        self.mean, self.std = mean, std
        self.window = kaiser_window(self.image_size, beta, self.device)
        self.lut = whitening_lut(mean, std, self.device)
        self.count = 0
        lib = L.get_lib()
        per_image = lib.ide3d_spectrum_scratch_bytes(1, self.channels, self.image_size, self.interp)
        self.native = per_image != L.UNSUPPORTED
        if not self.native:
            P = self.spectrum_size
            self.acc = torch.zeros([P, P], dtype=torch.float64, device=self.device)
            self.window2d = self.window.ger(self.window)[None, None]
            return
        if per_image < 0:
            L.check(per_image)
        self.chunk = max(1, SCRATCH_CAP_BYTES // per_image)
        self.acc = torch.zeros([self.spectrum_size // 2 + 1, self.spectrum_size], dtype=torch.float64, device=self.device)
        self._scratch = None

    def _scratch_for(self, n):
        need = L.get_lib().ide3d_spectrum_scratch_bytes(n, self.channels, self.image_size, self.interp)
        if self._scratch is None or self._scratch.numel() < need:
            self._scratch = torch.empty(max(int(need), 16), dtype=torch.uint8, device=self.device)
        return self._scratch, need

    def add(self, images):
        """Add a batch of uint8 images [B, C, N, N] (any strides) in index order."""
        images = _images(images)
        B, C, H, W = images.shape
        if C != self.channels or H != self.image_size or W != self.image_size:
            raise RuntimeError(f'ide3d_b200.spectra: images {tuple(images.shape)} do not match [*, {self.channels}, {self.image_size}, '
                               f'{self.image_size}]')
        if images.device != self.device:
            raise RuntimeError(f'ide3d_b200.spectra: images on {images.device}, spectrum on {self.device}')
        if not self.native:
            self._add_torch(images)
        else:
            lib = L.get_lib()
            for i in range(0, B, self.chunk):
                x = images[i:i + self.chunk]
                scratch, need = self._scratch_for(x.shape[0])
                s = x.stride()
                L.check(lib.ide3d_spectrum_accum(x.data_ptr(), x.shape[0], C, H, s[0], s[1], s[2], s[3], self.lut.data_ptr(),
                                                 self.window.data_ptr(), self.interp, self.acc.data_ptr(), scratch.data_ptr(), need,
                                                 L.stream_ptr(self.device)))
        self.count += B

    def _add_torch(self, images):
        """The reference's arithmetic (avg_spectra.py:164-166), one image at a time."""
        padding = self.spectrum_size - self.image_size
        for image in images.split(1):
            image = (image.to(torch.float64) - self.mean) / self.std
            image = torch.nn.functional.pad(image * self.window2d, [0, padding, 0, padding])
            self.acc += torch.fft.fftn(image, dim=[2, 3]).abs().square().mean(dim=[0, 1])

    def result(self):
        """float64 [P, P]: the average over the images added so far, in the reference's bin order."""
        if self.count == 0:
            raise RuntimeError('ide3d_b200.spectra: no images were added')
        if not self.native:
            return self.acc / self.count
        P = self.spectrum_size
        out = torch.empty([P, P], dtype=torch.float64, device=self.device)
        L.check(L.get_lib().ide3d_spectrum_finalize(self.acc.data_ptr(), self.image_size, self.interp, self.count, out.data_ptr(),
                                                    L.stream_ptr(self.device)))
        return out


def image_moments(images, moments):
    """moments (uint64 [3] on the images' device, stored as int64) += (number of values, sum x, sum x^2), exactly."""
    images = _images(images)
    L.require_cuda(moments)
    if moments.dtype not in (torch.int64, torch.uint64) or moments.shape != (3,) or moments.device != images.device:
        raise RuntimeError('ide3d_b200.spectra: moments must be a [3] 64-bit integer tensor on the images\' device')
    B, C, H, W = images.shape
    s = images.stride()
    L.check(L.get_lib().ide3d_image_moments(images.data_ptr(), B, C, H, W, s[0], s[1], s[2], s[3], moments.data_ptr(),
                                            L.stream_ptr(images.device)))
    return moments


def mean_std(moments):
    """(mean, std) from exact (count, sum x, sum x^2), with the reference's formula (avg_spectra.py:131-135) in float64."""
    n, s1, s2 = (int(v) for v in np.asarray(moments, dtype=np.uint64))
    m1, m2 = s1 / n, s2 / n
    return m1, float(np.sqrt(np.float64(m2) - np.float64(m1) ** 2))
