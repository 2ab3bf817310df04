"""Float64 numpy restatement of avg_spectra.py `calc` and `stats`, for the tests.

spectrum_pruned follows the kernel's decomposition (ide3d_spectrum_accum): with k = interp * m + r, each zero-padded length-P DFT of a
length-N row is interp twiddled length-N FFTs; rows first, keeping the half plane k2 <= P / 2, then columns; mean_c |Z|^2 is added
image by image and the half plane is mirrored at the end.  spectrum_direct is the plain np.fft.fft2 of the zero-padded plane, a second,
independent check.  Both take the whitening table and window of torch_utils/ops/spectra.py (whitening_lut, kaiser_window).
"""

import numpy as np
import torch

from .metrics import StandInMetricGenerator


class StandInSpectrumGenerator(StandInMetricGenerator):
    """The metrics' stand-in generator (512^2, c_dim 25) with the img_resolution attribute avg_spectra reads."""

    def __init__(self):
        super().__init__()
        self.img_resolution = self.g.img_resolution


def kaiser_window(image_size, beta):
    """The reference's window vector (float32 arithmetic), as float64."""
    w = torch.kaiser_window(image_size, periodic=False, beta=beta)
    w *= w.square().sum().rsqrt()
    return w.double().numpy()


def whitening_lut(mean, std):
    return (np.arange(256, dtype=np.float64) - mean) / std


def _whiten(images, lut, w):
    """uint8 [B, C, N, N] -> float64 lut[x] * (w[n1] w[n2])."""
    return lut[np.asarray(images)] * (w[:, None] * w[None, :])


def spectrum_pruned_sum(images, lut, w, interp, acc=None):
    """Half-plane sum [P / 2 + 1, P] (k2-major, as the kernel keeps it) of mean_c |X|^2 over the images, added in order to `acc`."""
    x = _whiten(images, lut, w)
    B, C, N, _ = x.shape
    P, H = N * interp, N * interp // 2 + 1
    n = np.arange(N)
    acc = np.zeros([H, P]) if acc is None else acc
    for b in range(B):
        pw = np.zeros([H, P])
        for c in range(C):
            Y = np.empty([N, H], dtype=np.complex128)                     # rows: Y[n1, k2], k2 <= P / 2
            for r in range(interp):
                t = np.fft.fft(x[b, c] * np.exp(-2j * np.pi * n * r / P)[None, :], axis=1)
                k2 = np.arange(N) * interp + r
                keep = k2 < H
                Y[:, k2[keep]] = t[:, keep]
            Z = np.empty([P, H], dtype=np.complex128)                     # columns: Z[k1, k2]
            for r in range(interp):
                Z[r::interp] = np.fft.fft(Y * np.exp(-2j * np.pi * n * r / P)[:, None], axis=0)
            pw += (Z.real ** 2 + Z.imag ** 2).T
        acc += pw / C
    return acc


def mirror(half, count):
    """[P / 2 + 1, P] half-plane sum -> [P, P] average in the reference's bin order."""
    H, P = half.shape
    out = np.empty([P, P])
    out[:, :H] = half.T
    k1 = (P - np.arange(P)) % P
    out[:, H:] = half[P - np.arange(H, P)][:, k1].T
    return out / count


def spectrum_pruned(images, lut, w, interp):
    return mirror(spectrum_pruned_sum(images, lut, w, interp), len(images))


def spectrum_direct(images, lut, w, interp):
    x = _whiten(images, lut, w)
    B, C, N, _ = x.shape
    P = N * interp
    acc = np.zeros([P, P])
    for b in range(B):
        X = np.fft.fft2(np.pad(x[b], [(0, 0), (0, P - N), (0, P - N)]), axes=(1, 2))
        acc += (np.abs(X) ** 2).mean(0)
    return acc / B


def moments(images):
    """Exact (count, sum x, sum x^2) as Python ints."""
    a = np.asarray(images, dtype=np.int64)
    return a.size, int(a.sum()), int((a * a).sum())
