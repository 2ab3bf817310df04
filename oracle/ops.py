"""Oracle (test infrastructure): CPU restatement of the StyleGAN custom ops on the hot path.

Follows (relative to the reference's torch_utils/ops):
  bias_act.py:91-120 (_bias_act_ref) and bias_act.cu:23-147 (gradient forms, clamp rule)
  upfirdn2d.py:70-115 (setup_filter), :167-211 (_upfirdn2d_ref), upfirdn2d.cpp:35-36 (output size)
  filtered_lrelu.py:121-153 (_filtered_lrelu_ref), filtered_lrelu.cpp:82-96 + filtered_lrelu.cu:494-505
  (2-bit sign tensor), conv2d_resample.py:46-141.
torch-CPU only; never imported by the product package.
"""

import math

import numpy as np
import torch
import torch.nn.functional as F

# name -> (function of (x, alpha), default alpha, default gain, plugin index)   bias_act.py:21-31
ACTIVATIONS = {
    'linear':   (lambda x, a: x,                          0.0, 1.0,          1),
    'relu':     (lambda x, a: F.relu(x),                  0.0, math.sqrt(2), 2),
    'lrelu':    (lambda x, a: F.leaky_relu(x, a),         0.2, math.sqrt(2), 3),
    'tanh':     (lambda x, a: torch.tanh(x),              0.0, 1.0,          4),
    'sigmoid':  (lambda x, a: torch.sigmoid(x),           0.0, 1.0,          5),
    'elu':      (lambda x, a: F.elu(x),                   0.0, 1.0,          6),
    'selu':     (lambda x, a: F.selu(x),                  0.0, 1.0,          7),
    'softplus': (lambda x, a: F.softplus(x),              0.0, 1.0,          8),
    'swish':    (lambda x, a: torch.sigmoid(x) * x,       0.0, math.sqrt(2), 9),
}


def bias_act(x, b=None, dim=1, act='linear', alpha=None, gain=None, clamp=None):
    """y = clamp(gain * act(x + b)); bias_act.py:91-120."""
    fn, def_alpha, def_gain, _ = ACTIVATIONS[act]
    alpha = float(def_alpha if alpha is None else alpha)
    gain = float(def_gain if gain is None else gain)
    if b is not None:
        assert b.ndim == 1 and b.shape[0] == x.shape[dim]
        x = x + b.reshape([-1 if i == dim else 1 for i in range(x.ndim)])
    y = fn(x, alpha)
    if gain != 1:
        y = y * gain
    if clamp is not None and clamp >= 0:
        y = y.clamp(-clamp, clamp)
    return y


def bias_act_grad(dy, x, b=None, dim=1, act='linear', alpha=None, gain=None, clamp=None, order=1, ddx=None):
    """First/second-order forms the plugin exposes as grad=1,2 (bias_act.cu:23-147):
    order 1: dx = dy * d/dx[forward];  order 2: d/dx of <ddx, dx> (dy held fixed).
    Computed with autograd on the forward restatement (double precision to avoid kinks' noise)."""
    xd = x.double().detach().requires_grad_(True)
    bd = None if b is None else b.double()
    y = bias_act(xd, bd, dim, act, alpha, gain, clamp)
    (dx,) = torch.autograd.grad(y, xd, dy.double(), create_graph=(order == 2))
    if order == 1:
        return dx.to(x.dtype)
    (d2,) = torch.autograd.grad(dx, xd, ddx.double(), allow_unused=True)
    d2 = torch.zeros_like(xd) if d2 is None else d2
    return d2.to(x.dtype)


# ----------------------------------------------------------------------------- upfirdn2d

def setup_filter(f, normalize=True, flip_filter=False, gain=1, separable=None):
    """upfirdn2d.py:70-115."""
    if f is None:
        f = 1
    f = torch.as_tensor(f, dtype=torch.float32)
    if f.ndim == 0:
        f = f[None]
    if separable is None:
        separable = (f.ndim == 1 and f.numel() >= 8)
    if f.ndim == 1 and not separable:
        f = torch.outer(f, f)
    if normalize:
        f = f / f.sum()
    if flip_filter:
        f = f.flip(list(range(f.ndim)))
    return f * (gain ** (f.ndim / 2))


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


def _pad4(p):
    if isinstance(p, int):
        p = [p, p]
    p = list(p)
    if len(p) == 2:
        p = [p[0], p[0], p[1], p[1]]
    return p


def upfirdn2d(x, f, up=1, down=1, padding=0, flip_filter=False, gain=1):
    """Zero-insert upsample -> pad/crop -> FIR -> decimate; upfirdn2d.py:167-211.  A 1-D ``f`` is a
    separable filter applied along x then y with sqrt(gain) each (:203-207)."""
    if f is None:
        f = torch.ones([1, 1], dtype=torch.float32)
    n, c, h, w = x.shape
    ux, uy = _pair(up)
    dx, dy = _pair(down)
    px0, px1, py0, py1 = _pad4(padding)
    z = x.reshape(n, c, h, 1, w, 1)
    z = F.pad(z, [0, ux - 1, 0, 0, 0, uy - 1])
    z = z.reshape(n, c, h * uy, w * ux)
    z = F.pad(z, [max(px0, 0), max(px1, 0), max(py0, 0), max(py1, 0)])
    z = z[:, :, max(-py0, 0): z.shape[2] - max(-py1, 0), max(-px0, 0): z.shape[3] - max(-px1, 0)]
    f = f * (gain ** (f.ndim / 2))
    f = f.to(x.dtype)
    if not flip_filter:
        f = f.flip(list(range(f.ndim)))
    if f.ndim == 2:
        z = F.conv2d(z, f[None, None].repeat(c, 1, 1, 1), groups=c)
    else:
        z = F.conv2d(z, f[None, None, None, :].repeat(c, 1, 1, 1), groups=c)
        z = F.conv2d(z, f[None, None, :, None].repeat(c, 1, 1, 1), groups=c)
    return z[:, :, ::dy, ::dx]


def upfirdn2d_direct(x, f2d, up, down, pad, flip, gain):
    """Closed form of SURVEY Appendix A.7 evaluated tap by tap in float64 (tiny inputs only) -- an
    independent second statement used to cross-check the conv-based one above.
    y[oy,ox] = gain * sum F[ky,kx] * X[(oy*dy+ky-py0)/uy, (ox*dx+kx-px0)/ux] over valid integer taps."""
    n, c, h, w = x.shape
    (ux, uy), (dx, dy) = up, down
    px0, px1, py0, py1 = pad
    fh, fw = f2d.shape
    ow = (w * ux + px0 + px1 - fw + dx) // dx
    oh = (h * uy + py0 + py1 - fh + dy) // dy
    X = x.double().numpy()
    Fk = f2d.double().numpy()
    if not flip:
        Fk = Fk[::-1, ::-1]
    y = np.zeros((n, c, oh, ow))
    for oy in range(oh):
        for ox in range(ow):
            acc = 0
            for ky in range(fh):
                ny = oy * dy + ky - py0
                if ny < 0 or ny % uy or ny // uy >= h:
                    continue
                for kx in range(fw):
                    nx = ox * dx + kx - px0
                    if nx < 0 or nx % ux or nx // ux >= w:
                        continue
                    acc = acc + Fk[ky, kx] * X[:, :, ny // uy, nx // ux]
            y[:, :, oy, ox] = acc
    return torch.from_numpy(y * gain).to(x.dtype)


def upsample2d(x, f, up=2, padding=0, flip_filter=False, gain=1):
    """upfirdn2d.py:313-348."""
    ux, uy = _pair(up)
    px0, px1, py0, py1 = _pad4(padding)
    fw, fh = f.shape[-1], f.shape[0]
    p = [px0 + (fw + ux - 1) // 2, px1 + (fw - ux) // 2, py0 + (fh + uy - 1) // 2, py1 + (fh - uy) // 2]
    return upfirdn2d(x, f, up=up, padding=p, flip_filter=flip_filter, gain=gain * ux * uy)


def downsample2d(x, f, down=2, padding=0, flip_filter=False, gain=1):
    """upfirdn2d.py:352-387."""
    dx, dy = _pair(down)
    px0, px1, py0, py1 = _pad4(padding)
    fw, fh = f.shape[-1], f.shape[0]
    p = [px0 + (fw - dx + 1) // 2, px1 + (fw - dx) // 2, py0 + (fh - dy + 1) // 2, py1 + (fh - dy) // 2]
    return upfirdn2d(x, f, down=down, padding=p, flip_filter=flip_filter, gain=gain)


def filter2d(x, f, padding=0, flip_filter=False, gain=1):
    """upfirdn2d.py:277-309."""
    px0, px1, py0, py1 = _pad4(padding)
    fw, fh = f.shape[-1], f.shape[0]
    p = [px0 + fw // 2, px1 + (fw - 1) // 2, py0 + fh // 2, py1 + (fh - 1) // 2]
    return upfirdn2d(x, f, padding=p, flip_filter=flip_filter, gain=gain)


# ----------------------------------------------------------------------------- filtered_lrelu

def filtered_lrelu(x, fu=None, fd=None, b=None, up=1, down=1, padding=0, gain=math.sqrt(2), slope=0.2,
                   clamp=None, flip_filter=False, return_signs=False):
    """filtered_lrelu.py:121-153.  With return_signs also returns the packed 2-bit sign tensor the
    plugin writes (filtered_lrelu.cpp:82-96): code 1 = value was negative, code 2 = value was clamped (clamp wins),
    4 elements per byte in x order, width padded to a multiple of 16 elements."""
    px0, px1, py0, py1 = _pad4(padding)
    t = bias_act(x, b)
    t = upfirdn2d(t, fu, up=up, padding=[px0, px1, py0, py1], gain=up ** 2, flip_filter=flip_filter)
    pre = t * gain
    t = bias_act(t, act='lrelu', alpha=slope, gain=gain, clamp=clamp)
    y = upfirdn2d(t, fd, down=down, flip_filter=flip_filter)
    if not return_signs:
        return y
    neg = (pre < 0)
    act = torch.where(neg, pre * slope, pre)
    clamped = (act.abs() > clamp) if clamp is not None else torch.zeros_like(neg)
    # filtered_lrelu.cu:1135-1145: s = 1 for a negative value, overwritten by s = 2 when the value clamps
    code = torch.where(clamped, torch.full_like(neg, 2, dtype=torch.uint8), neg.to(torch.uint8))
    n, c, sh, sw = code.shape
    swp = (sw + 15) // 16 * 16
    code = F.pad(code, [0, swp - sw])
    code = code.reshape(n, c, sh, swp // 4, 4)
    packed = code[..., 0] | (code[..., 1] << 2) | (code[..., 2] << 4) | (code[..., 3] << 6)
    return y, packed


# ----------------------------------------------------------------------------- conv2d_resample

def conv2d_resample(x, w, f=None, up=1, down=1, padding=0, groups=1, flip_weight=True, flip_filter=False):
    """conv2d_resample.py:46-141 restated the slow, obviously-correct way: upsample with the FIR
    (gain up^2), convolve, downsample with the FIR.  Mathematically identical to the reference's
    transposed-conv fast paths (:112-126)."""
    px0, px1, py0, py1 = _pad4(padding)
    fw = 1 if f is None else f.shape[-1]
    fh = 1 if f is None else f.shape[0]
    kw, kh = w.shape[-1], w.shape[-2]
    if up > 1:
        px0 += (fw + up - 1) // 2
        px1 += (fw - up) // 2
        py0 += (fh + up - 1) // 2
        py1 += (fh - up) // 2
    if down > 1:
        px0 += (fw - down + 1) // 2
        px1 += (fw - down) // 2
        py0 += (fh - down + 1) // 2
        py1 += (fh - down) // 2
    t = upfirdn2d(x, (f if up > 1 else None), up=up, padding=[px0, px1, py0, py1], gain=up ** 2,
                  flip_filter=flip_filter)
    wk = w if flip_weight else w.flip([2, 3])
    t = F.conv2d(t, wk.to(t.dtype), groups=groups)
    if down > 1:
        t = upfirdn2d(t, f, down=down, flip_filter=flip_filter)
    return t


def mask2color(masks, color_map):
    """dnnlib/seg_tools.py:75-82: argmax over dim 1, colour per class (classes without an entry stay 0)."""
    idx = torch.argmax(masks, dim=1).float()
    out = torch.zeros((idx.shape[0], idx.shape[1], idx.shape[2], 3), dtype=torch.float)
    for key, col in color_map.items():
        out[idx == key] = torch.tensor(col, dtype=torch.float)
    return out.permute(0, 3, 1, 2)
