"""Oracle (test infrastructure): seeded hybrid-encoder weights, the stand-in generator of the editing traces, the table formulation of
ide3d_seg_stem restated with torch on the CPU, and the CPU route of ide3d_b200.edit.

    encoder_state(E, seed)      every parameter of a HybridEncoder (reference or product: same names and shapes) drawn from a numpy
                                RandomState in state_dict order; buffers (the resample filters) keep their constructed values
    standin_generator()         oracle.projector's stand-in generator with num_ws = 10 (the released encoder's 8 geometry rows + 2),
                                512^2 images and a seeded mapping.w_avg
    seg_stem(mask, stem, conv1, skip)   ide3d_seg_stem's formulation for any C0: per-class tables in float64 rounded to fp32, then the
                                per-pixel sums (taps outside the image contribute nothing)
    seg_labels(seg_raw, size)   argmax of the bilinear upsampling (align_corners=False)
    cpu_edit_ops()              inside the context, the product's ops run on the CPU (oracle.backend.cpu_reference_ops) and the two
                                kernels of torch_utils/ops/seg_stem.py are the restatements above

tests/golden/make_edit_golden.py runs the reference's HybridEncoder, Painter step, infer_hybrid_encoder.test and face animation with
these; tests/test_edit.py replays them through ide3d_b200.encoder and ide3d_b200.edit.
"""

import contextlib
import math

import numpy as np
import torch
import torch.nn.functional as F

from . import backend
from . import projector as oproj

ENCODER_ARGS = dict(size=512, n_latents_app=2, n_latents_geo=8, w_dim=16)
ENCODER_SEED = 31
W_AVG_SEED = 32


def encoder_state(E, seed=ENCODER_SEED):
    """{name: tensor} for E.load_state_dict: weights ~ N(0, 1) (the reference's init), biases ~ 0.2 N(0, 1) so they count."""
    rs = np.random.RandomState(seed)
    params = dict(E.named_parameters())
    out = {}
    for name, v in E.state_dict().items():
        if name in params:
            scale = 0.2 if name.endswith('bias') else 1.0
            out[name] = torch.from_numpy((rs.randn(*v.shape) * scale).astype(np.float32))
        else:
            out[name] = v.detach().clone()
    return out


def standin_generator():
    G = oproj.StandInGenerator(z_dim=16, w_dim=ENCODER_ARGS['w_dim'], num_ws=10, img_resolution=512, render_size=16, seed=5)
    rs = np.random.RandomState(W_AVG_SEED)
    G.mapping.register_buffer('w_avg', torch.from_numpy((rs.randn(G.w_dim) * 0.3).astype(np.float32)))
    return G.eval()


def stem_tables(stem, conv1, skip, classes):
    """(L1 [9, classes + 2, C0], S [classes + 2, C1], f~ [4, 4]) as ide3d_seg_stem builds them: row `classes` is "no class", row
    `classes` + 1 (zeros) stands for taps outside the image."""
    w0 = stem.weight.detach().double().reshape(stem.weight.shape[0], classes)
    t = stem.weight_gain * (2 * w0.t() - w0.sum(1)) + stem.bias.detach().double()                # [classes, C0]
    t = torch.cat([t, (-stem.weight_gain * w0.sum(1) + stem.bias.detach().double())[None]])       # + no class
    w1 = conv1.weight.detach().double()                                                            # [C0, C0, 3, 3]
    l1 = conv1.weight_gain * torch.einsum('oiyx,ki->yxko', w1, t).reshape(9, t.shape[0], -1)
    s = skip.weight_gain * t @ skip.weight.detach().double().reshape(skip.weight.shape[0], -1).t()
    zero = lambda a: torch.cat([a, torch.zeros_like(a.narrow(-2, 0, 1))], -2)
    return zero(l1).float(), zero(s).float(), skip.resample_filter.detach().flip([0, 1]).float()


def seg_stem(mask, stem, conv1, skip):
    classes = stem.weight.shape[1]
    l1, s, f = stem_tables(stem, conv1, skip, classes)
    n, h, w = mask.shape
    ids = torch.where(mask.long() < classes, mask.long(), torch.full_like(mask, classes, dtype=torch.long))
    ids = F.pad(ids, (1, 1, 1, 1), value=classes + 1)                                              # [N, H + 2, W + 2]
    y1 = torch.zeros(n, h, w, l1.shape[2])
    for t in range(9):
        y1 += l1[t][ids[:, t // 3:t // 3 + h, t % 3:t % 3 + w]]
    y1 = y1 + conv1.bias.detach().float()
    y1 = torch.where(y1 > 0, y1, y1 * 0.2) * math.sqrt(2)
    sk = torch.zeros(n, h // 2, w // 2, s.shape[1])
    for a in range(16):
        ay, ax = a // 4, a % 4
        sk += f[ay, ax] * s[ids[:, ay:ay + h:2, ax:ax + w:2]]
    return y1.permute(0, 3, 1, 2), sk.permute(0, 3, 1, 2)


def seg_labels(seg_raw, size):
    return F.interpolate(seg_raw, size=tuple(size), mode='bilinear', align_corners=False).argmax(1).to(torch.uint8)


@contextlib.contextmanager
def cpu_edit_ops():
    from ide3d_b200.torch_utils.ops import seg_stem as S
    saved = (S.seg_stem, S.seg_labels)
    S.seg_stem, S.seg_labels = seg_stem, seg_labels
    try:
        with backend.cpu_reference_ops():
            yield
    finally:
        S.seg_stem, S.seg_labels = saved


# ------------------------------------------------------------------------------------------------ inputs of the golden trace
def golden_masks():
    """uint8 [3, 512, 512]: (0) 32^2 blocks of random classes 0..18 with one block in five an id >= 19 (19, 23, 200, 255);
    (1) a face-like layout whose hair, cloth and neck runs touch every border; (2) the same layout edited: a larger mouth and the
    hair cut (what a Painter stroke does).  Masks 1 and 2 stay within 0..18: the Painter's id_remap indexes a 19-entry table."""
    rs = np.random.RandomState(41)
    blocks = rs.randint(0, 19, size=(16, 16))
    odd = rs.rand(16, 16) < 0.2
    blocks[odd] = rs.choice([19, 23, 200, 255], size=int(odd.sum()))
    m0 = np.kron(blocks, np.ones((32, 32), np.int64))
    yy, xx = np.mgrid[0:512, 0:512]
    m1 = np.zeros((512, 512), np.int64)
    m1[:, :40] = 13
    m1[:40, :] = 13
    m1[470:, :] = 18
    m1[:, 490:] = 16
    face = (yy - 256) ** 2 / 180 ** 2 + (xx - 256) ** 2 / 140 ** 2 < 1
    m1[face] = 1
    m1[(yy - 210) ** 2 + (xx - 200) ** 2 < 15 ** 2] = 4
    m1[(yy - 210) ** 2 + (xx - 312) ** 2 < 15 ** 2] = 5
    m1[(yy > 240) & (yy < 300) & (np.abs(xx - 256) < 18)] = 2
    m1[(yy > 330) & (yy < 350) & (np.abs(xx - 256) < 50)] = 11
    m1[(yy > 350) & (yy < 368) & (np.abs(xx - 256) < 50)] = 12
    m2 = m1.copy()
    m2[(yy > 320) & (yy < 380) & (np.abs(xx - 256) < 70)] = 10
    m2[:20, :] = 0
    return torch.from_numpy(np.stack([m0, m1, m2]).astype(np.uint8))


def golden_images(n, seed=42):
    """[n, 3, 512, 512] smooth images in [-1, 1]."""
    rs = np.random.RandomState(seed)
    small = torch.from_numpy(rs.rand(n, 3, 16, 16).astype(np.float32))
    return F.interpolate(small, size=(512, 512), mode='bilinear', align_corners=False) * 2 - 1


def to_uint8(images):
    """[N, 3, H, W] in [-1, 1] -> the uint8 PNG bytes the golden scripts' inputs are saved as."""
    return ((images + 1) * 127.5).round().clamp(0, 255).to(torch.uint8)
