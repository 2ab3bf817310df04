"""Oracle (test infrastructure): seeded BiSeNet weights and the CPU route of ide3d_b200.finetune, with autograd.

    bisenet_state(net, seed)        every tensor of a BiSeNet state_dict (reference or product: same names) drawn from a numpy
                                    RandomState in state_dict order: convolutions ~ N(0, 2 / fan_in), BatchNorm weight / bias and
                                    running mean / var seeded too, so the eval-mode BatchNorm is not the identity
    seg_stem(mask, stem, conv1, skip)   ide3d_seg_stem and ide3d_seg_stem_bwd's formulation: per-class tables in float64 with autograd,
                                    gathered per pixel (taps outside the image contribute nothing), rounded to fp32 at the end
    seg_labels(seg_raw, size, align_corners=False)          argmax of F.interpolate(bilinear)
    seg_cross_entropy(seg_raw, mask, align_corners=False)   F.cross_entropy of F.interpolate(bilinear)
    cpu_finetune_ops()              inside the context, the product's ops run on the CPU (oracle.backend.cpu_reference_ops) and the
                                    kernels of torch_utils/ops/seg_stem.py and projection.seg_cross_entropy are the restatements above
    reference_step(...)             one fine-tuning step in the reference's own structure (for the GPU tests and the benchmark)

tests/golden/make_finetune_golden.py runs the reference's finetune() with these weights, oracle.edit's encoder weights and stand-in
generator; tests/test_finetune.py replays it through ide3d_b200.finetune.
"""

import contextlib
import math

import numpy as np
import torch
import torch.nn.functional as F

from . import backend

BISENET_SEED = 51


def bisenet_state(net, seed=BISENET_SEED):
    rs = np.random.RandomState(seed)
    out = {}
    for name, v in net.state_dict().items():
        shape = tuple(v.shape)
        if name.endswith('num_batches_tracked'):
            out[name] = v.clone()
            continue
        if v.ndim == 4:
            a = rs.randn(*shape) * math.sqrt(2.0 / (shape[1] * shape[2] * shape[3]))
        elif name.endswith('running_var'):
            a = 0.5 + rs.rand(*shape)
        elif name.endswith('weight'):
            a = 1.0 + 0.1 * rs.randn(*shape)
        else:                                                   # BatchNorm bias and running_mean
            a = 0.1 * rs.randn(*shape)
        out[name] = torch.from_numpy(a.astype(np.float32))
    return out


def seg_stem(mask, stem, conv1, skip):
    classes = stem.weight.shape[1]
    c0, c1 = stem.weight.shape[0], skip.weight.shape[0]
    w0 = stem.weight.double().reshape(c0, classes)
    t = stem.weight_gain * (2 * w0.t() - w0.sum(1)) + stem.bias.double()                          # [classes, C0]
    t = torch.cat([t, (-stem.weight_gain * w0.sum(1) + stem.bias.double())[None], torch.zeros(1, c0, dtype=torch.float64)])
    l1 = conv1.weight_gain * torch.einsum('oiyx,ki->yxko', conv1.weight.double(), t).reshape(9, classes + 2, c0)
    s = skip.weight_gain * t @ skip.weight.double().reshape(c1, c0).t()                             # [classes + 2, C1]
    f = skip.resample_filter.detach().flip([0, 1]).double()
    n, h, w = mask.shape
    ids = torch.where(mask.long() < classes, mask.long(), torch.full_like(mask, classes, dtype=torch.long))
    ids = F.pad(ids, (1, 1, 1, 1), value=classes + 1)
    y1 = sum(l1[k][ids[:, k // 3:k // 3 + h, k % 3:k % 3 + w]] for k in range(9)) + conv1.bias.double()
    y1 = torch.where(y1 > 0, y1, y1 * 0.2) * math.sqrt(2)
    sk = sum(f[a // 4, a % 4] * s[ids[:, a // 4:a // 4 + h:2, a % 4:a % 4 + w:2]] for a in range(16))
    return y1.float().permute(0, 3, 1, 2), sk.float().permute(0, 3, 1, 2)


def seg_labels(seg_raw, size, align_corners=False):
    return F.interpolate(seg_raw, size=tuple(size), mode='bilinear', align_corners=align_corners).argmax(1).to(torch.uint8)


def seg_cross_entropy(seg_raw, mask, align_corners=False):
    up = F.interpolate(seg_raw, size=tuple(mask.shape[-2:]), mode='bilinear', align_corners=align_corners)
    return F.cross_entropy(up, mask.long())


@contextlib.contextmanager
def cpu_finetune_ops():
    from ide3d_b200.torch_utils.ops import projection as P, seg_stem as S
    saved = (S.seg_stem, S.seg_labels, P.seg_cross_entropy)
    S.seg_stem, S.seg_labels, P.seg_cross_entropy = seg_stem, seg_labels, seg_cross_entropy
    try:
        with backend.cpu_reference_ops():
            yield
    finally:
        S.seg_stem, S.seg_labels, P.seg_cross_entropy = saved


REMAP = torch.tensor([0, 1, 6, 7, 4, 5, 2, 2, 10, 11, 12, 8, 9, 15, 3, 17, 16, 18, 13, 14])        # dnnlib/seg_tools.py:59


def reference_step(G, E, image, target_seg, code, label, parser, w_avg, n_geo=8):
    """One step of finetune_hybrid_encoder.py:155-183 in the reference's structure, on any device: the full E twice (the float
    target_seg map, then the {0, 1} scatter of the render's remapped parse), BiSeNet three times (twice on the render, once on the
    image) with the upsampled logits and torch's cross-entropy.  Returns the four loss terms; the caller runs the backward."""
    rec = E(image, target_seg) + w_avg.repeat(image.shape[0], 1, 1)
    rec[:, n_geo:] = code[:, n_geo:].detach().clone()
    loss = {'loss_ws': F.smooth_l1_loss(rec, code) * 10.0}
    img = G.synthesis(rec, c=label, noise_mode='const')
    loss['loss_gen_l2'] = F.mse_loss(img, image)
    logits = parser(img)[0]
    labels = parser(image)[0].argmax(1)
    loss['loss_real_entropy'] = torch.nn.CrossEntropyLoss()(logits, labels)
    parse = REMAP.to(image.device)[parser(img)[0].argmax(1, keepdim=True)]
    seg = torch.zeros(image.shape[0], 19, *image.shape[-2:], device=image.device).scatter_(1, parse, 1)
    loss['loss_real_cycle'] = F.smooth_l1_loss(rec, E(image, seg))
    return loss
