"""Fine-tune the hybrid encoder to one portrait (apps/finetune_hybrid_encoder.py:69-213): the step between pivotal tuning and the
Painter, which aligns the encoder's geometry rows with the tuned generator's pivot.

    run(G, E, image, code, label, *, parser, mask=None, steps=1000, lr=1e-5, start_from_latent_avg=True)
        -> (E_tuned, mask uint8 [H, W], losses {name: np.ndarray [steps]})

The generator is frozen; Adam(lr, betas (0.9, 0.99)) trains E.convs_seg and E.projector_seg for exactly `steps` updates.  Each step,
with the reference's weights and order:
    rec    = E(image, target_seg) + w_avg, rows n_latents_geo.. replaced by the pivot's
    loss_ws            10 * smooth_l1(rec, code)
    loss_gen_l2        mse(G.synthesis(rec, label, noise_mode='const'), image)
    loss_real_entropy  cross-entropy of BiSeNet's logits on the render, upsampled with align_corners=True, against the argmax of
                       BiSeNet on the image (no remap)
    loss_real_cycle    smooth_l1(rec, E(image, scatter(remap(argmax BiSeNet(render))))): the {0, 1} one-hot and no w_avg, as the
                       reference's parsing_img and second E call give it
target_seg is `mask` (uint8 ids, read as one_hot * 2 - 1) or, without one, the remapped parse of the image.  The returned mask is
the remapped parse of rec rendered with {'fov': 18, 'num_steps': 96} after the last step (the reference's mask.png).

What differs from the reference:
    - the shape rows come from E.geometry alone: the image branch of the first E call is never run, because the reference
      overwrites its rows with the pivot's; the split is E.n_latents_geo where the reference uses the literal 8 (the two agree for
      the released HybridEncoder(512, 10, 8));
    - the cycle's appearance rows E.appearance(image) are computed once, without grad: their weights are never stepped and the
      image does not change;
    - BiSeNet runs once per step on the render: the same logits feed the cross-entropy (ide3d_seg_xent_*_ac, without the
      upsampled logits) and the cycle's parse (ide3d_seg_labels_ac, then the remap), where the reference runs it twice; it runs
      once in total on the image, for the cross-entropy's labels and, without `mask`, target_seg;
    - both masks enter the encoder as uint8 ids through the one-byte stem kernel and its backward (encoder.HybridEncoder):
      target_seg as one_hot * 2 - 1, the cycle's parse as the {0, 1} one-hot;
    - masks are parsed at the image's size; the reference's face_parsing resizes to 512^2 first, a no-op at the released 512^2.
The caller's G and E are not modified: E_tuned is a copy, returned in eval mode without grad.
"""

import copy

import numpy as np
import torch
import torch.nn.functional as F

from . import edit as _edit
from .parsing import parse, remap_ids
from .torch_utils.ops import projection
from .torch_utils.ops import seg_stem as _seg_ops
from .training.triplane import invalidate_caches

RENDER_PARAMS = {'fov': 18, 'num_steps': 96}                                        # finetune_hybrid_encoder.py:205-208
LAMBDAS = {'loss_ws': 10.0, 'loss_gen_l2': 1.0, 'loss_real_entropy': 1.0, 'loss_real_cycle': 1.0}     # :144-147


def _one(what, t):
    if t.shape[0] != 1:
        raise ValueError(f'finetune: {what} must be a single portrait, got {t.shape[0]}')
    return t


def run(G, E, image, code, label, *, parser, mask=None, steps=1000, lr=1e-5, start_from_latent_avg=True):
    """image [3, H, W] or [1, 3, H, W] in [-1, 1] at the encoder's size; code: the pivot [1, num_ws, w_dim] (--target_code, e.g. from
    pti.run); label [1, 25]; parser: a parsing.BiSeNet (20 classes); mask: uint8 [H, W] class ids (--target_seg) or None."""
    _edit._check_pair(G, E)
    image = _one('image', _edit._check_image(E, image))
    dev = image.device
    code = _one('code', _edit._check_ws(G, code)).to(dev, torch.float32)
    label = _edit._check_label(label, 1).to(dev, torch.float32)
    if mask is not None:
        mask = _one('mask', _edit._check_masks(E, mask))
    steps = int(steps)
    if steps < 0:
        raise ValueError(f'finetune: steps must be >= 0, got {steps}')
    size = tuple(image.shape[-2:])
    G = copy.deepcopy(G).eval().requires_grad_(False)
    E = copy.deepcopy(E).eval().requires_grad_(False)
    params = list(E.convs_seg.parameters()) + list(E.projector_seg.parameters())
    for p in params:
        p.requires_grad_(True)
    opt = torch.optim.Adam(params, lr=lr, betas=(0.9, 0.99))
    w_avg = _edit._w_avg(G)
    n_geo = E.n_latents_geo

    with torch.no_grad():
        target_labels = _seg_ops.seg_labels(parser.logits(image), size, align_corners=True)
        target_seg = remap_ids(target_labels) if mask is None else mask
        app = E.appearance(image)
        app = app[0] if isinstance(app, tuple) else app

    history = []
    for _ in range(steps):
        opt.zero_grad()
        geo = E.geometry(target_seg)
        if start_from_latent_avg:
            geo = geo + w_avg
        rec = torch.cat((geo, code[:, n_geo:]), 1)
        img = G.synthesis(rec, c=label, noise_mode='const')
        logits = parser.logits(img)
        with torch.no_grad():
            cycle_seg = remap_ids(_seg_ops.seg_labels(logits, size, align_corners=True))
        cycle = torch.cat((E.geometry(cycle_seg, signed=False), app), 1)
        loss = {'loss_ws': F.smooth_l1_loss(rec, code) * LAMBDAS['loss_ws'],
                'loss_gen_l2': F.mse_loss(img, image) * LAMBDAS['loss_gen_l2'],
                'loss_real_entropy': projection.seg_cross_entropy(logits, target_labels, align_corners=True) * LAMBDAS['loss_real_entropy'],
                'loss_real_cycle': F.smooth_l1_loss(rec, cycle) * LAMBDAS['loss_real_cycle']}
        sum(loss.values()).backward()
        opt.step()
        history.append(torch.stack([v.detach() for v in loss.values()]))

    E.requires_grad_(False)
    with torch.no_grad():
        rec = torch.cat((E.geometry(target_seg) + w_avg, code[:, n_geo:]), 1)            # :201-203 adds w_avg unconditionally
        render = G.synthesis(rec, c=label, render_params=dict(RENDER_PARAMS), noise_mode='const')
        out_mask = parse(parser, render)[0]
    invalidate_caches(E)
    values = torch.stack(history).cpu().numpy() if history else np.zeros((0, len(LAMBDAS)), np.float32)
    return E, out_mask, {name: values[:, i] for i, name in enumerate(LAMBDAS)}
