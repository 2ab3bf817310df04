"""Edit portraits by semantic mask: the hybrid encoder's drivers.

    encode        apps/infer_hybrid_encoder.py:79-90    ws = E(image, mask) + w_avg; pivot= splices the pivot's appearance rows
    edit          Painter/run_UI.py:170-203 (run_deep_model with inversion=True), for K masks in one call: the masks' geometry rows
                  + w_avg followed by the pivot's appearance rows, then one synthesis
    reenact       apps/infer_face_animation.py:144-148 (and run_deep_model without inversion): B latents driven by F (mask, camera)
                  frames
    render_mask   the generator's own semantic render as a uint8 class-id mask at image resolution (ide3d_seg_labels): the starting
                  mask of an edit, where the reference parses the render with BiSeNet (apps/finetune_hybrid_encoder.py:209-213)

Masks are uint8 class ids [H, W] or [N, H, W] at the encoder's size; they take the encoder's one-byte stem (encoder.HybridEncoder).
Classes are COLOR_MAP's 19 (dnnlib/seg_tools.py): the generator's semantic logits, the encoder's input channels and render_mask's ids
are assumed to share that order, as the released generator and encoder do (both trained on the same 19-class CelebAMask-HQ parse).

What differs from the reference:
    - edit skips the pivot render (run_UI.py:193) and the image branch of E(gen_img, seg): the reference overwrites their result with
      the pivot's rows (:197-198), so an edit is the geometry branch plus one synthesis;
    - reenact renders the condition images of all frames with one backbone pass per latent (G.synthesis(..., views=F)) and encodes
      each mask once, not once per latent (the reference encodes target_seg.repeat(batch)).
"""

import torch

from .torch_utils.ops import seg_stem as _seg_ops

FRONTAL = [1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 2.7, 0, 0, 0, 1, 4.2647, 0, 0.5, 0, 4.2647, 0.5, 0, 0, 1]    # infer_face_animation.py:116
REENACT_RENDER_PARAMS = {'fov': 16, 'num_steps': 96}                                                  # infer_face_animation.py:139-142


def _device(m):
    return next(m.parameters()).device


def _check_pair(G, E):
    if E.n_latents_geo + E.n_latents_app != G.num_ws or E.w_dim != G.w_dim:
        raise ValueError(f'edit: the encoder writes {E.n_latents_geo} + {E.n_latents_app} rows of {E.w_dim}, the generator reads '
                         f'{G.num_ws} rows of {G.w_dim}')


def _check_masks(E, masks):
    masks = torch.as_tensor(masks)
    if masks.ndim == 2:
        masks = masks[None]
    if masks.dtype != torch.uint8 or masks.ndim != 3 or tuple(masks.shape[1:]) != (E.size, E.size) or masks.shape[0] < 1:
        raise ValueError(f'edit: masks must be uint8 [{E.size}, {E.size}] or [N, {E.size}, {E.size}] class ids, got {masks.dtype} '
                         f'{tuple(masks.shape)}')
    return masks.to(_device(E))


def _check_image(E, image):
    image = torch.as_tensor(image)
    if image.ndim == 3:
        image = image[None]
    if image.ndim != 4 or tuple(image.shape[1:]) != (3, E.size, E.size) or not image.is_floating_point():
        raise ValueError(f'edit: image must be float [3, {E.size}, {E.size}] or [N, 3, {E.size}, {E.size}] in [-1, 1], got '
                         f'{image.dtype} {tuple(image.shape)}')
    if image.numel() and (image.min() < -1 or image.max() > 1):
        raise ValueError(f'edit: image values must lie in [-1, 1], got [{image.min().item():.3g}, {image.max().item():.3g}]')
    return image.to(_device(E), torch.float32)


def _check_label(label, rows=None):
    label = torch.as_tensor(label)
    if label.ndim != 2 or label.shape[1] != 25 or (rows is not None and label.shape[0] not in (1, rows)):
        want = '[N, 25]' if rows is None else f'[1, 25] or [{rows}, 25]'
        raise ValueError(f'edit: label must be {want}, got {tuple(label.shape)}')
    return label


def _check_ws(G, ws):
    ws = torch.as_tensor(ws)
    if ws.ndim != 3 or tuple(ws.shape[1:]) != (G.num_ws, G.w_dim):
        raise ValueError(f'edit: ws must be [N, {G.num_ws}, {G.w_dim}], got {tuple(ws.shape)}')
    return ws


def _w_avg(G):
    return G.mapping.w_avg[None, None, :]


@torch.no_grad()
def encode(E, G, image, mask, *, pivot=None):
    """infer_hybrid_encoder.py:79-90 with start_from_latent_avg: ws = E(image, mask) + w_avg, [N, num_ws, w_dim].  pivot ([1 or N,
    num_ws, w_dim], --target_code): ws[:, n_latents_geo:] = pivot[:, n_latents_geo:] (the reference splices at the literal 8, which is
    n_latents_geo of the released HybridEncoder(512, 10, 8))."""
    _check_pair(G, E)
    image, mask = _check_image(E, image), _check_masks(E, mask)
    if image.shape[0] != mask.shape[0]:
        raise ValueError(f'edit: {image.shape[0]} images and {mask.shape[0]} masks')
    rec = E(image, mask)
    if isinstance(rec, tuple):
        rec = rec[0]
    ws = rec + _w_avg(G).repeat(*rec.shape[:2], 1)
    if pivot is not None:
        pivot = _check_ws(G, pivot).to(ws)
        if pivot.shape[0] not in (1, ws.shape[0]):
            raise ValueError(f'edit: pivot must have 1 or {ws.shape[0]} rows, got {pivot.shape[0]}')
        n = E.n_latents_geo
        ws = torch.cat((ws[:, :n], pivot[:, n:].expand(ws.shape[0], -1, -1)), 1)
    return ws


@torch.no_grad()
def edit(G, E, ws, label, masks):
    """Painter/run_UI.py:170-203 with inversion=True, for K masks in one call.  ws: the pivot [1, num_ws, w_dim] (projection / PTI);
    label [1, 25] or [K, 25]; masks uint8 [H, W] or [K, H, W].  -> (ws_edit [K, num_ws, w_dim], img [K, 3, res, res]) with
    ws_edit = cat(E.geometry(masks) + w_avg, ws[:, n_latents_geo:]) and img = G.synthesis(ws_edit, label, noise_mode='const').
    The split is E.n_latents_geo where the reference uses the literal 8: the two agree for the released HybridEncoder(512, 10, 8)
    (train_hybrid_encoder.py:208).  The pivot render and the image branch of E(gen_img, seg) are not run: the reference overwrites
    their rows with the pivot's."""
    _check_pair(G, E)
    masks = _check_masks(E, masks)
    k = masks.shape[0]
    ws = _check_ws(G, ws)
    if ws.shape[0] != 1:
        raise ValueError(f'edit: ws must be one pivot [1, {G.num_ws}, {G.w_dim}], got {tuple(ws.shape)}')
    label = _check_label(label, k).to(_device(G), torch.float32).expand(k, -1)
    geo = E.geometry(masks)
    geo = geo + _w_avg(G).repeat(k, geo.shape[1], 1)
    ws_edit = torch.cat((geo, ws.to(geo)[:, E.n_latents_geo:].expand(k, -1, -1)), 1)
    img = G.synthesis(ws_edit, c=label, noise_mode='const')
    return ws_edit, img


@torch.no_grad()
def reenact(G, E, ws, labels, masks, *, render_params=None, frames_per_call=8):
    """infer_face_animation.py:144-148 for B latents (ws [B, num_ws, w_dim]) and F frames (labels [F, 25], masks uint8 [F, H, W]):
    per frame, the latents' condition images from the frame's camera, their appearance rows, the frame mask's geometry rows, + w_avg,
    and the render from the frame's camera.  -> images [F, B, 3, res, res].
    render_params: those of both syntheses (default REENACT_RENDER_PARAMS, the reference's fov 16 and 96 steps).  The condition images
    of up to frames_per_call frames come from one G.synthesis(..., views=frames) call (one backbone pass per latent); each mask is
    encoded once for all latents."""
    _check_pair(G, E)
    masks = _check_masks(E, masks)
    f_total = masks.shape[0]
    labels = _check_label(labels, f_total)
    if labels.shape[0] != f_total:
        raise ValueError(f'edit: {f_total} masks and {labels.shape[0]} labels')
    ws = _check_ws(G, ws).to(_device(G), torch.float32)
    labels = labels.to(_device(G), torch.float32)
    rp = dict(REENACT_RENDER_PARAMS if render_params is None else render_params)
    b = ws.shape[0]
    n_geo = E.n_latents_geo
    out = []
    for f0 in range(0, f_total, int(frames_per_call)):
        fr = min(int(frames_per_call), f_total - f0)
        c = labels[f0:f0 + fr].repeat(b, 1)                                   # latent-major: row i * fr + j is frame j of latent i
        cond = G.synthesis(ws, c, noise_mode='const', render_params=rp, views=fr)
        app = E.appearance(cond)
        if isinstance(app, tuple):
            app = app[0]
        geo = E.geometry(masks[f0:f0 + fr])                                   # [fr, n_geo, w_dim], once per mask
        rec = torch.cat((geo.repeat(b, 1, 1), app), 1) + _w_avg(G)
        img = G.synthesis(rec, c, noise_mode='const', render_params=rp)
        out.append(img.reshape(b, fr, *img.shape[1:]).transpose(0, 1))
    return torch.cat(out)


@torch.no_grad()
def render_mask(G, ws, label, **synthesis_kwargs):
    """The generator's semantic render as class ids: uint8 [N, res, res] from G.synthesis(ws, label, return_seg='raw')'s render-resolution
    logits, upsampled and argmaxed per pixel by the rule of the frame and strip kernels (so a pixel's id is the class they colour); the
    upsampled logits are never built.  The ids index COLOR_MAP's classes (see the module docstring)."""
    ws = _check_ws(G, ws)
    label = _check_label(label, ws.shape[0]).to(_device(G), torch.float32).expand(ws.shape[0], -1)
    synthesis_kwargs.setdefault('noise_mode', 'const')
    _, seg_raw = G.synthesis(ws.to(_device(G), torch.float32), label, return_seg='raw', **synthesis_kwargs)
    return _seg_ops.seg_labels(seg_raw, (G.img_resolution, G.img_resolution))
