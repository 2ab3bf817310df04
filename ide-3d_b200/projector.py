"""Project a portrait into the generator: W / W+ projection, the mirrored view, camera refinement and a semantic-mask loss.

`project` is the first step of IDE-3D's editing workflow (README "Interactive editing", inversion/scripts/run_pti.py).  It follows
the reference's three projectors step for step -- inversion/training/projectors/w_projector_ide3d.py (W), w_plus_projector_ide3d.py
(W+) and w_projector_ide3d_join_view.py (the mirrored view) -- with the same schedules, random draws and order of operations:

    w statistics    z ~ RandomState(seed).randn(w_avg_samples, z_dim) mapped with c = label; w_avg, w_std of the first ws row
    noise           every noise_const buffer of the copied generator, randn_like in named_buffers order, renormalised after each step
    step            lr = initial_learning_rate * cosine ramp; w_noise = randn_like(w) * w_std * initial_noise_factor * ramp^2;
                    img -> (img + 1) * 255 / 2, 'area' down to 256; dist = sum((f_target - f_synth)^2);
                    loss = dist + regularize_noise_weight * noise_reg (+ seg_weight * seg_cross_entropy); Adam(betas 0.9, 0.999)

What differs from the reference loops:
    - the mirrored view is the second camera of ONE G.synthesis(..., views=2) call (one backbone pass instead of two);
    - the noise regulariser, its gradient and the renormalisation are two kernels over the whole buffer table
      (torch_utils.ops.projection; the reference runs a few hundred small torch kernels per step);
    - refine_camera (extension): a 6-vector (omega, t), zero at the start, gives cam2world' = [R(omega) | t] . cam2world (Rodrigues),
      optimised by its own Adam at camera_lr times the same ramp; the renderer's backward kernel supplies its gradient;
    - target_seg / seg_weight (extension, off by default): seg_weight * the cross-entropy of the render-resolution logits, upsampled
      to the mask inside the kernel, against a uint8 class map in dnnlib/seg_tools.py's 19-class order.

The swappable kernels are the module attributes of torch_utils.ops.projection (oracle/projector.py::cpu_projector_ops replaces them
with torch restatements to run the driver on the CPU).
"""

import copy
import os

import numpy as np
import torch
import torch.nn.functional as F

from .torch_utils.ops import projection

MIRROR_LABEL_INDICES = [1, 2, 3, 4, 8]           # w_projector_ide3d_join_view.py:72: the cam2world entries a left-right flip negates
NUM_CLASSES = 19                                  # dnnlib/seg_tools.py:35-55
# left/right class pairs of the 19-class map that a horizontal flip swaps: eyes, brows, ears
MIRROR_CLASSES = [0, 1, 2, 3, 5, 4, 7, 6, 9, 8, 10, 11, 12, 13, 14, 15, 16, 17, 18]
CAMERA_LR = 2e-3


def load_features(features, device):
    """The VGG16 feature network of the projectors: a path to its TorchScript file (the vgg16.pt the reference downloads), loaded
    with torch.jit.load, or any callable f(images [N,3,h,w] in 0..255, resize_images=False, return_lpips=True) -> [N, F]."""
    if isinstance(features, (str, os.PathLike)):
        if not os.path.isfile(features):
            raise FileNotFoundError(f'project: feature network {os.fspath(features)!r} not found (nothing is downloaded)')
        return torch.jit.load(os.fspath(features), map_location=device).eval()
    if not callable(features):
        raise TypeError(f'project: features must be a path or a callable, got {type(features).__name__}')
    return features


def mirror_label(label):
    """The label of the left-right mirrored camera, label[:, [1, 2, 3, 4, 8]] * -1 (differentiable in label)."""
    sign = torch.ones(label.shape[-1], dtype=label.dtype, device=label.device)
    sign[MIRROR_LABEL_INDICES] = -1
    return label * sign


def mirror_mask(mask):
    """The class map of the mirrored image: flipped along W, left/right pairs (4, 5), (6, 7), (8, 9) swapped."""
    lut = torch.tensor(MIRROR_CLASSES, dtype=mask.dtype, device=mask.device)
    return lut[torch.flip(mask, (-1,)).long()]


def rodrigues(omega):
    """Rotation matrix [3, 3] of the axis-angle vector omega [3]; exactly the identity for omega = 0, differentiable there."""
    th2 = (omega * omega).sum()
    small = th2 < 1e-6
    th = torch.where(small, torch.ones_like(th2), th2).sqrt()
    a = torch.where(small, 1 - th2 / 6, torch.sin(th) / th)                 # sin(th) / th
    b = torch.where(small, 0.5 - th2 / 24, (1 - torch.cos(th)) / (th * th))  # (1 - cos(th)) / th^2
    zero = torch.zeros_like(omega[0])
    k = torch.stack([zero, -omega[2], omega[1], omega[2], zero, -omega[0], -omega[1], omega[0], zero]).reshape(3, 3)
    return torch.eye(3, dtype=omega.dtype, device=omega.device) + a * k + b * (k @ k)


def refine_label(label, delta):
    """label [N, 25] with cam2world replaced by [R(delta[:3]) | delta[3:]] . cam2world.  A zero delta returns label bit for bit:
    the change D = ([R | t] - I) . cam2world is then exactly zero and is applied as `where(D == 0, M, M + D)`, with D's gradient
    passed straight through (x - (+0) keeps every bit of x, -0 included)."""
    m = label[:, :16].reshape(-1, 4, 4)
    top = torch.cat([rodrigues(delta[:3]) - torch.eye(3, dtype=delta.dtype, device=delta.device), delta[3:, None]], 1)
    d = torch.cat([top, torch.zeros_like(top[:1])], 0) @ m                    # [N, 4, 4]
    dd = d.detach()
    cam = torch.where(dd == 0, m, m + dd) - (dd - d)
    return torch.cat([cam.reshape(-1, 16), label[:, 16:]], 1)


def _check_mask(target_seg, res, device):
    mask = torch.as_tensor(target_seg)
    if mask.dtype != torch.uint8 or tuple(mask.shape) != (res, res):
        raise ValueError(f'project: target_seg must be a uint8 class map [{res}, {res}], got {mask.dtype} {tuple(mask.shape)}')
    if int(mask.max()) >= NUM_CLASSES:
        raise ValueError(f'project: target_seg has class {int(mask.max())}; the map has {NUM_CLASSES} classes (0..{NUM_CLASSES - 1})')
    return mask.to(device)


def _prepare(images):
    images = (images + 1) * (255 / 2)
    if images.shape[2] > 256:
        images = F.interpolate(images, size=(256, 256), mode='area')
    return images


def _target_images(target, device):
    images = target.unsqueeze(0).to(device).to(torch.float32)
    if images.shape[2] > 256:
        images = F.interpolate(images, size=(256, 256), mode='area')
    return images


def project(G, label, target, *, features, num_steps=1000, w_avg_samples=10000, initial_learning_rate=0.01, initial_noise_factor=0.05,
            lr_rampdown_length=0.25, lr_rampup_length=0.05, noise_ramp_length=0.75, regularize_noise_weight=1e5, initial_w=None,
            w_plus=False, mirror=False, refine_camera=False, camera_lr=CAMERA_LR, target_seg=None, seg_weight=0.0, seed=123,
            on_step=None):
    """Project `target` ([3, H, W], 0..255, H = W = G.img_resolution) rendered from camera `label` ([1, 25]) into G's latent space.

    -> (ws [1, num_ws, w_dim], label [1, 25]).  The W projector returns its single w repeated over G's num_ws rows (the reference
    hard-codes 18 rows, w_projector_ide3d.py:145); w_plus optimises and returns every row.  The label is the refined camera with
    refine_camera, else a copy of the input.  G is deep-copied and frozen; the caller's G is not modified.

    features: path to the VGG16 TorchScript file, or a callable with its contract (load_features).  initial_w: [1, 1 or num_ws,
    w_dim] start (numpy or tensor); w_avg otherwise.  mirror: also fit the target flipped along W from the mirrored camera.
    target_seg: uint8 [H, W] class map, used with seg_weight > 0.  The torch RNG draws (noise buffers, per-step w noise) come from the
    caller's seeded generator, as in the reference.  on_step(step, dist, loss): called after every optimiser step with 0-d tensors."""
    label = torch.as_tensor(label)
    res = G.img_resolution
    if tuple(target.shape) != (G.img_channels, res, res):
        raise ValueError(f'project: target must be [{G.img_channels}, {res}, {res}], got {tuple(target.shape)}')
    if label.ndim != 2 or tuple(label.shape) != (1, 25):
        raise ValueError(f'project: label must be [1, 25], got {tuple(label.shape)}')
    if seg_weight and target_seg is None:
        raise ValueError('project: seg_weight > 0 needs target_seg')
    device = next(G.parameters()).device
    label = label.to(device=device, dtype=torch.float32)
    use_seg = target_seg is not None and seg_weight > 0
    mask = _check_mask(target_seg, res, device) if target_seg is not None else None
    vgg16 = load_features(features, device)

    G = copy.deepcopy(G).eval().requires_grad_(False).to(device).float()
    num_ws = G.mapping.num_ws

    z_samples = np.random.RandomState(seed).randn(w_avg_samples, G.z_dim)
    w_samples = G.mapping(torch.from_numpy(z_samples).to(device), c=label.repeat(w_avg_samples, 1))
    w_samples = w_samples[:, :1, :].cpu().numpy().astype(np.float32)
    w_avg = np.mean(w_samples, axis=0, keepdims=True)
    w_std = (np.sum((w_samples - w_avg) ** 2) / w_avg_samples) ** 0.5

    start_w = w_avg if initial_w is None else (initial_w.detach().cpu().numpy() if torch.is_tensor(initial_w) else np.asarray(initial_w))
    if w_plus and start_w.shape[1] != num_ws:
        start_w = np.repeat(start_w, num_ws, axis=1)
    if not w_plus:
        start_w = start_w[:, :1]

    noise_bufs = [buf for name, buf in G.synthesis.named_buffers() if 'noise_const' in name]

    views = 2 if mirror else 1
    targets = [target]
    if mirror:
        targets.append(torch.flip(target, (2,)))
    target_features = [vgg16(_target_images(t, device), resize_images=False, return_lpips=True) for t in targets]
    if use_seg:
        mask_b = torch.stack([mask, mirror_mask(mask)]) if mirror else mask[None]

    w_opt = torch.tensor(start_w, dtype=torch.float32, device=device, requires_grad=True)
    optimizer = torch.optim.Adam([w_opt] + noise_bufs, betas=(0.9, 0.999), lr=initial_learning_rate)
    delta = cam_opt = None
    if refine_camera:
        delta = torch.zeros(6, dtype=torch.float32, device=device, requires_grad=True)
        cam_opt = torch.optim.Adam([delta], betas=(0.9, 0.999), lr=camera_lr)

    for buf in noise_bufs:
        buf[:] = torch.randn_like(buf)
        buf.requires_grad = True

    for step in range(num_steps):
        t = step / num_steps
        w_noise_scale = w_std * initial_noise_factor * max(0.0, 1.0 - t / noise_ramp_length) ** 2
        lr_ramp = min(1.0, (1.0 - t) / lr_rampdown_length)
        lr_ramp = 0.5 - 0.5 * np.cos(lr_ramp * np.pi)
        lr_ramp = lr_ramp * min(1.0, t / lr_rampup_length)
        for param_group in optimizer.param_groups:
            param_group['lr'] = initial_learning_rate * lr_ramp
        if cam_opt is not None:
            for param_group in cam_opt.param_groups:
                param_group['lr'] = camera_lr * lr_ramp

        w_noise = torch.randn_like(w_opt) * w_noise_scale
        ws = w_opt + w_noise if w_plus else (w_opt + w_noise).repeat([1, num_ws, 1])
        c = label if delta is None else refine_label(label, delta)
        if mirror:
            c = torch.cat([c, mirror_label(c)])
        out = G.synthesis(ws, c=c, noise_mode='const', force_fp32=True, views=views, return_seg='raw' if use_seg else False)
        synth_images, seg_raw = out if use_seg else (out, None)
        synth_images = _prepare(synth_images)
        dist = (target_features[0] - vgg16(synth_images[0:1], resize_images=False, return_lpips=True)).square().sum()
        if mirror:
            dist = dist + (target_features[1] - vgg16(synth_images[1:2], resize_images=False, return_lpips=True)).square().sum()

        reg_loss = projection.noise_regularizer(noise_bufs)
        loss = dist + reg_loss * regularize_noise_weight
        if use_seg:
            loss = loss + seg_weight * projection.seg_cross_entropy(seg_raw, mask_b)

        optimizer.zero_grad(set_to_none=True)
        if cam_opt is not None:
            cam_opt.zero_grad(set_to_none=True)
        loss.backward()
        optimizer.step()
        if cam_opt is not None:
            cam_opt.step()
        if on_step is not None:
            on_step(step, dist.detach(), loss.detach())
        projection.noise_normalize_(noise_bufs)

    ws = w_opt.detach() if w_plus else w_opt.detach().repeat([1, num_ws, 1])
    out_label = label.clone() if delta is None else refine_label(label, delta.detach()).detach()
    return ws, out_label
