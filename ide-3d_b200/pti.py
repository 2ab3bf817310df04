"""Pivotal tuning (PTI): fine-tune the generator around a projected pivot, then render the tuned generator from a free-view path.

This is the main path of inversion/scripts/run_pti.py after the projection:

    run                 SingleIDCoach.train (inversion/training/coaches/single_id_coach.py:18-89 with base_coach.py): project the
                        portrait (projector.project with the coach's arguments, base_coach.py:111-131), then tune
    tune                the tuning loop (:60-89): every weight of a copy of G trained by Adam at a fixed pivot w; per step
                        loss = l2_lambda * mse(render, target) + lpips_lambda * LPIPS(render, target), zero_grad, and a stop
                        before the backward once the step's LPIPS (summed over the views) is at most lpips_threshold
    free_view_frames    the --viz_video trajectory (run_pti.py:149-184) as uint8 frames

What differs from the reference loop:
    - mirror=True (the coach's 'ide3d_join_view') renders the camera and its mirror image with ONE G.synthesis(..., views=2) call;
    - LPIPS's head (normalise, difference, 1x1 conv, mean over every tapped layer) is one kernel call forward and one backward
      (torch_utils.ops.lpips), and the target's trunk features are computed once rather than every step (same values);
    - before returning, the tuned copy's inference caches (noise products, transposed weights, the style plan's constants and the
      packed decoder) are dropped explicitly: they are keyed on parameter versions, which a fused Adam step does not bump.

The shape of the tuned generator (--viz_mesh) needs nothing new: INTEGRATION.md shows backbone + renderer.sigma_grid + mrc.
The swappable head is torch_utils.ops.lpips.lpips_head (oracle/pti.py::cpu_pti_ops replaces it to run the driver on the CPU).
"""

import copy
import math

import numpy as np
import torch
import torch.nn.functional as F

from . import projector as _projector
from .training.triplane import invalidate_caches

PROJECTORS = {'w': {}, 'w_plus': dict(w_plus=True), 'join_view': dict(mirror=True)}   # the coach's ide3d / ide3d_plus / ide3d_join_view
INTRINSICS = [4.2647, 0, 0.5, 0, 4.2647, 0.5, 0, 0, 1]                             # run_pti.py:171
FREE_VIEW_PERIOD = 120                                                              # run_pti.py:156-157: 2 pi f / (0.5 * 240)


def _device(G):
    return next(G.parameters()).device


def _check_target(G, target):
    target = torch.as_tensor(target)
    if target.ndim == 3:
        target = target[None]
    res = G.img_resolution
    if tuple(target.shape) != (1, G.img_channels, res, res):
        raise ValueError(f'pti: target must be [{G.img_channels}, {res}, {res}] or [1, {G.img_channels}, {res}, {res}] in [-1, 1], '
                         f'got {tuple(target.shape)}')
    return target


def _check_label(label):
    label = torch.as_tensor(label)
    if tuple(label.shape) != (1, 25):
        raise ValueError(f'pti: label must be [1, 25], got {tuple(label.shape)}')
    return label


def tune(G, ws, label, target, *, lpips, steps=350, lr=3e-4, l2_lambda=1, lpips_lambda=1, lpips_threshold=0.06, mirror=False,
         on_step=None, adam_kwargs=None):
    """Pivotal tuning of a copy of G at the pivot ws ([1, num_ws, w_dim]) seen from label ([1, 25]) towards target ([3, H, W] or
    [1, 3, H, W], in [-1, 1]: the image the reference's data loader yields).  -> the tuned copy, in eval() and not requiring grad;
    the caller's G is not modified.

    lpips: a torch_utils.ops.lpips.LPIPS (or a callable with its contract: (x, y or target(y)) -> [N], and .target(y)).
    mirror: also fit the target flipped along W from projector.mirror_label(label); both views come from one synthesis call and the
    step's loss is the sum of the two.  on_step(step, l2 [views], lpips [views], loss): called for every evaluated step, the one that
    stops early included, with detached tensors.  adam_kwargs: extra torch.optim.Adam arguments (foreach=, fused=, ...)."""
    label = _check_label(label)
    target = _check_target(G, target)
    ws = torch.as_tensor(ws)
    if ws.ndim != 3 or ws.shape[0] != 1 or ws.shape[2] != G.w_dim:
        raise ValueError(f'pti: ws must be [1, num_ws, {G.w_dim}], got {tuple(ws.shape)}')
    if l2_lambda < 0 or lpips_lambda < 0:
        raise ValueError(f'pti: l2_lambda and lpips_lambda must be >= 0, got {l2_lambda} and {lpips_lambda}')
    device = _device(G)
    G = copy.deepcopy(G).eval().float().requires_grad_(True)
    ws = ws.detach().to(device=device, dtype=torch.float32)
    label = label.to(device=device, dtype=torch.float32)
    target = target.to(device=device, dtype=torch.float32)
    views = 2 if mirror else 1
    c = torch.cat([label, _projector.mirror_label(label)]) if mirror else label
    real = torch.cat([target, torch.flip(target, (3,))]) if mirror else target
    real_features = lpips.target(real)
    optimizer = torch.optim.Adam(G.parameters(), lr=lr, **(adam_kwargs or {}))

    for step in range(steps):
        images = G.synthesis(ws, c=c, noise_mode='const', force_fp32=True, views=views)
        l2 = [F.mse_loss(images[v:v + 1], real[v:v + 1]) for v in range(views)]
        lp = lpips(images, real_features)
        loss = lp_sum = None
        for v in range(views):                     # base_coach.calc_loss per view, then single_id_coach.py:72-76
            lv = 0.0
            if l2_lambda > 0:
                lv = lv + l2[v] * l2_lambda
            if lpips_lambda > 0:
                lv = lv + lp[v] * lpips_lambda
            loss = lv if loss is None else loss + lv
            lp_sum = lp[v] if lp_sum is None else lp_sum + lp[v]
        if on_step is not None:
            on_step(step, torch.stack(l2).detach(), lp.detach(), loss.detach())
        optimizer.zero_grad()
        if lp_sum <= lpips_threshold:
            break
        loss.backward()
        optimizer.step()

    optimizer.zero_grad()
    G.requires_grad_(False)
    invalidate_caches(G)
    return G


def run(G, label, target, *, features, lpips, projector='w', first_inv_steps=450, w_avg_samples=600, **tune_kw):
    """SingleIDCoach.train for one portrait: project target ([3, H, W] or [1, 3, H, W] in [-1, 1]) seen from label ([1, 25], OpenGL
    convention: the coach's get_label has already negated columns 1, 2, 5, 6, 9, 10 of the dataset's OpenCV pose) with the W, W+
    or join-view projector, then tune around the pivot.  -> (G_tuned, ws [1, num_ws, w_dim], label [1, 25]).

    features: the projector's VGG16 (projector.load_features); lpips: the tuning loss (tune).  tune_kw: tune's keyword arguments
    (steps, lr, lambdas, lpips_threshold, on_step, adam_kwargs); mirror follows the projector."""
    if projector not in PROJECTORS:
        raise ValueError(f'pti: projector must be one of {sorted(PROJECTORS)}, got {projector!r}')
    if 'mirror' in tune_kw:
        raise TypeError('pti.run: mirror follows the projector (join_view)')
    label = _check_label(label)
    target = _check_target(G, target)
    device = _device(G)
    id_image = torch.squeeze((target.to(device) + 1) / 2) * 255                     # base_coach.py:112
    ws, label = _projector.project(G, label, id_image, features=features, num_steps=first_inv_steps, w_avg_samples=w_avg_samples,
                                   **PROJECTORS[projector])
    G_tuned = tune(G, ws, label, target, lpips=lpips, mirror=projector == 'join_view', **tune_kw)
    return G_tuned, ws, label


def free_view_cameras(num_frames=240, device='cpu'):
    """c [num_frames, 25] of run_pti.py:155-171: yaw pi (0.5 + 0.1 cos(2 pi f / 120)), pitch pi (0.5 - 0.05 sin(2 pi f / 120)),
    radius 2.7, looking at the origin, the FFHQ intrinsics."""
    from .training.volumetric_rendering import create_cam2world_matrix, sample_camera_positions
    rows = []
    for f in range(num_frames):
        h = math.pi * (0.5 + 0.1 * math.cos(2 * math.pi * f / FREE_VIEW_PERIOD))
        v = math.pi * (0.5 - 0.05 * math.sin(2 * math.pi * f / FREE_VIEW_PERIOD))
        points, _, _ = sample_camera_positions(device=device, n=1, r=2.7, horizontal_mean=h, vertical_mean=v, mode=None)
        c = create_cam2world_matrix(-points, points, device=device).reshape(1, -1)
        rows.append(torch.cat((c, torch.tensor(INTRINSICS).reshape(1, -1).to(c)), -1))
    return torch.cat(rows)


@torch.no_grad()
def free_view_frames(G, ws, num_frames=240, chunk=24):
    """The --viz_video frames of run_pti.py:149-184 for the pivot ws ([1, num_ws, w_dim]): uint8 numpy [num_frames, H, W, 3],
    converted as layout_grid does ((img * 127.5 + 128).clamp(0, 255) -> uint8).  `chunk` cameras per G.synthesis(..., views=chunk)
    call: one backbone pass per chunk instead of one per frame.  With hash jitter, frame f uses the f-th seed the batch-1 loop would
    draw from the global torch RNG (one torch.randint per synthesis call), so the caller's seeding carries over."""
    if ws.ndim != 3 or ws.shape[0] != 1:
        raise ValueError(f'free_view_frames: ws must be [1, num_ws, w_dim], got {tuple(ws.shape)}')
    if num_frames < 1 or chunk < 1:
        raise ValueError(f'free_view_frames: num_frames and chunk must be >= 1, got {num_frames} and {chunk}')
    device = _device(G)
    ws = ws.to(device=device, dtype=torch.float32)
    cams = free_view_cameras(num_frames, device)
    render_params = {'fov': 18, 'num_steps': 96}                                   # run_pti.py:158-165 (a camera is given)
    perturb = {**G.rendering_kwargs}.get('perturb', 'hash')
    seeds = None
    if perturb in ('hash', True):
        seeds = torch.tensor([int(torch.randint(0, 2 ** 62, (1,)).item()) for _ in range(num_frames)], dtype=torch.int64)
    out = np.empty([num_frames, G.img_resolution, G.img_resolution, 3], dtype=np.uint8)
    for start in range(0, num_frames, chunk):
        k = min(chunk, num_frames - start)
        kw = {} if seeds is None else dict(seed=seeds[start:start + k])
        img = G.synthesis(ws, c=cams[start:start + k], render_params=render_params, noise_mode='const', views=k, **kw)
        out[start:start + k] = (img * 127.5 + 128).clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).cpu().numpy()
    return out
