"""Oracle (test infrastructure): run the product's *host-side* generator classes with every CUDA entry point
replaced by the CPU restatement.

Used by (a) the CPU tests of the generator's host logic (ws slicing, block walk, API contract) and (b) the
cpu_baseline / `--impl reference` legs of bench.py, where it stands in for "the reference's own PyTorch path on the
host cores": the same stock torch ops the reference runs on CPU (grid_sample-equivalent gather, linear, softplus,
cumprod, conv2d) chained exactly like oracle.renderer.render_frames.  Never imported by the product package.
"""

import contextlib

import torch

from . import ops as oops
from . import renderer as orr


def _decoder_from_renderer(r):
    """Dense oracle.Decoder equivalent to a TriPlaneRenderer's three heads."""
    heads = r.heads()
    H = heads[0][2].shape[0]
    w1 = torch.zeros(3 * H, 64)
    b1 = torch.zeros(3 * H)
    w2 = torch.zeros(52, 3 * H)
    b2 = torch.zeros(52)
    for i, (in_sel, off, hw1, hb1, hw2, hb2) in enumerate(heads):
        cols = slice(0, 32) if in_sel == 0 else slice(32, 64)
        w1[i * H:(i + 1) * H, cols] = hw1.detach().cpu()
        b1[i * H:(i + 1) * H] = hb1.detach().cpu()
        w2[off:off + hw2.shape[0], i * H:(i + 1) * H] = hw2.detach().cpu()
        b2[off:off + hw2.shape[0]] = hb2.detach().cpu()
    return orr.Decoder(w1, b1, w2, b2)


def _renderer_forward(self, img_v, seg_v, cam2world, img_size=64, num_steps=48, fov=18.0, ray_start=2.25, ray_end=3.3,
                      nerf_noise=0.0, perturb='hash', jitter_u=None, seed=None, clamp_mode='softplus', last_back=False,
                      white_back=False, max_depth=None, fill_mode=None, return_weights=False, hierarchical=False, n_importance=None,
                      importance_u=None):
    res = (img_size, img_size) if isinstance(img_size, int) else tuple(img_size)
    n = img_v.shape[0]
    if jitter_u is None and perturb == 'rand':
        jitter_u = torch.rand([n, res[0] * res[1], num_steps, 1])
    if jitter_u is None and perturb in ('hash', True) and seed is None:
        seed = int(torch.randint(0, 2 ** 62, (1,)).item())
    if perturb in (None, False, 'none'):
        seed = None
    if jitter_u is not None:
        jitter_u = jitter_u.reshape(n, res[0] * res[1], num_steps, 1).cpu()
    noise = torch.randn([n, res[0] * res[1], num_steps, 1]) if nerf_noise else None
    if hierarchical:
        assert not nerf_noise and fill_mode is None, 'oracle: hierarchical composition is defined without density noise / fill modes'
        rgb, depth, w, _ = orr.render_frames_hierarchical(
            img_v.float().cpu().contiguous(), seg_v.float().cpu().contiguous(), _decoder_from_renderer(self),
            cam2world.float().cpu().reshape(n, 4, 4), fov=fov, num_steps=num_steps, n_importance=n_importance, ray_start=ray_start,
            ray_end=ray_end, resolution=res, box_scale=self.box_scale, jitter_u=jitter_u, jitter_seed=seed,
            importance_u=None if importance_u is None else importance_u.cpu(), det=perturb in (None, False, 'none'),
            clamp_mode=clamp_mode, last_back=last_back, white_back=white_back, max_depth=max_depth)
        return rgb, depth, (w if return_weights else None)
    rgb, depth, w = orr.render_frames(img_v.float().cpu().contiguous(), seg_v.float().cpu().contiguous(),
                                      _decoder_from_renderer(self), cam2world.float().cpu().reshape(n, 4, 4), fov=fov,
                                      num_steps=num_steps, ray_start=ray_start, ray_end=ray_end, resolution=res,
                                      box_scale=self.box_scale, jitter_u=jitter_u, jitter_seed=seed,
                                      clamp_mode=clamp_mode, last_back=last_back, white_back=white_back,
                                      max_depth=max_depth, fill_mode=fill_mode, noise=noise, noise_std=float(nerf_noise or 0))
    return rgb, depth, (w if return_weights else None)


def _renderer_sample_voxel(self, img_v, seg_v, points, sigma_only=False):
    out = orr.sample_voxel(img_v.float().cpu().contiguous(), seg_v.float().cpu().contiguous(), _decoder_from_renderer(self),
                           points.float().cpu(), self.box_scale)
    return out[..., -1:] if sigma_only else out


@contextlib.contextmanager
def cpu_reference_ops(reference_layout=True):
    """Inside the context the product's op modules and renderer compute with the oracle on CPU tensors.
    reference_layout: activations stay NCHW as in the reference's fp32 path (inversion/networks.py:746) -- the GPU build's
    NHWC choice is a GPU layout decision and would only slow the CPU arm down; False keeps whatever the product is set to."""
    from ide3d_b200.torch_utils.ops import bias_act as p_ba, filtered_lrelu as p_fl, upfirdn2d as p_up
    from ide3d_b200.training import networks as p_nw, triplane as p_tp
    saved_layout = p_nw.CHANNELS_LAST
    if reference_layout:
        p_nw.CHANNELS_LAST = False

    def ba(x, b=None, dim=1, act='linear', alpha=None, gain=None, clamp=None, impl='cuda'):
        return oops.bias_act(x, b, dim, act, alpha, gain, clamp)

    def sba(x, scale=None, noise=None, b=None, act='linear', alpha=None, gain=None, clamp=None, next_scale=None, only_next=False):
        # the two reference ops the product fuses: fma (inversion/networks.py:104-105) then bias_act (:512)
        if scale is not None:
            x = x * scale.to(x.dtype).reshape(x.shape[0], -1, 1, 1)
        if noise is not None:
            x = x + noise.to(x.dtype)
        y = oops.bias_act(x, None if b is None else b.to(x.dtype), 1, act, alpha, gain, clamp)
        if next_scale is None:
            return y
        y2 = y * next_scale.to(y.dtype).reshape(y.shape[0], -1, 1, 1)      # `x * styles` of the next layer (:100)
        return y2 if only_next else (y, y2)

    def up(x, f, up=1, down=1, padding=0, flip_filter=False, gain=1, impl='cuda'):
        return oops.upfirdn2d(x, f, up=up, down=down, padding=padding, flip_filter=flip_filter, gain=gain)

    def fl(x, fu=None, fd=None, b=None, up=1, down=1, padding=0, gain=2 ** 0.5, slope=0.2, clamp=None, flip_filter=False, impl='cuda'):
        return oops.filtered_lrelu(x, fu, fd, b, up, down, padding, gain, slope, clamp, flip_filter)

    def upepi(x, f, padding=0, gain=1, flip_filter=False, scale=None, noise=None, b=None, act='linear', alpha=None, act_gain=None,
              clamp=None, next_scale=None, only_next=False):
        y = oops.upfirdn2d(x, f, padding=padding, flip_filter=flip_filter, gain=gain)       # conv2d_resample.py:125
        return sba(y, scale, noise, b, act, alpha, act_gain, clamp, next_scale, only_next)

    def upadd(x, f, y, b=None, up=2):
        out = oops.upsample2d(x, f, up=up) + y                   # networks.py:841-844
        return out if b is None else out + b.to(out.dtype).reshape(1, -1, 1, 1)

    R = p_tp.TriPlaneRenderer
    saved = (p_ba.bias_act, p_up.upfirdn2d, p_fl.filtered_lrelu, R.forward, R.sample_voxel, p_ba.scaled_bias_act, p_up.upsample2d_add,
             p_up.upfirdn2d_epilogue)
    p_ba.bias_act, p_up.upfirdn2d, p_fl.filtered_lrelu, p_ba.scaled_bias_act, p_up.upsample2d_add = ba, up, fl, sba, upadd
    p_up.upfirdn2d_epilogue = upepi
    R.forward, R.sample_voxel = _renderer_forward, _renderer_sample_voxel
    try:
        yield
    finally:
        p_nw.CHANNELS_LAST = saved_layout
        (p_ba.bias_act, p_up.upfirdn2d, p_fl.filtered_lrelu, R.forward, R.sample_voxel, p_ba.scaled_bias_act, p_up.upsample2d_add,
         p_up.upfirdn2d_epilogue) = saved
