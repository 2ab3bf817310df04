"""TriPlaneGenerator: the generator object the reference's tools call (`from training.triplane import
TriPlaneGenerator`, viz/renderer.py:196) -- restated, because the class source is not in the reference tree.

Contract reconstructed from the call sites (SURVEY.md §8b):
    G.z_dim, G.c_dim (25 = cam2world 16 + intrinsics 9), G.w_dim, G.img_resolution, G.img_channels,
    G.rendering_kwargs, G.neural_rendering_resolution, G.init_args / G.init_kwargs, G.backbone.num_ws
    G.mapping(z, c, truncation_psi=1, truncation_cutoff=None) -> ws [N, 18, w_dim];  G.mapping.w_avg
    G.synthesis(ws, c=None, render_params=None, noise_mode='const', force_fp32=False, return_seg=False,
                return_raw=False) -> img [N,3,512,512] | (img, seg [N,19,512,512]) | (img, img_raw)
        return_seg='raw' (extension): (img, seg_raw [N,19,R,R]), the render-resolution logits as a strided view of the
        ray-march output, not upsampled
    G.synthesis.voxel_block_resolutions / vb{res}(x, img, ws, condition_img=seg) -> (x, img, seg)
    G.synthesis.block_resolutions / b{res};  .num_ws, .w_dim, .render_size
    G.synthesis.renderer.sample_voxel(img_v, seg_v, points [N,P,3]) -> [N,P,52]       (extract_shapes.py:146)
Child order of `synthesis`: 7 backbone blocks, the renderer (3 decoder heads), 2 super-resolution blocks
(ide3d-nada/ZSSGAN/model/ZSSGAN_IDE3D.py:425-437) => 13 + 4 convs + final torgb = 18 ws.

What is this project's own choice (not recoverable from the reference, stated in DESIGN.md): the decoder heads
(texture -> 32 colour features; shape -> 19 semantic logits; shape -> sigma; 64 softplus hidden units each), the
world->plane scale 2/box_warp, stratified jitter by counter-hash, SR widths (128, 64) after EG3D.
"""

import math
import os
import weakref

import numpy as np
import torch

from .. import render
from ..torch_utils import misc, persistence
from . import networks
from .networks import FullyConnectedLayer, MappingNetwork, SegSynthesisBlock, SynthesisBlock

N_FEAT, N_SEG, N_OUT = 32, 19, 52
_STYLE_PLANS = weakref.WeakKeyDictionary()


# ================================================================================================ decoder
@persistence.persistent_class
class DecoderHead(torch.nn.Module):
    """features[32] -> softplus hidden -> out."""

    def __init__(self, in_features, hidden, out_features):
        super().__init__()
        self.fc1 = FullyConnectedLayer(in_features, hidden)
        self.fc2 = FullyConnectedLayer(hidden, out_features)

    def forward(self, f):
        return self.fc2(torch.nn.functional.softplus(self.fc1(f)))


# ================================================================================================ renderer
@persistence.persistent_class
class TriPlaneRenderer(torch.nn.Module):
    """Per-ray tri-plane sampling -> decoder -> alpha compositing, through the fused sm_90a kernels
    (ide3d_b200.render)."""

    def __init__(self, hidden=64, box_warp=1.0):
        super().__init__()
        self.tex_net = DecoderHead(N_FEAT, hidden, N_FEAT)      # texture planes -> colour features
        self.seg_net = DecoderHead(N_FEAT, hidden, N_SEG)       # shape planes   -> semantic logits
        self.sigma_net = DecoderHead(N_FEAT, hidden, 1)         # shape planes   -> density
        self.box_warp = box_warp
        self._packed = None
        self._packed_key = None

    @property
    def box_scale(self):
        return 2.0 / self.box_warp

    def heads(self):
        """[(in_sel, out_offset, w1, b1, w2, b2)] with the FC runtime gains folded in."""
        out = []
        for in_sel, off, head in ((0, 0, self.tex_net), (1, N_FEAT, self.seg_net), (1, N_FEAT + N_SEG, self.sigma_net)):
            w1, b1 = head.fc1.effective()
            w2, b2 = head.fc2.effective()
            out.append((in_sel, off, w1, b1, w2, b2))
        return out

    def packed(self):
        """Decoder parameters in the C-ABI head format; rebuilt when parameters move or change."""
        params = list(self.parameters())
        key = tuple((p.data_ptr(), p._version) for p in params)
        if self._packed is None or key != self._packed_key:
            self._packed = render.PackedDecoder(self.heads(), params[0].device)
            self._packed_key = key
        return self._packed

    def __getstate__(self):
        # the packed decoder holds ctypes structs of device pointers: copies and pickles rebuild it on their first call
        return dict(super().__getstate__(), _packed=None, _packed_key=None)

    as_planes = staticmethod(render.as_planes)

    def sample_voxel(self, img_v, seg_v, points, sigma_only=False):
        """Decode world-space points [N,P,3] -> [N,P,52] (or [N,P,1] sigma); extract_shapes.py:146."""
        return render.sample_voxel(img_v, seg_v, self.packed(), points, box_scale=self.box_scale, sigma_only=sigma_only)

    def sigma_grid(self, img_v, seg_v, grid_n=256, voxel_origin=(0, 0, 0), cube_length=2.0, pre_scale=0.9,
                   first=0, count=None):
        """Density on (a flat slab of) the voxel grid of extract_shapes.create_samples, points generated in-kernel."""
        return render.sigma_grid(img_v, seg_v, self.packed(), grid_n=grid_n, voxel_origin=voxel_origin,
                                 cube_length=cube_length, pre_scale=pre_scale, box_scale=self.box_scale,
                                 first=first, count=count)

    def forward(self, img_v, seg_v, cam2world, img_size=64, num_steps=48, fov=18.0, ray_start=2.25, ray_end=3.3,
                nerf_noise=0.0, perturb='hash', jitter_u=None, seed=None, clamp_mode='softplus', last_back=False,
                white_back=False, max_depth=None, fill_mode=None, return_weights=False, hierarchical=False, n_importance=None,
                importance_u=None, views=1):
        """-> feat [N, R, 51] (32 colour + 19 semantic), depth [N, R, 1], weights [N, R, S, 1] | None.
        views: frames per plane set; img_v / seg_v hold N / views sets and cam2world N rows, view j of set i being frame
        i * views + j.  seed: one int, or N per-frame seeds (frame f then jitters as a one-frame call with seed[f]).
        hierarchical: two-pass importance sampling (render.raymarch_hierarchical; sample_pdf, volumetric_rendering.py:224-265) with
        n_importance (default num_steps) extra samples per ray; gradients flow through the second pass, the importance depths are
        detached.  Off by default: whether the released generator samples
        hierarchically is not recoverable from the reference tree (SURVEY.md a8).
        perturb: 'hash' (in-kernel counter hash seeded from torch's CPU generator), 'rand' (torch.rand on the device,
        the draw the reference makes at volumetric_rendering.py:101), or None/False (no jitter)."""
        n = img_v.shape[0] * views
        res = (img_size, img_size) if isinstance(img_size, int) else tuple(img_size)
        if jitter_u is None and perturb == 'rand':
            jitter_u = torch.rand([n, res[0] * res[1], num_steps], device=img_v.device)
        if jitter_u is None and perturb in ('hash', True) and seed is None:
            seed = int(torch.randint(0, 2 ** 62, (1,)).item())      # keeps torch.manual_seed meaningful
        if perturb in (None, False, 'none'):
            seed = None
        noise = torch.randn([n, res[0] * res[1], num_steps], device=img_v.device) if nerf_noise else None
        # live parameters (differentiable) when a gradient can reach them, else the cached device copy
        train = torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters())
        if hierarchical:
            return render.raymarch_hierarchical(img_v, seg_v, self.heads() if train else self.packed(), cam2world, resolution=res, num_steps=num_steps,
                                                n_importance=n_importance, fov=fov, ray_start=ray_start, ray_end=ray_end,
                                                box_scale=self.box_scale, jitter_u=jitter_u, jitter_seed=seed, importance_u=importance_u,
                                                det=perturb in (None, False, 'none'), noise_std=float(nerf_noise or 0.0),
                                                clamp_mode=clamp_mode, last_back=last_back, white_back=white_back, max_depth=max_depth,
                                                fill_mode=fill_mode, return_weights=return_weights, views=views)
        return render.raymarch(img_v, seg_v, self.heads() if train else self.packed(), cam2world, resolution=res, num_steps=num_steps, fov=fov,
                               ray_start=ray_start, ray_end=ray_end, box_scale=self.box_scale, jitter_u=jitter_u,
                               jitter_seed=seed, noise=noise, noise_std=float(nerf_noise or 0.0), clamp_mode=clamp_mode,
                               last_back=last_back, white_back=white_back, max_depth=max_depth, fill_mode=fill_mode,
                               return_weights=return_weights, views=views)


def invalidate_caches(module):
    """Drop every inference constant cached under `module`: SynthesisLayer's noise products and transposed weights, the synthesis
    networks' style plans and the renderers' packed decoders; each is rebuilt on its next use.  Those caches key on
    (data_ptr, _version) of the parameters, and an in-place update that does not bump _version (torch.optim.Adam(fused=True) does
    not) leaves them stale: call this after changing weights that way."""
    for m in module.modules():
        m.__dict__.pop('_const_cache', None)
        if isinstance(m, SynthesisNetwork):
            _STYLE_PLANS.pop(m, None)
        if isinstance(m, TriPlaneRenderer):
            m._packed = m._packed_key = None


# ================================================================================================ synthesis
def _gather(t, index):
    """t[index] along dim 0 in one pass, keeping a channels_last layout (the fused skip passes and the chained convolutions expect it)."""
    if t.dim() == 4 and t.is_contiguous(memory_format=torch.channels_last) and not t.is_contiguous():
        return t.permute(0, 2, 3, 1).index_select(0, index).permute(0, 3, 1, 2)
    return t.index_select(0, index)


def upsample_seg(seg_raw, size):
    """Render-resolution semantic logits [N, 19, R, R] -> image resolution: bilinear, align_corners=False.  The rule of
    return_seg=True / return_dict; ide3d_video_frames (csrc/frames.cu) evaluates the same rule per pixel instead."""
    return torch.nn.functional.interpolate(seg_raw, size=size, mode='bilinear', align_corners=False)


@persistence.persistent_class
class SynthesisNetwork(torch.nn.Module):
    def __init__(self, w_dim, img_resolution=512, img_channels=3, plane_resolution=256, plane_channels=96,
                 render_size=64, channel_base=32768, channel_max=512, sr_channels=(128, 64), decoder_hidden=64,
                 box_warp=1.0, rendering_kwargs=None, conv_clamp=None, **block_kwargs):
        super().__init__()
        assert plane_resolution >= 4 and plane_resolution & (plane_resolution - 1) == 0
        self.w_dim, self.img_resolution, self.img_channels = w_dim, img_resolution, img_channels
        self.plane_resolution, self.plane_channels, self.render_size = plane_resolution, plane_channels, render_size
        self.rendering_kwargs = dict(ray_start=2.25, ray_end=3.3, fov=18.0, num_steps=48, nerf_noise=0.0,
                                     clamp_mode='softplus', white_back=False, last_back=False, perturb='hash')
        self.rendering_kwargs.update(rendering_kwargs or {})
        self.num_ws = 0

        # ---- tri-plane backbone: vb4 ... vb{plane_resolution}
        self.voxel_block_resolutions = [2 ** i for i in range(2, int(np.log2(plane_resolution)) + 1)]
        ch = {res: min(channel_base // res, channel_max) for res in self.voxel_block_resolutions}
        for res in self.voxel_block_resolutions:
            block = SegSynthesisBlock(ch[res // 2] if res > 4 else 0, ch[res], w_dim=w_dim, resolution=res,
                                      img_channels=plane_channels, seg_channels=plane_channels,
                                      is_last=(res == plane_resolution), conv_clamp=conv_clamp, **block_kwargs)
            self.num_ws += block.num_conv
            setattr(self, f'vb{res}', block)

        # ---- renderer (three decoder heads)
        self.renderer = TriPlaneRenderer(hidden=decoder_hidden, box_warp=box_warp)

        # ---- super-resolution head: 2 blocks, x2 each, fed with the feature image resized to img_resolution / 4
        self.sr_input_resolution = img_resolution // 4
        self.block_resolutions = [img_resolution // 2, img_resolution]
        cin = N_FEAT
        for res, cout in zip(self.block_resolutions, sr_channels):
            block = SynthesisBlock(cin, cout, w_dim=w_dim, resolution=res, img_channels=img_channels,
                                   is_last=(res == img_resolution), conv_clamp=conv_clamp, **block_kwargs)
            self.num_ws += block.num_conv
            if res == img_resolution:
                self.num_ws += block.num_torgb
            setattr(self, f'b{res}', block)
            cin = cout

    # ws slicing rule shared with extract_shapes.py:113-124: narrow num_conv+num_torgb, advance by num_conv
    def split_ws(self, ws):
        misc.assert_shape(ws, [None, self.num_ws, self.w_dim])
        ws = ws.to(torch.float32)
        voxel_ws, block_ws, idx = [], [], 0
        for res in self.voxel_block_resolutions:
            b = getattr(self, f'vb{res}')
            voxel_ws.append(ws.narrow(1, idx, b.num_conv + b.num_torgb))
            idx += b.num_conv
        for res in self.block_resolutions:
            b = getattr(self, f'b{res}')
            block_ws.append(ws.narrow(1, idx, b.num_conv + b.num_torgb))
            idx += b.num_conv
        return voxel_ws, block_ws

    def _blocks(self):
        return [getattr(self, f'vb{r}') for r in self.voxel_block_resolutions] + [getattr(self, f'b{r}') for r in self.block_resolutions]

    def _style_plan(self, ws, fp16_blocks=()):
        """All styles / demodulation coefficients of the call in two launches (networks.StylePlan) when the blocks run the fp32
        activation-scaled inference path on a CUDA device; None otherwise (every layer then computes its own, as the reference does).
        fp16_blocks: blocks that run on fp16 operands (networks.fp16_operands); their dcoefs carry each layer's 2^e."""
        if not (networks.STYLE_PLAN and ws.is_cuda) or (torch.is_grad_enabled() and (ws.requires_grad or any(p.requires_grad for p in self.parameters()))):
            return None
        blocks = self._blocks()
        if any(b.use_fp16 for b in blocks) or int(os.environ.get('IDE3D_FUSED_MODCONV_MIN_RES', networks.FUSED_MODCONV_MIN_RES)) <= max(b.resolution for b in blocks):
            return None
        plan = _STYLE_PLANS.get(self)                 # kept outside the module: the plan holds ctypes structs and is not picklable
        if plan is None:
            pairs, idx = [], 0
            for b in blocks:
                pairs.append((b, idx))
                idx += b.num_conv
            plan = _STYLE_PLANS[self] = networks.StylePlan(pairs)
        return plan.run(ws, fp16_blocks=fp16_blocks)

    def _chain_kwargs(self, blocks, block_kwargs):
        """Per-block keyword arguments that link consecutive blocks of one call (networks.FUSED_TORGB): every block but the last
        returns `x * styles` of the next block's conv0 (its only consumer) instead of x, the next block takes that as premodulated
        input, and the last block returns no x.  Needs the chained inference path in every block, which the style plan implies
        unless fused_modconv is forced; otherwise the blocks run unlinked."""
        plan = block_kwargs.get('style_plan')
        if plan is None or block_kwargs.get('fused_modconv') or not all(b.can_fold() for b in blocks):
            return [block_kwargs] * len(blocks)
        out = []
        for i, b in enumerate(blocks):
            kw = dict(block_kwargs, premodulated_x=i > 0 and b.in_channels != 0)
            if i + 1 < len(blocks):
                kw['x_next_styles'] = plan[blocks[i + 1].conv0][0]
            else:
                kw['drop_x'] = True
            out.append(kw)
        return out

    def prefix_blocks(self, rows):
        """How many leading backbone blocks read none of the ws `rows` (their split_ws slices, torgb row included)."""
        rows, idx = {int(r) for r in rows}, 0
        for k, res in enumerate(self.voxel_block_resolutions):
            b = getattr(self, f'vb{res}')
            if rows.intersection(range(idx, idx + b.num_conv + b.num_torgb)):
                return k
            idx += b.num_conv
        return len(self.voxel_block_resolutions)

    def backbone(self, voxel_ws, shared_prefix=None, **block_kwargs):
        x = img_v = seg_v = None
        blocks = [getattr(self, f'vb{res}') for res in self.voxel_block_resolutions]
        kws = self._chain_kwargs(blocks, block_kwargs)
        k = 0
        if shared_prefix is not None:
            # block k-1's torgb row is block k's conv0 row, so a prefix of un-mixed slices also fixes block k's conv0 styles within a
            # group: the prefix runs the plain call's chained kwargs on the groups' first latents, x * styles included
            k, first, inverse = shared_prefix
            plan = block_kwargs.get('style_plan')
            if plan is not None:
                layers = {m for b in blocks[:k] for m in b.modules()}
                plan = {layer: tuple(None if t is None else t.index_select(0, first) for t in sd)
                        for layer, sd in plan.items() if layer in layers}
            for block, cur_ws, kw in zip(blocks[:k], voxel_ws[:k], kws[:k]):
                kw = dict(kw) if plan is None else dict(kw, style_plan=plan)
                if kw.get('x_next_styles') is not None:
                    kw['x_next_styles'] = kw['x_next_styles'].index_select(0, first)
                x, img_v, seg_v = block(x, img_v, cur_ws.index_select(0, first), condition_img=seg_v, **kw)
            x, img_v, seg_v = (None if t is None else _gather(t, inverse) for t in (x, img_v, seg_v))
        for block, cur_ws, kw in zip(blocks[k:], voxel_ws[k:], kws[k:]):
            x, img_v, seg_v = block(x, img_v, cur_ws, condition_img=seg_v, **kw)
        return img_v, seg_v

    def superres(self, feat_img, block_ws, **block_kwargs):
        x, rgb = feat_img, feat_img[:, :self.img_channels]
        if x.shape[-1] != self.sr_input_resolution:
            size = (self.sr_input_resolution, self.sr_input_resolution)
            x = torch.nn.functional.interpolate(x, size=size, mode='bilinear', align_corners=False)
            rgb = torch.nn.functional.interpolate(rgb, size=size, mode='bilinear', align_corners=False)
        rgb = rgb.contiguous()
        blocks = [getattr(self, f'b{res}') for res in self.block_resolutions]
        for block, cur_ws, kw in zip(blocks, block_ws, self._chain_kwargs(blocks, block_kwargs)):
            x, rgb = block(x, rgb, cur_ws, **kw)
        return rgb

    def planes(self, ws, noise_mode='const', force_fp32=False, fused_modconv=None, shared_prefix=None, unlinked=False):
        """The tri-plane backbone of a synthesis call: -> (img_v, seg_v, style plan | None).  The plan holds every layer's styles and
        demodulation coefficients of the call; render_planes reads its super-resolution rows.  Arguments as forward's."""
        voxel_ws, _ = self.split_ws(ws)
        if shared_prefix is not None:
            k, groups = int(shared_prefix[0]), np.asarray(shared_prefix[1]).reshape(-1)
            if not 0 <= k <= len(self.voxel_block_resolutions) or groups.shape[0] != ws.shape[0]:
                raise ValueError(f'SynthesisNetwork: shared_prefix needs 0 <= k <= {len(self.voxel_block_resolutions)} and {ws.shape[0]} '
                                 f'group ids, got k={k} and {groups.shape[0]}')
            _, first, inverse = np.unique(groups, return_index=True, return_inverse=True)
            shared_prefix = None if k == 0 or len(first) == len(groups) else \
                (k, torch.from_numpy(first).to(ws.device), torch.from_numpy(inverse.reshape(-1)).to(ws.device))
        block_kwargs = dict(noise_mode=noise_mode, force_fp32=force_fp32, fused_modconv=fused_modconv)
        plan = None
        if unlinked:
            block_kwargs['unlinked'] = True
        else:
            # fp16 convolution operands in the tri-plane backbone only: the super-resolution blocks write the image itself, and there
            # one more rounding per convolution moves frames rendered at different batch sizes apart by 2 uint8 levels
            # (tests/test_gpu_multiview.py allows 1)
            backbone = [getattr(self, f'vb{r}') for r in self.voxel_block_resolutions]
            fp16 = networks.fp16_operands(backbone, force_fp32=force_fp32, fused_modconv=fused_modconv)
            plan = self._style_plan(ws, fp16_blocks=backbone if fp16 else ())
            if plan is not None:
                block_kwargs['style_plan'] = plan
                if fp16:
                    block_kwargs['fp16_operands'] = True
        img_v, seg_v = self.backbone(voxel_ws, shared_prefix=shared_prefix, **block_kwargs)
        return img_v, seg_v, plan

    def render_planes(self, img_v, seg_v, ws, c=None, render_params=None, noise_mode='const', force_fp32=False, return_seg=False,
                      return_raw=False, return_dict=False, fused_modconv=None, views=1, style_plan=None, unlinked=False,
                      **render_overrides):
        """Everything of a synthesis call after the backbone: the renderer and the super-resolution blocks, from the planes `planes`
        returned for these ws.  style_plan: the plan `planes` returned (its super-resolution rows are read).  The other arguments and
        the outputs are forward's; forward is planes followed by this call."""
        views = int(views)
        if views < 1:
            raise ValueError(f'SynthesisNetwork: views must be >= 1, got {views}')
        _, block_ws = self.split_ws(ws)
        sr_kwargs = dict(noise_mode=noise_mode, force_fp32=force_fp32, fused_modconv=fused_modconv)
        if unlinked:
            sr_kwargs['unlinked'] = True
        elif style_plan is not None:
            sr_kwargs['style_plan'] = style_plan
        if views > 1:
            # the per-view part: SR styles are functions of the ws row alone, so the plan's rows are repeated rather than recomputed
            block_ws = [w.repeat_interleave(views, 0) for w in block_ws]
            if 'style_plan' in sr_kwargs:
                rep = lambda t: None if t is None else t.repeat_interleave(views, 0)
                sr_layers = {m for r in self.block_resolutions for m in getattr(self, f'b{r}').modules()}
                sr_kwargs['style_plan'] = {layer: (rep(st), rep(dc)) for layer, (st, dc) in style_plan.items() if layer in sr_layers}

        kw = dict(self.rendering_kwargs)
        kw.update({k: v for k, v in (render_params or {}).items() if k in ('fov', 'num_steps', 'ray_start', 'ray_end',
                                                                          'nerf_noise', 'white_back', 'last_back',
                                                                          'clamp_mode', 'perturb', 'hierarchical', 'n_importance')})
        kw.update(render_overrides)
        n = ws.shape[0] * views
        if c is not None:
            if views > 1 and c.shape[0] != n:
                raise ValueError(f'SynthesisNetwork: c has {c.shape[0]} rows, expected ws rows x views = {n}')
            cam2world = c[:, :16].reshape(-1, 4, 4)
        else:   # no label: build the pose from the render params' means (frontal by default)
            from .volumetric_rendering import create_cam2world_matrix, sample_camera_positions
            rp = render_params or {}
            origin, _, _ = sample_camera_positions(ws.device, n=n, r=rp.get('radius', 2.7),
                                                   horizontal_mean=rp.get('h_mean', math.pi / 2),
                                                   vertical_mean=rp.get('v_mean', math.pi / 2), mode=None)
            cam2world = create_cam2world_matrix(-origin, origin, device=ws.device)
        R = self.render_size
        if views > 1:
            kw['views'] = views
        feat, depth, _ = self.renderer(img_v, seg_v, cam2world, img_size=R, **kw)
        maps = feat.permute(0, 2, 1).reshape(n, N_OUT - 1, R, R)
        # feat is [N, HW, 51]: already channels-last; keep that layout for the super-resolution blocks when they use it
        sr_fmt = torch.channels_last if networks.CHANNELS_LAST else torch.contiguous_format
        feat_img, seg_raw = maps[:, :N_FEAT].contiguous(memory_format=sr_fmt), maps[:, N_FEAT:]
        img = self.superres(feat_img, block_ws, **sr_kwargs)
        out_size = (self.img_resolution, self.img_resolution)
        if return_dict:
            return dict(image=img, image_raw=feat_img[:, :self.img_channels],
                        image_depth=depth.permute(0, 2, 1).reshape(n, 1, R, R),
                        image_seg=upsample_seg(seg_raw, out_size))
        if return_seg == 'raw':
            return img, seg_raw
        if return_seg:
            return img, upsample_seg(seg_raw, out_size)
        if return_raw:
            return img, feat_img[:, :self.img_channels]
        return img

    def forward(self, ws, c=None, render_params=None, noise_mode='const', force_fp32=False, return_seg=False,
                return_raw=False, return_dict=False, fused_modconv=None, views=1, shared_prefix=None, unlinked=False, **render_overrides):
        """views (extension): render every latent from `views` cameras with ONE backbone pass.  ws [N, num_ws, w_dim]; c [N * views, 25]
        in latent-major order (row i * views + j is view j of latent i); every output has N * views rows in that order.  The
        tri-plane backbone runs on the N latents, the renderer and the super-resolution blocks per view (their ws repeated per view).
        seed= (a render override) may then hold N * views per-frame jitter seeds.
        shared_prefix (extension) = (k, groups): groups holds N host ints, and latents with equal ids have equal ws rows for the first k
        backbone blocks (prefix_blocks gives k for a set of differing rows).  Those k blocks then run once per group, on the group's first
        latent, with the plain call's arithmetic, and their outputs are repeated per latent; the other blocks run per latent.  Only the
        prefix blocks' batch changes, and with it possibly cuDNN's algorithm choice.  Nothing shared (k == 0 or all ids distinct) is
        the plain call.
        unlinked (extension): every layer computes its own styles and returns its own output, and every block returns its x -- no style
        plan, no `x * styles` written for the next layer, no fp16 operands.  What forward hooks need to see each layer's output
        (viz.renderer's layer capture); the chained default computes the same function with fewer passes."""
        if int(views) < 1:
            raise ValueError(f'SynthesisNetwork: views must be >= 1, got {views}')
        img_v, seg_v, plan = self.planes(ws, noise_mode=noise_mode, force_fp32=force_fp32, fused_modconv=fused_modconv,
                                         shared_prefix=shared_prefix, unlinked=unlinked)
        return self.render_planes(img_v, seg_v, ws, c=c, render_params=render_params, noise_mode=noise_mode, force_fp32=force_fp32,
                                  return_seg=return_seg, return_raw=return_raw, return_dict=return_dict, fused_modconv=fused_modconv,
                                  views=views, style_plan=plan, unlinked=unlinked, **render_overrides)


# ================================================================================================ generator
@persistence.persistent_class
class TriPlaneGenerator(torch.nn.Module):
    def __init__(self, z_dim=512, c_dim=25, w_dim=512, img_resolution=512, img_channels=3, mapping_kwargs=None,
                 rendering_kwargs=None, **synthesis_kwargs):
        super().__init__()
        self.z_dim, self.c_dim, self.w_dim = z_dim, c_dim, w_dim
        self.img_resolution, self.img_channels = img_resolution, img_channels
        self.synthesis = SynthesisNetwork(w_dim=w_dim, img_resolution=img_resolution, img_channels=img_channels,
                                          rendering_kwargs=rendering_kwargs, **synthesis_kwargs)
        self.num_ws = self.synthesis.num_ws
        self.mapping = MappingNetwork(z_dim=z_dim, c_dim=c_dim, w_dim=w_dim, num_ws=self.num_ws, **(mapping_kwargs or {}))

    # attribute names other tools read (viz/renderer.py:201-202, :331)
    @property
    def rendering_kwargs(self):
        return self.synthesis.rendering_kwargs

    @property
    def neural_rendering_resolution(self):
        return self.synthesis.render_size

    @neural_rendering_resolution.setter
    def neural_rendering_resolution(self, v):
        self.synthesis.render_size = int(v)

    @property
    def backbone(self):
        return self.synthesis

    def forward(self, z, c, truncation_psi=1, truncation_cutoff=None, **synthesis_kwargs):
        ws = self.mapping(z, c, truncation_psi=truncation_psi, truncation_cutoff=truncation_cutoff)
        return self.synthesis(ws, c=c, **synthesis_kwargs)
