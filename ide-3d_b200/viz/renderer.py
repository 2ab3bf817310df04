"""Renderer: the frames of the reference's visualizer (viz/renderer.py), without its GUI.

    r = Renderer(); res = r.render(pkl=G, w0_seeds=[[0, 1]], yaw=0.3, render_type='image', do_backbone_caching=True)
    res.image (uint8 HWC numpy), res.stats (float32 [6]), res.layers, res.render_time, res.error (a string) ...

render(**args) takes the keywords of the reference's _render_impl (:239-273) and fills the same result fields; every exception is
caught and returned as res.error, a string with the traceback.

What it does as the reference does, quirks included:
  * Latents (:299-334): the seeds are list(set(w0 seeds + [stylemix_seed])) in that order, z = RandomState(seed).randn(z_dim), one
    mapping call with (trunc_psi, trunc_cutoff), w = sum_i weight_i (ws_i - w_avg), the rows stylemix_idx inside [0, G.backbone.num_ws)
    replaced by the stylemix seed's (ws - w_avg), then + w_avg.  Only the LAST entry of that seed list is mapped with the frontal
    conditioning label; every other seed is mapped with a zero label (the reference writes the label at the loop's leftover index).
  * Camera: pivot (0, 0, 0), radius 2.7, LookAtPoseSampler.sample(3.14/2 - yaw, 3.14/2 + pitch) (3.14, not pi), intrinsics from
    focal_length.  torch.manual_seed(random_seed) runs before the pose is sampled.
  * Ignored, as the reference ignores them: lookat_point, conditioning_yaw, conditioning_pitch, depth_mult, depth_importance_mult.
    input_transform / untransform need a StyleGAN3 synthesis.input: has_input_transform is False.
  * Display (:362-406): stats before any normalisation; image_depth normalised in place as the reference does, and the image taken
    from the normalised values; sel_channels falls back to 1 when larger than the map's channel count (the depth map has one).

Deviations:
  * Render types: synthesis runs with return_dict=True, so image_depth and image_raw show the depth and raw maps.  The reference's own
    call returns the image tensor alone and shows the RGB image for every render type.
  * Networks: `pkl` is a TriPlaneGenerator module (used in place, on this renderer's device) or a local state_dict file loaded as
    style_mixing.load_generator loads it; network pickles are refused.  Networks are cached per source.
  * Backbone caching (do_backbone_caching=True; accepted and ignored by the reference): the tri-plane backbone's planes are kept for
    one key -- the network, the ws bytes, noise_mode, force_fp32, random_seed and every synthesis parameter's (data_ptr, _version) --
    with torch's CPU and CUDA generator states as they stand after the backbone.  A frame with the same key (a camera drag, another
    render type or display setting) restores those states and runs only the ray-march and the super-resolution blocks, so it equals
    the uncached frame bit for bit for every noise mode.  A layer capture does not use the cache.  An in-place weight update that does
    not bump _version (see training.triplane.invalidate_caches) is not seen by the key.
  * Layer capture runs synthesis with unlinked=True, where every layer returns its own output (the chained default hands a block's
    `x * styles` to the next one).  The layer list is that of an unlinked call, cached per (synthesis, kwargs) as the reference does.
  * The display tail runs on sm_90a (torch_utils.ops.viz).  The FFT panel's colormap is `cmap` (uint8 [K, 3]); without one, viridis
    at 1024 entries is taken from matplotlib when it is installed, and otherwise the FFT view reports an error.
"""

import sys
import time
import traceback

import numpy as np
import torch

from .. import images, style_mixing
from ..dnnlib.util import EasyDict
from ..torch_utils.ops import viz as viz_ops
from ..training.volumetric_rendering import LookAtPoseSampler


def _error_text():
    _, value, _ = sys.exc_info()
    return str(value) if isinstance(value, _Captured) else traceback.format_exc()


class _Captured(Exception):
    pass


class _LayerFound(Exception):
    def __init__(self, out):
        super().__init__()
        self.out = out


def frontal_label():
    """The conditioning label the reference gives the last seed (viz/renderer.py:318), float32 [25]."""
    return np.asarray(images.FRONTAL, dtype=np.float32)


@torch.no_grad()
def latents(G, w0_seeds, stylemix_idx=(), stylemix_seed=0, trunc_psi=1, trunc_cutoff=0, device=None):
    """(w [1, num_ws, w_dim], labels float32 numpy [S, c_dim], the seed list) as viz/renderer.py:299-334 forms them (module docstring)."""
    device = G.mapping.w_avg.device if device is None else device
    seeds = list(set([seed for seed, _ in w0_seeds] + [stylemix_seed]))
    zs = np.zeros([len(seeds), G.z_dim], dtype=np.float32)
    cs = np.zeros([len(seeds), G.c_dim], dtype=np.float32)
    for i, seed in enumerate(seeds):
        zs[i] = np.random.RandomState(seed).randn(G.z_dim)
    cs[len(seeds) - 1] = frontal_label()
    w_avg = G.mapping.w_avg
    ws = G.mapping(z=torch.from_numpy(zs).to(device), c=torch.from_numpy(cs).to(device), truncation_psi=trunc_psi,
                   truncation_cutoff=trunc_cutoff) - w_avg
    by_seed = dict(zip(seeds, ws))
    w = torch.stack([by_seed[seed] * weight for seed, weight in w0_seeds]).sum(dim=0, keepdim=True)
    rows = style_mixing.valid_styles(stylemix_idx, G.backbone.num_ws)
    if rows:
        w[:, rows] = by_seed[stylemix_seed][rows].unsqueeze(0)
    w += w_avg
    return w, cs, seeds


def camera(yaw, pitch, focal_length, device):
    """c [1, 25]: the reference's pose (pivot (0, 0, 0), radius 2.7, 3.14/2 +- yaw / pitch) and intrinsics from focal_length."""
    pose = LookAtPoseSampler.sample(3.14 / 2 - yaw, 3.14 / 2 + pitch, torch.tensor((0, 0, 0)), radius=2.7)
    intrinsics = torch.tensor([[focal_length, 0, 0.5], [0, focal_length, 0.5], [0, 0, 1]])
    return torch.cat([pose.reshape(-1, 16), intrinsics.reshape(-1, 9)], 1).to(device)


def run_synthesis_net(net, *args, capture_layer=None, **kwargs):
    """net.synthesis(*args, **kwargs) with a forward hook on every module of net: -> (output, layers).  The naming rules of the
    reference's layer widget: the module's name ('output' for the root), ':k' for the k-th 4-D / 5-D tensor of a module that returns
    several, '_2', '_3' ... for names seen before; 5-D outputs are averaged over dim 2.  layers = [EasyDict(name, shape, dtype)] in call
    order.  When capture_layer names a layer, synthesis stops there and that tensor is the output."""
    names = {m: name for name, m in net.named_modules()}
    seen, layers = set(), []

    def hook(module, _inputs, outputs):
        outs = list(outputs) if isinstance(outputs, (tuple, list)) else [outputs]
        outs = [t for t in outs if isinstance(t, torch.Tensor) and t.ndim in (4, 5)]
        for k, t in enumerate(outs):
            if t.ndim == 5:
                t = t.mean(2)
            name = names[module] or 'output'
            if len(outs) > 1:
                name = f'{name}:{k}'
            if name in seen:
                n = 2
                while f'{name}_{n}' in seen:
                    n += 1
                name = f'{name}_{n}'
            seen.add(name)
            layers.append(EasyDict(name=name, shape=[int(s) for s in t.shape], dtype=str(t.dtype).split('.')[-1]))
            if name == capture_layer:
                raise _LayerFound(t)

    handles = [m.register_forward_hook(hook) for m in net.modules()]
    try:
        out = net.synthesis(*args, **kwargs)
    except _LayerFound as found:
        out = found.out
    finally:
        for h in handles:
            h.remove()
    return out, layers


def viridis():
    """matplotlib's viridis at 1024 entries, uint8 [1024, 3]; ImportError without matplotlib."""
    import matplotlib
    cmap = matplotlib.colormaps['viridis'] if hasattr(matplotlib, 'colormaps') else matplotlib.cm.get_cmap('viridis')
    return torch.from_numpy(np.ascontiguousarray(cmap(np.linspace(0, 1, num=1024), bytes=True)[:, :3]))


class Renderer:
    def __init__(self, device='cuda', cmap=None):
        """cmap: uint8 [K, 3] colormap of the FFT view (default viridis from matplotlib, see the module docstring)."""
        self._device = torch.device(device)
        self._networks = {}                 # {source: TriPlaneGenerator}
        self._pinned_bufs = {}              # {(shape, dtype): pinned host tensor}
        self._cmap = None if cmap is None else torch.as_tensor(cmap, dtype=torch.uint8).reshape(-1, 3).to(self._device)
        self._net_layers = {}               # {(synthesis, kwargs): [EasyDict]}
        self._backbone = None               # (key, img_v, seg_v, style plan, CPU RNG state, CUDA RNG state)
        self._cuda = self._device.type == 'cuda'
        if self._cuda:
            self._start_event = torch.cuda.Event(enable_timing=True)
            self._end_event = torch.cuda.Event(enable_timing=True)
        self._is_timing = False
        self._last_model_input = None

    def render(self, **args):
        """One frame: the reference's result fields (module docstring); every exception becomes res.error."""
        self._is_timing = True
        t0 = time.perf_counter()
        if self._cuda:
            self._start_event.record(torch.cuda.current_stream(self._device))
        res = EasyDict()
        try:
            self._render_impl(res, **args)
        except Exception:                   # noqa: BLE001 -- reported to the caller as res.error
            res.error = _error_text()
        if self._cuda:
            self._end_event.record(torch.cuda.current_stream(self._device))
        if 'image' in res:
            res.image = self.to_cpu(res.image).numpy()
        if 'stats' in res:
            res.stats = self.to_cpu(res.stats).numpy()
        if 'error' in res:
            res.error = str(res.error)
        if self._is_timing:
            if self._cuda:
                self._end_event.synchronize()
                res.render_time = self._start_event.elapsed_time(self._end_event) * 1e-3
            else:
                res.render_time = time.perf_counter() - t0
            self._is_timing = False
        return res

    def get_network(self, pkl):
        """The generator for `pkl` (a TriPlaneGenerator module, or a local state_dict file), on this renderer's device."""
        if pkl is None:
            raise _Captured('Renderer: no network given (pkl=)')
        net = self._networks.get(pkl)
        if net is None:
            if isinstance(pkl, torch.nn.Module):
                net = pkl
            else:
                try:
                    net = style_mixing.load_generator(str(pkl), 'cpu')
                except Exception as e:      # noqa: BLE001 -- the click message is the error text
                    raise _Captured(getattr(e, 'message', None) or str(e)) from None
            net = net.eval().requires_grad_(False).to(self._device)
            self._networks[pkl] = net
            self._ignore_timing()
        return net

    def _get_pinned_buf(self, ref):
        key = (tuple(ref.shape), ref.dtype)
        buf = self._pinned_bufs.get(key)
        if buf is None:
            buf = torch.empty(ref.shape, dtype=ref.dtype)
            buf = self._pinned_bufs[key] = buf.pin_memory() if self._cuda else buf
        return buf

    def to_device(self, buf):
        return self._get_pinned_buf(buf).copy_(buf).to(self._device)

    def to_cpu(self, buf):
        return self._get_pinned_buf(buf).copy_(buf).clone()

    def _ignore_timing(self):
        self._is_timing = False

    def colormap(self):
        """The FFT view's colormap on the device: the constructor's, else matplotlib's viridis (1024 entries)."""
        if self._cmap is None:
            try:
                lut = viridis()
            except ImportError:
                raise _Captured('Renderer: fft_show needs a colormap; pass Renderer(cmap=uint8 [K, 3]) or install matplotlib') from None
            self._cmap = lut.to(self._device)
        return self._cmap

    def _backbone_key(self, G, w, noise_mode, force_fp32, random_seed):
        params = tuple((t.data_ptr(), t._version) for t in list(G.synthesis.parameters()) + list(G.synthesis.buffers()))
        return (G, w.detach().cpu().numpy().tobytes(), noise_mode, bool(force_fp32), random_seed, params)

    def _synthesis(self, G, w, c, noise_mode, force_fp32, random_seed, caching):
        """The frame's synthesis maps (return_dict=True), through the backbone cache when `caching`."""
        syn = G.synthesis
        key = self._backbone_key(G, w, noise_mode, force_fp32, random_seed) if caching else None
        hit = self._backbone if caching and self._backbone is not None and self._backbone[0] == key else None
        if hit is not None:
            _, img_v, seg_v, plan, cpu_state, cuda_state = hit
            torch.set_rng_state(cpu_state)
            if self._cuda:
                torch.cuda.set_rng_state(cuda_state, self._device)
        else:
            self._backbone = None
            img_v, seg_v, plan = syn.planes(w, noise_mode=noise_mode, force_fp32=force_fp32)
            if caching:
                cuda_state = torch.cuda.get_rng_state(self._device) if self._cuda else None
                self._backbone = (key, img_v, seg_v, plan, torch.get_rng_state(), cuda_state)
        return syn.render_planes(img_v, seg_v, w, c, noise_mode=noise_mode, force_fp32=force_fp32, return_dict=True, style_plan=plan)

    def _render_impl(self, res,
                     pkl=None, w0_seeds=[[0, 1]], stylemix_idx=[], stylemix_seed=0, trunc_psi=1, trunc_cutoff=0, random_seed=0,
                     noise_mode='const', force_fp32=False, layer_name=None, sel_channels=3, base_channel=0, img_scale_db=0,
                     img_normalize=False, fft_show=False, fft_all=True, fft_range_db=50, fft_beta=8, input_transform=None,
                     untransform=False, yaw=0, pitch=0, lookat_point=(0, 0, 0.2), conditioning_yaw=0, conditioning_pitch=0,
                     focal_length=4.2647, render_type='image', do_backbone_caching=False, depth_mult=1, depth_importance_mult=1):
        # pylint: disable=dangerous-default-value,unused-argument
        G = self.get_network(pkl)
        res.img_resolution = G.img_resolution
        res.num_ws = G.synthesis.num_ws
        res.has_noise = any('noise_const' in name for name, _ in G.synthesis.named_buffers())
        res.has_input_transform = hasattr(G.synthesis, 'input') and hasattr(G.synthesis.input, 'transform')

        w, _, _ = latents(G, w0_seeds, stylemix_idx, stylemix_seed, trunc_psi, trunc_cutoff, device=self._device)
        synthesis_kwargs = EasyDict(noise_mode=noise_mode, force_fp32=force_fp32)
        torch.manual_seed(random_seed)
        c = camera(yaw, pitch, focal_length, w.device)
        self._last_model_input = w
        if layer_name is not None:
            out, _ = run_synthesis_net(G, w, c, capture_layer=layer_name, unlinked=True, return_dict=True, **synthesis_kwargs)
        else:
            out = self._synthesis(G, w, c, noise_mode, force_fp32, random_seed, do_backbone_caching)

        cache_key = (G.synthesis, tuple(sorted(synthesis_kwargs.items())))
        if cache_key not in self._net_layers:
            torch.manual_seed(random_seed)
            _, self._net_layers[cache_key] = run_synthesis_net(G, w, c, unlinked=True, **synthesis_kwargs)
        res.layers = self._net_layers[cache_key]

        out = (out[render_type] if isinstance(out, dict) else out)[0]
        lut = self.colormap() if fft_show else None
        res.image, res.stats = viz_ops.display(out, render_type=render_type, sel_channels=sel_channels, base_channel=base_channel,
                                               img_normalize=img_normalize, img_scale_db=img_scale_db, fft_show=fft_show, fft_all=fft_all,
                                               fft_range_db=fft_range_db, fft_beta=fft_beta, cmap=lut)
