"""Golden data of the visualizer's frames: the reference's own Renderer methods, loaded from its source and run on the CPU.

    python tests/golden/make_viz_golden.py [/path/to/reference]   -> tests/golden/viz.npz

From viz/renderer.py: _render_impl, _apply_cmap and run_synthesis_net.  They run as methods of a small host object on the CPU, with
_cmaps pre-filled with oracle.viz.index_lut (seeded, 1024 entries, each naming its index) under the name 'viridis', and with
oracle.viz.StandInGenerator as the network (a stand-in mapping with the reference's truncation rule and a synthesis that returns
seeded image / image_depth / image_raw maps).  Stored per case: the arguments, the mapping's z and labels, the ws and camera label
synthesis received, the map the display tail read (before normalisation), and the result's image and stats.  Also stored: the layer
list run_synthesis_net gives for a small CPU TriPlaneGenerator called with unlinked=True (under oracle.backend.cpu_reference_ops)."""

import ast
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

BASE = dict(w0_seeds=[[0, 1]], yaw=0.0, pitch=0.0)
CASES = {
    'default': dict(),
    'weights_repeat': dict(w0_seeds=[[3, 0.5], [7, 0.25], [3, 0.25]], yaw=0.3, pitch=-0.2),
    'stylemix_in': dict(w0_seeds=[[1, 1]], stylemix_idx=[0, 5, 17], stylemix_seed=9),
    'stylemix_out': dict(w0_seeds=[[1, 0.7], [2, 0.3]], stylemix_idx=[-1, 18, 30, 2], stylemix_seed=2),
    'trunc': dict(w0_seeds=[[4, 1]], trunc_psi=0.6, trunc_cutoff=8),
    'trunc_all': dict(w0_seeds=[[4, 1]], trunc_psi=0.6, trunc_cutoff=None, focal_length=3.1),
    'depth': dict(render_type='image_depth'),
    'depth_norm_db': dict(render_type='image_depth', img_normalize=True, img_scale_db=3),
    'raw_sel1': dict(render_type='image_raw', sel_channels=1, base_channel=2, img_normalize=True),
    'raw_sel_many': dict(render_type='image_raw', sel_channels=5, base_channel=1),
    'base_clamp': dict(sel_channels=2, base_channel=9, img_scale_db=-6),
    'fft_all': dict(fft_show=True, fft_all=True, yaw=-0.4),
    'fft_sel': dict(fft_show=True, fft_all=False, sel_channels=1, base_channel=1, fft_beta=4, fft_range_db=30),
    'fft_depth': dict(render_type='image_depth', fft_show=True, fft_beta=4, fft_range_db=30),
    'fft_raw_norm': dict(render_type='image_raw', fft_show=True, img_normalize=True, random_seed=5),
}


def _method(tree, name):
    return next(n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name == name)


def reference_methods(ref):
    """(_render_impl, _apply_cmap, run_synthesis_net, CaptureSuccess) from viz/renderer.py."""
    from ide3d_b200 import dnnlib
    from ide3d_b200.training.volumetric_rendering import LookAtPoseSampler
    tree = ast.parse(open(os.path.join(ref, 'viz', 'renderer.py')).read())
    cls = next(n for n in ast.walk(tree) if isinstance(n, ast.ClassDef) and n.name == 'CaptureSuccess')
    ns = {'np': np, 'torch': torch, 'dnnlib': dnnlib, 'LookAtPoseSampler': LookAtPoseSampler}
    body = [cls] + [_method(tree, n) for n in ('_render_impl', '_apply_cmap', 'run_synthesis_net')]
    exec(compile(ast.Module(body=body, type_ignores=[]), 'viz/renderer.py', 'exec'), ns)
    return ns['_render_impl'], ns['_apply_cmap'], ns['run_synthesis_net']


def host(G, lut, render_impl, apply_cmap, run_net):
    """The reference Renderer's state and helpers that _render_impl touches, on the CPU."""
    self = types.SimpleNamespace(_device=torch.device('cpu'), _cmaps={'viridis': lut}, _net_layers={}, _last_model_input=None)
    self.get_network = lambda pkl, key: G
    self.to_device = lambda buf: buf.clone()
    self._apply_cmap = lambda x, name='viridis': apply_cmap(self, x, name)
    self.run_synthesis_net = run_net
    self.render = lambda **args: (lambda res: (render_impl(self, res, **args), res)[1])(types.SimpleNamespace())
    return self


def small_generator():
    from ide3d_b200.training.triplane import TriPlaneGenerator
    torch.manual_seed(0)
    return TriPlaneGenerator(z_dim=32, w_dim=32, img_resolution=64, plane_resolution=32, render_size=16, channel_base=1024,
                             channel_max=32, sr_channels=(16, 8), mapping_kwargs=dict(num_layers=2)).eval().requires_grad_(False)


def main(ref=None):
    ref = ref or os.environ.get('IDE3D_REFERENCE', '/root/reference')
    from oracle import viz as ov
    from oracle.backend import cpu_reference_ops
    render_impl, apply_cmap, run_net = reference_methods(ref)
    lut = ov.index_lut()
    out = {'lut': lut.numpy()}
    for name, kw in CASES.items():
        G = ov.StandInGenerator()
        args = dict(BASE, **kw)
        res = host(G, lut, render_impl, apply_cmap, run_net).render(**args)
        (z, c_map), = G.mapping.calls
        (w, c_cam, maps), = G.synthesis.calls[:1]
        rt = args.get('render_type', 'image')
        out[f'{name}/args'] = np.array(json.dumps(args))
        out[f'{name}/z'], out[f'{name}/labels'] = z.numpy(), c_map.numpy()
        out[f'{name}/ws'], out[f'{name}/c'] = w.numpy(), c_cam.numpy()
        out[f'{name}/map'] = maps[rt][0].numpy()
        out[f'{name}/image'], out[f'{name}/stats'] = res.image.numpy(), res.stats.numpy()
    G = small_generator()
    with cpu_reference_ops(), torch.no_grad():
        ws = G.mapping(torch.randn(1, G.z_dim, generator=torch.Generator().manual_seed(1)), torch.zeros(1, G.c_dim))
        c = torch.zeros(1, 25)
        c[0, :16] = torch.eye(4).reshape(-1)
        c[0, 11] = 2.7
        _, layers = run_net(G, ws, c, noise_mode='const', force_fp32=False, unlinked=True)
    out['layers'] = np.array(json.dumps([(l.name, l.shape, l.dtype) for l in layers]))
    np.savez_compressed(os.path.join(HERE, 'viz.npz'), **out)
    print(f'wrote {os.path.join(HERE, "viz.npz")}: {len(CASES)} cases, {len(layers)} layers')


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else None)
