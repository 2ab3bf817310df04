#!/usr/bin/env python
"""Generate tests/golden/cli_*.npz by running the REFERENCE's own caller scripts (gen_images.py, gen_videos.py, extract_shapes.py,
imported unmodified) against this package on the CPU, and recording what they do with the generator.

    IDE3D_REFERENCE=/path/to/IDE-3D PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_cli_golden.py

The generator the scripts receive is wrapped in a recording proxy: every attribute the script reads from it (`G.z_dim`,
`generator.synthesis.voxel_block_resolutions`, ...) and every call it makes through it (`G.mapping(...)`, `G.synthesis(...)`,
`generator.synthesis.vb32(...)`, `generator.synthesis.renderer.sample_voxel(...)`, ...) is stored with its arguments, its result and
the CPU RNG state before the call.  tests/test_reference_cli.py replays that trace against a freshly built generator (cli_generator
below), so the exact API surface the reference scripts use stays pinned without the reference tree.  Also recorded: what the scripts
hand to their output writers (save_image tensors, video frames, the MRC writer's arguments and data).

cli_video_inputs.npz is separate: the (w, camera) pairs gen_interp_video's frame loop hands to G.synthesis, recorded with a stand-in
generator whose mapping is a fixed float64 function (video_stub_generator), replayed against ide3d_b200.video.interp_video_inputs.
"""

import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

KW = dict(seeds=[3, 1, 4, 1, 5, 9, 2, 6], w_frames=3, grid_dims=(2, 1), psi=0.7, truncation_cutoff=4)
FRAME_SHAPE = (3, 5, 7)
DEVICE = torch.device                                 # the scripts' hard-coded torch.device('cuda') is redirected while they run


def cli_generator():
    """The small random-init generator the script traces are recorded with (and replayed against)."""
    from ide3d_b200.training.triplane import TriPlaneGenerator
    torch.manual_seed(0)
    return TriPlaneGenerator(z_dim=32, w_dim=32, img_resolution=64, plane_resolution=32, render_size=16, channel_base=512,
                             channel_max=16, sr_channels=(8, 8), mapping_kwargs=dict(num_layers=2)).eval().requires_grad_(False)


def video_stub_generator(calls=None):
    """Stand-in generator: z_dim 32, six w's per sample from a fixed float64 map of z that also depends on psi and the cutoff;
    synthesis records its (ws, c) arguments."""
    M = torch.from_numpy(np.random.RandomState(7).randn(32, 32) / 8.0)

    class Stub:
        z_dim = 32

        def __init__(self):
            self._p = torch.nn.Parameter(torch.zeros(1, dtype=torch.float64))

        def parameters(self):
            return iter([self._p])

        @staticmethod
        def mapping(z, c, truncation_psi=1, truncation_cutoff=None, **kw):
            w = torch.tanh(z.double() @ M) * truncation_psi + 1e-3 * (truncation_cutoff or 0) + c.double()[:, :32].sum(1, keepdim=True)
            return w[:, None, :].repeat(1, 6, 1)

        @staticmethod
        def synthesis(ws, c, **kw):
            if calls is not None:
                calls.append((ws.detach().clone(), c.detach().clone()))
            n = ws.shape[0]
            return torch.zeros(n, 3, 4, 4), torch.zeros(n, 19, 4, 4)

    return Stub()


# ------------------------------------------------------------------------------------------------ trace encoding (JSON + arrays)
SAMPLE = 2048                                           # recorded elements per traced result tensor


class Arrays:
    """Tensors and arrays of a trace, one entry each (by object identity).  Inputs the script made itself are stored whole (a<i>);
    tensors that first appear as the RESULT of a traced call are stored as a fixed sample (s<i>: SAMPLE elements at seeded flat
    positions, shape in shape<i>) -- the replay feeds its own results into the later calls that consumed them and compares the sample.
    RNG states are stored once per distinct state."""

    def __init__(self):
        self.items, self.index, self.is_result, self.rng = [], {}, [], {}

    def add(self, x, result=False):
        key = id(x)
        if key not in self.index:
            self.index[key] = len(self.items)
            self.items.append(x)                        # keeps x alive: no id() reuse within a trace
            self.is_result.append(result)
        return self.index[key]

    def add_rng(self, state):
        key = bytes(state.numpy())
        if key not in self.rng:
            self.rng[key] = self.add(state)
        return self.rng[key]


def sample_positions(numel):
    return np.sort(np.random.RandomState(0).choice(numel, SAMPLE, replace=False)) if numel > SAMPLE else np.arange(numel)


def encode(x, arrays, result=False):
    if isinstance(x, Proxy):
        return {'generator': object.__getattribute__(x, '_path')}
    if isinstance(x, torch.Tensor):
        return {'tensor': arrays.add(x, result), 'dtype': str(x.dtype)}
    if isinstance(x, np.ndarray):
        return {'array': arrays.add(x)}
    if isinstance(x, DEVICE):
        return {'device': str(x)}
    if isinstance(x, torch.dtype):
        return {'torch_dtype': str(x)}
    if isinstance(x, (list, tuple)):
        return {'list' if isinstance(x, list) else 'tuple': [encode(v, arrays, result) for v in x]}
    if isinstance(x, dict):
        return {'dict': [[k, encode(v, arrays, result)] for k, v in x.items()]}
    if x is None or isinstance(x, (bool, int, float, str)):
        return x
    if isinstance(x, (np.integer, np.floating)):
        return x.item()
    return {'opaque': type(x).__name__}


def save_trace(path, events, arrays, **extra):
    blobs = {}
    for i, (a, res) in enumerate(zip(arrays.items, arrays.is_result)):
        a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
        if res:
            blobs[f's{i}'] = a.reshape(-1)[sample_positions(a.size)]
            blobs[f'shape{i}'] = np.array(a.shape, np.int64)
        else:
            blobs[f'a{i}'] = a
    np.savez_compressed(path, events=np.array(json.dumps(events)), **blobs, **extra)
    print(f'{path}: {len(events)} events, {len(arrays.items)} arrays, {os.path.getsize(path) / 1024:.0f} KB')


def _unwrap(x):
    if isinstance(x, Proxy):
        return object.__getattribute__(x, '_obj')
    if isinstance(x, (list, tuple)):
        return type(x)(_unwrap(v) for v in x)
    if isinstance(x, dict):
        return {k: _unwrap(v) for k, v in x.items()}
    return x


class Proxy:
    """Records attribute reads and calls made through it; sub-objects are wrapped with their attribute path."""

    def __init__(self, obj, path, events, arrays):
        for k, v in (('_obj', obj), ('_path', path), ('_events', events), ('_arrays', arrays)):
            object.__setattr__(self, k, v)

    def __getattr__(self, name):
        obj, path, events, arrays = (object.__getattribute__(self, k) for k in ('_obj', '_path', '_events', '_arrays'))
        v = getattr(obj, name)
        p = f'{path}.{name}' if path else name
        if v is None or isinstance(v, (torch.Tensor, bool, int, float, str, tuple, list)):
            events.append(['get', p, encode(v, arrays)])
            return v
        return Proxy(v, p, events, arrays)

    def __call__(self, *args, **kwargs):
        obj, path, events, arrays = (object.__getattribute__(self, k) for k in ('_obj', '_path', '_events', '_arrays'))
        args, kwargs = _unwrap(args), _unwrap(kwargs)
        rng = torch.get_rng_state()
        r = obj(*args, **kwargs)
        events.append(['call', path, encode(list(args), arrays), encode(kwargs, arrays), encode(r, arrays, result=True),
                       arrays.add_rng(rng)])
        if isinstance(r, torch.nn.Module):
            return Proxy(r, path.rpartition('.')[0] if r is getattr(obj, '__self__', None) else path + '()', events, arrays)
        return r


# ------------------------------------------------------------------------------------------------ recordings
def setup_reference(ref):
    sys.dont_write_bytecode = True
    sys.path.insert(0, ROOT)
    sys.path.insert(0, ref)
    for name in ('imageio', 'plyfile', 'skimage', 'skimage.measure', 'legacy'):
        sys.modules[name] = types.ModuleType(name)
    sys.modules['skimage'].measure = sys.modules['skimage.measure']
    import ide3d_b200.compat as compat
    compat.install()                                     # training.*, torch_utils.*, mrcfile -> this package
    import dnnlib                                        # the reference's own dnnlib
    import contextlib
    dnnlib.util.open_url = lambda *a, **k: contextlib.nullcontext(None)


def record_gen_images(out):
    import gen_images
    events, arrays = [], Arrays()
    G = Proxy(cli_generator(), '', events, arrays)
    sys.modules['legacy'].load_network_pkl = lambda f: {'G_ema': G}
    saved = {}
    gen_images.save_image = lambda t, path, **kw: saved.__setitem__(os.path.basename(path), t.clone())
    real_device = torch.device
    gen_images.torch.device = lambda *a, **k: real_device('cpu')          # the script hard-codes torch.device('cuda')
    try:
        gen_images.generate_images.callback(network_pkl='unused.pkl', seeds=[3], truncation_psi=0.7, noise_mode='const', outdir='unused')
    finally:
        gen_images.torch.device = real_device
    assert set(saved) == {'seed0003.png', 'seed0003_seg.png'}
    to8 = lambda t: ((t.clamp(-1, 1) + 1) * 127.5).round().to(torch.uint8).numpy()       # save_image(normalize=True, range=(-1, 1))
    save_trace(out, events, arrays, saved_img=to8(saved['seed0003.png']), saved_seg=to8(saved['seed0003_seg.png']))


def record_gen_videos(out):
    import gen_videos
    frames = []

    class _Writer:
        def append_data(self, a):
            frames.append(np.asarray(a))

        def close(self):
            pass

    sys.modules['imageio'].get_writer = lambda *a, **k: _Writer()
    events, arrays = [], Arrays()
    G = Proxy(cli_generator(), '', events, arrays)
    torch.manual_seed(0)
    gen_videos.gen_interp_video(G, 'unused.mp4', seeds=[0, 1], w_frames=2, grid_dims=(1, 1), psi=0.7, truncation_cutoff=4,
                                image_mode='image_seg', device=torch.device('cpu'))
    save_trace(out, events, arrays, frames=np.stack(frames))


def record_extract_shapes(out):
    import extract_shapes
    events, arrays = [], Arrays()
    G = Proxy(cli_generator(), '', events, arrays)
    z = torch.from_numpy(np.random.RandomState(0).randn(1, 32))
    label = torch.tensor([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 2.7, 0, 0, 0, 1, 4.2647, 0, 0.5, 0, 4.2647, 0.5, 0, 0, 1])[None].float()
    vox = extract_shapes.sample_generator_ide3d(G, None, z.float(), label, cube_length=1.0, voxel_resolution=12, psi=0.7, max_batch=500,
                                                h_stddev=0., v_stddev=0., num_steps=96)
    save_trace(out, events, arrays, voxels=vox)


def record_extract_shapes_main(out, ref):
    import runpy
    import tempfile
    from ide3d_b200 import mrc
    events, arrays = [], Arrays()
    G = Proxy(cli_generator(), '', events, arrays)
    sys.modules['legacy'].load_network_pkl = lambda f: {'G_ema': G}
    writes = []

    def new_mmap(name, **kw):                            # the script's MRC writer call, recorded; the file is written by ide3d_b200.mrc
        writes.append(kw)
        return mrc.new_mmap(name, **kw)

    sys.modules['mrcfile'] = types.SimpleNamespace(new_mmap=new_mmap)
    real_device = torch.device
    torch.device = lambda *a, **k: real_device('cpu')
    with tempfile.TemporaryDirectory() as tmp:
        argv = sys.argv
        sys.argv = ['extract_shapes.py', '--network', 'unused.pkl', '--seeds', '0', '--voxel_resolution', '10', '--cube_size', '1.0',
                    '--outdir', tmp]
        try:
            runpy.run_path(os.path.join(ref, 'extract_shapes.py'), run_name='__main__')
        finally:
            sys.argv = argv
            torch.device = real_device
        grid = np.load(os.path.join(tmp, '0.npy'))
        vol, hdr = mrc.read_mrc(os.path.join(tmp, '0.mrc'))
    assert len(writes) == 1 and np.array_equal(vol, grid.astype(np.float32)) and hdr['mode'] == 2
    save_trace(out, events, arrays, grid=grid, mrc_kwargs=np.array(json.dumps(encode(writes[0], Arrays()))))


def record_video_inputs(out):
    import gen_videos as gv

    class _Writer:
        def append_data(self, a):
            pass

        def close(self):
            pass

    sys.modules['imageio'].get_writer = lambda *a, **k: _Writer()
    calls = []
    gv.gen_interp_video(video_stub_generator(calls), 'unused.mp4', image_mode='image_seg', device=torch.device('cpu'), **KW)
    calls = calls[1:]                                    # the warm-up call (gen_videos.py:91)
    ws = torch.cat([w for w, _ in calls]).numpy()
    c = torch.cat([cc for _, cc in calls]).numpy()
    gw, gh = KW['grid_dims']
    n_frames = len(calls) // (gw * gh)
    frames = torch.randint(0, 255, (len(calls),) + FRAME_SHAPE, dtype=torch.uint8, generator=torch.Generator().manual_seed(0))
    grids = np.stack([gv.layout_grid(frames[f * gh * gw:(f + 1) * gh * gw], grid_w=gw, grid_h=gh, float_to_uint8=False)
                      for f in range(n_frames)])
    np.savez_compressed(out, ws=ws, c=c, frames=frames.numpy(), grids=grids)
    print(f'{out}: {len(calls)} (w, camera) pairs, {n_frames} frames')


def main():
    ref = os.environ.get('IDE3D_REFERENCE')
    if not ref or not os.path.isdir(ref):
        sys.exit('set IDE3D_REFERENCE to the reference IDE-3D tree')
    setup_reference(ref)
    torch.set_num_threads(4)
    from oracle.backend import cpu_reference_ops
    with torch.no_grad(), cpu_reference_ops():
        record_video_inputs(os.path.join(HERE, 'cli_video_inputs.npz'))
        record_gen_images(os.path.join(HERE, 'cli_gen_images.npz'))
        record_gen_videos(os.path.join(HERE, 'cli_gen_videos.npz'))
        record_extract_shapes(os.path.join(HERE, 'cli_extract_shapes.npz'))
        record_extract_shapes_main(os.path.join(HERE, 'cli_extract_shapes_main.npz'), ref)


if __name__ == '__main__':
    main()
