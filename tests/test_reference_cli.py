"""CPU: the reference's OWN caller scripts (gen_images.py, gen_videos.py, extract_shapes.py), replayed from recordings.

tests/golden/make_cli_golden.py ran the unmodified scripts against this package (through `compat.install()`, with the generator
wrapped in a recording proxy) and stored every attribute they read from the generator and every call they made through it --
arguments, results, CPU RNG state -- plus what they handed to their output writers.  Each test below rebuilds the same small
random-init generator, replays the trace call by call (a call's replayed results feed the later calls that consumed them; every
result is compared with the recorded one), and checks the script-level outputs against the recording.  The reference's video frame
loop is pinned the same way against ide3d_b200.video (cli_video_inputs.npz).

What the recordings stub, and why it does not touch the contract under test:
  * `legacy.load_network_pkl`  -> the small random-init TriPlaneGenerator (no checkpoint pickle exists offline)
  * `dnnlib.util.open_url`     -> dummy context manager (the "pickle path" is never read)
  * imageio / plyfile / skimage -> absent output-writer dependencies of the scripts; `mrcfile` is ide3d_b200.mrc (compat.install())
  * torch.device('cuda') inside the scripts -> 'cpu', and the CUDA entry points -> oracle (oracle.backend.cpu_reference_ops)
  * torchvision's save_image   -> recorder (the scripts call it with the removed `range=` keyword)"""

import importlib.util
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_golden


def _recipe():
    spec = importlib.util.spec_from_file_location('make_cli_golden', os.path.join(GOLDEN, 'make_cli_golden.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _close(actual, ref, what):
    ref = torch.as_tensor(ref).double()
    actual = torch.as_tensor(actual).double()
    assert actual.shape == ref.shape, (what, tuple(actual.shape), tuple(ref.shape))
    tol = 1e-3 * max(1.0, ref.abs().max().item()) if ref.numel() else 0.0
    err = (actual - ref).abs().max().item() if ref.numel() else 0.0
    assert err <= tol, f'{what}: max abs err {err:.3e} > {tol:.3e}'


class Trace:
    """Replays a recorded trace of generator attribute reads and calls (see tests/golden/make_cli_golden.py for the encoding)."""

    def __init__(self, name):
        self.z = load_golden(name)
        self.events = json.loads(str(self.z['events']))
        self.replayed = {}                         # array index -> the tensor the replay produced in its place
        self.results = []                          # (path, replayed result) of every call, in order

    def decode(self, x):
        if isinstance(x, dict):
            if 'tensor' in x:
                i = x['tensor']
                if i in self.replayed:
                    return self.replayed[i]
                return torch.from_numpy(np.array(self.z[f'a{i}']))
            if 'array' in x:
                return np.array(self.z[f'a{x["array"]}'])
            if 'device' in x:
                return torch.device(x['device'])
            if 'torch_dtype' in x:
                return getattr(torch, x['torch_dtype'].split('.')[-1])
            if 'list' in x:
                return [self.decode(v) for v in x['list']]
            if 'tuple' in x:
                return tuple(self.decode(v) for v in x['tuple'])
            if 'dict' in x:
                return {k: self.decode(v) for k, v in x['dict']}
            raise AssertionError(f'cannot decode {x}')
        return x

    def check_result(self, actual, rec, what):
        if isinstance(rec, dict) and 'tensor' in rec:
            i = rec['tensor']
            assert isinstance(actual, torch.Tensor), (what, type(actual))
            shape = tuple(self.z[f'shape{i}'])
            assert tuple(actual.shape) == shape, (what, tuple(actual.shape), shape)
            flat = actual.detach().reshape(-1)[torch.from_numpy(_recipe_mod.sample_positions(actual.numel()))]
            _close(flat, self.z[f's{i}'], what)
            self.replayed[i] = actual
        elif isinstance(rec, dict) and ('list' in rec or 'tuple' in rec):
            items = rec.get('list', rec.get('tuple'))
            assert isinstance(actual, (list, tuple)) and len(actual) == len(items), (what, type(actual))
            for k, (a, r) in enumerate(zip(actual, items)):
                self.check_result(a, r, f'{what}[{k}]')
        elif isinstance(rec, dict) and 'dict' in rec:
            for k, r in rec['dict']:
                self.check_result(actual[k], r, f'{what}[{k}]')
        elif isinstance(rec, dict) and 'opaque' in rec:
            assert type(actual).__name__ == rec['opaque'], (what, type(actual).__name__, rec['opaque'])
        else:
            assert actual == rec, (what, actual, rec)

    def replay(self, G):
        for ev in self.events:
            kind, path = ev[0], ev[1]
            target = G
            for name in filter(None, path.split('.')):
                target = getattr(target, name)
            if kind == 'get':
                self.check_result(target, ev[2], path)
                continue
            torch.set_rng_state(torch.from_numpy(np.array(self.z[f'a{ev[5]}'])))
            r = target(*self.decode(ev[2]), **self.decode(ev[3]))
            self.check_result(r, ev[4], path + '()')
            self.results.append((path, r))
        return self

    def outputs(self, path):
        return [r for p, r in self.results if p == path]


_recipe_mod = _recipe()


@pytest.fixture()
def replay_env():
    from oracle.backend import cpu_reference_ops
    with torch.no_grad(), cpu_reference_ops():
        yield _recipe_mod.cli_generator()


def _colorize(seg):
    """seg_tools.mask2color (reference dnnlib/seg_tools.py:75-82) with this package's colour table, on the CPU."""
    from ide3d_b200.dnnlib.seg_tools import COLOR_MAP
    lut = torch.tensor([COLOR_MAP.get(k, [0, 0, 0]) for k in range(seg.shape[1])], dtype=torch.float32)
    return lut[seg.argmax(1)].permute(0, 3, 1, 2)


def _sigma_grid(trace, res):
    return torch.cat([o[..., -1] for o in trace.outputs('synthesis.renderer.sample_voxel')], 1).reshape(res, res, res)


def test_gen_images_runs_unchanged(replay_env):
    """gen_images.py (seed 3, psi 0.7, three yaws): G.to / G.z_dim / G.mapping(z=, c=, truncation_psi=) / G.synthesis(ws, c=,
    render_params=, noise_mode=, return_seg=True) as the script calls them, and the two PNGs it writes."""
    tr = Trace('cli_gen_images').replay(replay_env)
    outs = tr.outputs('synthesis')
    assert len(outs) == 3                                                        # 3 yaws
    img = torch.cat([o[0] for o in outs])
    seg = (_colorize(torch.cat([o[1] for o in outs])) / 255. - 0.5) / 0.5
    assert img.shape == (3, 3, 64, 64) and seg.shape == (3, 3, 64, 64)
    assert torch.isfinite(img).all() and not torch.allclose(img[0], img[2])     # different yaws, different views
    to8 = lambda t: ((t.clamp(-1, 1) + 1) * 127.5).round().to(torch.int16)
    assert (to8(img) - torch.from_numpy(tr.z['saved_img']).short()).abs().max() <= 1
    assert torch.equal(to8(seg), torch.from_numpy(tr.z['saved_seg']).short())   # the colour table is the reference's


def test_extract_shapes_block_walk_runs_unchanged(replay_env):
    """extract_shapes.sample_generator_ide3d at 12^3: mapping, the synthesis block attributes it walks (num_ws, w_dim,
    voxel_block_resolutions, vb*/b* num_conv / num_torgb), vb* block calls with condition_img=, renderer.sample_voxel in chunks."""
    tr = Trace('cli_extract_shapes').replay(replay_env)
    vox = tr.z['voxels']
    assert vox.shape == (12, 12, 12) and np.isfinite(vox).all() and vox.std() > 0
    _close(_sigma_grid(tr, 12), vox, 'sigma grid')


def test_gen_videos_frame_loop_runs_unchanged(replay_env):
    """gen_videos.gen_interp_video (2 seeds x 2 frames, image_seg): the frames it hands to the video writer."""
    tr = Trace('cli_gen_videos').replay(replay_env)
    frames = tr.z['frames']
    assert frames.shape == (4, 64, 128, 3) and frames.dtype == np.uint8           # 2 keyframes x 2 frames; image | colourised mask
    outs = tr.outputs('synthesis')[1:]                                           # after the warm-up call (gen_videos.py:91)
    assert len(outs) == 4
    for f, (img, seg) in enumerate(outs):
        col = (_colorize(seg) / 255. - 0.5) / 0.5
        mine = (torch.cat((img, col), -1)[0] * 127.5 + 128).clamp(0, 255).to(torch.uint8).permute(1, 2, 0)
        assert (mine.short() - torch.from_numpy(frames[f]).short()).abs().max() <= 1, f


def test_extract_shapes_main_writes_mrc_through_the_shim(replay_env, tmp_path):
    """The script's __main__ block end to end (argparse -> stubbed pickle -> block walk -> sample_voxel chunks ->
    `mrcfile.new_mmap(...)` + np.save): the replayed grid is the saved one, and the MRC writer call the script made
    (same keywords, `with ... as m: m.data[:] = grid`) writes through ide3d_b200.mrc the same volume."""
    from ide3d_b200 import mrc
    tr = Trace('cli_extract_shapes_main').replay(replay_env)
    grid = tr.z['grid']
    assert grid.shape == (10, 10, 10)
    _close(_sigma_grid(tr, 10), grid, 'sigma grid')
    kw = tr.decode(json.loads(str(tr.z['mrc_kwargs'])))
    path = str(tmp_path / '0.mrc')
    with mrc.new_mmap(path, **kw) as m:
        m.data[:] = grid
    vol, hdr = mrc.read_mrc(path)
    assert np.array_equal(vol, grid.astype(np.float32)) and hdr['mode'] == 2


def test_batched_video_inputs_equal_the_reference_frame_loop():
    """ide3d_b200.video.interp_video_inputs computes, up front, exactly the (w, camera) pair the reference's frame loop hands to
    G.synthesis for every (frame, grid cell) (gen_videos.py:112-129), and layout_frames is layout_grid (gen_videos.py:24-38)
    applied per frame."""
    from ide3d_b200 import video
    ref = load_golden('cli_video_inputs')
    ws, c, (F, gh, gw) = video.interp_video_inputs(_recipe_mod.video_stub_generator(), device=torch.device('cpu'), **_recipe_mod.KW)
    assert (F, gh, gw) == (12, 1, 2) and ref['ws'].shape[0] == F * gh * gw == ws.shape[0] == c.shape[0]
    assert ws.dtype == torch.float64
    assert np.abs(ws.numpy() - ref['ws']).max() < 1e-9 and np.abs(c.numpy() - ref['c']).max() < 1e-6

    mine = video.layout_frames(torch.from_numpy(ref['frames']), F, gh, gw)
    for f in range(F):
        assert np.array_equal(mine[f].numpy(), ref['grids'][f])
