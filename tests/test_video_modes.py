"""CPU: the image_seg / image_depth modes of the batched video driver (gen_videos.py:129-139) with the CUDA entry points swapped for
the oracle (oracle.backend.cpu_reference_ops + oracle.frames.cpu_frame_ops), the reference's image_depth frame loop replayed from its
recording, and the C-ABI argument checks of ide3d_video_frames."""

import ctypes
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import ROOT
from oracle import frames as ofr
from oracle.backend import cpu_reference_ops
from test_reference_cli import Trace, _recipe_mod


@pytest.fixture(scope='module')
def G():
    from ide3d_b200.training.triplane import TriPlaneGenerator
    torch.manual_seed(0)
    return TriPlaneGenerator(z_dim=32, w_dim=32, img_resolution=64, plane_resolution=32, render_size=16, channel_base=1024,
                             channel_max=32, sr_channels=(16, 8), mapping_kwargs=dict(num_layers=2)).eval().requires_grad_(False)


def _colors(seg):
    """COLOR_MAP row of the argmax class, uint8 [N, 3, H, W] (the cell's right half: (c / 255 - 0.5) / 0.5 -> * 127.5 + 128 is c)."""
    from ide3d_b200.dnnlib.seg_tools import COLOR_MAP
    lut = torch.tensor([COLOR_MAP.get(k, [0, 0, 0]) for k in range(seg.shape[1])], dtype=torch.uint8)
    return lut[seg.argmax(1)].permute(0, 3, 1, 2)


def _decided(seg):
    """Pixels whose top-two class margin is clear of rounding: elsewhere two bilinear evaluations may pick different classes."""
    top2 = seg.topk(2, dim=1).values
    return (top2[:, 0] - top2[:, 1]) > 1e-5 * (1 + seg.abs().max())


def test_gen_videos_image_depth_frame_loop_replayed():
    """gen_videos.gen_interp_video (2 seeds x 2 frames, image_depth), replayed: the cells the script built and the frames it wrote
    are the oracle composition of the replayed G.synthesis outputs.  (The script's image_depth branch keeps the batch-1 axis, which
    its layout_grid cannot unpack; the recording drops that axis, as the image_seg branch does, see make_cli_depth_golden.py.)"""
    with torch.no_grad(), cpu_reference_ops():
        tr = Trace('cli_gen_videos_depth').replay(_recipe_mod.cli_generator())
    frames, cells = tr.z['frames'], tr.z['cells']
    assert frames.shape == (4, 64, 64, 3) and frames.dtype == np.uint8 and cells.shape == (4, 3, 64, 64)
    outs = tr.outputs('synthesis')[1:]                                           # after the warm-up call (gen_videos.py:91)
    assert len(outs) == 4
    img = torch.cat([o[0] for o in outs])
    mine = ofr.compose_frames(img, None, 'image_depth')
    assert mine.shape == (4, 3, 64, 64)
    for f in range(4):
        x = -img[f]
        cell = (x - x.min()) / (x.max() - x.min()) * 2 - 1
        assert (cell - torch.from_numpy(cells[f])).abs().max() <= 2e-3, f        # replayed synthesis within the trace tolerance
        assert cell.min() == -1 and cell.max() == 1                              # per-cell normalisation
    diff = (mine.permute(0, 2, 3, 1).short() - torch.from_numpy(frames).short()).abs()
    print(f'image_depth replay: max uint8 difference {int(diff.max())}, {int((diff > 0).sum())} / {diff.numel()} bytes differ')
    assert diff.max() <= 1


def test_return_seg_raw_is_the_render_resolution_view(G):
    """return_seg='raw' hands back the logits the 512^2 map is upsampled from, as a view of the ray-march output; the other returns
    are unchanged."""
    from ide3d_b200.training import triplane
    with torch.no_grad(), cpu_reference_ops():
        ws, c, _ = _inputs(G, 2)
        img, seg = G.synthesis(ws, c=c, noise_mode='const', perturb=None, return_seg=True)
        img2, raw = G.synthesis(ws, c=c, noise_mode='const', perturb=None, return_seg='raw')
    assert raw.shape == (2, 19, 16, 16) and not raw.is_contiguous() and raw.stride(1) == 1     # channel view of feat [N, R, 51]
    assert torch.equal(img, img2)
    assert torch.equal(seg, triplane.upsample_seg(raw, (64, 64)))


def _inputs(G, n):
    from ide3d_b200 import video
    ws, c, dims = video.interp_video_inputs(G, [0, 1, 2, 3], w_frames=2, grid_dims=(2, 1), truncation_cutoff=4, device=torch.device('cpu'))
    return ws[:n].float(), c[:n], dims


@pytest.mark.parametrize('image_mode', ['image_seg', 'image_depth'])
def test_render_interp_video_new_modes_on_cpu(G, image_mode):
    """render_interp_video(image_mode=...): [F, grid_h*H, grid_w*k*W, 3] grids in frame order, each cell where layout_grid puts it;
    the seg half is mask2color of an independently computed upsample, the depth cell the per-cell normalised negated image."""
    from ide3d_b200 import video
    k = 2 if image_mode == 'image_seg' else 1
    with torch.no_grad(), cpu_reference_ops(), ofr.cpu_frame_ops():
        grids = video.render_interp_video(G, seeds=[0, 1, 2, 3], w_frames=2, grid_dims=(2, 1), batch=2, truncation_cutoff=4,
                                          device=torch.device('cpu'), synthesis_kwargs=dict(perturb=None), image_mode=image_mode)
        ws, c, (F, gh, gw) = video.interp_video_inputs(G, [0, 1, 2, 3], w_frames=2, grid_dims=(2, 1), truncation_cutoff=4,
                                                       device=torch.device('cpu'))
        singles = [G.synthesis(ws[i:i + 1].float(), c=c[i:i + 1], noise_mode='const', perturb=None, return_seg=True) for i in (1, 2, 7)]
    assert grids.dtype == torch.uint8 and tuple(grids.shape) == (4, 64, 2 * k * 64, 3) and (F, gh, gw) == (4, 1, 2)
    for i, (img, seg) in zip((1, 2, 7), singles):
        f, xi = divmod(i, gw)                                                     # row index = (frame * grid_h + yi) * grid_w + xi
        cell = grids[f, :, xi * k * 64:(xi + 1) * k * 64].permute(2, 0, 1)
        if image_mode == 'image_depth':
            x = -img
            want = ofr.to_uint8((x - x.min()) / (x.max() - x.min()) * 2 - 1)[0]
            assert (cell.int() - want.int()).abs().max() <= 1, i
            continue
        assert (cell[:, :, :64].int() - ofr.to_uint8(img)[0].int()).abs().max() <= 1, i
        decided = _decided(seg)[0]
        assert decided.float().mean() > 0.99
        assert torch.equal(cell[:, :, 64:][:, decided], _colors(seg)[0][:, decided]), i


def test_driver_rejects_unknown_mode_and_kernel_wrapper_rejects_cpu(G):
    from ide3d_b200 import dist as idist, video
    with pytest.raises(ValueError):
        idist.stream_frames_sharded(G, torch.zeros(2, G.num_ws, G.w_dim), torch.zeros(2, 25), 0, 1, batch=2, image_mode='image_normal')
    with pytest.raises(ValueError):
        video.compose_frames(torch.zeros(1, 3, 8, 8), None, 'image')
    with pytest.raises(RuntimeError, match='CUDA'):
        video.compose_frames(torch.zeros(1, 3, 8, 8), torch.zeros(1, 19, 4, 4), 'image_seg')


# ------------------------------------------------------------------------------------------------ 2 ranks, gloo
def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    from ide3d_b200 import dist as idist
    from ide3d_b200.training.triplane import TriPlaneGenerator
    from oracle import frames as of
    from oracle.backend import cpu_reference_ops as cro
    r, w, dev = idist.init_from_env(backend='gloo')
    assert (r, w) == (rank, world) and dev.type == 'cpu'
    torch.manual_seed(0)                                   # identical replicas on every rank
    G = TriPlaneGenerator(z_dim=16, w_dim=16, img_resolution=32, plane_resolution=16, render_size=8, channel_base=256,
                          channel_max=16, sr_channels=(8, 8), mapping_kwargs=dict(num_layers=1)).eval().requires_grad_(False)
    F = 4
    z = torch.randn(F, 16)
    c = torch.tensor([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 2.7, 0, 0, 0, 1, 4.2647, 0, 0.5, 0, 4.2647, 0.5, 0, 0, 1.]).repeat(F, 1)
    res = {}
    with torch.no_grad(), cro(), of.cpu_frame_ops():
        ws = G.mapping(z, c)
        single = idist.stream_frames_sharded(G, ws, c, 0, 1, batch=2, image_mode='image_seg', num_steps=6, perturb=None).clone()
        distinct = all(not torch.equal(single[i], single[j]) for i in range(F) for j in range(i))
        for transport in ('nccl', 'shm'):
            got = idist.stream_frames_sharded(G, ws, c, rank, world, batch=2, transport=transport, image_mode='image_seg',
                                              num_steps=6, perturb=None)
            if rank == 0:
                res[transport] = (tuple(got.shape), int((got.int() - single.int()).abs().max()))
            else:
                res[transport] = None if got is None else 'rank 1 got frames'
    q.put((rank, distinct, res))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_two_rank_gloo_image_seg_frames_land_in_frame_order(monkeypatch):
    """stream_frames_sharded(image_mode='image_seg') over 2 ranks, both transports: the double-width frames of both ranks reach rank 0
    in frame order and equal a single-rank run."""
    monkeypatch.setenv('CUDA_VISIBLE_DEVICES', '')
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 29500 + ((os.getpid() + 997) % 2000)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=240) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, distinct, per in res:
        assert distinct, rank
        for transport, v in per.items():
            if rank == 0:
                assert v == ((4, 3, 32, 64), 0), (transport, v)
            else:
                assert v is None, (transport, v)


# ------------------------------------------------------------------------------------------------ C-ABI
def test_video_frames_abi_validates_before_touching_the_device(lib):
    from ide3d_b200 import _lib
    P = _lib.FramesParams
    call = lambda **kw: lib.ide3d_video_frames(ctypes.byref(P(**kw)), None)
    seg = dict(mode=_lib.FRAMES_IMAGE_SEG, n=2, height=8, width=8, seg_c=19, seg_h=4, seg_w=4)
    depth = dict(mode=_lib.FRAMES_IMAGE_DEPTH, n=2, height=8, width=8)
    assert lib.ide3d_video_frames(None, None) == _lib.INVALID and b'null params' in lib.ide3d_last_error()
    for bad in (dict(seg, mode=0), dict(seg, mode=3), dict(depth, n=0, mode=7)):
        assert call(**bad) == _lib.INVALID and b'mode' in lib.ide3d_last_error()
    for bad in (dict(seg, n=-1), dict(seg, height=0), dict(depth, width=0), dict(seg, seg_c=0), dict(seg, seg_h=0), dict(seg, seg_w=-3),
                dict(depth, n=70000)):
        assert call(**bad) == _lib.INVALID and b'sizes' in lib.ide3d_last_error(), bad
    assert call(**dict(seg, n=0)) == _lib.OK and call(**dict(depth, n=0)) == _lib.OK                # empty batch: nothing to do
    assert call(**seg) == _lib.INVALID and b'null' in lib.ide3d_last_error()                         # null tensors
    assert call(**depth) == _lib.INVALID and b'null' in lib.ide3d_last_error()
