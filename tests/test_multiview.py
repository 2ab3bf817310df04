"""CPU: the multi-view pieces behind ide3d_b200.images.render_multiview (gen_images.py:84-116 batched).

  * the driver's cameras and per-view jitter seeds against what the reference loop handed to G.synthesis (tests/golden/cli_gen_images.npz)
  * SynthesisNetwork(views=...) and per-frame seeds against one-row calls, through the oracle renderer
  * oracle/images.py against torchvision's make_grid + save_image (tests/golden/image_strips.npz)
  * a world-2 gloo run of the driver against the world-1 run
  * the C-ABI: the image-strip and new ray-march parameter checks"""

import ctypes
import json
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import GOLDEN, ROOT, load_golden


def _cli_generator():
    sys.path.insert(0, GOLDEN)
    try:
        import make_cli_golden
    finally:
        sys.path.remove(GOLDEN)
    return make_cli_golden.cli_generator()


def test_driver_seeds_and_cameras_match_the_reference_loop():
    """gen_images.py ran with seed 3: before each of its three G.synthesis calls the recording holds the CPU RNG state, and the renderer
    draws its jitter seed from that state; the driver derives the same three seeds without touching the global RNG, and builds the same
    three camera labels."""
    from ide3d_b200 import images
    z = load_golden('cli_gen_images')
    events = [e for e in json.loads(str(z['events'])) if e[0] == 'call' and e[1] == 'synthesis']
    assert len(events) == 3
    want_seeds, want_c = [], []
    saved = torch.get_rng_state()
    try:
        for ev in events:
            torch.set_rng_state(torch.from_numpy(np.array(z[f'a{ev[5]}'])))
            want_seeds.append(int(torch.randint(0, 2 ** 62, (1,)).item()))
            c_arg = dict(ev[3]['dict'])['c']
            want_c.append(np.array(z[f'a{c_arg["tensor"]}']))
    finally:
        torch.set_rng_state(saved)
    before = torch.get_rng_state()
    assert images.view_seeds(3, 3) == want_seeds
    assert torch.equal(torch.get_rng_state(), before)
    cams = images.view_cameras(images.YAWS, 'cpu')
    assert np.abs(cams.numpy() - np.concatenate(want_c)).max() <= 1e-6
    for ev, yaw in zip(events, images.YAWS):
        rp = dict(dict(ev[3]['dict'])['render_params']['dict'])
        assert rp == images.render_params(yaw)


def test_per_frame_hash_matches_one_frame_hash():
    """render_grad.hash_uniform_frames (the kernel's per-frame seed mode) row f equals the single-seed hash of a one-frame launch, and
    equals oracle.renderer.hash_uniform; coarse_depths with per-frame seeds equals the one-frame depths frame by frame."""
    from ide3d_b200 import render
    from ide3d_b200.render_grad import hash_uniform, hash_uniform_frames
    from oracle.renderer import hash_uniform as ohash
    seeds = [5, 2 ** 61 + 7, 123456789012345]
    u = hash_uniform_frames(64, seeds, 'cpu')
    for f, s in enumerate(seeds):
        assert torch.equal(u[f], hash_uniform(64, s, 'cpu'))
        assert np.array_equal(u[f].numpy(), ohash(np.arange(64, dtype=np.uint64), s))
    z = render.coarse_depths(3, (4, 2), 8, jitter_seed=torch.tensor(seeds), device='cpu')
    for f, s in enumerate(seeds):
        assert torch.equal(z[f], render.coarse_depths(1, (4, 2), 8, jitter_seed=s, device='cpu')[0])
    with pytest.raises(ValueError):
        render.coarse_depths(2, (4, 2), 8, jitter_seed=seeds, device='cpu')


@pytest.mark.parametrize('return_kind', ['image', 'seg', 'raw', 'dict'])
def test_synthesis_views_equal_one_row_calls(return_kind):
    """G.synthesis(ws, c, views=3, seed=[...]) under the oracle: one backbone pass on N rows, outputs equal to the one-row calls of
    every (latent, view) with its own seed."""
    from oracle.images import cpu_multiview_ops
    G = _cli_generator()
    from ide3d_b200 import images
    cams = images.view_cameras(images.YAWS, 'cpu')
    c = cams.repeat(2, 1)
    seeds = [11, 12, 13, 21, 22, 23]
    kw = dict(render_params=dict(num_steps=12), noise_mode='const')
    ret = dict(image={}, seg=dict(return_seg=True), raw=dict(return_seg='raw'), dict=dict(return_dict=True))[return_kind]
    calls = []
    hook = G.synthesis.vb4.register_forward_hook(lambda m, a, o: calls.append(a[2].shape[0]))
    try:
        with torch.no_grad(), cpu_multiview_ops():
            ws = G.mapping(torch.randn(2, G.z_dim, generator=torch.Generator().manual_seed(1)), cams[:1].repeat(2, 1))
            got = G.synthesis(ws, c=c, views=3, seed=seeds, **kw, **ret)
            assert calls == [2]
            want = [G.synthesis(ws[i // 3:i // 3 + 1], c=c[i:i + 1], seed=seeds[i], **kw, **ret) for i in range(6)]
    finally:
        hook.remove()
    flat = lambda o: [o[k] for k in sorted(o)] if isinstance(o, dict) else (list(o) if isinstance(o, (tuple, list)) else [o])
    got = flat(got)
    for k, g in enumerate(got):
        w = torch.cat([flat(o)[k] for o in want])
        assert g.shape == w.shape, (return_kind, k)
        assert (g - w).abs().max().item() <= 1e-5, (return_kind, k, (g - w).abs().max().item())


def test_views_argument_checks():
    G = _cli_generator()
    from oracle.images import cpu_multiview_ops
    ws = torch.zeros(2, G.num_ws, G.w_dim)
    with torch.no_grad(), cpu_multiview_ops():
        with pytest.raises(ValueError):
            G.synthesis(ws, c=torch.zeros(4, 25), views=3)
        with pytest.raises(ValueError):
            G.synthesis(ws, c=torch.zeros(2, 25), views=0)


@pytest.mark.parametrize('views', [1, 3])
def test_strip_oracle_matches_torchvision(views):
    """oracle/images.py (the torch restatement the kernel is checked against) equals torchvision's make_grid + save_image bytes, NaN
    pixel and out-of-range values included."""
    from oracle.images import compose_strips
    z = load_golden('image_strips')
    img, seg = torch.from_numpy(z[f'v{views}_img']), torch.from_numpy(z[f'v{views}_seg'])
    got_img, got_seg = compose_strips(img, seg, views)
    assert np.array_equal(got_img.numpy(), z[f'v{views}_out_img'])
    assert np.array_equal(got_seg.numpy(), z[f'v{views}_out_seg'])
    if views == 3:
        assert img.isnan().any() and (img.abs() > 1).any()
        assert got_img.shape == (2, 68, 3 * 66 + 2, 3) and (got_img[:, :2] == 0).all() and (got_img[:, :, 66:68] == 0).all()


def _mv_worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    from ide3d_b200 import dist as idist, images
    from oracle.images import cpu_multiview_ops
    r, w, dev = idist.init_from_env(backend='gloo')
    G = _cli_generator()
    seeds = [0, 1, 2, 3, 5]
    with cpu_multiview_ops():
        sharded = images.render_multiview(G, seeds, rank, world, psi=0.7, batch_seeds=2)
        single = images.render_multiview(G, seeds, 0, 1, psi=0.7, batch_seeds=3) if rank == 0 else None
    if rank == 0:
        diff = max(int(np.abs(a.astype(int) - b.astype(int)).max()) for a, b in zip(sharded, single))
        q.put((rank, sharded[0].shape, sharded[1].shape, diff, bool(np.array_equal(sharded[1], single[1]))))
    else:
        q.put((rank, None, None, 0 if sharded is None else 99, True))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_two_rank_gloo_multiview_driver(monkeypatch):
    """render_multiview sharded over two gloo ranks gives rank 0 the strips of the one-rank run (one uint8 level: the batch
    compositions differ, and so may the CPU convolution algorithms); the other rank gets None."""
    monkeypatch.setenv('CUDA_VISIBLE_DEVICES', '')
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 31500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_mv_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=240) for _ in procs], key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    (_, s_img, s_seg, diff, seg_equal), (_, _, _, other, _) = res
    assert tuple(s_img) == (5, 68, 3 * 66 + 2, 3) and tuple(s_seg) == tuple(s_img)
    assert diff <= 1 and seg_equal and other == 0, res


def test_render_multiview_writes_pngs(tmp_path):
    """The outdir form writes the reference's file names, and the PNGs hold the returned strips."""
    import PIL.Image
    from ide3d_b200 import images
    from oracle.images import cpu_multiview_ops
    G = _cli_generator()
    with cpu_multiview_ops():
        img, seg = images.render_multiview(G, [4, 7], yaws=(0.25, -0.25), outdir=str(tmp_path))
    assert img.shape == (2, 68, 2 * 66 + 2, 3) and img.dtype == np.uint8
    for k, s in enumerate([4, 7]):
        assert np.array_equal(np.asarray(PIL.Image.open(tmp_path / f'seed{s:04d}.png')), img[k])
        assert np.array_equal(np.asarray(PIL.Image.open(tmp_path / f'seed{s:04d}_seg.png')), seg[k])


def test_image_strips_rejects_bad_arguments(lib):
    from ide3d_b200 import _lib
    assert lib.ide3d_image_strips(None, None) == _lib.INVALID and b'null params' in lib.ide3d_last_error()
    p = _lib.StripsParams(seeds=1, views=9, height=8, width=8, seg_c=19, seg_h=4, seg_w=4)
    assert lib.ide3d_image_strips(ctypes.byref(p), None) == _lib.INVALID and b'bad sizes' in lib.ide3d_last_error()
    p.views = 3
    assert lib.ide3d_image_strips(ctypes.byref(p), None) == _lib.INVALID and b'null' in lib.ide3d_last_error()
    p.seeds = 0
    assert lib.ide3d_image_strips(ctypes.byref(p), None) == _lib.OK                  # empty: no-op


@pytest.mark.skipif(torch.cuda.is_available(), reason='passes fake device pointers: run only where no GPU can be reached')
@pytest.mark.parametrize('case', ['negative views', 'planes not frames / views', 'frames not a multiple of views'])
def test_raymarch_views_validation(lib, case):
    """views < 0 is rejected, and the frame count must be planes x views (message `batch mismatch`), in the forward and the backward."""
    from ide3d_b200 import _lib
    fake = 0x10000
    plane = lambda n: _lib.TriPlane(fake, n, 4, 4, 4 * 4 * 96, 1, 4 * 96, 96)
    p = _lib.RaymarchParams()
    p.tex, p.seg = plane(2), plane(2)
    p.dec.num_heads = 3
    for i, (in_sel, off, cnt) in enumerate([(0, 0, 32), (1, 32, 19), (1, 51, 1)]):
        p.dec.heads[i] = _lib.MlpHead(in_sel, 64, off, cnt, fake, fake, fake, fake)
    p.cam2world = p.out_feat = p.out_depth = fake
    p.n, p.res_w, p.res_h, p.num_steps, p.views = 6, 4, 4, 4, 3
    p.fov_deg, p.ray_start, p.ray_end, p.box_scale = 18.0, 2.25, 3.3, 2.0
    p.views, message = {'negative views': (-1, b'negative views'), 'planes not frames / views': (2, b'batch mismatch'),
                        'frames not a multiple of views': (4, b'batch mismatch')}[case]
    assert lib.ide3d_raymarch_fwd(ctypes.byref(p), None) == _lib.INVALID
    err = lib.ide3d_last_error()
    assert message in err
    f = ctypes.c_void_p(fake)
    assert lib.ide3d_raymarch_bwd(ctypes.byref(p), f, None, f, f, None, None) == _lib.INVALID and lib.ide3d_last_error() == err
