"""CPU: the style-mixing grid (ide3d_b200.style_mixing, apps/style_mixing.py batched).

  * mix_ws, num_range and the canvas order against the reference's own lines (tests/golden/style_mixing.npz)
  * the canvas contract of ide3d_style_grid (oracle/style_mixing.py) against the numpy port of the PIL paste loop, and that port
    against PIL
  * prefix_blocks, and SynthesisNetwork(shared_prefix=...) against the plain call through the CPU oracle
  * the command line refuses network pickles; a world-2 gloo run of render_grid against the world-1 run"""

import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import GOLDEN, ROOT, load_golden

CASES = ['overlap', 'single_row', 'single_col', 'out_of_range', 'psi']


def _cli_generator():
    sys.path.insert(0, GOLDEN)
    try:
        import make_cli_golden
    finally:
        sys.path.remove(GOLDEN)
    return make_cli_golden.cli_generator()


@pytest.mark.parametrize('case', CASES)
def test_mix_ws_matches_reference_lines(case):
    """Every cell's ws, in canvas order, equals what the reference's lines build from the same stand-in mapping, bit for bit."""
    from ide3d_b200 import style_mixing as sm
    from oracle.style_mixing import stand_in_generator
    z = load_golden('style_mixing')
    rows, cols = z[f'{case}/rows'].tolist(), z[f'{case}/cols'].tolist()
    styles = sm.num_range(str(z[f'{case}/styles_arg']))
    got = sm.mix_ws(stand_in_generator(seed=0), rows, cols, styles, psi=float(z[f'{case}/psi']))
    assert got.dtype == torch.float32 and np.array_equal(got.numpy(), z[f'{case}/ws'])
    assert sm.valid_styles(styles, 18) == z[f'{case}/styles_kept'].tolist()
    assert [list(c) for c in sm.cell_order(rows, cols)] == z[f'{case}/order'].tolist()


def test_num_range_matches_reference():
    from ide3d_b200 import style_mixing as sm
    z = load_golden('style_mixing')
    for key in z:
        if key.startswith('num_range/'):
            assert sm.num_range(key.split('/', 1)[1]) == z[key].tolist(), key


@pytest.mark.parametrize('views', [1, 3])
@pytest.mark.parametrize('rows,cols', [(1, 1), (3, 1), (1, 3), (3, 8)])
def test_grid_contract_matches_paste_loop(rows, cols, views):
    """The kernel's contract (cells in canvas order, any window of grid rows, any output strides) lays out what the reference's paste
    loop lays out: whole canvases, and the grid rows of a window written into a row-major buffer."""
    from ide3d_b200 import style_mixing as sm
    from oracle.style_mixing import paste_grid, style_grid, to_uint8
    H, W = 5, 7
    row_seeds, col_seeds = [10 + r for r in range(rows)], [20 + c for c in range(cols)]
    order = sm.cell_order(row_seeds, col_seeds)
    g = torch.Generator().manual_seed(rows * 10 + cols)
    img = torch.randn(len(order) * views, 3, H, W, generator=g) * 1.5
    img[0, 0, 0, 0] = float('nan')
    u8 = to_uint8(img).reshape(len(order), views, H, W, 3)
    image_dict = {key: u8[k].permute(1, 2, 3, 0).numpy() if views > 1 else u8[k, 0].numpy() for k, key in enumerate(order)}
    want = np.stack(paste_grid(image_dict, row_seeds, col_seeds, H, W))
    hc, wc = sm.canvas_shape(rows, cols, H, W)
    out = torch.full((views, hc, wc, 3), 7, dtype=torch.uint8)
    style_grid(img.contiguous(memory_format=torch.channels_last), 0, rows + 1, cols, views, out, H * wc * 3, hc * wc * 3)
    assert np.array_equal(out.numpy(), want)
    # grid rows 1 .. rows as a window into [rows, V, H, Wc, 3]
    part = torch.full((rows, views, H, wc, 3), 7, dtype=torch.uint8)
    style_grid(img[cols * views:], 1, rows, cols, views, part, views * H * wc * 3, H * wc * 3)
    assert np.array_equal(part.permute(1, 0, 2, 3, 4).reshape(views, rows * H, wc, 3).numpy(), want[:, H:])


def test_paste_port_matches_pil():
    import PIL.Image
    from oracle.style_mixing import paste_grid
    H, W, rows, cols = 4, 6, [3, 1], [2, 5, 8]
    rnd = np.random.RandomState(0)
    keys = [(c, c) for c in cols] + [(r, r) for r in rows] + [(r, c) for r in rows for c in cols]
    image_dict = {k: rnd.randint(0, 256, (H, W, 3)).astype(np.uint8) for k in keys}
    canvas = PIL.Image.new('RGB', (W * (len(cols) + 1), H * (len(rows) + 1)), 'black')
    for row_idx, row_seed in enumerate([0] + rows):
        for col_idx, col_seed in enumerate([0] + cols):
            if row_idx == 0 and col_idx == 0:
                continue
            key = (col_seed, col_seed) if row_idx == 0 else (row_seed, row_seed) if col_idx == 0 else (row_seed, col_seed)
            canvas.paste(PIL.Image.fromarray(image_dict[key], 'RGB'), (W * col_idx, H * row_idx))
    assert np.array_equal(paste_grid(image_dict, rows, cols, H, W)[0], np.asarray(canvas))


def test_prefix_blocks_follow_split_ws():
    """Backbone blocks of the released layout: vb4 reads ws 0-1, vb8 1-3, vb16 3-5, ..., vb256 11-13; the super-resolution blocks 13-17."""
    from ide3d_b200.training.triplane import SynthesisNetwork
    net = SynthesisNetwork(w_dim=8, img_resolution=64, plane_resolution=256, channel_base=2048, channel_max=8, sr_channels=(8, 8))
    assert net.num_ws == 18
    assert net.prefix_blocks(range(0, 7)) == 0
    assert net.prefix_blocks([2]) == 1
    assert net.prefix_blocks([8, 9]) == 4
    assert net.prefix_blocks([13]) == 6
    assert net.prefix_blocks(range(14, 18)) == 7
    assert net.prefix_blocks([]) == 7


def test_shared_prefix_matches_plain_call_on_the_oracle():
    """Through the CPU oracle: for every prefix length, shared_prefix gives the plain call's images (within CPU convolution
    batch effects), with and without views; groups that share nothing give the plain call exactly."""
    from oracle.images import cpu_multiview_ops
    from ide3d_b200 import images
    G = _cli_generator()
    syn = G.synthesis
    g = torch.Generator().manual_seed(3)
    rows = torch.randn(2, G.num_ws, G.w_dim, generator=g)
    ws = rows.repeat_interleave(3, 0)
    ws[1::3, 4:] = torch.randn(2, G.num_ws - 4, G.w_dim, generator=g)
    groups = [0, 0, 0, 1, 1, 1]
    for views in (1, 2):
        c = images.view_cameras((0, 0.3)[:views]).repeat(6, 1)
        kw = dict(c=c, views=views, seed=list(range(6 * views)), noise_mode='const')
        with torch.no_grad(), cpu_multiview_ops():
            want = syn(ws, **kw)
            for k in range(syn.prefix_blocks(range(4, G.num_ws)) + 1):
                got = syn(ws, shared_prefix=(k, groups), **kw)
                assert (got - want).abs().max().item() <= 1e-5, (views, k)
            assert torch.equal(syn(ws, shared_prefix=(2, list(range(6))), **kw), want)
            with pytest.raises(ValueError):
                syn(ws, shared_prefix=(len(syn.voxel_block_resolutions) + 1, groups), **kw)


def test_render_grid_renders_more_yaws_than_one_call_takes(monkeypatch):
    """Nine yaws run as calls of eight and one views; the first eight canvases are those of the eight-yaw grid (the same calls, the
    same per-view jitter seeds), and every canvas differs from its neighbour."""
    from ide3d_b200 import style_mixing as sm
    from oracle.images import cpu_multiview_ops
    from oracle.style_mixing import style_grid
    monkeypatch.setattr(sm, '_style_grid', style_grid)
    G = _cli_generator()
    yaws = tuple(-0.4 + 0.1 * j for j in range(9))
    with cpu_multiview_ops():
        nine = sm.render_grid(G, [1], [2], [5, 6], yaws=yaws, batch_cells=3)
        eight = sm.render_grid(G, [1], [2], [5, 6], yaws=yaws[:8], batch_cells=3)
    assert nine.shape == (9, 128, 128, 3)
    assert np.abs(nine[:8].astype(int) - eight.astype(int)).max() <= 1
    assert all((nine[j] != nine[j + 1]).any() for j in range(8))


def test_cli_refuses_network_pickles(tmp_path):
    from click.testing import CliRunner
    from ide3d_b200 import style_mixing as sm
    res = CliRunner().invoke(sm.main, ['--network', str(tmp_path / 'G.pkl'), '--rows', '1,2', '--cols', '3', '--outdir', str(tmp_path)])
    assert res.exit_code != 0 and 'pickles are not loaded' in res.output
    assert not any(tmp_path.iterdir())


def _grid_worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    from ide3d_b200 import dist as idist, style_mixing as sm
    from oracle.images import cpu_multiview_ops
    from oracle.style_mixing import style_grid
    idist.init_from_env(backend='gloo')
    G = _cli_generator()
    rendered = []
    synthesis = G.synthesis.forward

    def recording(ws, **kw):
        rendered.append(ws.clone())
        return synthesis(ws, **kw)

    G.synthesis.forward = recording
    sm._style_grid = style_grid
    args = ([1, 2, 3], [4, 1], [5, 6, 7], 0.7)
    with cpu_multiview_ops():
        sharded = sm.render_grid(G, *args, yaws=(0, 0.4), rank=rank, world=world, batch_cells=3)
        mine = torch.cat(rendered)
        single = sm.render_grid(G, *args, yaws=(0, 0.4), batch_cells=5) if rank == 0 else None
        want_ws = sm.mix_ws(G, *args)
    everyone = [None] * world
    dist.all_gather_object(everyone, mine)
    if rank == 0:
        got_ws = torch.cat(everyone)
        # every cell's ws was rendered by some rank (the padding repeats the last grid row), and nothing else was
        covered = all(any(torch.equal(w, r) for r in got_ws) for w in want_ws)
        foreign = sum(not any(torch.equal(r, w) for w in want_ws) for r in got_ws)
        diff = int(np.abs(sharded.astype(int) - single.astype(int)).max())
        q.put((rank, sharded.shape, diff, covered and foreign == 0))
    else:
        q.put((rank, None, 0 if sharded is None else 99, True))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_two_rank_gloo_render_grid(monkeypatch):
    """render_grid over two gloo ranks: rank 0 gets the one-rank canvases (one uint8 level: other batch compositions may pick
    other CPU convolution algorithms), the ranks together rendered exactly mix_ws's cells, and the other rank gets None."""
    monkeypatch.setenv('CUDA_VISIBLE_DEVICES', '')
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 33500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_grid_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=240) for _ in procs], key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    (_, shape, diff, cells_ok), (_, _, other, _) = res
    assert tuple(shape) == (2, 4 * 64, 3 * 64, 3)
    assert diff <= 1 and cells_ok and other == 0, res
