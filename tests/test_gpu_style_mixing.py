"""GPU: the style-mixing grid (ide3d_b200.style_mixing).

  * ide3d_style_grid against the reference's PIL paste loop (oracle/style_mixing.py) over torch-converted cells, bit for bit
  * SynthesisNetwork(shared_prefix=...): the per-latent blocks fed the repeated prefix activations are the plain call bit for bit, and
    the whole shared render is within one uint8 level of the plain one
  * render_grid against the reference's structure run through this package (one batch-1 synthesis per cell, then the paste loop), and
    reruns bit-identical"""

import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')


def _cells(n, h, w, layout, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(n, 3, h, w, generator=g) * 1.2).to(DEV)
    x[0, 1, 2, 3] = float('nan')
    if layout == 'channels_last':
        return x.contiguous(memory_format=torch.channels_last)
    if layout == 'strided':                          # a channel and column window of a wider tensor
        big = torch.randn(n, 5, h, w + 6, device=DEV)
        big[:, 1:4, :, 2:2 + w] = x
        return big[:, 1:4, :, 2:2 + w]
    return x


@pytest.mark.parametrize('layout', ['nchw', 'channels_last', 'strided'])
@pytest.mark.parametrize('views', [1, 3])
@pytest.mark.parametrize('rows,cols', [(1, 1), (1, 8), (3, 3), (8, 1), (8, 8)])
def test_grid_kernel_matches_paste_loop(rows, cols, views, layout):
    from ide3d_b200 import style_mixing as sm
    from oracle.style_mixing import paste_grid, to_uint8
    H, W = 24, 20
    row_seeds, col_seeds = list(range(100, 100 + rows)), list(range(200, 200 + cols))
    order = sm.cell_order(row_seeds, col_seeds)
    img = _cells(len(order) * views, H, W, layout, rows * 31 + cols)
    u8 = to_uint8(img).reshape(len(order), views, H, W, 3).cpu()
    image_dict = {key: u8[k].permute(1, 2, 3, 0).numpy() if views > 1 else u8[k, 0].numpy() for k, key in enumerate(order)}
    want = np.stack(paste_grid(image_dict, row_seeds, col_seeds, H, W))
    got = sm.compose_grid(img, rows, cols, views)
    assert got.shape == want.shape and got.dtype == torch.uint8
    assert np.array_equal(got.cpu().numpy(), want)


def test_grid_kernel_full_size_window():
    """512^2 cells, an 8 x 8 grid written as grid rows 3..5 into a row-major buffer: the same bytes as the whole canvas."""
    from ide3d_b200 import style_mixing as sm
    R, C, V = 8, 8, 1
    img = _cells(((R + 1) * (C + 1) - 1) * V, 512, 512, 'channels_last', 5)
    full = sm.compose_grid(img, R, C, V)
    wc = (C + 1) * 512
    part = torch.empty(3, V, 512, wc, 3, dtype=torch.uint8, device=DEV)
    first = 3 * (C + 1) - 1
    sm._style_grid(img[first:first + 3 * (C + 1)], 3, 3, C, V, part, V * 512 * wc * 3, 512 * wc * 3)
    assert torch.equal(part.reshape(3 * 512, wc, 3), full[0, 3 * 512:6 * 512])


def test_grid_kernel_refuses_bad_arguments(lib):
    from ide3d_b200 import _lib
    fake = ctypes.c_void_p(0x10000)
    bad = [((fake, 0, 1, 0, 1, 4, 4, 48, 16, 4, 1, fake, 0, 0), b'bad sizes'),
           ((fake, -1, 1, 1, 1, 4, 4, 48, 16, 4, 1, fake, 0, 0), b'bad sizes'),
           ((fake, 0, 1, 1, 0, 4, 4, 48, 16, 4, 1, fake, 0, 0), b'bad sizes'),
           ((fake, 0, 1, 1, 1, 0, 4, 48, 16, 4, 1, fake, 0, 0), b'bad sizes'),
           ((fake, 0, 1, 1 << 20, 1, 4, 1024, 48, 16, 4, 1, fake, 0, 0), b'canvas too large'),
           ((None, 0, 1, 1, 1, 4, 4, 48, 16, 4, 1, fake, 0, 0), b'null cells or output'),
           ((fake, 0, 1, 1, 1, 4, 4, 48, 16, 4, 1, None, 0, 0), b'null cells or output')]
    for args, msg in bad:
        assert lib.ide3d_style_grid(*args, None) == _lib.INVALID, args
        assert msg in lib.ide3d_last_error(), (args, lib.ide3d_last_error())
    assert lib.ide3d_style_grid(None, 0, 0, 1, 1, 4, 4, 48, 16, 4, 1, None, 0, 0, None) == _lib.OK          # no rows: a no-op
    with pytest.raises(RuntimeError, match='need'):
        from ide3d_b200 import style_mixing as sm
        sm.compose_grid(torch.zeros(5, 3, 4, 4, device=DEV), 2, 2)


@pytest.fixture(scope='module')
def bench_G():
    from ide3d_b200.compat import random_init_generator
    return random_init_generator(device=DEV, seed=0)


def _hooked_run(syn, ws, kw, k, inject=None):
    """syn(ws, **kw) with a hook at the entry of backbone block k (the renderer when k is the whole backbone) that records its
    activation inputs, or replaces them with `inject`."""
    blocks = [getattr(syn, f'vb{r}') for r in syn.voxel_block_resolutions]
    target = blocks[k] if k < len(blocks) else syn.renderer
    seen = {}

    def hook(mod, args, kwargs):
        if k < len(blocks):
            if inject is not None:
                return (inject['x'], inject['img'], args[2]) + args[3:], dict(kwargs, condition_img=inject['seg'])
            seen.update(x=args[0], img=args[1], seg=kwargs['condition_img'])
        else:
            if inject is not None:
                return (inject['img'], inject['seg']) + args[2:], kwargs
            seen.update(img=args[0], seg=args[1])
        return None

    h = target.register_forward_pre_hook(hook, with_kwargs=True)
    try:
        out = syn(ws, **kw)
    finally:
        h.remove()
    return out, seen


@pytest.mark.parametrize('views', [1, 3])
@pytest.mark.parametrize('mixed', [(0, 18), (8, 18), (14, 18)])
def test_shared_prefix_against_plain_call(bench_G, mixed, views):
    """The cells of a 2 x 2 grid (mix_ws, psi 0.7) whose ws differ from row `mixed[0]` on: prefix lengths 0, 4 (vb4-vb32) and 7 (the
    whole backbone).  The activations entering block k (the renderer for k = 7) are, gathered per cell, those of the plain call on
    the groups' first latents alone, bit for bit; the per-latent part fed them is the shared call bit for bit.  So the shared render is
    the plain call's arithmetic with the prefix at another batch size, and end to end it stays within one uint8 level of the plain
    call at the cells' batch size; groups that share nothing are the plain call."""
    from ide3d_b200 import images, style_mixing as sm
    from oracle.style_mixing import to_uint8
    G = bench_G
    syn = G.synthesis
    k = syn.prefix_blocks(range(*mixed))
    assert k == {0: 0, 8: 4, 14: 7}[mixed[0]]
    rows, cols = [3, 1], [1, 5]
    ws = sm.mix_ws(G, rows, cols, range(*mixed), psi=0.7)
    groups = [0, 1] + [2 + g for g in range(len(rows)) for _ in range(len(cols) + 1)]        # the column headers share nothing
    first = [0, 1, 2, 2 + len(cols) + 1]
    inverse = torch.tensor(groups, device=DEV)
    n = ws.shape[0]
    yaws = (-0.3, 0, 0.3)[:views] if views > 1 else (0,)
    cams = images.view_cameras(yaws, DEV)
    kw = dict(render_params=images.render_params(0), views=views, noise_mode='const')
    per = lambda idx: dict(kw, c=cams.repeat(len(idx), 1), seed=[j for i in idx for j in range(i * views, (i + 1) * views)])
    with torch.no_grad():
        plain = syn(ws, **per(range(n)))
        shared, acts = _hooked_run(syn, ws, dict(per(range(n)), shared_prefix=(k, groups)), k)
        _, prefix = _hooked_run(syn, ws[first], per(first), k)
        fed, _ = _hooked_run(syn, ws, per(range(n)), k, inject=acts)
        nothing = syn(ws, shared_prefix=(k, list(range(n))), **per(range(n)))
    for name, t in acts.items():
        assert t is None or torch.equal(t, prefix[name].index_select(0, inverse)), name
    assert torch.equal(fed, shared)
    assert torch.equal(nothing, plain)
    worst = int((to_uint8(shared).int() - to_uint8(plain).int()).abs().max())
    print(f'k={k} views={views}: shared vs plain {worst} uint8 levels, max |diff| {(shared - plain).abs().max().item():.2e}')
    assert worst <= 1
    if k == 0:
        assert torch.equal(shared, plain)


def _loop_grid(G, row_seeds, col_seeds, col_styles, psi, yaws):
    """style_mixing.py's structure through this package: one batch-1 synthesis per cell, the reference's conversion, the paste loop."""
    from ide3d_b200 import images, style_mixing as sm
    from oracle.style_mixing import paste_grid, to_uint8
    ws = sm.mix_ws(G, row_seeds, col_seeds, col_styles, psi=psi)
    cams = images.view_cameras(yaws, DEV)
    image_dict = {}
    for key, w in zip(sm.cell_order(row_seeds, col_seeds), ws):
        seeds = images.view_seeds(key[0], len(yaws))
        views = [to_uint8(G.synthesis(w[None], c=cams[j:j + 1], render_params=images.render_params(yaws[j]), noise_mode='const',
                                      seed=seeds[j]))[0].cpu().numpy() for j in range(len(yaws))]
        image_dict[key] = views[0] if len(yaws) == 1 else np.stack(views, -1)
    return np.stack(paste_grid(image_dict, row_seeds, col_seeds, G.img_resolution, G.img_resolution))


@pytest.mark.parametrize('styles,yaws', [('0-6', (0,)), ('8-17', (0,)), ('14-17', (-0.4, 0, 0.4))])
def test_render_grid_matches_batch1_loop(bench_G, styles, yaws):
    from ide3d_b200 import style_mixing as sm
    rows, cols = [3, 1, 4], [1, 5]
    with torch.no_grad():
        want = _loop_grid(bench_G, rows, cols, sm.num_range(styles), 0.7, yaws)
        got = sm.render_grid(bench_G, rows, cols, sm.num_range(styles), psi=0.7, yaws=yaws, batch_cells=6)
        again = sm.render_grid(bench_G, rows, cols, sm.num_range(styles), psi=0.7, yaws=yaws, batch_cells=6)
    assert got.shape == want.shape == (len(yaws), 4 * 512, 3 * 512, 3)
    worst = int(np.abs(got.astype(int) - want.astype(int)).max())
    print(f'styles {styles}, {len(yaws)} yaws: render_grid vs batch-1 loop {worst} uint8 levels, '
          f'{int((got != want).any(-1).sum())} pixels differ')
    assert worst <= 1
    assert np.array_equal(got, again)
