"""Style-mixing grids of a tri-plane generator: apps/style_mixing.py, batched and sharded.

The reference draws z = RandomState(seed).randn(z_dim) for every distinct seed, maps them in one call, truncates about w_avg
(style_mixing.py:89-95), then renders one cell per (row seed, column seed): the row seed's ws with the rows `col_styles` taken from
the column seed (:111-120), one batch-1 synthesis per cell, and pastes the uint8 images into a canvas with a black top-left cell,
the column seeds along the top and the row seeds down the left (:139-153).  With more than one frame per cell (STEP > 1) it writes
one canvas per frame.

Here:
  * mix_ws returns every cell's ws in canvas order (`cell_order`); render_grid renders them in batches of `batch_cells` with
    `views=len(yaws)` (up to 8 per call; one backbone pass per cell, the renderer and the super-resolution blocks per yaw, as
    images.render_multiview) and composes each batch's canvas rows in one launch (ide3d_style_grid).  Grid rows are the work units
    sharded over the ranks through dist.stream_sharded.
  * The backbone blocks that read no mixed ws row (SynthesisNetwork.prefix_blocks) give the same activations for a row seed's
    un-mixed cell and all its mixed cells; they run once per row seed (SynthesisNetwork shared_prefix).  Mixing only rows 14-17 (read
    by the super-resolution blocks alone) shares the whole backbone; row 13 is the last backbone block's ToRGB row as well.
  * Style rows outside [0, num_ws) are dropped, as viz/renderer.py:331 does; the reference script would raise an IndexError.

Deviations from the reference:
  * Conditioning label: the reference maps with c=None (style_mixing.py:92).  This generator's mapping is camera-conditioned, so
    the label is the frontal camera gen_images.py maps with (images.FRONTAL), unless `c` is given.
  * Cameras: the reference's StyleNeRF Renderer picks its own poses.  Here every cell is rendered from the yaws `yaws` (default
    the frontal view) with gen_images.py's cameras; view j of every cell uses the j-th jitter seed the gen_images loop would draw
    for the cell's row seed (images.view_seeds), so reruns are bit-identical.  mp4 encoding stays outside: several views give
    one PNG per view.
  * Generators come through the Python API or a local state_dict file; network pickles are refused, as in avg_spectra.py.
"""

import os
import re
import time
from typing import List

import click
import numpy as np
import torch

from . import _lib as L
from . import images

#----------------------------------------------------------------------------


def num_range(s: str) -> List[int]:
    '''Accept either a comma separated list of numbers 'a,b,c' or a range 'a-c' and return as a list of ints.'''
    m = re.match(r'^(\d+)-(\d+)$', s)
    if m:
        return list(range(int(m.group(1)), int(m.group(2)) + 1))
    return [int(x) for x in s.split(',')]


def valid_styles(col_styles, num_ws):
    """The style rows viz/renderer.py:331 keeps: those inside [0, num_ws), in the given order."""
    return [int(i) for i in col_styles if 0 <= int(i) < num_ws]


def cell_order(row_seeds, col_seeds):
    """(row seed, column seed) of every cell in canvas order: the column seeds' un-mixed cells (the top row after the black cell),
    then per row seed its un-mixed cell followed by its mixed cells.  Cell k fills grid slot k + 1 of the (R+1) x (C+1) grid."""
    cells = [(c, c) for c in col_seeds]
    for r in row_seeds:
        cells += [(r, r)] + [(r, c) for c in col_seeds]
    return cells


@torch.no_grad()
def mix_ws(G, row_seeds, col_seeds, col_styles, psi=1, c=None):
    """ws [(R+1)(C+1) - 1, num_ws, w_dim] of every cell in canvas order (cell_order), as style_mixing.py:89-114 forms them: one
    RandomState(seed).randn(z_dim) per distinct seed, one mapping call with label `c` (default: the frontal label, see the module
    docstring), w = w_avg + (w - w_avg) * psi, then a mixed cell is its row seed's w with the rows col_styles from its column seed."""
    row_seeds, col_seeds = [int(s) for s in row_seeds], [int(s) for s in col_seeds]
    if not row_seeds or not col_seeds:
        raise ValueError('mix_ws: need at least one row seed and one column seed')
    dev = G.mapping.w_avg.device
    all_seeds = list(set(row_seeds + col_seeds))
    all_z = np.stack([np.random.RandomState(seed).randn(G.z_dim) for seed in all_seeds])
    if c is None:
        c = torch.tensor(images.FRONTAL).float().reshape(1, -1)
    c = torch.as_tensor(c).float().reshape(-1, G.c_dim).to(dev)
    all_w = G.mapping(torch.from_numpy(all_z).to(dev), c.expand(len(all_seeds), -1) if c.shape[0] == 1 else c)
    w_avg = G.mapping.w_avg
    all_w = w_avg + (all_w - w_avg) * psi
    w_dict = {seed: w for seed, w in zip(all_seeds, list(all_w))}
    styles = valid_styles(col_styles, all_w.shape[1])
    out = []
    for r, col in cell_order(row_seeds, col_seeds):
        w = w_dict[r].clone()
        w[styles] = w_dict[col][styles]                 # a no-op for the un-mixed cells (r == col)
        out.append(w)
    return torch.stack(out)


#----------------------------------------------------------------------------


def canvas_shape(rows, cols, height, width):
    """(Hc, Wc) of the grid canvas for `rows` row seeds and `cols` column seeds."""
    return (rows + 1) * height, (cols + 1) * width


def _style_grid(img, first_row, rows, cols, views, out, out_stride_row, out_stride_view):
    L.require_cuda(img, out)
    L.forbid_grad('style_mixing.compose_grid', img)
    if img.dtype != torch.float32 or img.ndim != 4 or img.shape[1] != 3:
        raise RuntimeError(f'ide3d_b200.style_mixing.compose_grid: img must be float32 [cells * views, 3, H, W], got {img.dtype} '
                           f'{tuple(img.shape)}')
    need = (rows * (cols + 1) - (1 if first_row == 0 else 0)) * views
    if img.shape[0] != need:
        raise RuntimeError(f'ide3d_b200.style_mixing.compose_grid: {rows} grid rows of {cols} + 1 columns from row {first_row} with '
                           f'{views} views need {need} images, got {img.shape[0]}')
    h, w = img.shape[2:]
    sn, sc, sh, sw = img.stride()
    L.check(L.get_lib().ide3d_style_grid(img.data_ptr(), first_row, rows, cols, views, h, w, sn, sc, sh, sw, out.data_ptr(),
                                         out_stride_row, out_stride_view, L.stream_ptr(img.device)))
    return out


def compose_grid(img, rows, cols, views=1):
    """The grid canvases of style_mixing.py:100-153 in one launch (ide3d_style_grid).  img float32 [cells * views, 3, H, W], any
    strides, the (rows+1)(cols+1) - 1 cells in canvas order (cell_order), cell-major (row k * views + v is view v of cell k).
    -> uint8 [views, (rows+1) H, (cols+1) W, 3], one canvas per view.  CUDA tensors only."""
    views = int(views)
    if rows < 1 or cols < 1 or views < 1:
        raise ValueError(f'ide3d_b200.style_mixing.compose_grid: need rows, cols, views >= 1, got {rows}, {cols}, {views}')
    h, w = img.shape[-2:]
    hc, wc = canvas_shape(rows, cols, h, w)
    out = torch.empty([views, hc, wc, 3], dtype=torch.uint8, device=img.device)
    return _style_grid(img, 0, rows + 1, cols, views, out, h * wc * 3, hc * wc * 3)


@torch.no_grad()
def render_grid(G, row_seeds, col_seeds, col_styles, psi=1, noise_mode='const', yaws=(0,), rank=0, world=1, batch_cells=16, c=None):
    """style_mixing.py's grid as one batched, sharded call.  -> uint8 numpy [len(yaws), Hc, Wc, 3] on rank 0 (None on the other
    ranks), one canvas per yaw, (Hc, Wc) = canvas_shape(R, C, G.img_resolution, G.img_resolution).

    Cells are mix_ws's.  Grid rows are distributed over the ranks (dist.stream_sharded; the row list is padded to a multiple of
    world x rows-per-batch with repeats of the last row, rendered and dropped); each batch renders its cells in synthesis calls of at
    most batch_cells cells and images.MAX_VIEWS yaws (any number of yaws), the cells of one row seed sharing the backbone blocks before the first mixed row,
    and composes its canvas rows in one ide3d_style_grid launch.  noise_mode 'const' or 'none' gives what a batch-1 loop over the
    cells gives up to the batch size's effect on the convolution algorithms; 'random' draws noise per call."""
    from . import dist as idist
    row_seeds, col_seeds = [int(s) for s in row_seeds], [int(s) for s in col_seeds]
    V = len(yaws)
    if V < 1:
        raise ValueError('render_grid: need at least one yaw')
    # at most images.MAX_VIEWS views per synthesis call: more yaws run in several calls, each with its own backbone pass
    chunks = [slice(j, min(j + images.MAX_VIEWS, V)) for j in range(0, V, images.MAX_VIEWS)]
    R, Cn = len(row_seeds), len(col_seeds)
    dev = next(G.parameters()).device
    ws = mix_ws(G, row_seeds, col_seeds, col_styles, psi=psi, c=c)
    styles = valid_styles(col_styles, G.num_ws)
    k = G.synthesis.prefix_blocks(styles)
    cams = images.view_cameras(yaws, dev)
    rp = images.render_params(yaws[0])
    cells = cell_order(row_seeds, col_seeds)
    jitter = torch.tensor([images.view_seeds(r, V) for r, _ in cells], dtype=torch.int64)
    H = W = G.img_resolution
    wc = (Cn + 1) * W

    def row_cells(g):
        """Cell indices of grid row g, and their prefix groups: a row seed's cells share one, a column header is its own."""
        if g == 0:
            return list(range(Cn)), [-1 - j for j in range(Cn)]
        first = g * (Cn + 1) - 1
        return list(range(first, first + Cn + 1)), [g] * (Cn + 1)

    grid_rows = R + 1
    batch = max(1, min(int(batch_cells) // (Cn + 1), -(-grid_rows // world)))
    total = -(-grid_rows // (world * batch)) * world * batch
    padded = list(range(grid_rows)) + [grid_rows - 1] * (total - grid_rows)

    step = max(1, int(batch_cells))

    def render(idx):
        rows = [padded[i] for i in (range(idx.start, idx.stop) if isinstance(idx, slice) else idx.tolist())]
        sel, groups, spans = [], [], []
        for g in rows:
            s, gr = row_cells(g)
            spans.append((len(sel), len(sel) + len(s)))
            sel += s
            groups += [(g, x) for x in gr]
        imgs = []
        for i in range(0, len(sel), step):
            part = sel[i:i + step]
            grp = groups[i:i + step]
            ids = {key: n for n, key in enumerate(dict.fromkeys(grp))}
            per = []
            for ch in chunks:
                vc = ch.stop - ch.start
                img = G.synthesis(ws[part], c=cams[ch].repeat(len(part), 1), render_params=rp, noise_mode=noise_mode, views=vc,
                                  seed=jitter[part][:, ch].reshape(-1), shared_prefix=(k, [ids[key] for key in grp]))
                per.append(img.reshape(len(part), vc, *img.shape[1:]))
            imgs.append((per[0] if len(per) == 1 else torch.cat(per, 1)).flatten(0, 1))     # cell-major, views inner
        img = imgs[0] if len(imgs) == 1 else torch.cat(imgs)
        out = torch.empty([len(rows), V, H, wc, 3], dtype=torch.uint8, device=dev)
        # each run of consecutive grid rows is composed in one launch (the padding repeats the last row)
        a = 0
        for b in range(1, len(rows) + 1):
            if b == len(rows) or rows[b] != rows[b - 1] + 1:
                _style_grid(img[spans[a][0] * V:spans[b - 1][1] * V], rows[a], b - a, Cn, V, out[a:b], V * H * wc * 3, H * wc * 3)
                a = b
        return out

    host = idist.stream_sharded(render, total, (V, H, wc, 3), dev, rank, world, batch=batch, tag='style_grid')
    if host is None:
        return None
    rows_out = host[:grid_rows].numpy()                                # [R+1, V, H, Wc, 3]; the host buffer is reused by the next call
    return np.ascontiguousarray(rows_out.transpose(1, 0, 2, 3, 4)).reshape(V, grid_rows * H, wc, 3)


#----------------------------------------------------------------------------


def load_generator(network, device):
    """A TriPlaneGenerator from a local state_dict file (torch.save(G.state_dict())); network pickles are refused."""
    if network.lower().endswith('.pkl'):
        raise click.ClickException('--network: network pickles are not loaded here; pass a local state_dict file, or the generator '
                                   'module to ide3d_b200.style_mixing.render_grid (Python API)')
    from .compat import random_init_generator
    G = random_init_generator(device='cpu')
    G.load_state_dict(torch.load(network, map_location='cpu', weights_only=True))
    return G.to(device)


def save_grid(canvases, outdir, name='grid'):
    """Write the canvases as style_mixing.py:155-164 does: grid_<timestamp>.png for one view, else <outdir>/<name>_<timestamp>/NNNN.png
    (the reference's mp4 is left to an encoder of the user's choice).  -> the written paths."""
    import PIL.Image
    os.makedirs(outdir, exist_ok=True)
    timestamp = time.strftime('%Y%m%d.%H%M%S', time.localtime(time.time()))
    if len(canvases) == 1:
        paths = [os.path.join(outdir, f'grid_{timestamp}.png')]
    else:
        outdir = os.path.join(outdir, f'{name}_{timestamp}')
        os.makedirs(outdir, exist_ok=True)
        paths = [os.path.join(outdir, f'{step:04d}.png') for step in range(len(canvases))]
    for img, path in zip(canvases, paths):
        PIL.Image.fromarray(np.asarray(img), 'RGB').save(path)
    return paths


@click.command()
@click.option('--network', 'network', help='Generator state_dict file (network pickles are refused)', required=True)
@click.option('--rows', 'row_seeds', type=num_range, help='Random seeds to use for image rows', required=True)
@click.option('--cols', 'col_seeds', type=num_range, help='Random seeds to use for image columns', required=True)
@click.option('--styles', 'col_styles', type=num_range, help='Style layer range', default='0-6', show_default=True)
@click.option('--trunc', 'truncation_psi', type=float, help='Truncation psi', default=1, show_default=True)
@click.option('--noise-mode', help='Noise mode', type=click.Choice(['const', 'random', 'none']), default='const', show_default=True)
@click.option('--outdir', type=str, required=True)
@click.option('--yaws', type=str, help='Comma-separated camera yaws, one canvas per yaw (any number; up to 8 share one backbone pass)',
              default='0', show_default=True)
@click.option('--batch-cells', type=click.IntRange(min=1), help='Cells per synthesis call', default=16, show_default=True)
def main(network, row_seeds, col_seeds, col_styles, truncation_psi, noise_mode, outdir, yaws, batch_cells):
    """Generate a style-mixing grid of a tri-plane generator.

    \b
    python -m ide3d_b200.style_mixing --network=G.pt --outdir=out --rows=85,100,75,458,1500 --cols=55,821,1789,293 --styles=0-6
    """
    if network.lower().endswith('.pkl'):
        load_generator(network, 'cpu')                  # refuses before any device work
    from . import dist as idist
    rank, world, device = idist.init_from_env()
    G = load_generator(network, device)
    yaw_list = tuple(float(y) for y in yaws.split(','))
    canvases = render_grid(G, row_seeds, col_seeds, col_styles, psi=truncation_psi, noise_mode=noise_mode, yaws=yaw_list, rank=rank,
                           world=world, batch_cells=batch_cells)
    if rank == 0:
        name = os.path.basename(network).split('.')[0]
        for path in save_grid(canvases, outdir, name=name):
            print(path)


if __name__ == '__main__':
    main()  # pylint: disable=no-value-for-parameter
