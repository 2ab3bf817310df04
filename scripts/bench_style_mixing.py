"""Style-mixing grids: ide3d_b200.style_mixing.render_grid against the reference's structure run through this package.

    python scripts/bench_style_mixing.py [--rounds 3] [--cases geometry,split8,sr_rows,sr_rows_b36,yaws3]

Generator: compat.random_init_generator (the bench generator, 512^2).  Cases (seeds 0-7 by 8-15, psi 0.7, noise 'const'):
  geometry     styles 0-6, frontal view, batch_cells 16: no backbone block is shared (vb4 reads ws 0-1)
  split8       styles 8-17 (appearance), batch_cells 16: vb4-vb32 run once per row seed
  sr_rows      styles 14-17, batch_cells 16: the whole backbone runs once per row seed (one 9-cell grid row per call)
  sr_rows_b36  styles 14-17, batch_cells 36: four grid rows per call
  yaws3        styles 0-6, yaws -0.4, 0, 0.4: three canvases
Arms, alternated per round: `grid` = render_grid; `noshare` = render_grid with no backbone block shared (prefix_blocks -> 0), the
same calls otherwise; `loop` = apps/style_mixing.py's structure -- one batch-1 G.synthesis per cell and view, the reference's uint8
conversion, PIL's paste into the canvas.  All include the host copy of the canvases; none writes files.  Also timed:
ide3d_style_grid alone (CUDA events over 50 launches) on the 8 x 8 grid of 512^2 cells, with its bytes (cells read once, canvases
written once) over time against the 3.35 TB/s HBM3 data sheet figure.
Prints one JSON line per case and one for the kernel."""

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_PEAK = 3.35e12
CASES = {'geometry': ('0-6', (0.0,), 16), 'split8': ('8-17', (0.0,), 16), 'sr_rows': ('14-17', (0.0,), 16),
         'sr_rows_b36': ('14-17', (0.0,), 36), 'yaws3': ('0-6', (-0.4, 0.0, 0.4), 16)}


def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return out
    except Exception as e:                           # noqa: BLE001 -- the card's name is informational
        return f'unknown ({e})'


def loop_grid(G, rows, cols, styles, yaws):
    """apps/style_mixing.py:111-153 through this package: batch-1 synthesis per cell and view, conversion, PIL paste."""
    import PIL.Image
    from ide3d_b200 import images, style_mixing as sm
    dev = next(G.parameters()).device
    ws = sm.mix_ws(G, rows, cols, styles, psi=0.7)
    cams = images.view_cameras(yaws, dev)
    proc = lambda img: (img.permute(0, 2, 3, 1) * 127.5 + 128).clamp(0, 255).to(torch.uint8).cpu()
    image_dict = {}
    for key, w in zip(sm.cell_order(rows, cols), ws):
        seeds = images.view_seeds(key[0], len(yaws))
        image_dict[key] = [proc(G.synthesis(w[None], c=cams[j:j + 1], render_params=images.render_params(yaws[j]), noise_mode='const',
                                            seed=seeds[j]))[0].numpy() for j in range(len(yaws))]
    H = W = G.img_resolution
    canvases = []
    for step in range(len(yaws)):
        canvas = PIL.Image.new('RGB', (W * (len(cols) + 1), H * (len(rows) + 1)), 'black')
        for row_idx, row_seed in enumerate([0] + rows):
            for col_idx, col_seed in enumerate([0] + cols):
                if row_idx == 0 and col_idx == 0:
                    continue
                key = (col_seed, col_seed) if row_idx == 0 else (row_seed, row_seed) if col_idx == 0 else (row_seed, col_seed)
                canvas.paste(PIL.Image.fromarray(image_dict[key][step], 'RGB'), (W * col_idx, H * row_idx))
        canvases.append(np.asarray(canvas))
    return np.stack(canvases)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def kernel_time(views, res, R=8, C=8, iters=50):
    from ide3d_b200 import style_mixing as sm
    n = ((R + 1) * (C + 1) - 1) * views
    img = torch.randn(n, 3, res, res, device='cuda').contiguous(memory_format=torch.channels_last)
    for _ in range(3):
        sm.compose_grid(img, R, C, views)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        sm.compose_grid(img, R, C, views)
    b.record()
    b.synchronize()
    t = a.elapsed_time(b) / iters * 1e-3
    nbytes = n * 3 * res * res * 4 + views * (R + 1) * res * (C + 1) * res * 3
    return dict(views=views, grid=f'{R}x{C}', cell=res, us=round(t * 1e6, 1), bytes=nbytes, tb_s=round(nbytes / t / 1e12, 3),
                hbm_share=round(nbytes / t / HBM_PEAK, 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--cases', default=','.join(CASES))
    args = ap.parse_args()
    from ide3d_b200 import style_mixing as sm
    from ide3d_b200.compat import random_init_generator
    info = gpu_info()
    G = random_init_generator(device='cuda', seed=0)
    rows, cols = list(range(8)), list(range(8, 16))
    with torch.no_grad():
        for name in args.cases.split(','):
            styles, yaws, bc = CASES[name]
            st = sm.num_range(styles)
            grid = lambda: sm.render_grid(G, rows, cols, st, psi=0.7, yaws=yaws, batch_cells=bc)

            def noshare():
                G.synthesis.prefix_blocks = lambda _rows: 0
                try:
                    return grid()
                finally:
                    del G.synthesis.prefix_blocks

            arms = {'grid': grid, 'noshare': noshare, 'loop': lambda: loop_grid(G, rows, cols, st, yaws)}
            grid(), noshare(), loop_grid(G, rows[:1], cols[:2], st, yaws)          # warm-up: every shape the arms use
            times = {a: [] for a in arms}
            worst = {a: 0 for a in ('grid', 'noshare')}
            for _ in range(args.rounds):
                out = {}
                for a, fn in arms.items():
                    t, out[a] = timed(fn)
                    times[a].append(t)
                for a in worst:
                    worst[a] = max(worst[a], int(np.abs(out[a].astype(int) - out['loop'].astype(int)).max()))
            med = {a: float(np.median(v)) for a, v in times.items()}
            print(json.dumps(dict(case=name, styles=styles, yaws=list(yaws), batch_cells=bc, grid='8x8', cells=80,
                                  prefix_blocks=G.synthesis.prefix_blocks(st), **{f'{a}_s': [round(t, 3) for t in v] for a, v in times.items()},
                                  speedup_vs_loop=round(med['loop'] / med['grid'], 2), share_gain=round(med['noshare'] / med['grid'], 3),
                                  max_uint8_diff_vs_loop=worst, gpu=info)), flush=True)
        for views in (1, 3):
            print(json.dumps(dict(kernel='ide3d_style_grid', gpu=info, **kernel_time(views, G.img_resolution))), flush=True)


if __name__ == '__main__':
    main()
