#!/usr/bin/env python
"""Generate tests/golden/cli_gen_videos_depth.npz: the reference's gen_videos.gen_interp_video in image_mode='image_depth', run
unmodified against this package on the CPU and recorded with the proxy of make_cli_golden.py (same generator, same trace encoding).

    IDE3D_REFERENCE=/path/to/IDE-3D PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_cli_depth_golden.py

A recipe of its own, so that recording it leaves the other cli_*.npz files untouched (rewriting them changes their zip timestamps).
"""

import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))


def _recipe():
    spec = importlib.util.spec_from_file_location('make_cli_golden', os.path.join(HERE, 'make_cli_golden.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def record_gen_videos_depth(cli, out):
    import gen_videos
    frames = []

    class _Writer:
        def append_data(self, a):
            frames.append(np.asarray(a))

        def close(self):
            pass

    sys.modules['imageio'].get_writer = lambda *a, **k: _Writer()
    # The script's image_depth branch keeps the batch-1 axis (the image_seg branch drops it with `[0]`, gen_videos.py:135), so
    # layout_grid receives [cells, 1, 3, H, W] and fails to unpack it.  Record the cells as the script built them and apply the
    # script's own layout_grid to them with that axis dropped.
    layout_grid, cells = gen_videos.layout_grid, []

    def layout_grid_cells(img, **kw):
        cells.append(img.clone())
        return layout_grid(img[:, 0] if img.ndim == 5 else img, **kw)

    gen_videos.layout_grid = layout_grid_cells
    events, arrays = [], cli.Arrays()
    G = cli.Proxy(cli.cli_generator(), '', events, arrays)
    torch.manual_seed(0)
    try:
        gen_videos.gen_interp_video(G, 'unused.mp4', seeds=[0, 1], w_frames=2, grid_dims=(1, 1), psi=0.7, truncation_cutoff=4,
                                    image_mode='image_depth', device=torch.device('cpu'))
    finally:
        gen_videos.layout_grid = layout_grid
    assert all(tuple(c.shape) == (1, 1, 3, 64, 64) for c in cells), [tuple(c.shape) for c in cells]
    cli.save_trace(out, events, arrays, frames=np.stack(frames), cells=torch.cat(cells)[:, 0].numpy())


def main():
    ref = os.environ.get('IDE3D_REFERENCE')
    if not ref or not os.path.isdir(ref):
        sys.exit('set IDE3D_REFERENCE to the reference IDE-3D tree')
    cli = _recipe()
    cli.setup_reference(ref)
    torch.set_num_threads(4)
    from oracle.backend import cpu_reference_ops
    with torch.no_grad(), cpu_reference_ops():
        record_gen_videos_depth(cli, os.path.join(HERE, 'cli_gen_videos_depth.npz'))


if __name__ == '__main__':
    main()
