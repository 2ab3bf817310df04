"""render_mesh.py on the GPU: the shape saved by extract_shapes.py -> marching cubes -> a shaded turntable, one PNG per frame.

    python -m ide3d_b200.render_mesh --fname out/0.npy --outdir out [--size 256] [--sigma-threshold 10] [--w-frames 240]

The options are the reference script's (render_mesh.py:20-26).  Frames go to OUTDIR/<id>/<i:03d>.png, <id> being the file name up to
its first dot (the reference writes the same names under tmp/<id>/ and then encodes them into OUTDIR/render.mp4 with imageio; video
encoding stays outside this package, as in video.py).  Rendering details: ide3d_b200.mesh.render_turntable."""

import argparse
import os

import numpy as np
import torch


def main(argv=None):
    ap = argparse.ArgumentParser(description='Render the marching-cubes mesh of a density grid as turntable frames (GPU).')
    ap.add_argument('--fname', required=True, help='density grid .npy written by extract_shapes.py')
    ap.add_argument('--size', type=int, default=256, help='the mesh is divided by this (grid resolution)')
    ap.add_argument('--sigma-threshold', type=float, default=10.0, help='sigma threshold of marching cubes')
    ap.add_argument('--w-frames', type=int, default=240, help='number of frames')
    ap.add_argument('--outdir', required=True)
    ap.add_argument('--batch', type=int, default=8, help='frames rasterised per call')
    args = ap.parse_args(argv)

    from PIL import Image

    from . import mesh
    grid = torch.from_numpy(np.ascontiguousarray(np.load(args.fname), dtype=np.float32)).cuda()
    frames = mesh.render_turntable(grid, size=args.size, sigma_threshold=args.sigma_threshold, w_frames=args.w_frames, batch=args.batch)
    ident = os.path.basename(args.fname).split('.')[0]
    out = os.path.join(args.outdir, ident)
    os.makedirs(out, exist_ok=True)
    for i, frame in enumerate(frames.cpu().numpy()):
        Image.fromarray(frame).save(os.path.join(out, f'{i:03d}.png'))
    print(f'{len(frames)} frames -> {out}')
    return out


if __name__ == '__main__':
    main()
