#!/usr/bin/env python
"""BASELINE config 3: gen_videos.py grid=2x2, seeds 0-255, interpolated (w_frames=120 -> 7680 video frames x 4 cells = 30720 renders),
pose-batch shard over the ranks of one box (ide3d_b200.video / dist.stream_frames_sharded).  One process per GPU:

    python scripts/bench_video.py [--seeds 256] [--w-frames 120] [--chunk 1024]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29511 scripts/bench_video.py

The (w, camera) list of the whole video is computed up front exactly as gen_videos.py:66-140 does per frame (video.interp_video_inputs);
the renders are streamed in chunks (bounded host memory: the consumer -- the video writer -- takes frames in order).  Reports the host
input preparation separately from the render wall time (barrier + synchronize on both sides, max over ranks).  Rank 0 prints one JSON line."""
import argparse, json, os, sys, time
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--seeds', type=int, default=256)
    ap.add_argument('--w-frames', type=int, default=120)
    ap.add_argument('--chunk', type=int, default=1024, help='renders per streamed chunk (multiple of world * batch)')
    ap.add_argument('--batch', type=int, default=8)
    ap.add_argument('--image-mode', default='image', choices=['image', 'image_seg', 'image_depth'], help='gen_videos.py --image_mode')
    args = ap.parse_args()
    from ide3d_b200 import dist as idist, video
    from ide3d_b200.torch_utils import custom_ops
    from ide3d_b200.compat import random_init_generator
    import torch.distributed as tdist
    custom_ops.verbosity = 'none'
    rank, world, device = idist.init_from_env()
    torch.backends.cudnn.benchmark = True
    G = random_init_generator(device=device, seed=0)

    def barrier():
        if world > 1:
            tdist.barrier()
        torch.cuda.synchronize()

    t0 = time.perf_counter()
    with torch.no_grad():
        ws, c, (F, gh, gw) = video.interp_video_inputs(G, list(range(args.seeds)), w_frames=args.w_frames, grid_dims=(2, 2))
    ws, c = ws.to(torch.float32).pin_memory(), c.cpu().pin_memory()
    prep_s = time.perf_counter() - t0
    total = ws.shape[0]
    chunk = max(world * args.batch, args.chunk // (world * args.batch) * (world * args.batch))
    kw = dict(noise_mode='const', image_mode=args.image_mode)
    with torch.no_grad():
        idist.stream_frames_sharded(G, ws[:chunk], c[:chunk], rank, world, batch=args.batch, **kw)     # warm-up: cuDNN plans, buffers
        barrier()
        t0 = time.perf_counter()
        done, checksum = 0, 0
        while done < total:
            n = min(chunk, total - done)
            n -= n % (world * args.batch)
            if n == 0:
                break
            frames = idist.stream_frames_sharded(G, ws[done:done + n], c[done:done + n], rank, world, batch=args.batch, **kw)
            if rank == 0:
                checksum += int(frames[::97, :, ::64, ::64].sum())          # the consumer touches the frames (stand-in for the video writer)
            done += n
        barrier()
        render_s = time.perf_counter() - t0
    t = torch.tensor([render_s], dtype=torch.float64, device=device)
    if world > 1:
        tdist.all_reduce(t, op=tdist.ReduceOp.MAX)
    if rank == 0:
        print(json.dumps({'config': f'gen_videos grid=2x2 seeds=0-{args.seeds - 1} w_frames={args.w_frames} (BASELINE configs[2])', 'image_mode': args.image_mode, 'n_gpus': world,
                          'video_frames': F, 'renders': done, 'renders_per_s': done / float(t[0]), 'video_frames_per_s': done / 4 / float(t[0]),
                          'render_wall_s': float(t[0]), 'host_input_prep_s (scipy splines + mapping, per rank, untimed)': prep_s,
                          'chunk_renders': chunk, 'batch': args.batch, 'transport': 'shared page-locked /dev/shm buffer, each rank downloads its own frames' if world > 1 else 'pinned host buffer',
                          'frames_checksum': checksum}))
    if world > 1:
        tdist.barrier()
        tdist.destroy_process_group()


if __name__ == '__main__':
    main()
