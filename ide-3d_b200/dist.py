"""One process per GPU: shard independent work units, gather the results once.

The renderer has no exchange step (every frame is a pure function of its own (w, camera), every voxel of its own
coordinates), so there is no data-path collective: ranks take a strided share of the units -- the reference's own
idiom for metric evaluation, metrics/metric_utils.py:243 -- and a single all_gather (NCCL over NVLink on GPUs, gloo
in the CPU tests) brings the uint8 frames / sigma slabs together.  0.79 MB per 512^2 RGB frame: bandwidth-trivial.
"""

import os

import torch
import torch.distributed as dist

from . import video


def init_from_env(backend=None):
    """Initialise torch.distributed from torchrun's env (RANK / WORLD_SIZE / LOCAL_RANK / MASTER_*).
    Returns (rank, world, device)."""
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    use_cuda = torch.cuda.is_available()
    device = torch.device('cuda', local) if use_cuda else torch.device('cpu')
    if use_cuda:
        torch.cuda.set_device(device)
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
        os.environ.setdefault('MASTER_PORT', '29500')
        kw = dict(device_id=device) if use_cuda else {}
        dist.init_process_group(backend or ('nccl' if use_cuda else 'gloo'), rank=rank, world_size=world, **kw)
    return rank, world, device


def shard_indices(num_items, rank, world):
    """Strided share of range(num_items) for this rank (rank, rank+world, ...)."""
    return list(range(rank, num_items, world))


def slab_range(total, rank, world):
    """Contiguous [first, first+count) share of a flat voxel range (z-slab shard of the sigma grid)."""
    base, rem = divmod(total, world)
    first = rank * base + min(rank, rem)
    return first, base + (1 if rank < rem else 0)


def all_gather_padded(local, num_items, world):
    """Gather per-rank tensors produced for shard_indices(...) back into item order.
    local: [len(shard), ...] on this rank.  Returns [num_items, ...] on every rank."""
    if world == 1:
        return local
    per = (num_items + world - 1) // world
    pad = torch.zeros((per,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    pad[:local.shape[0]] = local
    out = torch.empty((world * per,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out, pad.contiguous())
    out = out.reshape((world, per) + tuple(local.shape[1:]))
    # item i lives at rank i % world, slot i // world
    idx = torch.arange(num_items, device=local.device)
    return out[idx % world, idx // world]


def all_gather_slabs(local, total, world):
    """Gather contiguous slabs (slab_range) into the flat [.., total] tensor (last dim is the sharded one)."""
    if world == 1:
        return local
    base, rem = divmod(total, world)
    per = base + (1 if rem else 0)
    pad = torch.zeros(tuple(local.shape[:-1]) + (per,), dtype=local.dtype, device=local.device)
    pad[..., :local.shape[-1]] = local
    out = torch.empty((world * pad.shape[0],) + tuple(pad.shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out, pad.contiguous())          # concatenation along dim 0 (gloo and nccl agree on this form)
    out = out.reshape((world,) + tuple(pad.shape))
    parts = [out[r][..., :base + (1 if r < rem else 0)] for r in range(world)]
    return torch.cat(parts, dim=-1)


@torch.no_grad()
def render_frames_sharded(G, ws, c, rank, world, batch=8, to_uint8=True, **synthesis_kwargs):
    """Render frames i = rank, rank+world, ... of (ws[i], c[i]) in batches and all-gather them in frame order.
    ws [F, num_ws, w_dim], c [F, 25] (host or device).  Returns uint8 [F, 3, H, W] (or float) on every rank."""
    F = ws.shape[0]
    mine = shard_indices(F, rank, world)
    dev = next(G.parameters()).device
    outs = []
    for i in range(0, len(mine), batch):
        sel = torch.as_tensor(mine[i:i + batch])
        img = G.synthesis(ws[sel].to(dev, non_blocking=True), c=c[sel].to(dev, non_blocking=True), **synthesis_kwargs)
        if isinstance(img, (tuple, list)):
            img = img[0]
        if to_uint8:
            img = (img * 127.5 + 128).clamp(0, 255).to(torch.uint8)
        outs.append(img)
    local = torch.cat(outs) if outs else torch.empty((0, G.img_channels, G.img_resolution, G.img_resolution),
                                                      dtype=torch.uint8 if to_uint8 else torch.float32, device=dev)
    return all_gather_padded(local, F, world)


_pinned = {}


def _pinned_buffer(shape, dtype):
    """Page-locked host buffer, cached per (shape, dtype): cudaHostAlloc costs milliseconds, a frame batch does not."""
    key = (tuple(shape), dtype)
    buf = _pinned.get(key)
    if buf is None:
        buf = _pinned[key] = torch.empty(shape, dtype=dtype, pin_memory=torch.cuda.is_available())
    return buf


_shared = {}


def _shm_free_bytes():
    try:
        st = os.statvfs('/dev/shm')
        return st.f_bavail * st.f_frsize
    except OSError:
        return 0


def _shared_frame_buffer(shape, rank, world, tag):
    """One uint8 frame buffer in /dev/shm that EVERY rank of the box maps (torch.from_file, shared) and page-locks
    (cudaHostRegister): each GPU then downloads its own frames straight into rank 0's result over its own PCIe link -- no
    collective, no second hop.  Cached per (shape, tag); rank 0 creates the file, one barrier makes it visible, and it is
    unlinked as soon as everybody has it mapped (the mapping keeps it alive)."""
    key = (tuple(shape), tag)
    buf = _shared.get(key)
    if buf is not None:
        return buf
    nbytes = 1
    for d in shape:
        nbytes *= int(d)
    path = f"/dev/shm/ide3d_b200_{os.environ.get('MASTER_PORT', '0')}_{os.getuid()}_{tag}_{nbytes}.bin"
    if rank == 0:
        with open(path, 'wb') as f:
            f.truncate(nbytes)
    dist.barrier()
    flat = torch.from_file(path, shared=True, size=nbytes, dtype=torch.uint8)
    if torch.cuda.is_available():
        rc = torch.cuda.cudart().cudaHostRegister(flat.data_ptr(), nbytes, 0)
        if int(rc) != 0:
            raise RuntimeError(f'ide3d_b200.dist: cudaHostRegister of the shared frame buffer failed ({rc})')
    dist.barrier()
    if rank == 0:
        os.unlink(path)
    buf = _shared[key] = flat.view(*shape)
    return buf


@torch.no_grad()
def stream_frames_sharded(G, ws, c, rank, world, batch=8, out=None, transport='auto', image_mode='image', **synthesis_kwargs):
    """The frame loop of gen_videos.py:127-139 as a pipeline: frames i = rank, rank+world, ... are rendered in batches and
    copied to page-locked HOST memory on a side stream while the next batch renders.  ws [F, num_ws, w_dim], c [F, 25] on
    the host (pinned for asynchronous uploads).  Returns uint8 [F, 3, H, k*W] on the host on rank 0, None elsewhere: image_mode
    (gen_videos.py:130-135) 'image' (k = 1), 'image_seg' (image | colourised semantic mask, k = 2) or 'image_depth' (the negated image
    min/max-normalised per frame, k = 1); the last two are composed by video.compose_frames from the render-resolution logits.
    F must be a multiple of world * batch.  The returned tensor is a cached buffer (pinned, or the shared one): it is valid until the
    next call with the same frame count -- consume or copy it before calling again (pass `out=` to get a private copy).

    transport (world > 1; how the frames of the other ranks reach rank 0's host memory):
      'shm'   every rank downloads its own frames into ONE shared, page-locked /dev/shm buffer (all ranks on one box): `world`
              PCIe links in parallel, ranks never wait for each other inside the loop, one barrier at the end.  Default on CUDA.
      'nccl'  one all_gather of the batch's uint8 frames per batch on the compute stream, rank 0 downloads everything (the
              round-1 path; also what the gloo CPU tests exercise, and the only choice across boxes)."""
    F = ws.shape[0]
    assert F % (world * batch) == 0, 'stream_frames_sharded: F must be a multiple of world * batch'
    if image_mode not in video.FRAME_WIDTH:
        raise ValueError(f'stream_frames_sharded: image_mode must be one of {sorted(video.FRAME_WIDTH)}, got {image_mode!r}')
    width = video.FRAME_WIDTH[image_mode] * G.img_resolution
    dev = next(G.parameters()).device

    def render(idx):
        w_b, c_b = ws[idx], c[idx]
        if image_mode == 'image_seg':
            img, seg_raw = G.synthesis(w_b.to(dev, non_blocking=True), c=c_b.to(dev, non_blocking=True), return_seg='raw', **synthesis_kwargs)
            return video.compose_frames(img, seg_raw, image_mode)
        img = G.synthesis(w_b.to(dev, non_blocking=True), c=c_b.to(dev, non_blocking=True), **synthesis_kwargs)
        if isinstance(img, (tuple, list)):
            img = img[0]
        if image_mode == 'image_depth':
            return video.compose_frames(img, None, image_mode)
        return (img * 127.5 + 128).clamp(0, 255).to(torch.uint8).contiguous()

    return stream_sharded(render, F, (G.img_channels, G.img_resolution, width), dev, rank, world, batch=batch, out=out,
                          transport=transport, tag='frames')


def stream_sharded(render, num_items, item_shape, dev, rank, world, batch=8, out=None, transport='auto', tag='frames'):
    """The pipeline of stream_frames_sharded for any per-item uint8 product: render(idx) -> uint8 [batch, *item_shape] on `dev` for the
    items idx (a slice when world == 1, else an index tensor) of this rank's share i = rank, rank+world, ...; the batches reach rank 0's
    host memory by `transport` while the next batch renders.  num_items must be a multiple of world * batch.  Returns uint8
    [num_items, *item_shape] on the host on rank 0 (a cached buffer, or `out`), None elsewhere.  `tag` names the shared buffer."""
    F = num_items
    assert F % (world * batch) == 0, 'stream_sharded: the item count must be a multiple of world * batch'
    cuda = dev.type == 'cuda'
    shape = (F,) + tuple(item_shape)
    if transport == 'auto':
        transport = 'shm' if (cuda and world > 1 and os.path.isdir('/dev/shm')) else 'nccl'
        if transport == 'shm':
            # the shared buffer must fit /dev/shm (containers often cap it): rank 0 looks, everybody follows its decision
            need = 1
            for d in shape:
                need *= int(d)
            ok = torch.zeros(1, dtype=torch.int32, device=dev)
            if rank == 0 and ((shape, tag) in _shared or _shm_free_bytes() > need + (64 << 20)):
                ok += 1
            dist.broadcast(ok, src=0)
            if int(ok.item()) == 0:
                transport = 'nccl'
    host = None
    if world > 1 and transport == 'shm':
        host = _shared_frame_buffer(shape, rank, world, tag)
    elif rank == 0:
        host = out if out is not None else _pinned_buffer(shape, torch.uint8)
    copy_stream = torch.cuda.Stream(dev) if cuda else None
    per_rank = F // world
    for b0 in range(0, per_rank, batch):
        if world == 1:
            idx = slice(b0, b0 + batch)                                      # views of the pinned inputs: asynchronous H2D
        else:
            idx = torch.arange(rank + world * b0, rank + world * (b0 + batch), world)
        img = render(idx)
        if world > 1 and transport == 'shm':
            # my items k of this batch are global items rank + world * (b0 + k): one asynchronous copy per item into the shared buffer
            if cuda:
                copy_stream.wait_stream(torch.cuda.current_stream(dev))
                with torch.cuda.stream(copy_stream):
                    for k in range(batch):
                        host[rank + world * (b0 + k)].copy_(img[k], non_blocking=True)
                img.record_stream(copy_stream)
            else:
                for k in range(batch):
                    host[rank + world * (b0 + k)].copy_(img[k])
            continue
        if world > 1:
            allf = torch.empty((world,) + tuple(img.shape), dtype=img.dtype, device=dev)
            dist.all_gather_into_tensor(allf.view((world * img.shape[0],) + tuple(img.shape[1:])), img)
            img = allf.transpose(0, 1).reshape((world * batch,) + tuple(img.shape[1:]))     # item order: j * world + r
        if rank == 0:
            lo = world * b0
            if cuda:
                copy_stream.wait_stream(torch.cuda.current_stream(dev))
                with torch.cuda.stream(copy_stream):
                    host[lo:lo + world * batch].copy_(img, non_blocking=True)
                img.record_stream(copy_stream)
            else:
                host[lo:lo + world * batch].copy_(img)
    if cuda:
        if copy_stream is not None:
            copy_stream.synchronize()
        torch.cuda.current_stream(dev).synchronize()
    if world > 1 and transport == 'shm':
        dist.barrier()                                   # every rank's items are in the shared buffer
        if rank != 0:
            return None
        if out is not None:
            out.copy_(host)
            return out
    return host


@torch.no_grad()
def sigma_grid_sharded(G, img_v, seg_v, rank, world, grid_n=256, cube_length=1.0, voxel_origin=(0, 0, 0)):
    """extract_shapes' density grid, flat voxel range split into contiguous z-slabs over the ranks, one all_gather."""
    total = grid_n ** 3
    first, count = slab_range(total, rank, world)
    local = G.synthesis.renderer.sigma_grid(img_v, seg_v, grid_n=grid_n, voxel_origin=voxel_origin,
                                            cube_length=cube_length, first=first, count=count)
    return all_gather_slabs(local, total, world)
