"""Create ZIP/PNG datasets: the reference's dataset_tool.py, with the Lanczos resize on the device and the semantic masks of the encoder's
real branch.

    python -m ide3d_b200.dataset_tool --source DIR|ZIP --dest DIR|ZIP [--max-images N] [--transform center-crop|center-crop-wide]
                                      [--resolution WxH] [--ext png|jpg] [--seg-dest DIR|ZIP --parser BISENET.pth] [--workers N]

The options, messages, errors and outputs are the reference's (dataset_tool.py:324-460): archive names 00000/img00000000.png, PNGs
stored with compress_level=0 (JPEG at quality 100, under the same .png names), a dataset.json of [archive_name, label] pairs, ZIP_STORED
archives or an empty folder.  Its quirks are kept:
  - a folder source keys labels by basename and drops an unlabeled image before numbering; a zip source keys them by archive name and
    drops nothing, so one missing label makes `labels` null;
  - --max-images counts the folder iterator's dropped images; a center-crop-wide image that is too small is dropped after numbering;
  - the checks (square, RGB or grayscale, power of two, equal attributes) run on the first image written, then on every later one.

Differences:
  - PIL.Image.resize(LANCZOS) runs as ide3d_resample_u8, bit for bit; decoding and encoding run in `--workers` processes, and the
    results are written in source order, so an error stops the tool at the image the reference stops at.  A CUDA device is required.
  - LSUN LMDB, CIFAR-10 and MNIST sources are refused: they are not portrait data.  Images must be 8-bit.
  - --seg-dest PATH --parser PATH (no reference script): for every image written, the 512 x 512 uint8 class-id mask of the reference's
    dnnlib/seg_tools.face_parsing (x / 127.5 - 1, bilinear resize to 512^2 with align_corners=True, BiSeNet, argmax, id_remap) as an
    L PNG under the same archive name, so that train_encoder.PortraitDataset(dest, seg_dest, resolution) reads the pairs.  The mask is
    taken from the pixels before encoding (for --ext jpg, before the JPEG coding).
"""

import collections
import io
import json
import multiprocessing
import os
import re
import sys
import zipfile
from pathlib import Path
from typing import Optional, Tuple

import click
import numpy as np
import PIL.Image
import torch
import torch.nn.functional as F
from tqdm import tqdm

from . import parsing
from .torch_utils.ops import resample as _resample

MASK_SIZE = 512
DEFAULT_BATCH = 8


def error(msg):
    print('Error: ' + msg)
    sys.exit(1)


def parse_tuple(s: str) -> Tuple[int, int]:
    m = re.match(r'^(\d+)[x,](\d+)$', s)
    if m:
        return (int(m.group(1)), int(m.group(2)))
    raise ValueError(f'cannot parse tuple {s}')


def maybe_min(a: int, b: Optional[int]) -> int:
    return min(a, b) if b is not None else a


def file_ext(name) -> str:
    return str(name).split('.')[-1]


def is_image_ext(fname) -> bool:
    return f'.{file_ext(fname).lower()}' in PIL.Image.EXTENSION


# --------------------------------------------------------------------------------------------------------------------------- sources
# A source is (max_idx, entries): the reference iterator's files in its order, each (file, label, dropped).  Nothing is decoded here.

def _read_labels(f):
    labels = json.load(f)['labels']
    return {x[0]: x[1] for x in labels} if labels is not None else {}


def open_image_folder(source_dir, *, max_images):
    input_images = [str(f) for f in sorted(Path(source_dir).rglob('*')) if is_image_ext(f) and os.path.isfile(f)]
    labels = {}
    meta_fname = os.path.join(source_dir, 'dataset.json')
    if os.path.isfile(meta_fname):
        with open(meta_fname, 'r') as file:
            labels = _read_labels(file)
        print("labels:\n", len(labels))
    max_idx = maybe_min(len(input_images), max_images)
    entries = []
    for idx, fname in enumerate(input_images):
        arch_fname = os.path.basename(os.path.relpath(fname, source_dir).replace('\\', '/'))
        if len(labels) > 0 and arch_fname not in labels:
            entries.append((fname, arch_fname, True))       # decoded, reported and dropped: no index, no --max-images check
            continue
        entries.append((fname, labels.get(arch_fname), False))
        if idx >= max_idx - 1:
            break
    return max_idx, ('folder', None), entries


def open_image_zip(source, *, max_images):
    with zipfile.ZipFile(source, mode='r') as z:
        input_images = [str(f) for f in sorted(z.namelist()) if is_image_ext(f)]
        labels = {}
        if 'dataset.json' in z.namelist():
            with z.open('dataset.json', 'r') as file:
                labels = _read_labels(file)
    max_idx = maybe_min(len(input_images), max_images)
    entries = [(fname, labels.get(fname), False) for fname in input_images[:max(max_idx, 1)]]
    return max_idx, ('zip', source), entries


def open_dataset(source, *, max_images):
    if os.path.isdir(source):
        if source.rstrip('/').endswith('_lmdb'):
            error(f'LSUN LMDB sources are not supported ({source}); convert the images to a folder or zip first')
        return open_image_folder(source, max_images=max_images)
    elif os.path.isfile(source):
        if os.path.basename(source) in ('cifar-10-python.tar.gz', 'train-images-idx3-ubyte.gz'):
            error(f'CIFAR-10 and MNIST sources are not supported ({source}); this tool prepares portrait image folders and zips')
        elif file_ext(source) == 'zip':
            return open_image_zip(source, max_images=max_images)
        else:
            assert False, 'unknown archive type'
    else:
        error(f'Missing input file or directory: {source}')


def open_dest(dest: str):
    if file_ext(dest) == 'zip':
        if os.path.dirname(dest) != '':
            os.makedirs(os.path.dirname(dest), exist_ok=True)
        zf = zipfile.ZipFile(file=dest, mode='w', compression=zipfile.ZIP_STORED)
        return '', zf.writestr, zf.close
    if os.path.isdir(dest) and len(os.listdir(dest)) != 0:
        error('--dest folder must be empty')
    os.makedirs(dest, exist_ok=True)

    def folder_write_bytes(fname, data):
        os.makedirs(os.path.dirname(fname), exist_ok=True)
        with open(fname, 'wb') as fout:
            fout.write(data.encode('utf8') if isinstance(data, str) else data)
    return dest, folder_write_bytes, lambda: None


# ------------------------------------------------------------------------------------------------------------------- worker processes
_zip_cache = {}


def _decode(kind, archive, fname):
    """np.array(PIL.Image.open(file)), as the reference's iterators decode."""
    if kind == 'folder':
        return np.array(PIL.Image.open(fname))
    z = _zip_cache.get(archive)
    if z is None:
        z = _zip_cache[archive] = zipfile.ZipFile(archive, mode='r')
    with z.open(fname, 'r') as file:
        return np.array(PIL.Image.open(file))


def _encode(img, mode, ext):
    image_bits = io.BytesIO()
    img = PIL.Image.fromarray(img, mode)
    if ext == 'png':
        img.save(image_bits, format='png', compress_level=0, optimize=False)
    else:
        img.save(image_bits, format='jpeg', quality=100)
    return image_bits.getvalue()


class _Done:
    def __init__(self, fn, args):
        try:
            self.value, self.exc = fn(*args), None
        except Exception as e:  # re-raised by get(), where the pool would raise it
            self.value, self.exc = None, e

    def get(self):
        if self.exc is not None:
            raise self.exc
        return self.value


class _InProcess:
    """The pool interface with no worker processes (--workers 0)."""

    def apply_async(self, fn, args):
        return _Done(fn, args)

    def terminate(self):
        pass


# --------------------------------------------------------------------------------------------------------------------------- transform
class _Plan:
    """What the reference's transform does with one image: drop it (out_shape None), keep it (resize None) or resize src (a view of the
    decoded image, or PIL's 'RGB' reading of it) to `resize` = (width, height), into a zeroed width x width canvas at row `row0` for
    center-crop-wide.  out_shape is the shape the reference's transform returns, which is all the attribute checks read."""

    def __init__(self, img, src=None, resize=None, out_shape=None, canvas=None, row0=0):
        self.img, self.src, self.resize, self.out_shape, self.canvas, self.row0 = img, src, resize, out_shape, canvas, row0
        self.pixels = None


def _as_rgb(img):
    """PIL.Image.fromarray(img, 'RGB') as the reference's crop transforms call it: an RGB view, or PIL's own reading and error."""
    if img.dtype == np.uint8 and img.ndim == 3 and img.shape[2] == 3:
        return img
    return np.array(PIL.Image.fromarray(img, 'RGB'))


def plan_transform(transform, width, height, img):
    if img.dtype != np.uint8:
        raise ValueError(f'dataset_tool: only 8-bit images are supported, got {img.dtype} pixels')
    h, w = img.shape[:2]
    if transform is None:                                   # scale()
        if width == w and height == h:
            return _Plan(img, out_shape=img.shape)
        ww, hh = (width if width is not None else w), (height if height is not None else h)
        shape = (hh, ww) + img.shape[2:]
        if img.ndim == 2 or img.shape[2] == 3:
            return _Plan(img, src=img, resize=(ww, hh), out_shape=shape)
        PIL.Image.fromarray(img)                            # raises where the reference raises
        return _Plan(img, out_shape=shape)                  # LA / RGBA: the channel check stops the tool before any pixel is used
    if transform == 'center-crop':
        crop = np.min(img.shape[:2])
        src = _as_rgb(img[(h - crop) // 2:(h + crop) // 2, (w - crop) // 2:(w + crop) // 2])
        return _Plan(img, src=src, resize=(width, height), out_shape=(height, width, 3))
    ch = int(np.round(width * h / w))                       # center-crop-wide
    if w < width or ch < height:
        return _Plan(img)
    src = _as_rgb(img[(h - ch) // 2:(h + ch) // 2])
    rows = range(width)[(width - height) // 2:(width + height) // 2]
    if len(rows) != height:                                 # the reference's canvas assignment fails: fail the same way
        np.zeros([width, width, 3], dtype=np.uint8)[(width - height) // 2:(width + height) // 2, :] = np.zeros([height, width, 3], np.uint8)
    return _Plan(img, src=src, resize=(width, height), out_shape=(width, width, 3), canvas=width, row0=rows.start)


def _device():
    if not torch.cuda.is_available():
        error('dataset_tool needs a CUDA device: the Lanczos resize runs only as the ide3d_resample_u8 kernel')
    return torch.device('cuda', torch.cuda.current_device())


def _run_device(plans, device, parser):
    """Resize every plan with a `resize` on the device, in runs of equal source shape; fill plan.pixels (numpy HWC uint8).  With a parser,
    returns the face_parsing mask of every plan's output pixels (uint8 [512, 512] each), else None."""
    pin = device.type == 'cuda'
    i = 0
    out_dev = []
    while i < len(plans):
        p = plans[i]
        j = i + 1
        if p.resize is not None:
            while (j < len(plans) and plans[j].resize == p.resize and plans[j].canvas == p.canvas and plans[j].src.shape == p.src.shape):
                j += 1
            n = j - i
            host = torch.empty((n,) + tuple(p.src.shape[:2]) + (p.src.shape[2] if p.src.ndim == 3 else 1,), dtype=torch.uint8,
                               pin_memory=pin)
            for k in range(n):
                host[k].numpy().reshape(plans[i + k].src.shape)[...] = plans[i + k].src
            src = host.to(device, non_blocking=True)
            ww, hh = p.resize
            if p.canvas is None:
                dst = torch.empty([n, hh, ww, src.shape[3]], dtype=torch.uint8, device=device)
                out = dst
            else:
                out = torch.zeros([n, p.canvas, p.canvas, 3], dtype=torch.uint8, device=device)
                dst = out[:, p.row0:p.row0 + hh]
            _resample.resample_u8(src, dst)
            res = out.cpu().numpy()
            for k in range(n):
                plans[i + k].pixels = res[k] if res.shape[3] == 3 else res[k, :, :, 0]
            out_dev.extend(out[k] for k in range(n))
        else:
            p.pixels = p.img
            out_dev.append(None)
        i = j
    if parser is None:
        return None
    imgs = torch.stack([o if o is not None else torch.from_numpy(np.ascontiguousarray(p.pixels)).to(device)
                        for o, p in zip(out_dev, plans)])
    return face_parsing_masks(parser, imgs).cpu().numpy()


@torch.no_grad()
def face_parsing_masks(parser, images):
    """dnnlib/seg_tools.face_parsing(x / 127.5 - 1, parser) of uint8 images [N, H, W, 3] as uint8 class ids [N, 512, 512] (id_remap
    applied).  The align_corners=True resize to 512^2 is skipped at 512^2, where it is the identity."""
    x = images.permute(0, 3, 1, 2).to(torch.float32) / 127.5 - 1
    if x.shape[-2:] != (MASK_SIZE, MASK_SIZE):
        x = F.interpolate(x, size=(MASK_SIZE, MASK_SIZE), mode='bilinear', align_corners=True)
    return parsing.parse(parser, x)


# ---------------------------------------------------------------------------------------------------------------------------- driver
def convert(source, dest, max_images=None, transform=None, resolution=None, ext='png', seg_dest=None, parser=None, workers=None,
            batch=None, fail=None):
    """The reference's convert_dataset body.  `fail(msg)` reports a usage error (click's ctx.fail on the command line)."""
    fail = fail or error
    if dest == '':
        fail('--dest output filename or directory must not be an empty string')
    if (seg_dest is None) != (parser is None):
        fail('--seg-dest and --parser must be given together')
    PIL.Image.init()
    workers = min(8, os.cpu_count() or 1) if workers is None else workers
    batch = batch or DEFAULT_BATCH
    # the workers only decode and encode: they never touch the device, so forking them is safe after CUDA is initialised
    pool = multiprocessing.get_context('fork').Pool(workers) if workers > 0 else _InProcess()
    try:
        _convert(pool, workers, source, dest, max_images, transform, resolution, ext, seg_dest, parser, batch)
    finally:
        pool.terminate()


def _convert(pool, workers, source, dest, max_images, transform, resolution, ext, seg_dest, parser, batch):
    num_files, (kind, archive), entries = open_dataset(source, max_images=max_images)
    archive_root_dir, save_bytes, close_dest = open_dest(dest)
    if seg_dest is not None:
        seg_root_dir, save_seg, close_seg = open_dest(seg_dest)
    if resolution is None:
        resolution = (None, None)
    width, height = resolution
    if transform is not None and (width is None or height is None):
        error('must specify --resolution=WxH when using ' + transform + ('transform' if transform == 'center-crop' else ' transform'))
    device = _device()
    net = parsing.BiSeNet.load(parser).to(device) if parser is not None else None

    window = max(2 * batch, 4 * workers)
    decodes = collections.deque()
    todo = iter(entries)

    def refill():
        while len(decodes) < window:
            e = next(todo, None)
            if e is None:
                return
            decodes.append((e, pool.apply_async(_decode, (kind, archive, e[0]))))

    writes = collections.deque()                            # (archive_fname, image bytes result, mask bytes result or None)

    def flush(keep):
        while len(writes) > keep:
            name, data, mask = writes.popleft()
            save_bytes(os.path.join(archive_root_dir, name), data.get())
            if mask is not None:
                save_seg(os.path.join(seg_root_dir, name), mask.get())

    dataset_attrs = None
    labels = []
    idx = 0
    progress = tqdm(total=num_files)
    refill()
    while decodes:
        # one batch: decode and plan in source order; stop at the first image whose transform or checks fail
        group, failure = [], None
        while decodes and len(group) < batch and failure is None:
            (fname, label, dropped), res = decodes.popleft()
            refill()
            try:
                img = res.get()
            except Exception as e:
                failure = e
                break
            if dropped:
                print("Label nout found:", label, None)
                continue
            idx_str = f'{idx:08d}'
            archive_fname = f'{idx_str[:5]}/img{idx_str}.png'
            idx += 1
            progress.update(1)
            try:
                plan = plan_transform(transform, width, height, img)
            except Exception as e:
                failure = e
                break
            if plan.out_shape is None:
                continue
            shape = plan.out_shape
            channels = shape[2] if len(shape) == 3 else 1
            cur_image_attrs = {'width': shape[1], 'height': shape[0], 'channels': channels}
            if dataset_attrs is None:
                dataset_attrs = cur_image_attrs
                w, h = dataset_attrs['width'], dataset_attrs['height']
                if w != h:
                    failure = f'Image dimensions after scale and crop are required to be square.  Got {w}x{h}'
                elif dataset_attrs['channels'] not in [1, 3]:
                    failure = 'Input images must be stored as RGB or grayscale'
                elif w != 2 ** int(np.floor(np.log2(w))):
                    failure = 'Image width/height after scale and crop are required to be power-of-two'
                elif net is not None and channels != 3:
                    failure = '--seg-dest needs RGB images: BiSeNet parses three channels'
            elif dataset_attrs != cur_image_attrs:
                err = [f'  dataset {k}/cur image {k}: {dataset_attrs[k]}/{cur_image_attrs[k]}' for k in dataset_attrs.keys()]
                failure = f'Image {archive_fname} attributes must be equal across all images of the dataset.  Got:\n' + '\n'.join(err)
            if failure is not None:
                break
            group.append((archive_fname, label, plan))
        if group:
            plans = [p for _, _, p in group]
            masks = _run_device(plans, device, net)
            for k, (archive_fname, label, plan) in enumerate(group):
                data = pool.apply_async(_encode, (plan.pixels, {1: 'L', 3: 'RGB'}[dataset_attrs['channels']], ext))
                mask = pool.apply_async(_encode, (masks[k], 'L', 'png')) if masks is not None else None
                writes.append((archive_fname, data, mask))
                labels.append([archive_fname, label] if label is not None else None)
            flush(window)
        if failure is not None:
            flush(0)
            progress.close()
            if isinstance(failure, str):
                error(failure)
            raise failure
    flush(0)
    progress.close()
    metadata = {'labels': labels if all(x is not None for x in labels) else None}
    save_bytes(os.path.join(archive_root_dir, 'dataset.json'), json.dumps(metadata))
    close_dest()
    if seg_dest is not None:
        close_seg()


@click.command()
@click.pass_context
@click.option('--source', help='Directory or archive name for input dataset', required=True, metavar='PATH')
@click.option('--dest', help='Output directory or archive name for output dataset', required=True, metavar='PATH')
@click.option('--max-images', help='Output only up to `max-images` images', type=int, default=None)
@click.option('--transform', help='Input crop/resize mode', type=click.Choice(['center-crop', 'center-crop-wide']))
@click.option('--resolution', help='Output resolution (e.g., \'512x512\')', metavar='WxH', type=parse_tuple)
@click.option('--ext', help='Output format', type=click.Choice(['png', 'jpg']), default="png")
@click.option('--seg-dest', help='Output directory or archive for the 512x512 semantic masks', metavar='PATH', default=None)
@click.option('--parser', help='BiSeNet state_dict for --seg-dest (e.g. segNet-20Class.pth)', metavar='PATH', default=None)
@click.option('--workers', help='Decode/encode worker processes  [default: min(8, CPUs)]', type=click.IntRange(min=0), default=None)
def convert_dataset(ctx, source, dest, max_images, transform, resolution, ext, seg_dest, parser, workers):
    """Convert an image folder or zip into a dataset archive usable with StyleGAN2 ADA PyTorch (the reference's dataset_tool.py).

    \b
    --source path/                      Recursively load all images from path/
    --source dataset.zip                Recursively load all images from dataset.zip
    --dest /path/to/dir                 Save output files under /path/to/dir
    --dest /path/to/dataset.zip         Save output files into /path/to/dataset.zip

    Images are stored as uncompressed PNG (or JPEG at quality 100 with --ext jpg), with the source's dataset.json labels carried over.
    Output images must be square with the same power-of-two size; --resolution resizes (Lanczos, bit-identical to PIL) and
    --transform=center-crop / center-crop-wide crop first.  --seg-dest with --parser also writes each image's 512x512 BiSeNet
    class-id mask under the same archive name.
    """
    convert(source, dest, max_images=max_images, transform=transform, resolution=resolution, ext=ext, seg_dest=seg_dest,
            parser=parser, workers=workers, fail=ctx.fail)


if __name__ == "__main__":
    convert_dataset()  # pylint: disable=no-value-for-parameter
