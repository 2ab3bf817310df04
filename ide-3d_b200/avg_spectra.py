"""Compare average power spectra between real and generated images, or between multiple generators (the reference's avg_spectra.py).

    python -m ide3d_b200.avg_spectra stats   --source=DATASET [--num=INT] [--seed=INT]
    python -m ide3d_b200.avg_spectra calc    --source=DATASET --dest=NPZ --mean=FLOAT --std=FLOAT [--num --seed --beta --interp]
    python -m ide3d_b200.avg_spectra heatmap NPZ [--save --dpi --smooth]
    python -m ide3d_b200.avg_spectra slices  NPZ... [--save --dpi --smooth]

The commands, options, defaults, messages and the .npz (`spectrum` float64 [P, P] in unshifted bin order, `image_size`) are the
reference's, so files written by either tool plot with the other.  Differences:

- The hot paths are sm_90a kernels (torch_utils/ops/spectra.py): `calc` accumulates with a pruned float64 FFT of the non-zero N x N
  block and never builds the zero-padded P x P plane; `stats` sums x and x^2 as exact 64-bit integers, where the reference's float64
  sums start rounding above 2^53.  Images arrive in batches, as uint8, through a pinned non-blocking copy.
- A network pickle on the command line is refused: checkpoint pickles are not loaded by this package.  The Python API takes a
  generator module instead: stream_source_images(G, num, seed, device).
- Generated image idx draws from RandomState(seed + idx): z = randn(1, z_dim), then the label.  The reference's label is a random
  one-hot, which for this generator's 25-value camera label is a degenerate pose with zero intrinsics.  Here, with c_dim == 25 the label
  is `labels.get_label(randint(len(labels)))` when a labelled dataset is given and the frontal conditioning camera otherwise; c_dim == 0
  gives an empty label; any other c_dim keeps the reference's one-hot.  Images are rendered `batch` at a time.
- heatmap / slices: the plotted arrays come from construct_heatmap and slice_curves; matplotlib is imported only to draw.
"""

import os

import click
import numpy as np
import scipy.ndimage
import torch

from . import dnnlib
from .torch_utils.ops import spectra as ops

# The frontal conditioning camera of the reference's generation scripts (cam2world of a camera at radius 2.7 on +z, then the
# normalised intrinsics).
FRONTAL_CAMERA = [1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 2.7, 0, 0, 0, 1, 4.2647, 0, 0.5, 0, 4.2647, 0.5, 0, 0, 1]

#----------------------------------------------------------------------------
# Generator draws.


def generator_draw(z_dim, c_dim, seed, labels=None):
    """(z float64 [1, z_dim], c float32 [1, c_dim]) of the image with RandomState seed `seed` (the reference passes seed + idx)."""
    rnd = np.random.RandomState(seed)
    z = rnd.randn(1, z_dim)
    c = np.zeros([1, c_dim], dtype=np.float32)
    if c_dim == 25:
        c[0] = labels.get_label(rnd.randint(len(labels))) if labels is not None else FRONTAL_CAMERA
    elif c_dim > 0:
        c[:, rnd.randint(c_dim)] = 1
    return z, c


def _generator_stream(G, num, seed, device, batch, labels):
    def render(first, count):
        draws = [generator_draw(G.z_dim, G.c_dim, first + i, labels) for i in range(count)]
        z = torch.from_numpy(np.concatenate([d[0] for d in draws])).to(device)
        c = torch.from_numpy(np.concatenate([d[1] for d in draws])).to(device)
        with torch.no_grad():
            return (G(z=z, c=c) * 127.5 + 128).clamp(0, 255).to(torch.uint8)

    _ = render(seed, min(batch, num))  # warm up
    return (render(seed + i, min(batch, num - i)) for i in range(0, num, batch))

#----------------------------------------------------------------------------
# Setup an iterator for streaming images, in uint8 NCHW format, based on the
# respective command line options.


def stream_source_images(source, num, seed, device, data_loader_kwargs=None, batch=32, labels=None):  # => num_images, image_size, image_iter
    """image_iter yields uint8 [B, C, N, N] batches on `device`, in image order.  `source` is a dataset zip or directory, or (Python
    API) a generator module with z_dim, c_dim, img_resolution and G(z=, c=) -> [B, C, N, N] in [-1, 1]."""
    if isinstance(source, torch.nn.Module):
        if num is None:
            raise click.ClickException('--num is required when --source points to network pickle')
        return num, source.img_resolution, _generator_stream(source, num, seed, device, batch, labels)

    ext = source.split('.')[-1].lower()
    if data_loader_kwargs is None:
        data_loader_kwargs = dict(pin_memory=True, num_workers=3, prefetch_factor=2)

    if ext == 'pkl':
        raise click.ClickException('--source: network pickles are not loaded here; pass the generator module to '
                                   'ide3d_b200.avg_spectra.stream_source_images (Python API) instead')

    elif ext == 'zip' or os.path.isdir(source):
        from .training import dataset
        dataset_obj = dataset.ImageFolderDataset(path=source, max_size=num, random_seed=seed)
        if num is not None and num != len(dataset_obj):
            raise click.ClickException(f'--source contains fewer than {num} images')
        num_images, resolution = len(dataset_obj), dataset_obj.resolution
        dataset_obj.close()  # forked loader workers must not share the parent's open zip file; each opens its own
        data_loader = torch.utils.data.DataLoader(dataset_obj, batch_size=batch, **data_loader_kwargs)
        image_iter = (image.to(device, non_blocking=True) for image, _label in data_loader)
        return num_images, resolution, image_iter

    else:
        raise click.ClickException('--source must point to network pickle, dataset zip, or directory')

#----------------------------------------------------------------------------
# The two accumulations, as functions of an image stream.


def compute_stats(image_iter, device):
    """(mean, std) of a uint8 image stream from exact integer moments."""
    moments = torch.zeros([3], dtype=torch.int64, device=device)
    for images in image_iter:
        ops.image_moments(images, moments)
    return ops.mean_std(moments.cpu().numpy().view(np.uint64))


def compute_spectrum(image_iter, image_size, mean, std, beta, interp, device):
    """float64 [P, P] average power spectrum of a uint8 image stream (P = image_size * interp)."""
    acc = None
    for images in image_iter:
        if acc is None:
            acc = ops.Spectrum(image_size, images.shape[1], mean, std, beta=beta, interp=interp, device=device)
        acc.add(images)
    return acc.result()


def save_spectrum(dest, spectrum, image_size):
    if os.path.dirname(dest):
        os.makedirs(os.path.dirname(dest), exist_ok=True)
    np.savez(dest, spectrum=np.asarray(spectrum, dtype=np.float64), image_size=image_size)

#----------------------------------------------------------------------------
# Load average power spectrum from the specified .npz file and construct
# the corresponding heatmap for visualization.


def construct_heatmap(npz_file, smooth):
    npz_data = np.load(npz_file)
    spectrum = npz_data['spectrum']
    image_size = npz_data['image_size']
    hmap = np.log10(spectrum) * 10  # dB
    hmap = np.fft.fftshift(hmap)
    hmap = np.concatenate([hmap, hmap[:1, :]], axis=0)
    hmap = np.concatenate([hmap, hmap[:, :1]], axis=1)
    if smooth > 0:
        sigma = spectrum.shape[0] / image_size * smooth
        hmap = scipy.ndimage.gaussian_filter(hmap, sigma=sigma, mode='nearest')
    return hmap, image_size


def slice_curves(hmap, image_size):
    """The 0 and 45 degree slices `slices` plots: dict(freqs0, slice0, freqs45, slice45)."""
    hmap_size = hmap.shape[0]
    hmap_center = hmap_size // 2
    hmap_range = np.arange(hmap_center, hmap_size)
    return dict(freqs0=np.linspace(0, image_size / 2, num=(hmap_size // 2 + 1), endpoint=True),
                slice0=hmap[hmap_center, hmap_range],
                freqs45=np.linspace(0, image_size / np.sqrt(2), num=(hmap_size // 2 + 1), endpoint=True),
                slice45=hmap[hmap_range, hmap_range])


def _set_spawn():
    if torch.multiprocessing.get_start_method(allow_none=True) is None:
        torch.multiprocessing.set_start_method('spawn')


def _show_or_save(plt, save):
    if save is None:
        plt.show()
    else:
        if os.path.dirname(save):
            os.makedirs(os.path.dirname(save), exist_ok=True)
        plt.savefig(save)

#----------------------------------------------------------------------------


@click.group()
def main():
    """Compare average power spectra between real and generated images,
    or between multiple generators.

    Example:

    \b
    # Calculate dataset mean and std, needed in subsequent steps.
    python -m ide3d_b200.avg_spectra stats --source=~/datasets/ffhq-512x512.zip

    \b
    # Calculate average spectrum for the training data.
    python -m ide3d_b200.avg_spectra calc --source=~/datasets/ffhq-512x512.zip \\
        --dest=tmp/training-data.npz --mean=112.684 --std=69.509

    \b
    # Display results.
    python -m ide3d_b200.avg_spectra heatmap tmp/training-data.npz
    python -m ide3d_b200.avg_spectra slices tmp/training-data.npz tmp/generator.npz

    \b
    # Save as PNG.
    python -m ide3d_b200.avg_spectra heatmap tmp/training-data.npz --save=tmp/training-data.png --dpi=300
    python -m ide3d_b200.avg_spectra slices tmp/training-data.npz tmp/generator.npz --save=tmp/slices.png --dpi=300
    """

#----------------------------------------------------------------------------


@main.command()
@click.option('--source', help='Network pkl, dataset zip, or directory', metavar='[PKL|ZIP|DIR]', required=True)
@click.option('--num', help='Number of images to process  [default: all]', metavar='INT', type=click.IntRange(min=1))
@click.option('--seed', help='Random seed for selecting the images', metavar='INT', type=click.IntRange(min=0), default=0, show_default=True)
def stats(source, num, seed, device=torch.device('cuda')):
    """Calculate dataset mean and standard deviation needed by 'calc'."""
    _set_spawn()
    _num_images, _image_size, image_iter = stream_source_images(source=source, num=num, seed=seed, device=device)
    mean, std = compute_stats(image_iter, device)
    print(f'--mean={mean:g} --std={std:g}')
    return mean, std

#----------------------------------------------------------------------------


@main.command()
@click.option('--source', help='Network pkl, dataset zip, or directory', metavar='[PKL|ZIP|DIR]', required=True)
@click.option('--dest', help='Where to store the result', metavar='NPZ', required=True)
@click.option('--mean', help='Dataset mean for whitening', metavar='FLOAT', type=float, required=True)
@click.option('--std', help='Dataset standard deviation for whitening', metavar='FLOAT', type=click.FloatRange(min=0), required=True)
@click.option('--num', help='Number of images to process  [default: all]', metavar='INT', type=click.IntRange(min=1))
@click.option('--seed', help='Random seed for selecting the images', metavar='INT', type=click.IntRange(min=0), default=0, show_default=True)
@click.option('--beta', help='Shape parameter for the Kaiser window', metavar='FLOAT', type=click.FloatRange(min=0), default=8, show_default=True)
@click.option('--interp', help='Frequency-domain interpolation factor', metavar='INT', type=click.IntRange(min=1), default=4, show_default=True)
def calc(source, dest, mean, std, num, seed, beta, interp, device=torch.device('cuda')):
    """Calculate average power spectrum and store it in .npz file."""
    _set_spawn()
    _num_images, image_size, image_iter = stream_source_images(source=source, num=num, seed=seed, device=device)
    spectrum = compute_spectrum(image_iter, image_size, mean, std, beta, interp, device)
    save_spectrum(dest, spectrum.cpu().numpy(), image_size)

#----------------------------------------------------------------------------


@main.command()
@click.argument('npz-file', nargs=1)
@click.option('--save', help='Save the plot and exit', metavar='[PNG|PDF|...]')
@click.option('--dpi', help='Figure resolution', metavar='FLOAT', type=click.FloatRange(min=1), default=100, show_default=True)
@click.option('--smooth', help='Amount of smoothing', metavar='FLOAT', type=click.FloatRange(min=0), default=1.25, show_default=True)
def heatmap(npz_file, save, smooth, dpi):
    """Visualize 2D heatmap based on the given .npz file."""
    hmap, image_size = construct_heatmap(npz_file=npz_file, smooth=smooth)
    import matplotlib.pyplot as plt

    # Setup plot.
    plt.figure(figsize=[6, 4.8], dpi=dpi, tight_layout=True)
    freqs = np.linspace(-0.5, 0.5, num=hmap.shape[0], endpoint=True) * image_size
    ticks = np.linspace(freqs[0], freqs[-1], num=5, endpoint=True)
    levels = np.linspace(-40, 20, num=13, endpoint=True)

    # Draw heatmap.
    plt.xlim(ticks[0], ticks[-1])
    plt.ylim(ticks[0], ticks[-1])
    plt.xticks(ticks)
    plt.yticks(ticks)
    plt.contourf(freqs, freqs, hmap, levels=levels, extend='both', cmap='Blues')
    plt.gca().set_aspect('equal')
    plt.colorbar(ticks=levels)
    plt.contour(freqs, freqs, hmap, levels=levels, extend='both', linestyles='solid', linewidths=1, colors='midnightblue', alpha=0.2)
    _show_or_save(plt, save)

#----------------------------------------------------------------------------


@main.command()
@click.argument('npz-files', nargs=-1, required=True)
@click.option('--save', help='Save the plot and exit', metavar='[PNG|PDF|...]')
@click.option('--dpi', help='Figure resolution', metavar='FLOAT', type=click.FloatRange(min=1), default=100, show_default=True)
@click.option('--smooth', help='Amount of smoothing', metavar='FLOAT', type=click.FloatRange(min=0), default=0, show_default=True)
def slices(npz_files, save, dpi, smooth):
    """Visualize 1D slices based on the given .npz files."""
    cases = [dnnlib.EasyDict(npz_file=npz_file) for npz_file in npz_files]
    for c in cases:
        c.hmap, c.image_size = construct_heatmap(npz_file=c.npz_file, smooth=smooth)
        c.label = os.path.splitext(os.path.basename(c.npz_file))[0]

    # Check consistency.
    image_size = cases[0].image_size
    hmap_size = cases[0].hmap.shape[0]
    if any(c.image_size != image_size or c.hmap.shape[0] != hmap_size for c in cases):
        raise click.ClickException('All .npz must have the same resolution')
    for c in cases:
        c.curves = slice_curves(c.hmap, c.image_size)
    import matplotlib.pyplot as plt

    # Setup plot.
    plt.figure(figsize=[12, 4.6], dpi=dpi, tight_layout=True)
    freqs0, freqs45 = cases[0].curves['freqs0'], cases[0].curves['freqs45']
    xticks0 = np.linspace(freqs0[0], freqs0[-1], num=9, endpoint=True)
    xticks45 = np.round(np.linspace(freqs45[0], freqs45[-1], num=9, endpoint=True))
    yticks = np.linspace(-50, 30, num=9, endpoint=True)

    # Draw 0 degree slice.
    plt.subplot(1, 2, 1)
    plt.title('0° slice')
    plt.xlim(xticks0[0], xticks0[-1])
    plt.ylim(yticks[0], yticks[-1])
    plt.xticks(xticks0)
    plt.yticks(yticks)
    for c in cases:
        plt.plot(freqs0, c.curves['slice0'], label=c.label)
    plt.grid()
    plt.legend(loc='upper right')

    # Draw 45 degree slice.
    plt.subplot(1, 2, 2)
    plt.title('45° slice')
    plt.xlim(xticks45[0], xticks45[-1])
    plt.ylim(yticks[0], yticks[-1])
    plt.xticks(xticks45)
    plt.yticks(yticks)
    for c in cases:
        plt.plot(freqs45, c.curves['slice45'], label=c.label)
    plt.grid()
    plt.legend(loc='upper right')
    _show_or_save(plt, save)

#----------------------------------------------------------------------------


if __name__ == "__main__":
    main()  # pylint: disable=no-value-for-parameter
