"""H100: the average power spectrum (ide3d_spectrum_accum / _finalize) and image moments (ide3d_image_moments) of avg_spectra against
float64 numpy, and `calc` / `stats` end to end against the CPU golden of the reference's avg_spectra.py.

Kernel against numpy: every bin within TOL * max|S| of np.fft.fft2 of the zero-padded plane (oracle.spectra.spectrum_direct, the same
whitening table and window).  Both sides are float64 FFTs whose rounding grows with log2(P) * 2^-53 relative to the largest values, so
the bound is relative to max|S|.  Measured on an H100 80GB HBM3 (700 W): at most 8.2e-16 (N = 1024, interp 4), so TOL has four
decades of margin.
"""

import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, load_golden

sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
import make_spectra_golden as sg  # noqa: E402

pytestmark = pytest.mark.gpu

TOL = 1e-11                # measured <= 8.2e-16
REL_GOLDEN = 1e-7          # the reference rounds the 2-D window to float32 (tests/test_spectra.py); measured 1.3e-8
REL_GEN = 1e-5             # the batched device render may round a few uint8 pixels the other way; measured 4.6e-7


def _images(b, c, n, seed, layout='nchw', dev='cuda'):
    """Smooth random images plus noise (a spectrum spanning many decades, like photographs), uint8, NCHW or an NHWC view."""
    g = torch.Generator().manual_seed(seed)
    base = torch.nn.functional.interpolate(torch.rand(b, c, 6, 6, generator=g), size=(n, n), mode='bicubic', align_corners=False)
    x = (base * 200 + torch.rand(b, c, n, n, generator=g) * 40).clamp(0, 255).to(torch.uint8)
    if layout == 'nhwc':
        return x.permute(0, 2, 3, 1).contiguous().to(dev).permute(0, 3, 1, 2)
    return x.to(dev)


def _kernel_vs_numpy(n, interp, c, layout, b=3, beta=8.0):
    from oracle import spectra as osp
    from ide3d_b200.torch_utils.ops import spectra as ops
    x = _images(b, c, n, seed=n * 10 + interp + c, layout=layout)
    acc = ops.Spectrum(n, c, 112.684, 69.509, beta=beta, interp=interp, device='cuda')
    assert acc.native
    acc.add(x)
    got = acc.result().cpu().numpy()
    ref = osp.spectrum_direct(x.cpu().numpy(), acc.lut.cpu().numpy(), acc.window.cpu().numpy(), interp)
    err = float(np.abs(got - ref).max() / np.abs(ref).max())
    print(f'N={n} interp={interp} C={c} {layout}: max |S - ref| / max|S| = {err:.2e}')
    assert err <= TOL
    return err


@pytest.mark.parametrize('layout', ['nchw', 'nhwc'])
@pytest.mark.parametrize('c', [1, 3])
@pytest.mark.parametrize('interp', [1, 2, 4, 8])
@pytest.mark.parametrize('n', [16, 64])
def test_accum_small(n, interp, c, layout):
    _kernel_vs_numpy(n, interp, c, layout)


@pytest.mark.parametrize('n, c, layout', [(512, 3, 'nchw'), (512, 1, 'nhwc'), (1024, 3, 'nhwc')])
def test_accum_production(n, c, layout):
    """512^2 at interp 4 (P = 2048) and the reference's FFHQ-1024 example (P = 4096)."""
    _kernel_vs_numpy(n, 4, c, layout, b=2 if n == 512 else 1)


def test_batch_split_and_rerun_bit_identical():
    from ide3d_b200.torch_utils.ops import spectra as ops
    x = _images(8, 3, 64, seed=3)

    def run(splits):
        acc = ops.Spectrum(64, 3, 100.0, 50.0, interp=4)
        i = 0
        for s in splits:
            acc.add(x[i:i + s])
            i += s
        return acc.result()

    one = run([1] * 8)
    assert torch.equal(one, run([3, 3, 2]))
    assert torch.equal(one, run([8]))
    assert torch.equal(one, run([8]))
    acc = ops.Spectrum(64, 3, 100.0, 50.0, interp=4)      # a chunked call (scratch cap) gives the same bits
    acc.chunk = 3
    acc.add(x)
    assert torch.equal(one, acc.result())


def test_moments_exact():
    from ide3d_b200.torch_utils.ops import spectra as ops
    x = torch.randint(0, 256, (6, 3, 256, 256), dtype=torch.uint8, generator=torch.Generator().manual_seed(1))
    a = x.numpy().astype(np.int64)
    want = [a.size, int(a.sum()), int((a * a).sum())]
    for view in (x.cuda(), x.permute(0, 2, 3, 1).contiguous().cuda().permute(0, 3, 1, 2)):
        m = torch.zeros(3, dtype=torch.int64, device='cuda')
        ops.image_moments(view[:4], m)
        ops.image_moments(view[4:], m)
        assert [int(v) for v in m.cpu()] == want
    # above 2^53 a float64 sum rounds; the 64-bit integer counters stay exact
    m = torch.tensor([0, (1 << 62) - 5, 0], dtype=torch.int64, device='cuda')
    ops.image_moments(torch.full((1, 1, 16, 16), 255, dtype=torch.uint8, device='cuda'), m)
    assert int(m[1]) == (1 << 62) - 5 + 256 * 255


def test_refused_shapes_and_fallback(lib):
    from ide3d_b200 import _lib
    from ide3d_b200.torch_utils.ops import spectra as ops
    from oracle import spectra as osp
    for c, n, interp in ((3, 48, 4), (3, 16, 3), (3, 1024, 8), (5, 16, 1), (3, 2048, 1), (3, 8, 2)):
        assert lib.ide3d_spectrum_scratch_bytes(1, c, n, interp) == _lib.UNSUPPORTED
        assert lib.ide3d_spectrum_accum(None, 1, c, n, 0, 0, 0, 0, None, None, interp, None, None, 0, None) == _lib.UNSUPPORTED
    assert lib.ide3d_spectrum_accum(None, 1, 3, 16, 0, 0, 0, 0, None, None, 4, None, None, 0, None) == _lib.INVALID
    x = _images(2, 3, 48, seed=9)
    acc = ops.Spectrum(48, 3, 112.684, 69.509, interp=3)
    assert not acc.native
    acc.add(x)
    got = acc.result().cpu().numpy()
    ref = osp.spectrum_direct(x.cpu().numpy(), acc.lut.cpu().numpy(), acc.window.cpu().numpy(), 3)
    assert np.abs(got - ref).max() <= TOL * np.abs(ref).max()


@pytest.fixture(scope='module')
def data(tmp_path_factory):
    return sg.setup(str(tmp_path_factory.mktemp('spectra')))


def _rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


@pytest.mark.parametrize('res', sg.SIZES)
def test_calc_and_stats_match_reference(data, res):
    from ide3d_b200 import avg_spectra
    golden = load_golden('spectra')
    dev = torch.device('cuda')
    kw = dict(data_loader_kwargs=dict(pin_memory=True, num_workers=0), batch=7)
    worst = 0.0
    for kind, path in zip(('dir', 'zip'), data[res]):
        _, _, it = avg_spectra.stream_source_images(path, None, 0, dev, **kw)
        assert f'--mean={{:g}} --std={{:g}}'.format(*avg_spectra.compute_stats(it, dev)) == str(golden[f'stats_{res}_{kind}'])
        for interp in sg.INTERPS:
            for beta in sg.BETAS:
                num, size, it = avg_spectra.stream_source_images(path, None, 0, dev, **kw)
                spec = avg_spectra.compute_spectrum(it, size, sg.MEAN, sg.STD, beta, interp, dev).cpu().numpy()
                worst = max(worst, _rel(spec, golden[f'calc_{res}_i{interp}_b{beta:g}']))
    _, size, it = avg_spectra.stream_source_images(data[res][1], 7, 3, dev, **kw)
    worst = max(worst, _rel(avg_spectra.compute_spectrum(it, size, sg.MEAN, sg.STD, 8.0, 2, dev).cpu().numpy(), golden[f'calc_{res}_sub']))
    print(f'{res}^2 datasets: max |S - reference| / max|S| = {worst:.2e}')
    assert worst < REL_GOLDEN


def test_cli_calc_and_stats(data, tmp_path):
    """The command line as a user runs it (DataLoader workers, pinned copies); its .npz reads back through construct_heatmap."""
    from ide3d_b200 import avg_spectra
    golden = load_golden('spectra')
    res, zpath = sg.SIZES[-1], data[sg.SIZES[-1]][1]
    env = dict(os.environ, PYTHONPATH=ROOT)
    run = lambda *a: subprocess.run([sys.executable, '-m', 'ide3d_b200.avg_spectra', *a], cwd=ROOT, env=env, capture_output=True,
                                    text=True, timeout=600)
    r = run('stats', f'--source={zpath}')
    assert r.returncode == 0, r.stderr
    assert r.stdout.strip().splitlines()[-1] == str(golden[f'stats_{res}_zip'])
    dest = str(tmp_path / 'out' / 'spec.npz')
    r = run('calc', f'--source={zpath}', f'--dest={dest}', f'--mean={sg.MEAN}', f'--std={sg.STD}')
    assert r.returncode == 0, r.stderr
    with np.load(dest) as z:
        assert z['spectrum'].dtype == np.float64 and int(z['image_size']) == res
        assert _rel(z['spectrum'], golden[f'calc_{res}_i4_b8']) < REL_GOLDEN
    hmap, image_size = avg_spectra.construct_heatmap(dest, 0)
    ref = 10 ** (golden['hmap_s0'] / 10)
    assert image_size == res and hmap.shape == ref.shape
    assert np.abs(10 ** (hmap / 10) - ref).max() < REL_GOLDEN * ref.max()


def test_generator_source_matches_reference():
    from ide3d_b200 import avg_spectra
    from oracle import spectra as osp
    golden = load_golden('spectra')
    g = sg.GEN
    dev = torch.device('cuda')
    G = osp.StandInSpectrumGenerator().to(dev)
    num, size, it = avg_spectra.stream_source_images(G, g['num'], g['seed'], dev, batch=2)
    assert (num, size) == (g['num'], 512)
    spec = avg_spectra.compute_spectrum(it, size, sg.MEAN, sg.STD, g['beta'], g['interp'], dev).cpu().numpy()
    errs = (_rel(spec[::7, ::7], golden['calc_gen_sub']), _rel(spec.sum(0), golden['calc_gen_sum0']), _rel(spec.sum(1), golden['calc_gen_sum1']))
    print(f'generator: max |S - reference| / max|S| over the stored bins and sums = {max(errs):.2e}')
    assert max(errs) < REL_GEN
