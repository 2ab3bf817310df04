"""CPU: avg_spectra against the reference's own avg_spectra.py (tests/golden/make_spectra_golden.py): the float64 oracle of the kernel's
pruned transform reproduces the reference's `calc` and `stats`, construct_heatmap and slice_curves match it, the generator draw rule,
the .npz layout, and the command line's refusals.

The reference rounds the 2-D window w[n1] w[n2] to float32 before multiplying; the oracle (like the kernel) keeps the product in float64.
Measured on the CPU, that moves the spectra by at most 1.3e-8 of max|S| (datasets) and 7.8e-10 (generator); the tolerance is 1e-7.
"""

import os
import sys

import numpy as np
import pytest
import torch
from click.testing import CliRunner

from conftest import ROOT, load_golden

sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
import make_spectra_golden as sg  # noqa: E402

from ide3d_b200 import avg_spectra  # noqa: E402
from ide3d_b200.torch_utils.ops import spectra as ops  # noqa: E402
from ide3d_b200.training.dataset import ImageFolderDataset  # noqa: E402
from oracle import spectra as osp  # noqa: E402

REL = 1e-7


@pytest.fixture(scope='module')
def golden():
    return load_golden('spectra')


@pytest.fixture(scope='module')
def data(tmp_path_factory):
    return sg.setup(str(tmp_path_factory.mktemp('spectra')))


def dataset_images(path, num=None, seed=0):
    d = ImageFolderDataset(path=path, max_size=num, random_seed=seed)
    return np.stack([d[i][0] for i in range(len(d))])


def generator_images(num, seed):
    G = osp.StandInSpectrumGenerator()
    out = []
    for idx in range(num):
        z, c = avg_spectra.generator_draw(G.z_dim, G.c_dim, seed + idx)
        with torch.no_grad():
            out.append((G(z=torch.from_numpy(z), c=torch.from_numpy(c)) * 127.5 + 128).clamp(0, 255).to(torch.uint8).numpy())
    return np.concatenate(out)


def rel_err(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


@pytest.mark.parametrize('res', sg.SIZES)
def test_oracle_reproduces_reference_calc(data, golden, res):
    for kind, path in zip(('dir', 'zip'), data[res]):
        x = dataset_images(path)
        for interp in sg.INTERPS:
            for beta in sg.BETAS:
                ref = golden[f'calc_{res}_i{interp}_b{beta:g}']
                lut, w = osp.whitening_lut(sg.MEAN, sg.STD), osp.kaiser_window(res, beta)
                pruned = osp.spectrum_pruned(x, lut, w, interp)
                assert pruned.shape == ref.shape == (res * interp, res * interp)
                assert rel_err(pruned, ref) < REL, (kind, interp, beta)
                assert rel_err(pruned, osp.spectrum_direct(x, lut, w, interp)) < 1e-13
    sub = dataset_images(data[res][1], num=7, seed=3)
    assert rel_err(osp.spectrum_pruned(sub, osp.whitening_lut(sg.MEAN, sg.STD), osp.kaiser_window(res, 8.0), 2), golden[f'calc_{res}_sub']) < REL


def test_oracle_reproduces_reference_generator_calc(golden):
    g = sg.GEN
    x = generator_images(g['num'], g['seed'])
    spec = osp.spectrum_pruned(x, osp.whitening_lut(sg.MEAN, sg.STD), osp.kaiser_window(512, g['beta']), g['interp'])
    assert rel_err(spec[::7, ::7], golden['calc_gen_sub']) < REL
    assert rel_err(spec.sum(0), golden['calc_gen_sum0']) < REL and rel_err(spec.sum(1), golden['calc_gen_sum1']) < REL


@pytest.mark.parametrize('res', sg.SIZES)
def test_stats_match_reference(data, golden, res):
    for kind, path in zip(('dir', 'zip'), data[res]):
        m = osp.moments(dataset_images(path))
        mean, std = ops.mean_std(np.array(m, dtype=np.uint64))
        assert f'--mean={mean:g} --std={std:g}' == str(golden[f'stats_{res}_{kind}'])


def test_heatmap_and_slices_match_reference(golden, tmp_path):
    res = sg.SIZES[-1]
    npz = str(tmp_path / 'spec.npz')
    avg_spectra.save_spectrum(npz, golden[f'calc_{res}_i4_b8'], res)
    for smooth in (0.0, 1.25):
        hmap, image_size = avg_spectra.construct_heatmap(npz, smooth)
        assert image_size == res
        np.testing.assert_array_equal(hmap, golden[f'hmap_s{smooth:g}'])
        curves = avg_spectra.slice_curves(hmap, image_size)
        for key in ('slice0', 'slice45', 'freqs0', 'freqs45'):
            np.testing.assert_array_equal(curves[key], golden[f'{key}_s{smooth:g}'])


def test_npz_layout(tmp_path):
    dest = str(tmp_path / 'sub' / 'x.npz')
    avg_spectra.save_spectrum(dest, np.ones([64, 64], dtype=np.float64), 16)
    with np.load(dest) as z:
        assert sorted(z.files) == ['image_size', 'spectrum']
        assert z['spectrum'].dtype == np.float64 and z['spectrum'].shape == (64, 64)
        assert z['image_size'].dtype.kind == 'i' and int(z['image_size']) == 16


def test_generator_draw_rule(data):
    seed, zd = 11, 16
    rnd = np.random.RandomState(seed)
    z_ref = rnd.randn(1, zd)
    for c_dim in (25, 0, 10):
        z, c = avg_spectra.generator_draw(zd, c_dim, seed)
        np.testing.assert_array_equal(z, z_ref)
        assert c.shape == (1, c_dim)
    _, c = avg_spectra.generator_draw(zd, 25, seed)
    np.testing.assert_array_equal(c[0], np.array(avg_spectra.FRONTAL_CAMERA, dtype=np.float32))
    _, c = avg_spectra.generator_draw(zd, 10, seed)
    assert c.sum() == 1 and c[0, rnd.randint(10)] == 1            # the reference's one-hot: the draw after z
    labels = ImageFolderDataset(path=data[16][1], use_labels=True)
    _, c = avg_spectra.generator_draw(zd, 25, seed, labels=labels)
    r = np.random.RandomState(seed)
    r.randn(1, zd)
    np.testing.assert_array_equal(c[0], labels.get_label(r.randint(len(labels))))


def test_cli_refusals(data, tmp_path):
    run = lambda *args: CliRunner().invoke(avg_spectra.main, list(args))
    dest = f'--dest={tmp_path / "o.npz"}'
    r = run('calc', '--source=net.pkl', dest, '--mean=1', '--std=1')
    assert r.exit_code == 1 and 'network pickles are not loaded here' in r.output and 'stream_source_images' in r.output
    r = run('stats', '--source=net.pkl')
    assert r.exit_code == 1 and 'network pickles are not loaded here' in r.output
    r = run('calc', f'--source={tmp_path / "missing.txt"}', dest, '--mean=1', '--std=1')
    assert r.exit_code == 1 and '--source must point to network pickle, dataset zip, or directory' in r.output
    r = run('calc', f'--source={data[16][1]}', dest, '--mean=1', '--std=1', '--num=50')
    assert r.exit_code == 1 and '--source contains fewer than 50 images' in r.output
    assert run('calc', f'--source={data[16][1]}', '--mean=1', '--std=1').exit_code == 2                  # --dest is required
    assert run('calc', f'--source={data[16][1]}', dest, '--mean=1', '--std=-1').exit_code == 2           # std >= 0
    assert run('calc', f'--source={data[16][1]}', dest, '--mean=1', '--std=1', '--interp=0').exit_code == 2
    assert run('stats', f'--source={data[16][1]}', '--num=0').exit_code == 2
    a, b = str(tmp_path / 'a.npz'), str(tmp_path / 'b.npz')
    avg_spectra.save_spectrum(a, np.ones([32, 32]), 16)
    avg_spectra.save_spectrum(b, np.ones([64, 64]), 32)
    r = run('slices', a, b)
    assert r.exit_code == 1 and 'All .npz must have the same resolution' in r.output
    assert not os.path.exists(str(tmp_path / 'o.npz'))


def test_cpu_tensors_are_refused():
    with pytest.raises(RuntimeError, match='CUDA'):
        ops.Spectrum(16, 3, 0.0, 1.0, device='cpu')
    with pytest.raises(RuntimeError, match='CUDA'):
        ops.image_moments(torch.zeros(1, 3, 16, 16, dtype=torch.uint8), torch.zeros(3, dtype=torch.int64))
