"""CPU: the visualizer's frames (ide3d_b200.viz.renderer) against tests/golden/viz.npz, the reference's own Renderer methods run over
oracle.viz's stand-in generator (tests/golden/make_viz_golden.py).

  * latents and camera: the ws and labels the reference forms, bit for bit, quirks included
  * oracle.viz.display (the tail's contract, FFT in float64): image bytes and stats of the reference, FFT colormap indices within 1
    and equal at >= 99.9 % of the pixels
  * the layer list of an unlinked call equals the reference's run_synthesis_net on a small CPU generator
  * errors come back as res.error strings"""

import json

import numpy as np
import pytest
import torch

from conftest import load_golden


@pytest.fixture(scope='module')
def golden():
    return load_golden('viz')


def _cases(golden):
    return sorted({k.split('/')[0] for k in golden if '/' in k})


def _args(golden, name):
    return json.loads(str(golden[f'{name}/args']))


def test_latents_and_camera_match_reference(golden):
    from ide3d_b200.viz import renderer as R
    from oracle import viz as ov
    for name in _cases(golden):
        a = _args(golden, name)
        G = ov.StandInGenerator()
        w, labels, _ = R.latents(G, a['w0_seeds'], a.get('stylemix_idx', []), a.get('stylemix_seed', 0), a.get('trunc_psi', 1),
                                 a.get('trunc_cutoff', 0), device='cpu')
        (z, c), = G.mapping.calls
        assert np.array_equal(z.numpy(), golden[f'{name}/z']), name
        assert np.array_equal(labels, golden[f'{name}/labels']) and np.array_equal(c.numpy(), golden[f'{name}/labels']), name
        assert np.array_equal(w.numpy(), golden[f'{name}/ws']), name
        torch.manual_seed(a.get('random_seed', 0))
        cam = R.camera(a.get('yaw', 0), a.get('pitch', 0), a.get('focal_length', 4.2647), 'cpu')
        assert np.array_equal(cam.numpy(), golden[f'{name}/c']), name
    # the label quirk: one seed list entry, the last, carries the frontal label
    labels = golden['weights_repeat/labels']
    assert (labels[:-1] == 0).all() and np.array_equal(labels[-1], R.frontal_label())


def test_oracle_tail_matches_reference(golden):
    from oracle import viz as ov
    lut = torch.from_numpy(golden['lut'])
    for name in _cases(golden):
        a = _args(golden, name)
        kw = {k: a[k] for k in ('render_type', 'sel_channels', 'base_channel', 'img_normalize', 'img_scale_db', 'fft_show', 'fft_all',
                                'fft_range_db', 'fft_beta') if k in a}
        img, stats = ov.display(torch.from_numpy(golden[f'{name}/map']), cmap=lut, **kw)
        ref_img, ref_stats = golden[f'{name}/image'], golden[f'{name}/stats']
        assert img.shape == ref_img.shape, name
        np.testing.assert_allclose(stats.numpy(), ref_stats, rtol=1e-6, atol=1e-6 * np.abs(ref_stats[4:]).max(), err_msg=name)
        W = golden[f'{name}/map'].shape[-1]
        if not a.get('fft_show'):
            assert np.array_equal(img.numpy(), ref_img), name
            continue
        assert np.array_equal(img[:, :W].numpy(), ref_img[:, :W]), name
        d = np.abs(ov.decode(img[:, W:].numpy()) - ov.decode(ref_img[:, W:]))
        assert d.max() <= 1 and (d == 0).mean() >= 0.999, (name, d.max(), (d == 0).mean())


def test_layer_list_matches_reference(golden):
    from ide3d_b200.viz import renderer as R
    from oracle.backend import cpu_reference_ops
    from golden.make_viz_golden import small_generator
    G = small_generator()
    with cpu_reference_ops(), torch.no_grad():
        ws = G.mapping(torch.randn(1, G.z_dim, generator=torch.Generator().manual_seed(1)), torch.zeros(1, G.c_dim))
        c = torch.zeros(1, 25)
        c[0, :16] = torch.eye(4).reshape(-1)
        c[0, 11] = 2.7
        _, layers = R.run_synthesis_net(G, ws, c, noise_mode='const', force_fp32=False, unlinked=True)
        out, _ = R.run_synthesis_net(G, ws, c, capture_layer='synthesis.vb16:1', noise_mode='const', unlinked=True)
    ref = [(n, s, d) for n, s, d in json.loads(str(golden['layers']))]
    assert [(l.name, l.shape, l.dtype) for l in layers] == ref
    assert list(out.shape) == next(s for n, s, _ in ref if n == 'synthesis.vb16:1')


def test_errors_surface_as_strings(tmp_path):
    from ide3d_b200.viz.renderer import Renderer
    r = Renderer(device='cpu')
    res = r.render(pkl=str(tmp_path / 'G.pkl'))
    assert isinstance(res.error, str) and 'network pickles are not loaded' in res.error and 'image' not in res
    res = r.render(pkl=str(tmp_path / 'missing.pt'))
    assert isinstance(res.error, str) and 'No such file' in res.error
    from oracle.viz import StandInGenerator
    res = r.render(pkl=StandInGenerator())                  # fails inside synthesis: the traceback is the error text
    assert isinstance(res.error, str) and res.error.startswith('Traceback') and res.num_ws == 18
    res = r.render()
    assert res.error == 'Renderer: no network given (pkl=)' and res.render_time >= 0
