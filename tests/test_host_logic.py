"""CPU: host-side logic of the generator / plugin shims with the CUDA entry points swapped for the oracle
(oracle.backend.cpu_reference_ops) -- API contract reconstructed from the reference's call sites (SURVEY.md §8b)."""

import math
import os
import sys

import numpy as np
import pytest
import torch

from oracle.backend import cpu_reference_ops

LABEL = [1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 2.7, 0, 0, 0, 1, 4.2647, 0, 0.5, 0, 4.2647, 0.5, 0, 0, 1]   # gen_images.py:87


@pytest.fixture(scope='module')
def G():
    from ide3d_b200.training.triplane import TriPlaneGenerator
    torch.manual_seed(0)
    return TriPlaneGenerator(z_dim=32, w_dim=32, img_resolution=64, plane_resolution=32, render_size=16, channel_base=1024,
                             channel_max=32, sr_channels=(16, 8), mapping_kwargs=dict(num_layers=2)).eval().requires_grad_(False)


def test_full_size_generator_has_the_reference_layer_structure():
    """7 backbone blocks (3 children each: conv0?, conv1, torgb), 3 renderer heads, 2 SR blocks, 18 ws
    (ide3d-nada/ZSSGAN/model/ZSSGAN_IDE3D.py:425-437; apps/train_hybrid_encoder.py:40-43)."""
    from ide3d_b200.training.triplane import TriPlaneGenerator
    g = TriPlaneGenerator()
    s = g.synthesis
    assert g.num_ws == s.num_ws == g.mapping.num_ws == g.backbone.num_ws == 18
    assert (g.z_dim, g.c_dim, g.w_dim, g.img_resolution, g.img_channels) == (512, 25, 512, 512, 3)
    assert s.voxel_block_resolutions == [4, 8, 16, 32, 64, 128, 256] and s.block_resolutions == [256, 512]
    assert s.render_size == g.neural_rendering_resolution == 64
    layers = [l for child in s.children() for l in child.children()]
    names = [type(l).__name__ for l in layers]
    assert len(layers) == 29 and names[:2] == ['SynthesisLayer', 'ToRGBLayer']
    assert names[20:23] == ['DecoderHead'] * 3                                   # the "nerf" layers, idx 20-22
    conv_inds = [0, 2, 3, 5, 6, 8, 9, 11, 12, 14, 15, 17, 18, 23, 24, 26, 27]
    rgb_inds = [1, 4, 7, 10, 13, 16, 19, 25, 28]
    assert all(names[i] == 'SynthesisLayer' for i in conv_inds) and all(names[i] == 'ToRGBLayer' for i in rgb_inds)
    assert g.rendering_kwargs['ray_start'] == 2.25 and g.rendering_kwargs['ray_end'] == 3.3 and g.rendering_kwargs['fov'] == 18.0
    assert set(g.init_kwargs) == set() and g.init_args == ()
    assert any('noise_const' in n for n, _ in s.named_buffers())


def test_synthesis_contract(G):
    z = torch.randn(2, G.z_dim)
    c = torch.tensor(LABEL).repeat(2, 1)
    with cpu_reference_ops():
        ws = G.mapping(z, c, truncation_psi=0.7, truncation_cutoff=4)
        assert ws.shape == (2, G.num_ws, G.w_dim)
        img = G.synthesis(ws, c=c, noise_mode='const', render_params=dict(num_steps=8, h_mean=1.2, fov=18))
        img2, seg = G.synthesis(ws, c=c, noise_mode='const', return_seg=True, render_params=dict(num_steps=8))
        img3, raw = G.synthesis(ws, c, return_raw=True, force_fp32=True, num_steps=8)
        d = G.synthesis(ws, c=c, return_dict=True, num_steps=8)
        img_nolabel = G.synthesis(ws, render_params=dict(num_steps=8, h_mean=math.pi / 2, v_mean=math.pi / 2), perturb=None)
        img_label = G.synthesis(ws, c=c, num_steps=8, perturb=None)
    assert img.shape == img2.shape == img3.shape == (2, 3, 64, 64) and seg.shape == (2, 19, 64, 64) and raw.shape == (2, 3, 16, 16)
    assert set(d) >= {'image', 'image_raw', 'image_depth'} and d['image_depth'].shape == (2, 1, 16, 16)
    assert torch.isfinite(img).all() and torch.isfinite(seg).all()
    # the frontal label IS the pose sample_camera_positions(pi/2, pi/2, r=2.7) builds: both routes agree
    assert torch.allclose(img_nolabel, img_label, atol=1e-5)


def test_layout_and_chaining_switches_do_not_change_values(G):
    """The GPU build's host-side choices -- NHWC activations, epilogues that pre-modulate the next layer, activation scaling
    instead of weight modulation -- are re-orderings of the reference arithmetic (inversion/networks.py:97-129)."""
    from ide3d_b200.training import networks as nw
    z = torch.randn(2, G.z_dim, generator=torch.Generator().manual_seed(3))
    c = torch.tensor(LABEL).repeat(2, 1)
    outs = {}
    saved = (nw.CHANNELS_LAST, nw.CHAIN_MODULATION)
    try:
        with cpu_reference_ops(reference_layout=False):
            ws = G.mapping(z, c)
            for cl, chain, fused in ((True, True, None), (False, True, None), (True, False, None), (False, False, True)):
                nw.CHANNELS_LAST, nw.CHAIN_MODULATION = cl, chain
                outs[(cl, chain, fused)] = G.synthesis(ws, c=c, noise_mode='const', num_steps=8, perturb=None, fused_modconv=fused)
    finally:
        nw.CHANNELS_LAST, nw.CHAIN_MODULATION = saved
    ref = outs[(False, False, True)]                     # the reference's eval path: NCHW, grouped weight-modulated convs
    for k, v in outs.items():
        assert torch.allclose(v, ref, atol=2e-4, rtol=1e-4), (k, (v - ref).abs().max().item())


def test_block_walk_of_extract_shapes(G):
    """The exact loop of extract_shapes.py:113-147 runs against the generator."""
    from ide3d_b200.torch_utils import misc
    z = torch.randn(1, G.z_dim)
    c = torch.tensor(LABEL)[None]
    with cpu_reference_ops():
        ws = G.mapping(z, c, truncation_psi=0.5)
        misc.assert_shape(ws, [None, G.synthesis.num_ws, G.synthesis.w_dim])
        voxel_block_ws, block_ws, w_idx = [], [], 0
        for res in G.synthesis.voxel_block_resolutions:
            block = getattr(G.synthesis, f'vb{res}')
            voxel_block_ws.append(ws.narrow(1, w_idx, block.num_conv + block.num_torgb))
            w_idx += block.num_conv
        for res in G.synthesis.block_resolutions:
            block = getattr(G.synthesis, f'b{res}')
            block_ws.append(ws.narrow(1, w_idx, block.num_conv + block.num_torgb))
            w_idx += block.num_conv
        assert w_idx + 1 == G.synthesis.num_ws
        x_v = img_v = seg_v = None
        for res, cur_ws in zip(G.synthesis.voxel_block_resolutions, voxel_block_ws):
            x_v, img_v, seg_v = getattr(G.synthesis, f'vb{res}')(x_v, img_v, cur_ws, condition_img=seg_v)
        assert img_v.shape == seg_v.shape == (1, 96, 32, 32)
        samples = torch.rand(1, 250, 3) - 0.5
        out = G.synthesis.renderer.sample_voxel(img_v, seg_v, samples[:, 0:100]).reshape(samples.size(0), -1, 52)
        assert out.shape == (1, 100, 52)
        a, b = G.synthesis.split_ws(ws)
        assert all(torch.equal(x, y) for x, y in zip(a + b, voxel_block_ws + block_ws))


def test_compat_aliases_and_persistence(G):
    import ide3d_b200.compat as compat
    saved = {k: sys.modules.get(k) for k in list(sys.modules) if k.split('.')[0] in ('training', 'torch_utils')}
    try:
        names = compat.install()
        from training.triplane import TriPlaneGenerator as A                       # noqa: the reference's import lines
        from training.volumetric_rendering import LookAtPoseSampler, create_cam2world_matrix, sample_camera_positions  # noqa
        from torch_utils.ops import bias_act, filtered_lrelu, upfirdn2d             # noqa
        from torch_utils import custom_ops, misc, persistence                      # noqa
        assert 'training.triplane' in names and A is type(G).__mro__[0] or issubclass(type(G), A.__mro__[1])
    finally:
        for k in list(sys.modules):
            if k.split('.')[0] in ('training', 'torch_utils'):
                del sys.modules[k]
        sys.modules.update({k: v for k, v in saved.items() if v is not None})
    # viz/renderer.py:199 style re-instantiation
    G2 = type(G)(*G.init_args, **G.init_kwargs)
    assert G2.num_ws == G.num_ws and sum(p.numel() for p in G2.parameters()) == sum(p.numel() for p in G.parameters())


def test_pose_helpers_cpu():
    from ide3d_b200.training.volumetric_rendering import LookAtPoseSampler, create_cam2world_matrix, sample_camera_positions
    o, phi, theta = sample_camera_positions('cpu', n=3, r=2.7, horizontal_mean=math.pi / 2, vertical_mean=math.pi / 2, mode=None)
    m = create_cam2world_matrix(-o, o, device='cpu')
    assert torch.allclose(m[0].reshape(-1), torch.tensor(LABEL[:16]), atol=1e-6)
    la = LookAtPoseSampler.sample(math.pi / 2, math.pi / 2, torch.tensor([0, 0, 0.]), radius=2.7)
    assert torch.allclose(la, m[:1], atol=1e-6)
    torch.manual_seed(1)
    for mode in ('uniform', 'normal', 'hybrid', 'truncated_gaussian', 'spherical_uniform'):
        o, _, _ = sample_camera_positions('cpu', n=4, r=1.5, mode=mode)
        assert torch.allclose(o.norm(dim=-1), torch.full((4,), 1.5), atol=1e-5)


def test_setup_filter_matches_oracle():
    from ide3d_b200.torch_utils.ops import upfirdn2d as up
    from oracle import ops as oops
    for taps, kw in (([1, 3, 3, 1], {}), ([1, 2, 1], dict(gain=4)), (list(range(1, 13)), {}), ([[1, 2], [3, 4]], dict(flip_filter=True)), (None, {})):
        assert torch.equal(up.setup_filter(taps, **kw), oops.setup_filter(taps, **kw))


def test_mrc_writer_round_trip_and_mrcfile_shim(tmp_path):
    """extract_shapes.py:191-192 writes the sigma grid as a mode-2 MRC volume; ide3d_b200.mrc does it without `mrcfile`."""
    from ide3d_b200 import mrc
    vol = np.random.RandomState(0).randn(5, 7, 9).astype(np.float32)
    path = str(tmp_path / 'grid.mrc')
    with mrc.new_mmap(path, overwrite=True, shape=vol.shape, mrc_mode=2) as m:          # the reference's exact call shape
        m.data[:] = vol
    assert os.path.getsize(path) == 1024 + vol.size * 4
    back, hdr = mrc.read_mrc(path)
    assert np.array_equal(back, vol) and (hdr['nx'], hdr['ny'], hdr['nz'], hdr['mode']) == (9, 7, 5, 2)
    assert hdr['nversion'] == 20140 and abs(hdr['dmean'] - vol.mean()) < 1e-6 and hdr['dmax'] == vol.max()
    with pytest.raises(ValueError):
        with mrc.new_mmap(path, shape=vol.shape):
            pass
    mrc.write_mrc(path, torch.from_numpy(vol).double(), voxel_size=0.5)
    back2, hdr2 = mrc.read_mrc(path)
    assert np.array_equal(back2, vol) and hdr2['cella'] == (4.5, 3.5, 2.5)


def test_render_interp_video_batched_driver(G):
    """gen_videos' frame loop as one batched, sharded call: frame grids come back in frame order with the cells side by side."""
    from ide3d_b200 import video
    with cpu_reference_ops():
        grids = video.render_interp_video(G, seeds=[0, 1, 2, 3], w_frames=2, grid_dims=(2, 1), batch=2, truncation_cutoff=4,
                                          device=torch.device('cpu'), synthesis_kwargs=dict(perturb=None))
        ws, c, (F, gh, gw) = video.interp_video_inputs(G, [0, 1, 2, 3], w_frames=2, grid_dims=(2, 1), truncation_cutoff=4, device=torch.device('cpu'))
        one = G.synthesis(ws[2:3].float(), c=c[2:3], noise_mode='const', perturb=None)          # frame 1, cell 0
    assert grids.dtype == torch.uint8 and tuple(grids.shape) == (4, 64, 128, 3) and (F, gh, gw) == (4, 1, 2)
    want = (one[0] * 127.5 + 128).clamp(0, 255).to(torch.uint8).permute(1, 2, 0)
    assert (grids[1, :, :64].int() - want.int()).abs().max() <= 1


def test_conv2d_gradfix_gradient_penalty():
    """conv2d_gradfix (torch_utils/ops/conv2d_gradfix.py:66-198): gradients of gradients (R1 / path-length penalties) and the
    no_weight_gradients() switch.  For y = conv(x, w): d/dx sum(y * r) = conv_transpose(r, w), so the penalty P = |dL/dx|^2 is an explicit
    function of w; its autograd gradient through the module must equal the gradient of that explicit form."""
    from ide3d_b200.torch_utils.ops import conv2d_gradfix as cg
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 3, 9, 9, generator=g, dtype=torch.float64, requires_grad=True)
    w = torch.randn(4, 3, 3, 3, generator=g, dtype=torch.float64, requires_grad=True)
    r = torch.randn(2, 4, 9, 9, generator=g, dtype=torch.float64)
    y = cg.conv2d(x, w, padding=1)
    (gx,) = torch.autograd.grad((y * r).sum(), x, create_graph=True)
    gx.square().sum().backward()
    w2 = w.detach().clone().requires_grad_(True)
    torch.nn.functional.conv_transpose2d(r, w2, padding=1).square().sum().backward()
    assert torch.allclose(w.grad, w2.grad, rtol=1e-10, atol=1e-10)
    # transposed convolution: same statement with the roles swapped
    wt = torch.randn(3, 4, 3, 3, generator=g, dtype=torch.float64, requires_grad=True)
    yt = cg.conv_transpose2d(x, wt, stride=2, padding=1)
    rt = torch.randn(*yt.shape, generator=g, dtype=torch.float64)
    (gxt,) = torch.autograd.grad((yt * rt).sum(), x, create_graph=True)
    gxt.square().sum().backward()
    wt2 = wt.detach().clone().requires_grad_(True)
    torch.nn.functional.conv2d(rt, wt2, stride=2, padding=1).square().sum().backward()
    assert torch.allclose(wt.grad, wt2.grad, rtol=1e-10, atol=1e-10)
    # no_weight_gradients(): the input gradient is unchanged, the weight receives nothing (first and second order)
    w3 = w.detach().clone().requires_grad_(True)
    x3 = x.detach().clone().requires_grad_(True)
    with cg.no_weight_gradients():
        y3 = cg.conv2d(x3, w3, padding=1)
        (gx3,) = torch.autograd.grad((y3 * r).sum(), x3, create_graph=True)
    assert torch.allclose(gx3, gx.detach()) and w3.grad is None
    assert torch.autograd.grad(gx3.square().sum(), [w3, x3], allow_unused=True)[0] is None      # nothing reaches the weight, at any order
    assert cg.weight_gradients_disabled is False


def test_seg_block_loads_reference_style_torgb_toseg_state_dict():
    """ADVICE r1 (low): a state_dict with separate torgb / toseg layers (the in-repo reference class, inversion/networks.py:1093-1134) is
    merged into the block's single [img | seg] ToRGB when the two affines are tied, and refused loudly when they are not."""
    from ide3d_b200.training.networks import SegSynthesisBlock
    torch.manual_seed(0)
    blk = SegSynthesisBlock(8, 8, w_dim=16, resolution=8, img_channels=6, seg_channels=6, is_last=False)
    sd = blk.state_dict()
    w, b = sd.pop('torgb.weight'), sd.pop('torgb.bias')
    ref = dict(sd)
    ref['torgb.weight'], ref['torgb.bias'] = w[:6].clone(), b[:6].clone() + 0.5
    ref['toseg.weight'], ref['toseg.bias'] = w[6:].clone() * 2, b[6:].clone() - 0.5
    ref['toseg.affine.weight'], ref['toseg.affine.bias'] = sd['torgb.affine.weight'].clone(), sd['torgb.affine.bias'].clone()
    other = SegSynthesisBlock(8, 8, w_dim=16, resolution=8, img_channels=6, seg_channels=6, is_last=False)
    other.load_state_dict(dict(ref))
    assert torch.equal(other.torgb.weight[:6], w[:6]) and torch.equal(other.torgb.weight[6:], w[6:] * 2)
    assert torch.equal(other.torgb.bias, torch.cat([b[:6] + 0.5, b[6:] - 0.5]))
    bad = dict(ref)
    bad['toseg.affine.bias'] = bad['toseg.affine.bias'] + 1
    with pytest.raises(RuntimeError, match='toseg'):
        SegSynthesisBlock(8, 8, w_dim=16, resolution=8, img_channels=6, seg_channels=6, is_last=False).load_state_dict(bad)


def test_coarse_depths_and_torch_hash_match_the_oracle_on_cpu():
    """render.coarse_depths (the depths of the first pass of the hierarchical render, computed on the host side of the kernel) equals the
    oracle's initial_rays + perturb z values, with injected uniforms and with the counter hash (integer-exact twin of the kernel's)."""
    import numpy as np
    from ide3d_b200 import render, render_grad
    from oracle import renderer as orr
    n, res, S = 2, (5, 4), 11
    R = res[0] * res[1]
    seed = 0x0123_4567_89AB_CDEF
    u_ref = torch.from_numpy(orr.hash_uniform(np.arange(n * R * S, dtype=np.uint64), seed)).reshape(n, R, S)
    assert torch.equal(render_grad.hash_uniform(n * R * S, seed, 'cpu').reshape(n, R, S), u_ref)
    pts, zv, d = orr.initial_rays(n, S, 18.0, res, 2.25, 3.3)
    _, z_ref = orr.perturb(pts, zv, d, u_ref.unsqueeze(-1))
    z = render.coarse_depths(n, res, S, 2.25, 3.3, jitter_seed=seed, device='cpu')
    assert z.shape == (n, R, S) and (z - z_ref.reshape(n, R, S)).abs().max() <= 1e-6
    g = torch.Generator().manual_seed(0)
    u = torch.rand(n, R, S, generator=g)
    _, z_ref2 = orr.perturb(pts, zv, d, u.unsqueeze(-1))
    assert (render.coarse_depths(n, res, S, 2.25, 3.3, jitter_u=u, device='cpu') - z_ref2.reshape(n, R, S)).abs().max() <= 1e-6
    assert torch.equal(render.coarse_depths(1, res, S, 2.25, 3.3, device='cpu')[0, 0], torch.linspace(2.25, 3.3, S))
