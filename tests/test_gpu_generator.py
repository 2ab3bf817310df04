"""GPU parity of the WHOLE synthesis path: TriPlaneGenerator.synthesis on cuda (NHWC backbone, chained epilogues, TMA FIR,
fused skip step, tensor-core / fp32 ray-march, SR blocks) against the same module evaluated by the CPU oracle in the reference's
layout (oracle.backend.cpu_reference_ops: NCHW, reference op chain).  cuDNN tf32 is switched off for the comparison so that
the convolutions are fp32 on both sides.  Tolerances are relative to max|tensor| (2.5 ... 5.9 here): 1e-4 on the 128^2 image and
semantic maps and on the 32^2 feature image, 2e-5 on depth, 1 uint8 level on the final frames -- the same for NHWC / NCHW, chained /
unchained epilogues and the optional matmul form of the 1x1 convolutions."""

import pytest
import torch

from conftest import assert_close
from oracle.backend import cpu_reference_ops

pytestmark = pytest.mark.gpu
LABEL = [1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 2.7, 0, 0, 0, 1, 4.2647, 0, 0.5, 0, 4.2647, 0.5, 0, 0, 1]


@pytest.fixture(scope='module')
def case():
    from ide3d_b200.training.triplane import TriPlaneGenerator
    torch.manual_seed(0)
    G = TriPlaneGenerator(z_dim=32, w_dim=32, img_resolution=128, plane_resolution=64, render_size=32, channel_base=2048, channel_max=64,
                          sr_channels=(32, 32), mapping_kwargs=dict(num_layers=2)).eval().requires_grad_(False)
    for name, p in G.named_parameters():                        # non-trivial noise so that the noise path is exercised
        if name.endswith('noise_strength'):
            p.data.fill_(0.1)
    z = torch.randn(2, G.z_dim, generator=torch.Generator().manual_seed(5))
    c = torch.tensor(LABEL).repeat(2, 1)
    c[1, 3] = 0.15                                              # second camera slightly off-axis
    kw = dict(noise_mode='const', num_steps=24, perturb=None)
    with torch.no_grad(), cpu_reference_ops():
        ws = G.mapping(z, c, truncation_psi=0.7)
        ref = G.synthesis(ws, c=c, return_dict=True, **kw)
    return G, ws, c, kw, ref


@pytest.mark.parametrize('channels_last,chain,mm', [(True, True, False), (True, True, True), (False, True, False), (True, False, False)])
def test_synthesis_on_gpu_matches_cpu_oracle(case, channels_last, chain, mm):
    from ide3d_b200.training import networks as nw
    G, ws, c, kw, ref = case
    Gd = G.cuda()
    saved = (nw.CHANNELS_LAST, nw.CHAIN_MODULATION, nw.CONV1X1_AS_MATMUL, torch.backends.cudnn.allow_tf32)
    try:
        nw.CHANNELS_LAST, nw.CHAIN_MODULATION, nw.CONV1X1_AS_MATMUL = channels_last, chain, mm
        torch.backends.cudnn.allow_tf32 = False
        with torch.no_grad():
            out = Gd.synthesis(ws.cuda(), c=c.cuda(), return_dict=True, **kw)
    finally:
        nw.CHANNELS_LAST, nw.CHAIN_MODULATION, nw.CONV1X1_AS_MATMUL, torch.backends.cudnn.allow_tf32 = saved
        G.cpu()
    report = {}
    for key, tol in (('image_raw', 1e-4), ('image_depth', 2e-5), ('image', 1e-4), ('image_seg', 1e-4)):
        a, b = out[key].float().cpu(), ref[key].float()
        scale = max(1.0, b.abs().max().item())
        report[key] = ((a - b).abs().max().item(), scale, tol)
    print('synthesis parity (max abs err, scale, tol):', report)
    for key, (err, scale, tol) in report.items():
        assert err <= tol * scale, (key, report)
    to8 = lambda t: (t * 127.5 + 128).clamp(0, 255).to(torch.uint8).int()
    assert (to8(out['image'].float().cpu()) - to8(ref['image'])).abs().max() <= 1


@pytest.mark.parametrize('channels_last', [True, False])
def test_blocks_on_gpu_reproduce_recorded_reference_classes(channels_last):
    """tests/golden/networks.npz (outputs of the reference's own MappingNetwork / SynthesisBlock / SegSynthesisBlock, see
    tests/test_oracle_golden.py) replayed through the CUDA path: same state_dicts, sm_90a ops, fp32 convolutions."""
    import numpy as np
    from conftest import load_golden
    from ide3d_b200.training import networks as nw
    g = load_golden('networks')
    T_ = lambda k: torch.from_numpy(np.asarray(g[k])).cuda()
    sd = lambda prefix: {k[len(prefix) + 1:]: torch.from_numpy(np.asarray(g[k])) for k in g if k.startswith(prefix + '/')}
    saved = (nw.CHANNELS_LAST, torch.backends.cudnn.allow_tf32)
    try:
        nw.CHANNELS_LAST, torch.backends.cudnn.allow_tf32 = channels_last, False
        with torch.no_grad():
            mm = nw.MappingNetwork(z_dim=16, c_dim=25, w_dim=12, num_ws=5, num_layers=2).eval()
            mm.load_state_dict(sd('map'))
            mm.cuda()
            assert (mm(T_('map_z'), T_('map_c'), truncation_psi=0.7, truncation_cutoff=3) - T_('map_ws')).abs().max() < 1e-5
            for tag, in_ch in (('b0', 0), ('b1', 16)):
                mb = nw.SynthesisBlock(in_ch, 8, w_dim=12, resolution=16, img_channels=6, is_last=False).eval()
                mb.load_state_dict(sd(tag))
                mb.cuda()
                xo, io = mb(T_(f'{tag}_x') if in_ch else None, T_(f'{tag}_img').clone() if in_ch else None, T_(f'{tag}_ws'), noise_mode='const')
                for got, key in ((xo, f'{tag}_eval_x'), (io, f'{tag}_eval_img')):
                    ref = T_(key)
                    assert (got.float() - ref).abs().max() <= 1e-4 * max(1.0, ref.abs().max().item()), (key, channels_last)
            ms = nw.SegSynthesisBlock(16, 8, w_dim=12, resolution=16, img_channels=6, seg_channels=4, is_last=False).eval()
            ms.load_state_dict(sd('seg'))
            ms.cuda()
            outs = ms(T_('seg_x'), T_('seg_img').clone(), T_('seg_ws'), condition_img=T_('seg_seg').clone(), noise_mode='const')
            for got, key in zip(outs, ('seg_out_x', 'seg_out_img', 'seg_out_seg')):
                ref = T_(key)
                assert (got.float() - ref).abs().max() <= 1e-4 * max(1.0, ref.abs().max().item()), (key, channels_last)
    finally:
        nw.CHANNELS_LAST, torch.backends.cudnn.allow_tf32 = saved


def test_stream_frames_matches_batch_loop_and_lands_in_pinned_host_memory(case):
    """dist.stream_frames_sharded (H2D from pinned inputs, render, uint8, D2H on a side stream overlapping the next batch) returns the
    same frames as the plain batch loop render_frames_sharded; result lives in page-locked host memory."""
    from ide3d_b200 import dist as idist
    G, ws, c, kw, ref = case
    Gd = G.cuda()
    try:
        ws4, c4 = ws.repeat(2, 1, 1).pin_memory(), c.repeat(2, 1).pin_memory()
        skw = dict(noise_mode='const', num_steps=24, perturb=None)
        streamed = idist.stream_frames_sharded(Gd, ws4, c4, 0, 1, batch=2, **skw)
        looped = idist.render_frames_sharded(Gd, ws4.cuda(), c4.cuda(), 0, 1, batch=4, **skw)
    finally:
        G.cpu()
    assert streamed.dtype == torch.uint8 and streamed.device.type == 'cpu' and streamed.is_pinned() and tuple(streamed.shape) == (4, 3, 128, 128)
    assert (streamed.int() - looped.cpu().int()).abs().max() <= 1            # batch 2 vs batch 4: cuDNN may pick different algorithms
    # the two halves are the same inputs rendered as two batches of the same size: bit-identical (scripts/determinism.py: every stage
    # is run-to-run bit-equal under all cudnn.benchmark / cudnn.deterministic settings; a one-level difference comes only from
    # comparing DIFFERENT batch sizes, above)
    assert torch.equal(streamed[:2], streamed[2:])


def test_style_plan_matches_per_layer_styles():
    """networks.StylePlan (ide3d_style_plan: every style vector and demodulation coefficient of the call in two launches) against the
    per-layer computation it replaces (FullyConnectedLayer affine + the dcoefs reduction of modulated_conv2d): same values, same image."""
    from ide3d_b200.compat import random_init_generator
    from ide3d_b200.training import networks
    G = random_init_generator(device='cuda', seed=3, img_resolution=128, plane_resolution=64, render_size=16, channel_max=64)
    torch.manual_seed(0)
    # non-trivial affine biases / noise strengths so that every term of the formula is exercised
    with torch.no_grad():
        for m in G.synthesis.modules():
            if isinstance(m, (networks.SynthesisLayer, networks.ToRGBLayer)):
                m.affine.bias.add_(0.3 * torch.randn_like(m.affine.bias))
    saved_tf32, torch.backends.cudnn.allow_tf32 = torch.backends.cudnn.allow_tf32, False      # TF32 convolutions amplify 1e-7 input differences to 1e-3
    z = torch.randn(3, G.z_dim, device='cuda')
    c = torch.eye(4, device='cuda').reshape(1, 16).repeat(3, 1); c[:, 11] = 2.7
    c = torch.cat([c, torch.zeros(3, 9, device='cuda')], 1)
    with torch.no_grad():
        ws = G.mapping(z, c)
        ws = ws + 0.1 * torch.randn_like(ws)                      # a different w per layer
        plan = G.synthesis._style_plan(ws)
        assert plan is not None
        voxel_ws, block_ws = G.synthesis.split_ws(ws)
        blocks = [getattr(G.synthesis, f'vb{r}') for r in G.synthesis.voxel_block_resolutions] + [getattr(G.synthesis, f'b{r}') for r in G.synthesis.block_resolutions]
        for blk, bws in zip(blocks, voxel_ws + block_ws):
            w_iter = iter(bws.unbind(1))
            layers = ([blk.conv0] if blk.in_channels != 0 else []) + [blk.conv1]
            for layer in layers:
                w = next(w_iter)
                s_ref = layer.affine(w)
                d_ref = (s_ref.square() @ layer.weight.square().sum(dim=[2, 3]).t() + 1e-8).rsqrt()
                s, d = plan[layer]
                assert_close(s, s_ref, 1e-5 * float(s_ref.abs().max()), what='styles'); assert_close(d, d_ref, 1e-5 * float(d_ref.abs().max()), what='dcoefs')
            s, d = plan[blk.torgb]
            assert d is None
            assert_close(s, blk.torgb.styles(next(w_iter)), 1e-6, what='torgb styles')
        a = G.synthesis(ws, c=c, perturb=None)
        saved, networks.STYLE_PLAN = networks.STYLE_PLAN, False
        try:
            b = G.synthesis(ws, c=c, perturb=None)
        finally:
            networks.STYLE_PLAN = saved
            torch.backends.cudnn.allow_tf32 = saved_tf32
    assert_close(a, b, 2e-5 * float(b.abs().max()), what='image with / without the style plan')
