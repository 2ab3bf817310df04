"""Oracle (test infrastructure): seeded loss networks and portraits for the encoder-training traces, the CPU route of
ide3d_b200.train_encoder, and one training step in the reference script's own structure.

    VGG_CFG / standin_vgg19()       torchvision's VGG19 feature layout (the same 37 modules, so the taps (2, 7, 12, 21, 30) fall on
                                    the same ReLUs) at an eighth of its widths, drawn under torch.manual_seed(VGG_SEED): the full
                                    network at 512^2 would make a CPU trace take minutes
    irse50_state(net, seed)         every tensor of an IR-SE50 state_dict (reference or product: same names) from a numpy RandomState,
                                    BatchNorm statistics and PReLU slopes included
    write_portraits(root, n, seed)  n portraits in the script's dataset layout: images/img%08d.png with dataset.json (OpenCV labels),
                                    segs/img%08d.png class ids (some >= 19), at 512^2 except image 1 (448^2, resized on load)
    cpu_train_ops()                 inside the context, the product's kernels are torch restatements (oracle.finetune.cpu_finetune_ops,
                                    the LPIPS head and the VGG L1 head in torch ops) so train_encoder runs on the CPU
    reference_step(...)             one step of train_hybrid_encoder.py:254-334 in the script's structure: the full E twice per branch,
                                    BiSeNet twice per image, the float one-hot masks and torch's heads

tests/golden/make_encoder_train_golden.py runs the reference's train() with these; tests/test_train_encoder.py replays it.
"""

import contextlib
import json
import math
import os

import numpy as np
import torch
import torch.nn.functional as F

from . import finetune as of

VGG_SEED = 61
IRSE_SEED = 62
VGG_CFG = [8, 8, 'M', 16, 16, 'M', 32, 32, 32, 32, 'M', 64, 64, 64, 64, 'M', 64, 64, 64, 64, 'M']
OPENCV_FLIP = [1, 2, 5, 6, 9, 10]


def standin_vgg19():
    import torchvision
    state = torch.random.get_rng_state()
    torch.manual_seed(VGG_SEED)
    try:
        net = torchvision.models.VGG(torchvision.models.vgg.make_layers(VGG_CFG), init_weights=True)
    finally:
        torch.random.set_rng_state(state)
    for m in net.features:                                  # the default init zeroes the biases; seeded biases make them count
        if isinstance(m, torch.nn.Conv2d):
            with torch.no_grad():
                m.bias.copy_(torch.linspace(-0.05, 0.05, m.bias.numel()))
    return net.eval()


def irse50_state(net, seed=IRSE_SEED):
    rs = np.random.RandomState(seed)
    out = {}
    for name, v in net.state_dict().items():
        shape = tuple(v.shape)
        if name.endswith('num_batches_tracked'):
            out[name] = v.clone()
            continue
        if v.ndim == 4:
            a = rs.randn(*shape) * math.sqrt(1.0 / (shape[1] * shape[2] * shape[3]))
        elif v.ndim == 2:
            a = rs.randn(*shape) * math.sqrt(1.0 / shape[1])
        elif name.endswith('running_var'):
            a = 0.5 + rs.rand(*shape)
        elif name.endswith('weight') and 'res_layer.2' not in name and 'input_layer.2' not in name:
            a = 1.0 + 0.1 * rs.randn(*shape)
        elif name.endswith('weight'):                        # PReLU slopes
            a = 0.25 + 0.05 * rs.randn(*shape)
        else:
            a = 0.1 * rs.randn(*shape)
        out[name] = torch.from_numpy(a.astype(np.float32))
    return out


def write_portraits(root, n=6, seed=71):
    """(images dir, segs dir, OpenGL labels [n, 25]).  Images are smooth random colour fields; masks are blocky class ids."""
    from PIL import Image
    rs = np.random.RandomState(seed)
    img_dir, seg_dir = os.path.join(root, 'images'), os.path.join(root, 'segs')
    os.makedirs(img_dir)
    os.makedirs(seg_dir)
    labels = {}
    opengl = []
    for i in range(n):
        size = 448 if i == 1 else 512
        coarse = torch.from_numpy(rs.rand(1, 3, 8, 8).astype(np.float32))
        img = F.interpolate(coarse, size=(size, size), mode='bicubic', align_corners=False).clamp(0, 1)[0]
        Image.fromarray((img.permute(1, 2, 0).numpy() * 255).round().astype(np.uint8)).save(os.path.join(img_dir, f'img{i:08d}.png'))
        ids = np.kron(rs.randint(0, 21, size=(16, 16)), np.ones((size // 16, size // 16), np.int64)).astype(np.uint8)
        Image.fromarray(ids).save(os.path.join(seg_dir, f'img{i:08d}.png'))
        yaw, pitch = 0.3 * rs.randn(), 0.1 * rs.randn()
        cam = np.eye(4)
        cam[:3, :3] = np.array([[math.cos(yaw), 0, math.sin(yaw)], [0, 1, 0], [-math.sin(yaw), 0, math.cos(yaw)]]) @ \
            np.array([[1, 0, 0], [0, math.cos(pitch), -math.sin(pitch)], [0, math.sin(pitch), math.cos(pitch)]])
        cam[:3, 3] = cam[:3, 2] * 2.7
        label = np.concatenate([cam.reshape(-1), [4.2647, 0, 0.5, 0, 4.2647, 0.5, 0, 0, 1]])
        opengl.append(label.copy())
        label[OPENCV_FLIP] *= -1
        labels[f'img{i:08d}.png'] = label.tolist()
    with open(os.path.join(img_dir, 'dataset.json'), 'w') as f:
        json.dump({'labels': list(labels.items())}, f)
    return img_dir, seg_dir, np.array(opengl, np.float32)


@contextlib.contextmanager
def cpu_train_ops():
    from ide3d_b200.torch_utils.ops import lpips as LP, vgg_loss as V
    saved = (LP.lpips_head, V.feat_l1)
    LP.lpips_head, V.feat_l1 = LP.lpips_head_torch, V.feat_l1_torch
    try:
        with of.cpu_finetune_ops():
            yield
    finally:
        LP.lpips_head, V.feat_l1 = saved


def reference_step(G, E, parser, *, lambdas, w_avg, z=None, cam=None, real=None, start_from_latent_avg=False, vgg=None, lpips=None,
                   id_net=None, truncation=1.0):
    """train_hybrid_encoder.py:254-334 in the script's structure on any device, for explicit inputs (as train_encoder.step_losses
    takes them): E's full forward on the float one-hot maps (twice per branch), BiSeNet on the upsampled logits twice per image, the
    VGG head as per-layer F.l1_loss, the ID features of the target extracted per call.  Returns the loss terms; vgg / lpips / id_net
    are the product's modules, called the script's way."""
    from ide3d_b200.torch_utils.ops import vgg_loss as V
    remap = of.REMAP.to(w_avg.device)
    out = {}

    def scatter(ids):
        return torch.zeros(ids.shape[0], 19, *ids.shape[-2:], device=ids.device).scatter_(1, ids, 1)

    def parse(img):
        return remap[parser(img)[0].argmax(1, keepdim=True)]

    def cycle(rec, img, rec_img):
        return F.smooth_l1_loss(rec, E(img, scatter(parse(rec_img))))

    if z is not None:
        front = torch.tensor([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 2.7, 0, 0, 0, 1, 4.2647, 0, 0.5, 0, 4.2647, 0.5, 0, 0, 1],
                             dtype=torch.float32, device=z.device).reshape(1, -1).repeat(len(z), 1)
        w = G.mapping(z, front)
        if truncation < 1.0:
            w = w_avg + (w - w_avg) * truncation
        gen_img = G.synthesis(w, c=cam, noise_mode='const')
        with torch.no_grad():
            gen_seg = scatter(parse(gen_img)) * 2 - 1
        rec = E(gen_img, gen_seg)
        if start_from_latent_avg:
            rec = rec + w_avg.repeat(rec.shape[0], 1, 1)
        out['loss_ws'] = F.smooth_l1_loss(rec, w).mean() * 50.
        rec_img = G.synthesis(rec, c=cam, noise_mode='const')
        out['loss_gen_l2'] = F.mse_loss(rec_img, gen_img) * lambdas['l2']
        out['loss_gen_entropy'] = torch.nn.CrossEntropyLoss()(parser(rec_img)[0], parser(gen_img)[0].argmax(1)) * lambdas['entropy']
        out['loss_cycle'] = cycle(rec, gen_img, rec_img) * lambdas['cycle']
    if real is not None:
        img_u8, ids, label = real
        img = img_u8.to(torch.float32) / 127.5 - 1
        seg = F.one_hot(ids.long().clamp(max=19), 20)[..., :19].permute(0, 3, 1, 2).float() * 2 - 1
        rec = E(img, seg)
        if start_from_latent_avg:
            rec = rec + w_avg
        rec_img = G.synthesis(rec, c=label, noise_mode='const')
        if vgg is not None:
            with torch.no_grad():
                target = vgg.trunk(img)
            out['loss_vgg'] = V.feat_l1_torch(vgg.trunk(rec_img), target, vgg.weights)[0] * lambdas['vgg']
        out['loss_real_l2'] = F.mse_loss(rec_img, img) * lambdas['l2']
        if lpips is not None:
            out['loss_lpips'] = lpips(rec_img, img).sum() / img.shape[0] * lambdas['lpips']
        if id_net is not None:
            f_hat, f_y = id_net.extract_feats(rec_img), id_net.extract_feats(img).detach()
            out['loss_id'] = sum(1 - f_hat[i].dot(f_y[i]) for i in range(len(img))) / len(img) * lambdas['id']
        out['loss_real_entropy'] = torch.nn.CrossEntropyLoss()(parser(rec_img)[0], parser(img)[0].argmax(1)) * lambdas['entropy']
        out['loss_real_cycle'] = cycle(rec, img, rec_img) * lambdas['cycle']
    return out
