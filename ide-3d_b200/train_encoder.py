"""Train the hybrid encoder for a generator (apps/train_hybrid_encoder.py:155-392): the step that makes the HybridEncoder the rest of the
editing workflow (edit.encode / edit.edit, finetune.run) needs, for any generator.

    train(G, E=None, *, parser, steps, batch=8, lr=1e-4, lambdas=None, truncation=1.0, start_from_latent_avg=False, train_gen=True,
          train_real=False, dataset=None, vgg=None, lpips=None, id_net=None, rank=0, world=1, seed=0, snapshot_every=0, outdir=None,
          resume=None) -> (E_trained, losses {name: np.ndarray [steps]})
    step_losses(G, enc, *, parser, lambdas, ...)   one step's loss terms from explicit latents, cameras and real batch
    PortraitDataset(path, seg_path, resolution)    the script's dataset layout as (uint8 [3, H, W], uint8 ids [H, W], float32 [25])
    cam_sampler(batch, device, generator=None)     the script's camera draw (:72-78)

lambdas take the script's names (vgg, l2, adv, lpips, id, entropy, cycle), 0 by default; loss_ws keeps its fixed weight 50.  adv must
be 0: the script computes no adversarial term.  E=None builds HybridEncoder(G.img_resolution, G.num_ws - 8, 8, G.w_dim) on the CPU
under torch.manual_seed(seed) (:181, :208) without touching the global RNG.  Adam(lr, betas (0.9, 0.99)) trains every parameter of E.
parser is a parsing.BiSeNet; vgg a torch_utils.ops.vgg_loss.VGGLoss, lpips a torch_utils.ops.lpips.LPIPS, id_net an arcface.IDLoss,
each required only when its lambda is non-zero.  Per step, with the script's weights and order:
    synthetic (:254-289)  z ~ randn(batch, w_dim) mapped with the frontal label (truncated towards w_avg when truncation < 1), a
                          gaussian camera (stddev 0.3 / 0.155, r 2.7), gen_img = G.synthesis(w, c, noise_mode='const'):
                          loss_ws 50 smooth_l1(rec, w), loss_gen_l2, loss_gen_entropy, loss_cycle
    real (:292-334)       one batch of the dataset: loss_vgg, loss_real_l2, loss_lpips (LPIPS's mean over the batch), loss_id,
                          loss_real_entropy, loss_real_cycle
rec = E(img, seg) (+ w_avg with start_from_latent_avg); the cycle compares rec with E(img, remapped parse of rec's render).

What differs from the script (each exact, or a change of rounding only):
    - BiSeNet runs once per image: without grad on gen_img / real_img, giving the cross-entropy's labels (no remap) and the encoder's
      mask (remapped); with grad on the render, whose logits feed both the align_corners=True cross-entropy (ide3d_seg_xent_*_ac)
      and the cycle's parse.  The script runs it twice on each;
    - masks enter the encoder as uint8 ids through the one-byte stem and its backward: the target as one_hot * 2 - 1, the cycle's
      parse as the {0, 1} one-hot (signed=False); masks are parsed at the image's size (face_parsing's resize to 512^2 is a no-op at
      the released 512^2);
    - E's image branch runs once per branch: the cycle reuses the appearance tensor itself, not detached.  The cycle's two gradient
      contributions to those rows are equal and opposite and cancel at the tensor, where the script's cancel in param.grad; the
      loss value, including the w_avg offset those rows carry with start_from_latent_avg, is unchanged;
    - the real branch's targets are computed once per step: the VGG features (no-grad in the script too), LPIPS.target(real_img)
      and the ID features of real_img, which the script's IDLoss extracts twice;
    - a term whose lambda is 0 is not computed and is recorded as 0 (the script multiplies it by 0); the render is skipped when no
      term needs it, and BiSeNet on real_img when the cross-entropy's lambda is 0;
    - dead code is dropped: return_raw=True and its F.interpolate (unused), the discriminator, tensorboard and the sample grids;
    - snapshots are torch.save'd dicts (encoder-snapshot-{step:06d}.pt: E's state_dict and constructor arguments, the Adam state, the
      step count, every rank's two stream states, the data position and the run's seed, world, batch and branches), not pickles that
      embed class source; `resume=` continues from one, each rank from its own streams, and refuses a run with other parameters.
Multiple GPUs: one process per GPU (dist.init_from_env), E wrapped in DistributedDataParallel, each rank taking batch // world
samples.  At world == 1 and seed == 0 the latent, camera and data streams equal the script's draw for draw.  At world > 1 the script
trains every rank on the same latents and real images (np.random.seed(0) on every rank, InfiniteSampler(rank=local_rank), always 0);
only its cameras differ.  Here rank r draws latents and cameras from seed + r and reads its own share of the sampler.  The loop draws
from its own np.random.RandomState and a device torch.Generator and never reseeds the global RNGs.
The caller's G and E are not modified: E_trained is a copy, returned in eval mode without grad.
"""

import copy
import json
import math
import os
import zipfile

import numpy as np
import torch
import torch.nn.functional as F

from .encoder import HybridEncoder
from .parsing import remap_ids
from .torch_utils.misc import InfiniteSampler
from .torch_utils.ops import projection
from .torch_utils.ops import seg_stem as _seg_ops
from .training.triplane import invalidate_caches
from .training.volumetric_rendering import create_cam2world_matrix, sample_camera_positions

LAMBDAS = ('vgg', 'l2', 'adv', 'lpips', 'id', 'entropy', 'cycle')
GEN_LOSSES = ('loss_ws', 'loss_gen_l2', 'loss_gen_entropy', 'loss_cycle')
REAL_LOSSES = ('loss_vgg', 'loss_real_l2', 'loss_lpips', 'loss_id', 'loss_real_entropy', 'loss_real_cycle')
WS_WEIGHT = 50.0                                                                   # :272
INTRINSICS = (4.2647, 0, 0.5, 0, 4.2647, 0.5, 0, 0, 1)
FRONTAL = (1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 2.7, 0, 0, 0, 1) + INTRINSICS          # :257
LABEL_FLIP = [1, 2, 5, 6, 9, 10]                                                   # training/dataset_seg.py:314, OpenCV -> OpenGL


def cam_sampler(batch, device, generator=None):
    """[batch, 25] camera labels: gaussian yaw / pitch around the front (stddev 0.3 / 0.155) on a sphere of radius 2.7 (:72-78)."""
    pts, _, _ = sample_camera_positions(device, n=batch, r=2.7, horizontal_mean=0.5 * math.pi, vertical_mean=0.5 * math.pi,
                                        horizontal_stddev=0.3, vertical_stddev=0.155, mode='gaussian', generator=generator)
    c = create_cam2world_matrix(-pts, pts, device=device).reshape(batch, -1)
    return torch.cat((c, torch.tensor(INTRINSICS, device=c.device).reshape(1, -1).repeat(batch, 1).to(c)), -1)


# ------------------------------------------------------------------------------------------------------------------------------ data
class _Files:
    """A directory or a zip, by relative name."""

    def __init__(self, path):
        self.path = os.fspath(path)
        if os.path.isdir(self.path):
            self.zip = None
            self.names = {os.path.relpath(os.path.join(root, f), start=self.path) for root, _, files in os.walk(self.path) for f in files}
        elif os.path.splitext(self.path)[1].lower() == '.zip':
            self.zip = zipfile.ZipFile(self.path)
            self.names = set(self.zip.namelist())
        else:
            raise IOError(f'PortraitDataset: {self.path!r} must be a directory or a zip')

    def open(self, name):
        return self.zip.open(name, 'r') if self.zip is not None else open(os.path.join(self.path, name), 'rb')

    def images(self):
        """Image names in sorted order, those numbered >= 140000 left out (dataset_seg.py:227-229, non_rebalance)."""
        import PIL.Image
        PIL.Image.init()
        names = sorted(n for n in self.names if os.path.splitext(n)[1].lower() in PIL.Image.EXTENSION)
        for n in names:
            if not n[-12:-4].isdigit():
                raise ValueError(f'PortraitDataset: {n!r} does not end in an 8-digit number, as dataset_tool.py names images')
        return [n for n in names if int(n[-12:-4]) < 140000]


class PortraitDataset(torch.utils.data.Dataset):
    """CameraLabeledDataset(load_seg=True, use_labels=True, xflip=False) of training/dataset_seg.py:160-395: images from `path` (a
    directory or zip), seg PNGs from the parallel `seg_path`, camera labels from path's dataset.json with the OpenCV -> OpenGL sign flip.
    Images are PIL-resized to `resolution` when their size differs, seg maps with NEAREST.  item i -> (uint8 [3, H, W], uint8 class ids
    [H, W], float32 [25]); the script's float64 one-hot is never built: ids stand for one_hot * 2 - 1 in the encoder, an id >= 19 for -1
    in every channel.  The seg zip is read from seg_path (the script's zip branch reads the image zip instead)."""

    def __init__(self, path, seg_path, resolution):
        self.resolution = int(resolution)
        self._img, self._seg = _Files(path), _Files(seg_path)
        self._image_names, self._seg_names = self._img.images(), self._seg.images()
        if not self._image_names:
            raise IOError(f'PortraitDataset: no image files in {self._img.path!r}')
        if len(self._seg_names) != len(self._image_names):
            raise ValueError(f'PortraitDataset: {len(self._image_names)} images but {len(self._seg_names)} seg maps')
        if 'dataset.json' not in self._img.names:
            raise ValueError(f'PortraitDataset: {self._img.path!r} has no dataset.json with the camera labels')
        with self._img.open('dataset.json') as f:
            labels = json.load(f)['labels']
        if labels is None:
            raise ValueError('PortraitDataset: dataset.json has no labels')
        labels = dict(labels)
        labels = np.array([labels[n.replace('\\', '/')] for n in self._image_names])
        if labels.ndim != 2 or labels.shape[1] != 25:
            raise ValueError(f'PortraitDataset: camera labels must be [N, 25], got {labels.shape}')
        labels[:, LABEL_FLIP] *= -1
        self.labels = labels.astype(np.float32)

    def __len__(self):
        return len(self._image_names)

    def _read(self, files, name, seg):
        import PIL.Image
        with files.open(name) as f:
            im = PIL.Image.open(f)
            if seg:
                im = im.convert('L')
            if im.size != (self.resolution, self.resolution):
                im = im.resize((self.resolution, self.resolution), **({'resample': PIL.Image.NEAREST} if seg else {}))
            return np.array(im)

    def __getitem__(self, idx):
        image = self._read(self._img, self._image_names[idx], False)
        if image.ndim != 3 or image.shape[2] != 3:
            raise ValueError(f'PortraitDataset: {self._image_names[idx]!r} is not an RGB image ({image.shape})')
        seg = self._read(self._seg, self._seg_names[idx], True)
        return (torch.from_numpy(np.ascontiguousarray(image.transpose(2, 0, 1))), torch.from_numpy(seg),
                torch.from_numpy(self.labels[idx].copy()))


# ------------------------------------------------------------------------------------------------------------------------------ step
class _Encode(torch.nn.Module):
    """The encoder's two branches behind one forward, so that every use goes through DistributedDataParallel's forward."""

    def __init__(self, E):
        super().__init__()
        self.E = E

    def forward(self, branch, x, signed=True):
        if branch == 'geometry':
            return self.E.geometry(x, signed=signed)
        app = self.E.appearance(x)
        return app[0] if isinstance(app, tuple) else app


def _parse(parser, img):
    """BiSeNet without grad: (argmax ids for the cross-entropy, the remapped mask for the encoder)."""
    with torch.no_grad():
        labels = _seg_ops.seg_labels(parser.logits(img), tuple(img.shape[-2:]), align_corners=True)
    return labels, remap_ids(labels)


def _render_terms(G, enc, parser, rec, app, img, labels, label, lam, names, perceptual=None, perceptual_lambdas=()):
    """The render of rec and the terms computed from it: perceptual(render) (the real branch's VGG / LPIPS / ID), then the l2,
    entropy and cycle terms under `names`.  The render is skipped when every lambda that needs it is 0."""
    l2, entropy, cycle = names
    zero = rec.new_zeros(())
    out = {l2: zero, entropy: zero, cycle: zero}
    if not (lam['l2'] or lam['entropy'] or lam['cycle'] or any(lam[k] for k in perceptual_lambdas)):
        return out
    rec_img = G.synthesis(rec, c=label, noise_mode='const')
    if perceptual is not None:
        out.update(perceptual(rec_img))
    if lam['l2']:
        out[l2] = F.mse_loss(rec_img, img) * lam['l2']
    if lam['entropy'] or lam['cycle']:
        logits = parser.logits(rec_img)
        if lam['entropy']:
            out[entropy] = projection.seg_cross_entropy(logits, labels, align_corners=True) * lam['entropy']
        if lam['cycle']:
            with torch.no_grad():
                parse = remap_ids(_seg_ops.seg_labels(logits, tuple(img.shape[-2:]), align_corners=True))
            out[cycle] = F.smooth_l1_loss(rec, torch.cat((enc('geometry', parse, signed=False), app), 1)) * lam['cycle']
    return out


def step_losses(G, enc, *, parser, lambdas, z=None, cam=None, real=None, truncation=1.0, start_from_latent_avg=False, vgg=None,
                lpips=None, id_net=None):
    """One step's loss terms {name: 0-d tensor}, in the script's order, for explicit inputs: z [B, w_dim] and cam [B, 25] (the
    synthetic branch, skipped when z is None) and real = (uint8 images [B, 3, H, W], uint8 ids [B, H, W], labels [B, 25]) (the real
    branch, skipped when None), all on G's device.  enc(branch, x, signed=True) runs E's 'geometry' or 'appearance' branch (an _Encode,
    or one wrapped in DistributedDataParallel).  The caller sums the terms and runs the backward."""
    lam = {k: float(lambdas.get(k, 0.0)) for k in LAMBDAS}
    w_avg = G.mapping.w_avg[None, None, :]
    out = {}

    def encode(img, seg):
        app = enc('appearance', img)
        rec = torch.cat((enc('geometry', seg), app), 1)
        return (rec + w_avg if start_from_latent_avg else rec), app

    if z is not None:
        with torch.no_grad():
            front = torch.tensor(FRONTAL, dtype=torch.float32, device=z.device).reshape(1, -1).repeat(len(z), 1)
            w = G.mapping(z, front)
            if truncation < 1.0:
                w = w_avg + (w - w_avg) * truncation
            gen_img = G.synthesis(w, c=cam, noise_mode='const')
            labels, seg = _parse(parser, gen_img)
        rec, app = encode(gen_img, seg)
        out['loss_ws'] = F.smooth_l1_loss(rec, w) * WS_WEIGHT
        out.update(_render_terms(G, enc, parser, rec, app, gen_img, labels, cam, lam, GEN_LOSSES[1:]))

    if real is not None:
        img_u8, seg, label = real
        img = img_u8.to(torch.float32) / 127.5 - 1.
        labels = _parse(parser, img)[0] if lam['entropy'] else None        # the cross-entropy's targets, its only use
        with torch.no_grad():
            t_vgg = vgg.target(img) if lam['vgg'] else None
            t_lpips = lpips.target(img) if lam['lpips'] else None
            t_id = id_net.target(img) if lam['id'] else None
        rec, app = encode(img, seg)
        zero = rec.new_zeros(())

        def perceptual(rec_img):
            return {'loss_vgg': vgg(rec_img, t_vgg) * lam['vgg'] if lam['vgg'] else zero,
                    'loss_lpips': lpips(rec_img, t_lpips).mean() * lam['lpips'] if lam['lpips'] else zero,
                    'loss_id': id_net(rec_img, t_id) * lam['id'] if lam['id'] else zero}

        terms = {'loss_vgg': zero, 'loss_lpips': zero, 'loss_id': zero}
        terms.update(_render_terms(G, enc, parser, rec, app, img, labels, label, lam, REAL_LOSSES[1:2] + REAL_LOSSES[4:],
                                   perceptual, ('vgg', 'lpips', 'id')))
        out.update({k: terms[k] for k in REAL_LOSSES})
    return out


# ------------------------------------------------------------------------------------------------------------------------------ loop
def _encoder_args(E):
    return dict(size=E.size, n_latents_app=E.n_latents_app, n_latents_geo=E.n_latents_geo, w_dim=E.w_dim, add_dim=E.add_dim,
                input_img_dim=E.convs_img[0].weight.shape[1], input_seg_dim=E.input_seg_dim)


def _np_state(rs):
    name, keys, pos, has_gauss, gauss = rs.get_state()
    return dict(name=name, keys=torch.from_numpy(keys.astype(np.int64)), pos=int(pos), has_gauss=int(has_gauss), gauss=float(gauss))


def _set_np_state(rs, s):
    rs.set_state((s['name'], s['keys'].numpy().astype(np.uint32), s['pos'], s['has_gauss'], s['gauss']))


def _rank_states(rs, gen, world):
    """Every rank's (numpy, device generator) stream state, in rank order, on every rank."""
    mine = dict(np_rng=_np_state(rs), torch_rng=gen.get_state())
    if world == 1:
        return [mine]
    import torch.distributed as dist
    states = [None] * world
    dist.all_gather_object(states, mine)
    return states


def _check_lambdas(lambdas):
    lambdas = dict(lambdas or {})
    unknown = sorted(set(lambdas) - set(LAMBDAS))
    if unknown:
        raise ValueError(f'train_encoder: unknown lambdas {unknown}; the names are {LAMBDAS}')
    if lambdas.get('adv', 0.0) != 0.0:
        raise ValueError('train_encoder: lambdas["adv"] must be 0 (the script computes no adversarial term)')
    return {k: float(lambdas.get(k, 0.0)) for k in LAMBDAS}


def train(G, E=None, *, parser, steps, batch=8, lr=1e-4, lambdas=None, truncation=1.0, start_from_latent_avg=False, train_gen=True,
          train_real=False, dataset=None, vgg=None, lpips=None, id_net=None, rank=0, world=1, seed=0, snapshot_every=0, outdir=None,
          resume=None):
    """Run `steps` training steps (after the resumed snapshot's, with resume=) and return (E_trained, {name: np.ndarray [steps]}) with
    this rank's loss terms of the active branches.  At world > 1 the process group must be initialised (dist.init_from_env)."""
    import torch.distributed as dist
    lam = _check_lambdas(lambdas)
    steps, batch, world, rank = int(steps), int(batch), int(world), int(rank)
    if steps < 0:
        raise ValueError(f'train_encoder: steps must be >= 0, got {steps}')
    if not (train_gen or train_real):
        raise ValueError('train_encoder: train_gen or train_real must be set')
    if world < 1 or not 0 <= rank < world or batch < world:
        raise ValueError(f'train_encoder: rank {rank} of world {world} with batch {batch} (each rank takes batch // world >= 1)')
    if world > 1 and not (dist.is_available() and dist.is_initialized()):
        raise ValueError('train_encoder: world > 1 needs an initialised process group (dist.init_from_env)')
    if train_real:
        if dataset is None:
            raise ValueError('train_encoder: train_real needs a dataset (PortraitDataset)')
        for key, module in (('vgg', vgg), ('lpips', lpips), ('id', id_net)):
            if lam[key] and module is None:
                raise ValueError(f'train_encoder: lambdas["{key}"] = {lam[key]} needs the {key} module')
    if snapshot_every and outdir is None:
        raise ValueError('train_encoder: snapshot_every needs an outdir')

    dev = next(G.parameters()).device
    G = copy.deepcopy(G).eval().requires_grad_(False)
    snap = torch.load(os.fspath(resume), map_location='cpu', weights_only=True) if resume is not None else None
    if snap is not None:
        if E is not None:
            raise ValueError('train_encoder: resume= rebuilds the encoder from the snapshot; pass E=None')
        run = dict(seed=seed, world=world, batch=batch, train_gen=bool(train_gen), train_real=bool(train_real))
        saved = {k: snap['run'][k] for k in run}
        if saved != run:
            raise ValueError(f'train_encoder: the snapshot was written by a run with {saved}, this one has {run}: its random streams '
                             f'and data shares would not continue')
        with torch.random.fork_rng(devices=[]):
            E = HybridEncoder(**snap['encoder_args'])
        E.load_state_dict(snap['encoder'])
    elif E is None:
        with torch.random.fork_rng(devices=[]):
            torch.manual_seed(seed)
            E = HybridEncoder(G.img_resolution, G.num_ws - 8, 8, G.w_dim)
    else:
        E = copy.deepcopy(E)
    if E.n_latents_geo + E.n_latents_app != G.num_ws or E.w_dim != G.w_dim:
        raise ValueError(f'train_encoder: the encoder gives {E.n_latents_geo} + {E.n_latents_app} rows of {E.w_dim}, the generator '
                         f'takes {G.num_ws} of {G.w_dim}')
    E = E.to(dev).train().requires_grad_(True)
    opt = torch.optim.Adam(E.parameters(), lr=lr, betas=(0.9, 0.99))
    enc = _Encode(E)
    if world > 1:
        from torch.nn.parallel import DistributedDataParallel
        enc = DistributedDataParallel(enc, device_ids=[dev] if dev.type == 'cuda' else None, broadcast_buffers=False)

    local = batch // world
    rs = np.random.RandomState(seed + rank)
    gen = torch.Generator(dev).manual_seed(seed + rank)
    start, consumed = 0, 0
    if snap is not None:
        opt.load_state_dict(snap['optimizer'])
        _set_np_state(rs, snap['streams'][rank]['np_rng'])
        gen.set_state(snap['streams'][rank]['torch_rng'])
        start, consumed = int(snap['step']), int(snap['items'])
    data = None
    if train_real:
        data = iter(InfiniteSampler(dataset, rank=rank, num_replicas=world, seed=seed))
        for _ in range(consumed):
            next(data)

    history = []
    for i in range(start, start + steps):
        opt.zero_grad(set_to_none=True)
        z = cam = real = None
        if train_gen:
            z = torch.from_numpy(rs.randn(local, G.w_dim)).to(torch.float32).to(dev)
            cam = cam_sampler(local, dev, gen)
        if train_real:
            items = [dataset[int(next(data))] for _ in range(local)]
            consumed += local
            real = tuple(torch.stack([it[k] for it in items]).to(dev) for k in range(3))
        loss = step_losses(G, enc, parser=parser, lambdas=lam, z=z, cam=cam, real=real, truncation=truncation,
                           start_from_latent_avg=start_from_latent_avg, vgg=vgg, lpips=lpips, id_net=id_net)
        sum(loss.values()).backward()
        opt.step()
        history.append(torch.stack([v.detach().float() for v in loss.values()]))
        if snapshot_every and (i + 1) % snapshot_every == 0:
            streams = _rank_states(rs, gen, world)                  # collective: every rank takes part
            if rank == 0:
                os.makedirs(outdir, exist_ok=True)
                torch.save(dict(encoder=E.state_dict(), encoder_args=_encoder_args(E), optimizer=opt.state_dict(), step=i + 1,
                                items=consumed, streams=streams,
                                run=dict(seed=seed, world=world, batch=batch, train_gen=bool(train_gen), train_real=bool(train_real))),
                           os.path.join(outdir, f'encoder-snapshot-{i + 1:06d}.pt'))
            if world > 1:
                dist.barrier()                                     # the file is complete before any rank goes on

    E = E.eval().requires_grad_(False)
    invalidate_caches(E)
    names = (GEN_LOSSES if train_gen else ()) + (REAL_LOSSES if train_real else ())
    values = torch.stack(history).cpu().numpy() if history else np.zeros((0, len(names)), np.float32)
    return E, {name: values[:, k] for k, name in enumerate(names)}
