"""Golden data of avg_spectra: the reference's own avg_spectra.py, loaded from its AST and run on the CPU.

    python tests/golden/make_spectra_golden.py [/path/to/reference]   -> tests/golden/spectra.npz

The module is executed without its matplotlib and legacy imports (neither is needed by `stats`, `calc` or construct_heatmap).
`stats` and `calc` run with device='cpu' and a DataLoader without pinning or workers.  Sources:
  - the oracle.metrics.write_dataset images, as a directory and as a zip, at 16^2 and 32^2: stats, and calc at interp 1, 2 and 4 with
    beta 8 and 2 (plus one --num=7 --seed=3 subset).  The directory's spectra equal the zip's bit for bit; only the zip's are stored;
  - oracle.spectra.StandInSpectrumGenerator (the metrics' stand-in, 512^2) as a network pickle, with generate_image's label replaced by the camera rule of
    ide3d_b200.avg_spectra (c_dim 25 without a dataset: the frontal conditioning camera), 3 images at interp 2.  Its [1024, 1024]
    spectrum is stored as every 7th bin in each direction plus the row and column sums;
  - construct_heatmap of one spectrum at smooth 0 and 1.25, and the two slices the `slices` command plots.
"""

import ast
import io
import os
import pickle
import sys
import tempfile
import types
from contextlib import redirect_stdout

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

FRONTAL_CAMERA = [1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 2.7, 0, 0, 0, 1, 4.2647, 0, 0.5, 0, 4.2647, 0.5, 0, 0, 1]
SIZES = (16, 32)
INTERPS = (1, 2, 4)
BETAS = (8.0, 2.0)
MEAN, STD = 112.5, 61.25
GEN = dict(num=3, seed=5, interp=2, beta=8.0)


def camera_label(rnd, c_dim):
    c = np.zeros([1, c_dim], dtype=np.float32)
    if c_dim == 25:
        c[0] = FRONTAL_CAMERA
    elif c_dim > 0:
        c[:, rnd.randint(c_dim)] = 1
    return torch.from_numpy(c)


class _LabelRule(ast.NodeTransformer):
    """In generate_image: `c = torch.zeros(...)` and the one-hot `if` become `c = camera_label(rnd, G.c_dim).to(device)`."""

    def visit_FunctionDef(self, node):
        self.generic_visit(node)
        if node.name != 'generate_image':
            return node
        body = []
        for st in node.body:
            src = ast.unparse(st)
            if src.startswith('c = torch.zeros'):
                body.append(ast.parse('c = camera_label(rnd, G.c_dim).to(device)').body[0])
            elif src.startswith('if G.c_dim > 0'):
                continue
            else:
                body.append(st)
        node.body = body
        return node


def load_reference(ref):
    """The reference module's namespace, minus the matplotlib and legacy imports, with the label rule in generate_image."""
    tree = ast.parse(open(os.path.join(ref, 'avg_spectra.py')).read())
    tree.body = [n for n in tree.body if not (isinstance(n, (ast.Import, ast.ImportFrom)) and
                                             any(a.name in ('matplotlib.pyplot', 'legacy') for a in n.names))]
    tree = ast.fix_missing_locations(_LabelRule().visit(tree))
    mp = types.SimpleNamespace(set_start_method=lambda *a, **k: None)
    ns = dict(__name__='ref_avg_spectra', camera_label=camera_label,
              legacy=types.SimpleNamespace(load_network_pkl=lambda f: {'G_ema': pickle.load(f)}))
    exec(compile(tree, 'avg_spectra.py', 'exec'), ns)
    ns['torch'] = types.SimpleNamespace(**{k: getattr(torch, k) for k in dir(torch) if not k.startswith('__')})
    ns['torch'].multiprocessing = mp
    stream = ns['stream_source_images']
    ns['stream_source_images'] = lambda **kw: stream(data_loader_kwargs=dict(pin_memory=False, num_workers=0), **kw)
    ns['tqdm'] = types.SimpleNamespace(tqdm=lambda it, total=None: it)
    return ns


def setup(tmp):
    """The datasets (dir and zip per size) under `tmp`: {size: (dir, zip)}."""
    from oracle import metrics as om
    return {res: om.write_dataset(os.path.join(tmp, f'ffhq-{res}'), res=res, seed=res) for res in SIZES}


def save_generator(path):
    from oracle import spectra as osp
    with open(path, 'wb') as f:
        pickle.dump(osp.StandInSpectrumGenerator(), f)
    return path


def main(ref=None):
    ref = ref or os.environ.get('IDE3D_REFERENCE', '/root/reference')
    sys.path.insert(0, ref)
    torch.set_num_threads(4)
    ns = load_reference(ref)
    tmp = tempfile.mkdtemp()
    data = setup(tmp)
    cpu = torch.device('cpu')
    out = {}

    def calc(source, tag, **kw):
        dest = os.path.join(tmp, tag + '.npz')
        ns['calc'].callback(source=source, dest=dest, device=cpu, **kw)
        with np.load(dest) as z:
            return z['spectrum'], z['image_size']

    for res, (ds_dir, ds_zip) in data.items():
        for kind, path in (('dir', ds_dir), ('zip', ds_zip)):
            buf = io.StringIO()
            with redirect_stdout(buf):
                ns['stats'].callback(source=path, num=None, seed=0, device=cpu)
            out[f'stats_{res}_{kind}'] = np.array(buf.getvalue().strip())
        for interp in INTERPS:
            for beta in BETAS:
                tag = f'calc_{res}_i{interp}_b{beta:g}'
                kw = dict(mean=MEAN, std=STD, num=None, seed=0, beta=beta, interp=interp)
                (spec_dir, _), (out[tag], out[tag + '_image_size']) = calc(ds_dir, tag + '_dir', **kw), calc(ds_zip, tag, **kw)
                assert np.array_equal(spec_dir, out[tag])
        out[f'calc_{res}_sub'], _ = calc(ds_zip, f'calc_{res}_sub', mean=MEAN, std=STD, num=7, seed=3, beta=8.0, interp=2)

    pkl = save_generator(os.path.join(tmp, 'standin.pkl'))
    spec, out['calc_gen_image_size'] = calc(pkl, 'calc_gen', mean=MEAN, std=STD, num=GEN['num'], seed=GEN['seed'], beta=GEN['beta'],
                                            interp=GEN['interp'])
    out['calc_gen_sub'], out['calc_gen_sum0'], out['calc_gen_sum1'] = spec[::7, ::7], spec.sum(0), spec.sum(1)

    npz = os.path.join(tmp, f'calc_{SIZES[-1]}_i4_b8.npz')
    for smooth in (0.0, 1.25):
        hmap, image_size = ns['construct_heatmap'](npz_file=npz, smooth=smooth)
        out[f'hmap_s{smooth:g}'] = hmap
        # the arrays slices() plots (avg_spectra.py:231-234, 247, 259)
        hmap_size = hmap.shape[0]
        hmap_center = hmap_size // 2
        hmap_range = np.arange(hmap_center, hmap_size)
        out[f'slice0_s{smooth:g}'] = hmap[hmap_center, hmap_range]
        out[f'slice45_s{smooth:g}'] = hmap[hmap_range, hmap_range]
        out[f'freqs0_s{smooth:g}'] = np.linspace(0, image_size / 2, num=(hmap_size // 2 + 1), endpoint=True)
        out[f'freqs45_s{smooth:g}'] = np.linspace(0, image_size / np.sqrt(2), num=(hmap_size // 2 + 1), endpoint=True)
    np.savez_compressed(os.path.join(HERE, 'spectra.npz'), **out)
    print({k: (v.shape if v.ndim else v) for k, v in out.items()})


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else None)
