"""Golden data of dataset_tool: the reference's own dataset_tool.py command, imported from the reference tree, run on seeded sources.

    python tests/golden/make_dataset_tool_golden.py [/path/to/reference]   -> tests/golden/dataset_tool.npz

make_sources(root) writes the sources (the tests rebuild them with the same function):
  folder_labeled/   six RGB PNGs of assorted sizes, one in a subfolder, and a dataset.json that labels all but one (by basename)
  zip_labeled.zip   the same images under imgs/, with a dataset.json keyed by archive name that misses one image, plus one image
                    too narrow for the center-crop-wide case
  folder_plain/     four 16x16 RGB PNGs, no dataset.json
  folder_gray/      three 32x32 L PNGs
  folder_mixed/     a 16x16 and a 32x32 RGB PNG
CASES runs the command once per entry; for each it records the exit code, stdout (tqdm writes to stderr), the exception if one
escaped, the archive names written, every written image's decoded pixels and the dataset.json text.  Error cases write to a folder,
so that the images written before the error are recorded too.  JPEG pixels depend on the libjpeg inside Pillow: the Pillow version is
recorded with them.
"""

import importlib.util
import json
import os
import sys
import tempfile
import zipfile

import numpy as np
import PIL
import PIL.Image

HERE = os.path.dirname(os.path.abspath(__file__))

# name -> (source, dest kind, extra arguments)
CASES = {
    'folder_scale_zip': ('folder_labeled', 'zip', ['--resolution', '32x32']),
    'folder_scale_jpg': ('folder_labeled', 'zip', ['--resolution', '32x32', '--ext', 'jpg']),
    'folder_crop_max': ('folder_labeled', 'dir', ['--transform', 'center-crop', '--resolution', '16x16', '--max-images', '3']),
    'zip_crop_wide': ('zip_labeled.zip', 'zip', ['--transform', 'center-crop-wide', '--resolution', '32x16']),
    'zip_crop': ('zip_labeled.zip', 'dir', ['--transform', 'center-crop', '--resolution', '64x64', '--max-images', '4']),
    'plain_copy': ('folder_plain', 'zip', []),
    'plain_copy_jpg': ('folder_plain', 'dir', ['--ext', 'jpg']),
    'plain_up': ('folder_plain', 'zip', ['--resolution', '32x32']),
    'gray_scale': ('folder_gray', 'zip', ['--resolution', '16x16']),
    'err_square': ('folder_labeled', 'dir', ['--resolution', '32x16']),
    'err_pow2': ('folder_labeled', 'dir', ['--resolution', '24x24']),
    'err_mixed': ('folder_mixed', 'dir', []),
    'err_gray_crop': ('folder_gray', 'dir', ['--transform', 'center-crop', '--resolution', '16x16']),
    'err_no_resolution': ('folder_plain', 'dir', ['--transform', 'center-crop-wide']),
}

# the PNG case whose pixels a JPEG case encodes
JPEG_OF = {'folder_scale_jpg': 'folder_scale_zip', 'plain_copy_jpg': 'plain_copy'}


def _smooth(rng, h, w, c):
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    ph = rng.uniform(0, 2 * np.pi, size=[c, 2])
    img = [(np.sin(xx / rng.uniform(2, 9) + ph[i, 0]) + np.cos(yy / rng.uniform(2, 9) + ph[i, 1])) * 60 + 128 for i in range(c)]
    img = np.stack(img, -1) + rng.normal(0, 12, size=[h, w, c])
    img = np.clip(np.round(img), 0, 255).astype(np.uint8)
    return img[:, :, 0] if c == 1 else img


def _png(path, img):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    PIL.Image.fromarray(img).save(path, format='png')


def make_sources(root, seed=7):
    rng = np.random.default_rng(seed)
    sizes = [(40, 48), (48, 40), (64, 64), (37, 53), (64, 70), (50, 50)]       # (h, w)
    names = ['a.png', 'b.png', 'c.png', 'd.png', 'sub/e.png', 'f.png']
    imgs = [_smooth(rng, h, w, 3) for h, w in sizes]
    labeled = os.path.join(root, 'folder_labeled')
    for n, im in zip(names, imgs):
        _png(os.path.join(labeled, n), im)
    labels = [[os.path.basename(n), [float(i), i * 0.5]] for i, n in enumerate(names) if n != 'c.png']
    with open(os.path.join(labeled, 'dataset.json'), 'w') as f:
        json.dump({'labels': labels}, f)

    narrow = _smooth(rng, 40, 24, 3)                                        # narrower than the 32-wide center-crop-wide output
    with zipfile.ZipFile(os.path.join(root, 'zip_labeled.zip'), 'w') as z:
        entries = [(f'imgs/{os.path.basename(n)}', im) for n, im in zip(names, imgs)] + [('imgs/b_narrow.png', narrow)]
        for n, im in entries:
            z.writestr(n, _png_bytes(im))
        z.writestr('dataset.json', json.dumps({'labels': [[n, i] for i, (n, _) in enumerate(entries) if n != 'imgs/d.png']}))

    for i in range(4):
        _png(os.path.join(root, 'folder_plain', f'p{i}.png'), _smooth(rng, 16, 16, 3))
    for i in range(3):
        _png(os.path.join(root, 'folder_gray', f'g{i}.png'), _smooth(rng, 32, 32, 1))
    _png(os.path.join(root, 'folder_mixed', 'm0.png'), _smooth(rng, 16, 16, 3))
    _png(os.path.join(root, 'folder_mixed', 'm1.png'), _smooth(rng, 32, 32, 3))


def _png_bytes(img):
    import io
    b = io.BytesIO()
    PIL.Image.fromarray(img).save(b, format='png')
    return b.getvalue()


def read_dest(path):
    """{archive name: decoded pixels} and the dataset.json text of a written dataset (zip or folder)."""
    files = {}
    if path.endswith('.zip'):
        if not zipfile.is_zipfile(path):
            return {}, ''
        with zipfile.ZipFile(path) as z:
            for n in z.namelist():
                files[n] = z.read(n)
    elif os.path.isdir(path):
        for d, _, fs in os.walk(path):
            for f in fs:
                p = os.path.join(d, f)
                files[os.path.relpath(p, path).replace('\\', '/')] = open(p, 'rb').read()
    import io
    out = {n: np.array(PIL.Image.open(io.BytesIO(b))) for n, b in files.items() if n != 'dataset.json'}
    return out, files.get('dataset.json', b'').decode()


def case_args(root, out, name):
    src, kind, extra = CASES[name]
    dest = os.path.join(out, name + ('.zip' if kind == 'zip' else ''))
    return dest, ['--source', os.path.join(root, src), '--dest', dest] + extra


def run_case(command, root, out, name, extra_args=()):
    """Invoke a click command on one case: (record dict, dest path)."""
    from click.testing import CliRunner
    dest, args = case_args(root, out, name)
    r = CliRunner(mix_stderr=False).invoke(command, args + list(extra_args))
    exc = '' if r.exception is None or isinstance(r.exception, SystemExit) else f'{type(r.exception).__name__}: {r.exception}'
    rec = dict(exit_code=r.exit_code, stdout=r.stdout, exception=exc)
    rec['images'], rec['json'] = read_dest(dest) if os.path.exists(dest) else ({}, '')
    return rec


def load_reference(ref):
    spec = importlib.util.spec_from_file_location('reference_dataset_tool', os.path.join(ref, 'dataset_tool.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main(ref=None):
    ref = ref or os.environ.get('IDE3D_REFERENCE', '/root/reference')
    mod = load_reference(ref)
    out = {'pillow_version': np.array(PIL.__version__)}
    with tempfile.TemporaryDirectory() as tmp:
        root, dests = os.path.join(tmp, 'src'), os.path.join(tmp, 'out')
        make_sources(root)
        for name in CASES:
            rec = run_case(mod.convert_dataset, root, dests, name)
            out[f'{name}/exit_code'] = np.array(rec['exit_code'])
            out[f'{name}/stdout'] = np.array(rec['stdout'].replace(root, '<src>'))
            out[f'{name}/exception'] = np.array(rec['exception'])
            out[f'{name}/json'] = np.array(rec['json'])
            out[f'{name}/names'] = np.array(sorted(rec['images']), dtype=str)
            for n, px in rec['images'].items():
                out[f'{name}/px/{n}'] = px
            print(name, rec['exit_code'], repr(rec['exception']), len(rec['images']), rec['stdout'][-120:].replace('\n', '|'))
    np.savez_compressed(os.path.join(HERE, 'dataset_tool.npz'), **out)


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else None)
