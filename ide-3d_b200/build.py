"""Build libide3d_b200.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

    python ide-3d_b200/build.py [--force] [--verbose]

No torch involvement: plain `nvcc -c` per translation unit (in parallel) and one `nvcc -shared` link.
The result lands in ide-3d_b200/lib/libide3d_b200.so (git-ignored build product).
"""

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OBJ = os.path.join(HERE, '_build_tuning' if os.environ.get('IDE3D_BUILD_TUNING', '0') == '1' else '_build')
LIBDIR = os.path.join(HERE, 'lib')
LIB = os.path.join(LIBDIR, 'libide3d_b200_tuning.so' if os.environ.get('IDE3D_BUILD_TUNING', '0') == '1' else 'libide3d_b200.so')
TUNING = os.environ.get('IDE3D_BUILD_TUNING', '0') == '1'      # experiment switches (A/B scripts only)
UNITS = ['capi', 'raymarch', 'raymarch_bwd', 'raymarch_tc', 'voxel', 'voxel_tc', 'stages', 'style_plan', 'mcubes', 'raster', 'frames', 'strips', 'projector', 'lpips', 'seg_stem', 'bias_act', 'upfirdn2d', 'filtered_lrelu', 'filtered_lrelu_fused', 'knn', 'spectra', 'resample', 'style_grid', 'viz']
NVCC_FLAGS = ['-O3', '-std=c++17', '--expt-relaxed-constexpr', '-gencode', 'arch=compute_90a,code=sm_90a',
              '-lineinfo', '-Xcompiler', '-fPIC', '-Xptxas', '-v'] + (['-DIDE3D_TUNING'] if TUNING else [])


def _nvcc():
    for cand in (os.environ.get('NVCC'), shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError('nvcc not found (set NVCC=/path/to/nvcc)')


def _sources():
    return [u for u in UNITS if os.path.exists(os.path.join(CSRC, u + '.cu'))]


def _digest():
    h = hashlib.sha256(' '.join(NVCC_FLAGS).encode())
    names = sorted(os.listdir(CSRC)) + ['../../include/ide3d_b200.h']
    for n in names:
        p = os.path.join(CSRC, n)
        if os.path.isfile(p):
            h.update(n.encode())
            h.update(open(p, 'rb').read())
    return h.hexdigest()


def _compile(nvcc, unit, verbose):
    src = os.path.join(CSRC, unit + '.cu')
    obj = os.path.join(OBJ, unit + '.o')
    cmd = [nvcc, '-c'] + NVCC_FLAGS + [src, '-o', obj]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    with open(os.path.join(OBJ, unit + '.log'), 'w') as f:
        f.write(' '.join(cmd) + '\n' + r.stdout)
    if r.returncode != 0:
        raise RuntimeError(f'nvcc failed on {unit}.cu:\n{r.stdout[-6000:]}')
    if verbose:
        print(r.stdout)
    return obj


def build(force=False, verbose=False):
    """Compile if the sources changed since the last build; return the library path."""
    os.makedirs(OBJ, exist_ok=True)
    os.makedirs(LIBDIR, exist_ok=True)
    stamp = os.path.join(LIBDIR, 'build_tuning.sha256' if TUNING else 'build.sha256')
    digest = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read().strip() == digest:
        return LIB
    nvcc = _nvcc()
    units = _sources()
    with ThreadPoolExecutor(max_workers=min(8, len(units))) as ex:
        objs = list(ex.map(lambda u: _compile(nvcc, u, verbose), units))
    cmd = [nvcc, '-shared', '-gencode', 'arch=compute_90a,code=sm_90a', '-o', LIB] + objs + ['-lcudart']
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError('link failed:\n' + r.stdout)
    with open(stamp, 'w') as f:
        f.write(digest)
    return LIB


if __name__ == '__main__':
    path = build(force='--force' in sys.argv, verbose='--verbose' in sys.argv)
    print(path)
