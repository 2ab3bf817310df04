#!/usr/bin/env python
"""Build the REFERENCE's own CUDA plugins (torch_utils/ops/{upfirdn2d,bias_act,filtered_lrelu}) for sm_90a, unmodified, so that
they can be timed on the H100 beside this package's kernels (BASELINE.md config 5).

    IDE3D_REFERENCE=/path/to/IDE-3D python baseline/build_ref_plugins.py     # no GPU needed (nvcc cross-compiles)

Outputs ONLY into baseline/_ref/ (git-ignored):
    baseline/_ref/torch_utils/...   an untouched copy of the reference's torch_utils package (Python wrappers + plugin sources)
    baseline/_ref/dnnlib/...        (torch_utils imports dnnlib)
    baseline/_ref/plugins/<name>/<name>.so   the three pybind modules, compiled from those sources with the reference's own
                                    flags (--use_fast_math, custom_ops.py:136) plus -gencode arch=compute_90a,code=sm_90a
Nothing from the reference is committed to this repository.  On the GPU machine scripts/bench_ops.py imports the copies and
pre-seeds custom_ops._cached_plugins with the prebuilt modules, so the reference's Python op wrappers dispatch to the
reference's own kernels exactly as custom_ops.get_plugin would after its JIT build (custom_ops.py:68-69, :154)."""
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get('IDE3D_REFERENCE', '')
OUT = os.path.join(HERE, '_ref')
PLUGINS = {
    'bias_act_plugin': ['bias_act.cpp', 'bias_act.cu'],
    'upfirdn2d_plugin': ['upfirdn2d.cpp', 'upfirdn2d.cu'],
    'filtered_lrelu_plugin': ['filtered_lrelu.cpp', 'filtered_lrelu_wr.cu', 'filtered_lrelu_rd.cu', 'filtered_lrelu_ns.cu'],
}


def build(verbose=False):
    if not os.path.isdir(REF):
        print(f'[ref-plugins] {REF} absent: nothing to build (prebuilt files are used as they are)')
        return False
    os.makedirs(OUT, exist_ok=True)
    for pkg in ('torch_utils', 'dnnlib'):
        dst = os.path.join(OUT, pkg)
        if not os.path.isdir(dst):
            shutil.copytree(os.path.join(REF, pkg), dst, ignore=shutil.ignore_patterns('__pycache__'))
    os.environ.setdefault('TORCH_CUDA_ARCH_LIST', '10.0')
    from torch.utils import cpp_extension
    src_dir = os.path.join(OUT, 'torch_utils', 'ops')
    for name, srcs in PLUGINS.items():
        bdir = os.path.join(OUT, 'plugins', name)
        if os.path.exists(os.path.join(bdir, name + '.so')):
            continue
        os.makedirs(bdir, exist_ok=True)
        cpp_extension.load(name=name, sources=[os.path.join(src_dir, s) for s in srcs], build_directory=bdir, verbose=verbose,
                           extra_cuda_cflags=['--use_fast_math', '-gencode', 'arch=compute_90a,code=sm_90a'], is_python_module=False)
        print(f'[ref-plugins] built {name}')
    return True


if __name__ == '__main__':
    build(verbose='-v' in sys.argv)
