"""CPU: the C-ABI library builds/loads without a GPU and exports every symbol include/ide3d_b200.h declares
(no compute calls here), and the product refuses CPU tensors instead of falling back."""

import ctypes
import os
import re

import pytest
import torch

from conftest import ROOT


def header_functions():
    src = open(os.path.join(ROOT, 'include', 'ide3d_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(ide3d_[a-z0-9_]+)\s*\(', src)))


def test_library_exports_every_declared_symbol(lib):
    names = header_functions()
    assert len(names) >= 16
    for n in names:
        assert hasattr(lib, n), f'{n} declared in include/ide3d_b200.h but not exported by libide3d_b200.so'
    from ide3d_b200 import _lib
    assert sorted(_lib.exported_symbols()) == names
    assert lib.ide3d_abi_version() == 1


def test_struct_sizes_match_header():
    """ctypes mirrors of the parameter structs must have the C layout (compile a probe with gcc)."""
    import subprocess, tempfile
    from ide3d_b200 import _lib
    probe = r'''
    #include <stdio.h>
    #include "ide3d_b200.h"
    int main(void) { printf("%zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(ide3d_fir_epilogue), sizeof(ide3d_upfirdn2d_params), sizeof(ide3d_filtered_lrelu_params),
        sizeof(ide3d_filtered_lrelu_act_params), sizeof(ide3d_triplane), sizeof(ide3d_mlp_head), sizeof(ide3d_decoder),
        sizeof(ide3d_raymarch_params)); return 0; }'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, 'p.c')
        open(c, 'w').write(probe)
        exe = os.path.join(d, 'p')
        subprocess.run(['gcc', '-I', os.path.join(ROOT, 'include'), c, '-o', exe], check=True)
        sizes = [int(v) for v in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    ours = [ctypes.sizeof(t) for t in (_lib.FirEpilogue, _lib.UpfirParams, _lib.FlreluParams, _lib.FlreluActParams, _lib.TriPlane,
                                       _lib.MlpHead, _lib.Decoder, _lib.RaymarchParams)]
    assert ours == sizes


def test_invalid_arguments_return_status_not_crash(lib):
    from ide3d_b200 import _lib
    assert lib.ide3d_raymarch_fwd(None, None) == _lib.INVALID
    assert b'null params' in lib.ide3d_last_error()
    assert lib.ide3d_upfirdn2d(None, None) == _lib.INVALID
    assert lib.ide3d_bias_act(None, None, None, None, None, None, 0, 0, 1, 0.0, 1.0, -1.0, 16, 0, 1, None) == _lib.INVALID
    # the fused extensions validate before they touch the device as well
    assert lib.ide3d_modconv_epilogue(None, None, None, None, None, None, None, 0, 1, 0.0, 1.0, -1.0, 1, 4, 16, 1, 0, None) == _lib.INVALID
    assert lib.ide3d_modconv_epilogue(None, None, None, None, None, None, None, 0, 1, 0.0, 1.0, -1.0, 0, 4, 16, 1, 0, None) == _lib.OK   # empty: no-op
    assert lib.ide3d_upfirdn2d_add(None, None, 0, 0, 0, None, None) == _lib.INVALID and b'null add' in lib.ide3d_last_error()
    assert lib.ide3d_upfirdn2d_epilogue(None, None, None) == _lib.INVALID and b'null epilogue' in lib.ide3d_last_error()
    assert lib.ide3d_mask2color(None, 1, 0, 4, 4, 0, 0, 0, 0, None, None, 0, None) == _lib.INVALID
    assert lib.ide3d_mask2color(None, 0, 19, 4, 4, 0, 0, 0, 0, None, None, 0, None) == _lib.OK                                           # empty batch


def _fake_raymarch_params(_lib):
    """Well-formed ide3d_raymarch_params for a 4x4 three-head render whose pointers are fake (never dereferenced)."""
    fake = 0x10000
    plane = lambda: _lib.TriPlane(fake, 1, 4, 4, 4 * 4 * 96, 1, 4 * 96, 96)
    p = _lib.RaymarchParams()
    p.tex, p.seg = plane(), plane()
    p.dec.num_heads = 3
    for i, (in_sel, off, cnt) in enumerate([(0, 0, 32), (1, 32, 19), (1, 51, 1)]):
        p.dec.heads[i] = _lib.MlpHead(in_sel, 64, off, cnt, fake, fake, fake, fake)
    p.cam2world = p.out_feat = p.out_depth = fake
    p.n, p.res_w, p.res_h, p.num_steps = 1, 4, 4, 4
    p.fov_deg, p.ray_start, p.ray_end, p.box_scale = 18.0, 2.25, 3.3, 2.0
    p.jitter_mode, p.clamp_mode = _lib.JITTER_NONE, _lib.CLAMP_SOFTPLUS
    return p


def _set(path, value):
    def apply(p):
        *parents, leaf = path.split('.')
        obj = p
        for name in parents:
            obj = getattr(obj, name)
        setattr(obj, leaf, value)
    return apply


RAYMARCH_BROKEN = {
    'tex null data': (_set('tex.data', None), b'tex: null data'),
    'seg null data': (_set('seg.data', None), b'seg: null data'),
    'seg empty': (_set('seg.h', 0), b'seg: empty tri-plane'),
    'plane sizes differ': (_set('seg.w', 8), b'tex/seg plane sizes differ'),
    'tex batch': (_set('tex.n', 2), b'batch mismatch'),
    'seg batch': (_set('seg.n', 2), b'batch mismatch'),
    'empty render': (_set('num_steps', 0), b'empty render'),
    'null cam2world': (_set('cam2world', None), b'null camera/output'),
    'clamp mode': (_set('clamp_mode', 7), b'Need to choose clamp mode'),
    'jitter mode 4': (_set('jitter_mode', 4), b'bad jitter mode'),
    'jitter mode -1': (_set('jitter_mode', -1), b'bad jitter mode'),
    'tensor jitter missing': (_set('jitter_mode', 1), b'jitter / depth tensor missing'),
    'z_vals missing': (_set('jitter_mode', 3), b'jitter / depth tensor missing'),
    '2^32 samples': (lambda p: (_set('res_w', 65536)(p), _set('res_h', 65536)(p), _set('num_steps', 1)(p)), b'more than 2^32 samples'),
}


@pytest.mark.skipif(torch.cuda.is_available(), reason='passes fake device pointers: run only where no GPU can be reached')
@pytest.mark.parametrize('case', sorted(RAYMARCH_BROKEN))
def test_raymarch_entry_points_share_validation(lib, case):
    """ide3d_raymarch_fwd and ide3d_raymarch_bwd reject the same malformed parameters with the same status and message,
    before anything reaches the device."""
    from ide3d_b200 import _lib
    breaker, message = RAYMARCH_BROKEN[case]
    p = _fake_raymarch_params(_lib)
    breaker(p)
    fake = ctypes.c_void_p(0x10000)
    assert lib.ide3d_raymarch_fwd(ctypes.byref(p), None) == _lib.INVALID
    fwd_error = lib.ide3d_last_error()
    assert message in fwd_error
    assert lib.ide3d_raymarch_bwd(ctypes.byref(p), fake, None, fake, fake, None, None) == _lib.INVALID
    assert lib.ide3d_last_error() == fwd_error


@pytest.mark.parametrize('option, error', [(dict(clamp_mode='bogus'), ValueError), (dict(fill_mode='bogus'), NotImplementedError)])
def test_raymarch_backward_checks_options_like_forward(option, error):
    from ide3d_b200 import render
    planes, cam = torch.randn(1, 96, 4, 4), torch.eye(4).reshape(1, 16)
    heads = [(0, 0, torch.zeros(64, 32), torch.zeros(64), torch.zeros(32, 64), torch.zeros(32))]
    with pytest.raises(error) as fwd:
        render.raymarch(planes, planes, heads, cam, resolution=4, num_steps=4, **option)
    with pytest.raises(error) as bwd:
        render.raymarch_backward(planes, planes, heads, cam, torch.zeros(1, 16, 51), None, resolution=4, num_steps=4, **option)
    assert str(bwd.value) == str(fwd.value)


def test_product_has_no_cpu_path():
    from ide3d_b200.torch_utils.ops import bias_act, filtered_lrelu, upfirdn2d
    from ide3d_b200 import render
    x = torch.randn(1, 2, 4, 4)
    with pytest.raises(RuntimeError):
        bias_act.bias_act(x, act='lrelu')
    with pytest.raises(RuntimeError):
        upfirdn2d.upsample2d(x, upfirdn2d.setup_filter([1, 3, 3, 1]))
    with pytest.raises(RuntimeError):
        filtered_lrelu.filtered_lrelu(x)
    with pytest.raises(NotImplementedError):
        bias_act.bias_act(x, act='lrelu', impl='ref')
    with pytest.raises(RuntimeError):
        render.as_planes(torch.randn(1, 96, 4, 4))


def test_product_never_imports_oracle():
    """Static check: nothing under ide-3d_b200/ mentions the oracle package as an import."""
    pkg = os.path.join(ROOT, 'ide-3d_b200')
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(('.py', '.cu', '.cuh')):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r'^\s*(from|import)\s+oracle\b', src, flags=re.M), f'{f} imports oracle'
