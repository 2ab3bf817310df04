"""CPU: the ctypes mirror in ide3d_b200/_lib.py conforms to include/ide3d_b200.h -- struct pairing and layouts, constants,
prototypes -- and the library exports every declared function (no compute calls here); the entry points reject malformed
arguments, and the product refuses CPU tensors instead of falling back."""

import ctypes
import os
import re
import subprocess

import pytest
import torch

from conftest import ROOT
from ide3d_b200 import _lib

HEADER = os.path.join(ROOT, 'include', 'ide3d_b200.h')

# header struct -> its ctypes mirror in _lib
STRUCTS = {
    'ide3d_upfirdn2d_params': 'UpfirParams', 'ide3d_fir_epilogue': 'FirEpilogue', 'ide3d_filtered_lrelu_params': 'FlreluParams',
    'ide3d_filtered_lrelu_act_params': 'FlreluActParams', 'ide3d_triplane': 'TriPlane', 'ide3d_mlp_head': 'MlpHead',
    'ide3d_decoder': 'Decoder', 'ide3d_raymarch_params': 'RaymarchParams', 'ide3d_frames_params': 'FramesParams',
    'ide3d_strips_params': 'StripsParams', 'ide3d_raster_params': 'RasterParams', 'ide3d_style_layer': 'StyleLayer',
    'ide3d_noise_table': 'NoiseTable', 'ide3d_seg_xent_params': 'SegXentParams', 'ide3d_lpips_layer': 'LpipsLayer',
    'ide3d_lpips_params': 'LpipsParams', 'ide3d_feat_l1_layer': 'FeatL1Layer', 'ide3d_feat_l1_params': 'FeatL1Params',
    'ide3d_seg_stem_params': 'SegStemParams', 'ide3d_seg_stem_bwd_params': 'SegStemBwdParams', 'ide3d_seg_labels_params': 'SegLabelsParams',
}

# _lib name -> header name of every constant _lib copies from the header
CONSTANTS = {name: 'IDE3D_' + name for name in (
    'ABI_VERSION', 'OK', 'UNSUPPORTED', 'INVALID', 'CUDA_ERROR', 'F32', 'F16', 'F64', 'JITTER_NONE', 'JITTER_TENSOR', 'JITTER_HASH',
    'JITTER_ZVALS', 'CLAMP_SOFTPLUS', 'CLAMP_RELU', 'FRAMES_IMAGE_SEG', 'FRAMES_IMAGE_DEPTH', 'FRAMES_PARTIALS', 'NOISE_MAX_BUFFERS',
    'LPIPS_MAX_LAYERS', 'FEAT_L1_MAX_LAYERS', 'SEG_STEM_MAX_CLASSES')}


def _header():
    return re.sub(r'/\*.*?\*/', '', open(HEADER).read(), flags=re.S)


def header_functions():
    """name -> (return type, [parameter declarations]) of every function the header declares."""
    protos = re.findall(r'^([A-Za-z_][\w \t*]*?)\s*\b(ide3d_\w+)\s*\(([^)]*)\)\s*;', _header(), flags=re.M)
    return {name: (ret, [] if params.strip() == 'void' else [p.strip() for p in params.split(',')]) for ret, name, params in protos}


def c_kind(decl):
    """'int', 'int64', 'uint64', 'float', 'ptr', or 'ptr:ide3d_x' for a pointer to header struct ide3d_x."""
    words = [w for w in re.findall(r'\w+|\*|\[', decl) if w != 'const']
    if '*' in words or '[' in words:
        return f'ptr:{words[0]}' if words[0] in STRUCTS else 'ptr'
    return {'int': 'int', 'int64_t': 'int64', 'uint64_t': 'uint64', 'float': 'float', 'ide3d_stream_t': 'ptr'}[words[0]]


def ctypes_kind(t):
    if t in (ctypes.c_void_p, ctypes.c_char_p):
        return 'ptr'
    if issubclass(t, ctypes._Pointer):
        paired = {getattr(_lib, py): c for c, py in STRUCTS.items()}
        return f'ptr:{paired[t._type_]}' if t._type_ in paired else 'ptr'
    return {ctypes.c_int: 'int', ctypes.c_int64: 'int64', ctypes.c_uint64: 'uint64', ctypes.c_float: 'float'}[t]


@pytest.fixture(scope='module')
def probe(tmp_path_factory):
    """Compile and run a C program that prints, from the header, every value the ctypes mirror claims: `key value...` lines."""
    lines = []
    for c_name, py_name in STRUCTS.items():
        lines.append(f'printf("{c_name} %zu %zu\\n", sizeof({c_name}), _Alignof({c_name}));')
        for field, _ in getattr(_lib, py_name)._fields_:
            lines.append(f'printf("{c_name}.{field} %zu %zu\\n", offsetof({c_name}, {field}), sizeof((({c_name}*)0)->{field}));')
    for c_name in list(CONSTANTS.values()) + ['IDE3D_PRECISION_' + k.upper() for k in _lib.PRECISION]:
        lines.append(f'printf("{c_name} %lld\\n", (long long){c_name});')
    d = tmp_path_factory.mktemp('abi_probe')
    (d / 'probe.c').write_text('#include <stddef.h>\n#include <stdio.h>\n#include "ide3d_b200.h"\nint main(void) {\n'
                               + '\n'.join(lines) + '\nreturn 0;\n}\n')
    subprocess.run(['gcc', '-std=c11', '-I', os.path.dirname(HEADER), str(d / 'probe.c'), '-o', str(d / 'probe')], check=True)
    out = subprocess.run([str(d / 'probe')], capture_output=True, text=True, check=True).stdout
    return {key: [int(v) for v in vals] for key, *vals in (line.split() for line in out.splitlines())}


def test_structs_pair_with_header():
    declared = re.findall(r'\btypedef\s+struct\s+(ide3d_\w+)', _header())
    assert sorted(declared) == sorted(STRUCTS)
    mirrors = [name for name, v in vars(_lib).items() if isinstance(v, type) and issubclass(v, ctypes.Structure)]
    assert sorted(mirrors) == sorted(STRUCTS.values())


def test_struct_sizes_match_header(probe):
    """Every struct's size and alignment, and every field's offset and size, are the C layout."""
    want = {}
    for c_name, py_name in STRUCTS.items():
        cls = getattr(_lib, py_name)
        want[c_name] = [ctypes.sizeof(cls), ctypes.alignment(cls)]
        for field, t in cls._fields_:
            want[f'{c_name}.{field}'] = [getattr(cls, field).offset, ctypes.sizeof(t)]
    assert {k: probe[k] for k in want} == want


def test_constants_match_header(probe):
    want = {c_name: [getattr(_lib, name)] for name, c_name in CONSTANTS.items()}
    want.update({'IDE3D_PRECISION_' + k.upper(): [v] for k, v in _lib.PRECISION.items()})
    assert {k: probe[k] for k in want} == want


def test_prototypes_match_header():
    """The table declares exactly the header's functions, each with the return kind and the parameter kinds of its prototype."""
    declared = header_functions()
    assert sorted(declared) == sorted(set(re.findall(r'\b(ide3d_\w+)\s*\(', _header())))      # the parser missed no declaration
    assert sorted(declared) == sorted(_lib.SIGNATURES)
    for name, (ret, params) in declared.items():
        restype, argtypes = _lib.SIGNATURES[name]
        assert ctypes_kind(restype) == c_kind(ret), name
        mine = [ctypes_kind(t) for t in argtypes or []]
        theirs = [c_kind(p) for p in params]
        assert len(mine) == len(theirs), name
        # c_void_p stands for any pointer; POINTER(S) must point to the struct of the prototype
        assert all(m == t or (m == 'ptr' and t.startswith('ptr:')) for m, t in zip(mine, theirs)), (name, mine, theirs)


def test_library_exports_every_declared_symbol(lib):
    for n in _lib.exported_symbols():
        assert hasattr(lib, n), f'{n} declared in include/ide3d_b200.h but not exported by libide3d_b200.so'
    assert lib.ide3d_abi_version() == _lib.ABI_VERSION


def test_invalid_arguments_return_status_not_crash(lib):
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
    breaker, message = RAYMARCH_BROKEN[case]
    p = _fake_raymarch_params(_lib)
    breaker(p)
    fake = ctypes.c_void_p(0x10000)
    assert lib.ide3d_raymarch_fwd(ctypes.byref(p), None) == _lib.INVALID
    fwd_error = lib.ide3d_last_error()
    assert message in fwd_error
    assert lib.ide3d_raymarch_bwd(ctypes.byref(p), fake, None, fake, fake, None, None) == _lib.INVALID
    assert lib.ide3d_last_error() == fwd_error


@pytest.mark.skipif(torch.cuda.is_available(), reason='passes fake device pointers: run only where no GPU can be reached')
@pytest.mark.parametrize('field', ['x_c', 'x_n', 'y_w', 'y_h'])
def test_filtered_lrelu_rejects_empty_output(lib, field):
    """ide3d_filtered_lrelu refuses a call with no output elements before anything reaches the device."""
    p = _lib.FlreluParams()
    p.x = p.fu = p.fd = p.y = 0x10000
    p.dtype, p.up, p.down, p.fu_w, p.fd_w = _lib.F32, 2, 2, 12, 12
    p.x_w = p.x_h = p.x_c = p.x_n = p.y_w = p.y_h = 4
    setattr(p, field, 0)
    assert lib.ide3d_filtered_lrelu(ctypes.byref(p), None) == _lib.INVALID
    assert b'y is empty' in lib.ide3d_last_error()


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
