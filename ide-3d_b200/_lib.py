"""ctypes binding of libide3d_b200.so (include/ide3d_b200.h).

The library is the product: there is no CPU path and no fallback.  If the shared object is missing or a
tensor is not on a CUDA device the calls raise -- loudly -- instead of computing something else.
"""

import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('IDE3D_B200_LIB') or os.path.join(_HERE, 'lib', 'libide3d_b200.so')      # (override: A/B runs against a tuning build)

ABI_VERSION = 1                                        # IDE3D_ABI_VERSION
OK, UNSUPPORTED, INVALID, CUDA_ERROR = 0, -1, -2, -3
F32, F16, F64 = 0, 1, 2
JITTER_NONE, JITTER_TENSOR, JITTER_HASH, JITTER_ZVALS = 0, 1, 2, 3
CLAMP_SOFTPLUS, CLAMP_RELU = 0, 1
PRECISION = {'auto': 0, 'fp32': 1, 'tc': 2}

_DTYPES = {torch.float32: F32, torch.float16: F16, torch.float64: F64}


def dtype2(a, b):
    """IDE3D_DTYPE2(a, b): the mixed-format code of the epilogues and the skip add (torch dtypes in, int out)."""
    return _DTYPES[a] | ((_DTYPES[b] + 1) << 4)


class UpfirParams(C.Structure):
    _fields_ = [('x', C.c_void_p), ('f', C.c_void_p), ('y', C.c_void_p), ('dtype', C.c_int),
                ('up_x', C.c_int), ('up_y', C.c_int), ('down_x', C.c_int), ('down_y', C.c_int),
                ('pad_x0', C.c_int), ('pad_y0', C.c_int), ('flip', C.c_int), ('gain', C.c_float),
                ('in_w', C.c_int), ('in_h', C.c_int), ('in_c', C.c_int), ('in_n', C.c_int),
                ('in_stride_w', C.c_int64), ('in_stride_h', C.c_int64), ('in_stride_c', C.c_int64), ('in_stride_n', C.c_int64),
                ('f_w', C.c_int), ('f_h', C.c_int), ('f_stride_w', C.c_int64), ('f_stride_h', C.c_int64),
                ('out_w', C.c_int), ('out_h', C.c_int),
                ('out_stride_w', C.c_int64), ('out_stride_h', C.c_int64), ('out_stride_c', C.c_int64), ('out_stride_n', C.c_int64)]


class FirEpilogue(C.Structure):
    _fields_ = [('scale', C.c_void_p), ('noise', C.c_void_p), ('b', C.c_void_p), ('scale2', C.c_void_p), ('y2', C.c_void_p),
                ('act', C.c_int), ('alpha', C.c_float), ('gain', C.c_float), ('clamp', C.c_float), ('noise_batch', C.c_int64)]


class StyleLayer(C.Structure):
    _fields_ = [('affine_w', C.c_void_p), ('affine_b', C.c_void_p), ('wsq', C.c_void_p), ('w_gain', C.c_float), ('b_gain', C.c_float),
                ('out_scale', C.c_float), ('w_index', C.c_int), ('in_ch', C.c_int), ('out_ch', C.c_int),
                ('style_off', C.c_int64), ('dcoef_off', C.c_int64)]


class FlreluParams(C.Structure):
    _fields_ = [('x', C.c_void_p), ('b', C.c_void_p), ('fu', C.c_void_p), ('fd', C.c_void_p), ('y', C.c_void_p),
                ('s', C.c_void_p), ('dtype', C.c_int), ('up', C.c_int), ('down', C.c_int),
                ('fu_w', C.c_int), ('fu_h', C.c_int), ('fd_w', C.c_int), ('fd_h', C.c_int),
                ('pad_x0', C.c_int), ('pad_y0', C.c_int), ('flip', C.c_int),
                ('gain', C.c_float), ('slope', C.c_float), ('clamp', C.c_float),
                ('x_w', C.c_int), ('x_h', C.c_int), ('x_c', C.c_int), ('x_n', C.c_int),
                ('x_stride_w', C.c_int64), ('x_stride_h', C.c_int64), ('x_stride_c', C.c_int64), ('x_stride_n', C.c_int64),
                ('y_w', C.c_int), ('y_h', C.c_int),
                ('y_stride_w', C.c_int64), ('y_stride_h', C.c_int64), ('y_stride_c', C.c_int64), ('y_stride_n', C.c_int64),
                ('s_w', C.c_int), ('s_h', C.c_int), ('s_ofs_x', C.c_int), ('s_ofs_y', C.c_int),
                ('write_signs', C.c_int), ('read_signs', C.c_int)]


class FlreluActParams(C.Structure):
    _fields_ = [('x', C.c_void_p), ('s', C.c_void_p), ('dtype', C.c_int),
                ('x_w', C.c_int), ('x_h', C.c_int), ('x_c', C.c_int), ('x_n', C.c_int),
                ('x_stride_w', C.c_int64), ('x_stride_h', C.c_int64), ('x_stride_c', C.c_int64), ('x_stride_n', C.c_int64),
                ('s_w', C.c_int), ('s_h', C.c_int), ('s_ofs_x', C.c_int), ('s_ofs_y', C.c_int),
                ('gain', C.c_float), ('slope', C.c_float), ('clamp', C.c_float),
                ('write_signs', C.c_int), ('read_signs', C.c_int)]


class TriPlane(C.Structure):
    _fields_ = [('data', C.c_void_p), ('n', C.c_int), ('h', C.c_int), ('w', C.c_int),
                ('stride_n', C.c_int64), ('stride_c', C.c_int64), ('stride_h', C.c_int64), ('stride_w', C.c_int64)]


class MlpHead(C.Structure):
    _fields_ = [('in_sel', C.c_int), ('hidden', C.c_int), ('out_offset', C.c_int), ('out_count', C.c_int),
                ('w1', C.c_void_p), ('b1', C.c_void_p), ('w2', C.c_void_p), ('b2', C.c_void_p)]


class Decoder(C.Structure):
    _fields_ = [('num_heads', C.c_int), ('heads', MlpHead * 4)]


class RaymarchParams(C.Structure):
    _fields_ = [('tex', TriPlane), ('seg', TriPlane), ('dec', Decoder), ('cam2world', C.c_void_p),
                ('n', C.c_int), ('res_w', C.c_int), ('res_h', C.c_int), ('num_steps', C.c_int),
                ('fov_deg', C.c_float), ('ray_start', C.c_float), ('ray_end', C.c_float), ('box_scale', C.c_float),
                ('jitter_mode', C.c_int), ('jitter_u', C.c_void_p), ('jitter_seed', C.c_uint64),
                ('clamp_mode', C.c_int), ('last_back', C.c_int), ('white_back', C.c_int), ('max_depth', C.c_float),
                ('fill_weight', C.c_int), ('noise_std', C.c_float), ('noise', C.c_void_p),
                ('out_feat', C.c_void_p), ('out_depth', C.c_void_p), ('out_weights', C.c_void_p), ('precision', C.c_int),
                ('views', C.c_int), ('jitter_seeds', C.c_void_p)]


class RasterParams(C.Structure):
    _fields_ = [('vertices', C.c_void_p), ('triangles', C.c_void_p), ('normals', C.c_void_p), ('cam2world', C.c_void_p),
                ('num_vertices', C.c_int64), ('num_triangles', C.c_int64), ('num_frames', C.c_int), ('width', C.c_int), ('height', C.c_int),
                ('yfov_deg', C.c_float), ('znear', C.c_float), ('base', C.c_float), ('ambient', C.c_float), ('diffuse', C.c_float),
                ('background', C.c_int), ('rgb', C.c_void_p), ('ids', C.c_void_p), ('scratch', C.c_void_p), ('scratch_bytes', C.c_int64)]


FRAMES_IMAGE_SEG, FRAMES_IMAGE_DEPTH = 1, 2
FRAMES_PARTIALS = 64                                   # IDE3D_FRAMES_PARTIALS


class FramesParams(C.Structure):
    _fields_ = [('image', C.c_void_p), ('n', C.c_int), ('height', C.c_int), ('width', C.c_int),
                ('image_stride_n', C.c_int64), ('image_stride_c', C.c_int64), ('image_stride_h', C.c_int64), ('image_stride_w', C.c_int64),
                ('seg', C.c_void_p), ('seg_c', C.c_int), ('seg_h', C.c_int), ('seg_w', C.c_int),
                ('seg_stride_n', C.c_int64), ('seg_stride_c', C.c_int64), ('seg_stride_h', C.c_int64), ('seg_stride_w', C.c_int64),
                ('lut', C.c_void_p), ('mode', C.c_int), ('out', C.c_void_p), ('scratch', C.c_void_p)]


class StripsParams(C.Structure):
    _fields_ = [('image', C.c_void_p), ('seeds', C.c_int), ('views', C.c_int), ('height', C.c_int), ('width', C.c_int),
                ('image_stride_n', C.c_int64), ('image_stride_c', C.c_int64), ('image_stride_h', C.c_int64), ('image_stride_w', C.c_int64),
                ('seg', C.c_void_p), ('seg_c', C.c_int), ('seg_h', C.c_int), ('seg_w', C.c_int),
                ('seg_stride_n', C.c_int64), ('seg_stride_c', C.c_int64), ('seg_stride_h', C.c_int64), ('seg_stride_w', C.c_int64),
                ('lut', C.c_void_p), ('out_image', C.c_void_p), ('out_seg', C.c_void_p)]


NOISE_MAX_BUFFERS = 64                                 # IDE3D_NOISE_MAX_BUFFERS


class NoiseTable(C.Structure):
    _fields_ = [('count', C.c_int), ('sides', C.c_int * NOISE_MAX_BUFFERS), ('bufs', C.c_void_p * NOISE_MAX_BUFFERS),
                ('grads', C.c_void_p * NOISE_MAX_BUFFERS), ('scratch', C.c_void_p), ('scratch_floats', C.c_int64)]


class SegXentParams(C.Structure):
    _fields_ = [('seg', C.c_void_p), ('n', C.c_int), ('classes', C.c_int), ('in_h', C.c_int), ('in_w', C.c_int),
                ('seg_stride_n', C.c_int64), ('seg_stride_c', C.c_int64), ('seg_stride_h', C.c_int64), ('seg_stride_w', C.c_int64),
                ('mask', C.c_void_p), ('out_h', C.c_int), ('out_w', C.c_int), ('lse', C.c_void_p), ('partials', C.c_void_p),
                ('loss', C.c_void_p), ('grad_loss', C.c_void_p), ('grad_seg', C.c_void_p)]


LPIPS_MAX_LAYERS = 8                                   # IDE3D_LPIPS_MAX_LAYERS


class LpipsLayer(C.Structure):
    _fields_ = [('c', C.c_int), ('h', C.c_int), ('w', C.c_int), ('x', C.c_void_p), ('x_stride', C.c_int64 * 4),
                ('y', C.c_void_p), ('y_stride', C.c_int64 * 4), ('lin', C.c_void_p),
                ('grad_x', C.c_void_p), ('gx_stride', C.c_int64 * 4), ('grad_y', C.c_void_p), ('gy_stride', C.c_int64 * 4)]


class LpipsParams(C.Structure):
    _fields_ = [('n', C.c_int), ('num_layers', C.c_int), ('layers', LpipsLayer * LPIPS_MAX_LAYERS), ('value', C.c_void_p),
                ('scratch', C.c_void_p), ('scratch_bytes', C.c_int64), ('grad_value', C.c_void_p)]


FEAT_L1_MAX_LAYERS = 8                                 # IDE3D_FEAT_L1_MAX_LAYERS


class FeatL1Layer(C.Structure):
    _fields_ = [('c', C.c_int), ('h', C.c_int), ('w', C.c_int), ('weight', C.c_float), ('x', C.c_void_p), ('x_stride', C.c_int64 * 4),
                ('y', C.c_void_p), ('y_stride', C.c_int64 * 4), ('grad_x', C.c_void_p), ('gx_stride', C.c_int64 * 4)]


class FeatL1Params(C.Structure):
    _fields_ = [('n', C.c_int), ('num_layers', C.c_int), ('dtype', C.c_int), ('layers', FeatL1Layer * FEAT_L1_MAX_LAYERS),
                ('value', C.c_void_p), ('scratch', C.c_void_p), ('scratch_bytes', C.c_int64), ('grad_value', C.c_void_p)]


SEG_STEM_MAX_CLASSES = 31                              # IDE3D_SEG_STEM_MAX_CLASSES


class SegStemParams(C.Structure):
    _fields_ = [('mask', C.c_void_p), ('n', C.c_int), ('h', C.c_int), ('w', C.c_int),
                ('mask_stride_n', C.c_int64), ('mask_stride_h', C.c_int64), ('mask_stride_w', C.c_int64),
                ('classes', C.c_int), ('c0', C.c_int), ('c1', C.c_int),
                ('w0', C.c_void_p), ('b0', C.c_void_p), ('wg0', C.c_float), ('w1', C.c_void_p), ('b1', C.c_void_p), ('wg1', C.c_float),
                ('ws', C.c_void_p), ('wgs', C.c_float), ('fir', C.c_void_p), ('tables', C.c_void_p), ('y1', C.c_void_p), ('skip', C.c_void_p)]


class SegStemBwdParams(C.Structure):
    _fields_ = [('fwd', SegStemParams), ('grad_y1', C.c_void_p), ('grad_skip', C.c_void_p), ('grad_w0', C.c_void_p),
                ('grad_b0', C.c_void_p), ('grad_w1', C.c_void_p), ('grad_b1', C.c_void_p), ('grad_ws', C.c_void_p),
                ('scratch', C.c_void_p), ('scratch_bytes', C.c_int64)]


class SegLabelsParams(C.Structure):
    _fields_ = [('seg', C.c_void_p), ('n', C.c_int), ('classes', C.c_int), ('in_h', C.c_int), ('in_w', C.c_int),
                ('seg_stride_n', C.c_int64), ('seg_stride_c', C.c_int64), ('seg_stride_h', C.c_int64), ('seg_stride_w', C.c_int64),
                ('out_h', C.c_int), ('out_w', C.c_int), ('out', C.c_void_p)]


_vp, _i32, _i64, _f32, _P = C.c_void_p, C.c_int, C.c_int64, C.c_float, C.POINTER

# Every function include/ide3d_b200.h declares: name -> (restype, argtypes), in header order.  argtypes None leaves the
# (void) entry points as ctypes loads them.
SIGNATURES = {
    'ide3d_abi_version': (_i32, None),
    'ide3d_last_error': (C.c_char_p, None),
    'ide3d_launch_count': (C.c_uint64, None),
    'ide3d_bias_act': (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _f32, _f32, _f32, _i64, _i64, _i64, _vp]),
    'ide3d_modconv_epilogue': (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _f32, _f32, _f32, _i64, _i64, _i64, _i64, _i32,
                                      _vp]),
    'ide3d_modconv_epilogue_rgb': (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i32, _i32, _f32, _f32,
                                          _f32, _i64, _i64, _i64, _i64, _vp]),
    'ide3d_upfirdn2d': (_i32, [_P(UpfirParams), _vp]),
    'ide3d_upfirdn2d_add': (_i32, [_P(UpfirParams), _vp, _i64, _i64, _i64, _vp, _vp]),
    'ide3d_upfirdn2d_epilogue': (_i32, [_P(UpfirParams), _P(FirEpilogue), _vp]),
    'ide3d_filtered_lrelu': (_i32, [_P(FlreluParams), _vp]),
    'ide3d_filtered_lrelu_act': (_i32, [_P(FlreluActParams), _vp]),
    'ide3d_raymarch_fwd': (_i32, [_P(RaymarchParams), _vp]),
    'ide3d_raymarch_bwd': (_i32, [_P(RaymarchParams), _vp, _vp, _vp, _vp, _P(C.c_void_p), _vp]),
    'ide3d_raymarch_bwd_cam': (_i32, [_P(RaymarchParams), _vp, _vp, _vp, _vp, _P(C.c_void_p), _vp, _vp]),
    'ide3d_sample_voxel': (_i32, [_P(TriPlane), _P(TriPlane), _P(Decoder), _vp, _i64, _f32, _i32, _vp, _vp]),
    'ide3d_sigma_grid': (_i32, [_P(TriPlane), _P(TriPlane), _P(Decoder), _i32, _P(C.c_float * 3), _f32, _f32, _f32, _i64, _i64,
                                _vp, _vp]),
    'ide3d_planes_to_nhwc': (_i32, [_vp, _i32, _i32, _i32, _i32, _i64, _i64, _i64, _i64, _vp, _vp]),
    'ide3d_initial_rays': (_i32, [_i32, _i32, _f32, _i32, _i32, _f32, _f32, _vp, _vp, _vp, _vp]),
    'ide3d_transform_points': (_i32, [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp]),
    'ide3d_sample_triplane': (_i32, [_P(TriPlane), _vp, _i64, _vp, _vp]),
    'ide3d_integrate': (_i32, [_vp, _vp, _vp, _vp, _f32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _f32, _i32, _vp, _vp, _vp, _vp]),
    'ide3d_sample_pdf': (_i32, [_vp, _vp, _vp, _i32, _i32, _i32, _f32, _vp, _vp]),
    'ide3d_mask2color': (_i32, [_vp, _i32, _i32, _i32, _i32, _i64, _i64, _i64, _i64, _vp, _vp, _i32, _vp]),
    'ide3d_video_frames': (_i32, [_P(FramesParams), _vp]),
    'ide3d_image_strips': (_i32, [_P(StripsParams), _vp]),
    'ide3d_mc_classify': (_i32, [_vp, _i32, _i32, _i32, _f32, _vp, _vp, _vp]),
    'ide3d_mc_emit': (_i32, [_vp, _i32, _i32, _i32, _f32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    'ide3d_mesh_normals': (_i32, [_vp, _vp, _i64, _vp, _vp, _vp, _vp]),
    'ide3d_raster_scratch_bytes': (_i64, [_i32, _i32, _i32, _i64, _i64]),
    'ide3d_raster': (_i32, [_P(RasterParams), _vp]),
    'ide3d_style_plan': (_i32, [_vp, _i32, _i32, _i32, _P(StyleLayer), _i32, _vp, _vp, _vp]),
    'ide3d_noise_reg': (_i32, [_P(NoiseTable), _vp, _vp, _vp]),
    'ide3d_noise_normalize': (_i32, [_P(NoiseTable), _vp]),
    'ide3d_seg_xent_fwd': (_i32, [_P(SegXentParams), _vp]),
    'ide3d_seg_xent_bwd': (_i32, [_P(SegXentParams), _vp]),
    'ide3d_seg_xent_fwd_ac': (_i32, [_P(SegXentParams), _vp]),
    'ide3d_seg_xent_bwd_ac': (_i32, [_P(SegXentParams), _vp]),
    'ide3d_lpips_scratch_bytes': (_i64, [_P(LpipsParams)]),
    'ide3d_lpips_fwd': (_i32, [_P(LpipsParams), _vp]),
    'ide3d_lpips_bwd': (_i32, [_P(LpipsParams), _vp]),
    'ide3d_feat_l1_scratch_bytes': (_i64, [_P(FeatL1Params)]),
    'ide3d_feat_l1_fwd': (_i32, [_P(FeatL1Params), _vp]),
    'ide3d_feat_l1_bwd': (_i32, [_P(FeatL1Params), _vp]),
    'ide3d_seg_stem_scratch_bytes': (_i64, [_i32, _i32]),
    'ide3d_seg_stem': (_i32, [_P(SegStemParams), _vp]),
    'ide3d_seg_stem_bwd_scratch_bytes': (_i64, [_i32, _i32, _i32, _i32, _i32]),
    'ide3d_seg_stem_bwd': (_i32, [_P(SegStemBwdParams), _vp]),
    'ide3d_seg_labels': (_i32, [_P(SegLabelsParams), _vp]),
    'ide3d_seg_labels_ac': (_i32, [_P(SegLabelsParams), _vp]),
}


_lib = None


class _StreamHandle(int):
    """cudaStream_t as an int that remembers which device it belongs to (see _GuardedLib)."""
    device = None


class _GuardedLib:
    """Every ide3d_* entry point takes the stream as its LAST argument, and every caller builds it with
    stream_ptr(tensor.device).  The wrapper makes that device current around the call -- the OptionalCUDAGuard(device_of(x))
    of the reference plugins (upfirdn2d.cpp:34, bias_act.cpp:54) -- so the launch and the SM-count / occupancy queries inside
    the library refer to the tensors' own device even when another one is current."""

    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if not name.startswith('ide3d_'):
            return fn

        def call(*args):
            dev = getattr(args[-1], 'device', None) if args else None
            if dev is None:
                return fn(*args)
            with torch.cuda.device(dev):
                return fn(*args)

        call.__name__ = name
        self.__dict__[name] = call
        return call


def get_lib():
    """Load the shared library once.  Raises if it has not been built (python ide-3d_b200/build.py)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f'ide3d_b200: CUDA library not built ({LIB_PATH} missing); run '
                           f'`python {os.path.join(_HERE, "build.py")}` -- there is no CPU fallback')
    lib = C.CDLL(LIB_PATH, mode=os.RTLD_NOW)       # every symbol resolved at load: a half-built library fails here, loudly
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    if lib.ide3d_abi_version() != ABI_VERSION:
        raise RuntimeError('ide3d_b200: ABI version mismatch between _lib.py and libide3d_b200.so')
    _lib = _GuardedLib(lib)
    return _lib


def exported_symbols():
    """Names declared in include/ide3d_b200.h (used by the CPU test that checks the .so exports them)."""
    return list(SIGNATURES)


def check(rc, allow_unsupported=False):
    """Status -> exception, mirroring the reference's TORCH_CHECK behaviour (RuntimeError)."""
    if rc == OK or (allow_unsupported and rc == UNSUPPORTED):
        return rc
    msg = get_lib().ide3d_last_error().decode(errors='replace')
    raise RuntimeError(f'ide3d_b200: {msg} (status {rc})')


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and (not isinstance(t, torch.Tensor) or t.device.type != 'cuda'):
            raise RuntimeError('ide3d_b200: tensors must reside on a CUDA device -- this package has no CPU path '
                               '(the CPU restatement lives in oracle/ and is test infrastructure only)')


def forbid_grad(name, *tensors):
    """The stage free functions write into fresh buffers through ctypes: their outputs carry no grad_fn.  Fail up front
    instead of silently cutting the graph when a caller tries to back-propagate through them (the reference module is a
    differentiable implementation); the differentiable route is render.raymarch / render_grad.RaymarchFunction."""
    if torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in tensors):
        raise RuntimeError(f'ide3d_b200.{name}: inputs require grad, but this stage kernel is forward-only -- use '
                           f'ide3d_b200.render.raymarch (fused forward, render_grad backward) or wrap the call in torch.no_grad()')


def dtype_code(t):
    try:
        return _DTYPES[t.dtype]
    except KeyError:
        raise RuntimeError(f'ide3d_b200: unsupported dtype {t.dtype}') from None


def ptr(t):
    return None if t is None else t.data_ptr()


def stream_ptr(device=None):
    """Current stream of `device` as a cudaStream_t handle that carries the device (the guard in _GuardedLib reads it)."""
    h = _StreamHandle(torch.cuda.current_stream(device).cuda_stream)
    h.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    return h


def launch_count():
    return int(get_lib().ide3d_launch_count())


def triplane_view(t):
    """[N, 96, H, W] float32 tensor (any strides) -> TriPlane struct."""
    if t.ndim != 4 or t.shape[1] != 96 or t.dtype != torch.float32:
        raise RuntimeError(f'ide3d_b200: tri-plane tensor must be float32 [N, 96, H, W], got {tuple(t.shape)} {t.dtype}')
    s = t.stride()
    return TriPlane(t.data_ptr(), t.shape[0], t.shape[2], t.shape[3], s[0], s[1], s[2], s[3])
