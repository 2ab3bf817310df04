"""CPU: the C entry of the epilogue with ToRGB folded in (ide3d_modconv_epilogue_rgb) validates its arguments
before it touches a device -- malformed calls return IDE3D_INVALID, shapes without a kernel IDE3D_UNSUPPORTED (the caller then
composes the separate passes)."""

from ide3d_b200 import _lib

FAKE = 0x10000          # 16-byte aligned, never dereferenced: every call below returns during validation


def call(lib, x=FAKE, scale=None, noise=None, b=None, yscale=None, y=FAKE, scale2=None, y2=None, wrgb=None, srgb=None, brgb=None, rgb=None,
         o=0, dtype=0, act=3, n=2, c=64, hw=256, noise_batch=1):
    return lib.ide3d_modconv_epilogue_rgb(x, scale, noise, b, yscale, y, scale2, y2, wrgb, srgb, brgb, rgb, o, dtype, act, 0.2, 1.4142135,
                                          -1.0, n, c, hw, noise_batch, None)


def test_argument_validation(lib):
    assert call(lib, n=0) == _lib.OK                                                     # empty: no-op
    assert call(lib, n=-1) == _lib.INVALID
    assert call(lib, x=None) == _lib.INVALID
    assert call(lib, y=None) == _lib.INVALID and b'no output' in lib.ide3d_last_error()
    assert call(lib, y2=FAKE) == _lib.INVALID and b'scale2 and y2' in lib.ide3d_last_error()
    assert call(lib, y=None, yscale=FAKE, y2=FAKE, scale2=FAKE) == _lib.INVALID and b'yscale without y' in lib.ide3d_last_error()
    assert call(lib, rgb=FAKE, wrgb=FAKE, srgb=FAKE, o=5) == _lib.INVALID
    assert call(lib, rgb=FAKE, srgb=FAKE, o=3) == _lib.INVALID                           # no weight
    assert call(lib, noise=FAKE, noise_batch=3) == _lib.INVALID
    assert call(lib, act=10) == _lib.INVALID
    assert call(lib, y=FAKE + 4) == _lib.INVALID and b'16-byte' in lib.ide3d_last_error()
    assert call(lib, rgb=FAKE + 2, wrgb=FAKE, srgb=FAKE, o=3) == _lib.INVALID


def test_shapes_without_a_kernel(lib):
    assert call(lib, dtype=1) == _lib.UNSUPPORTED                                        # fp16
    assert call(lib, c=6) == _lib.UNSUPPORTED
    assert call(lib, c=516) == _lib.UNSUPPORTED
    assert call(lib, rgb=FAKE, wrgb=FAKE, srgb=FAKE, o=3, c=1028) == _lib.UNSUPPORTED
