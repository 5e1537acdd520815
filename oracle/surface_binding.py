"""ctypes binding of oracle/libsurface_harness.so -- TEST INFRASTRUCTURE ONLY; needs a GPU to render.

Renders through vr_render_surface (and the surface form of vr_draw_probe) into a cudaArray, as the C++ drop-in
launch_renderer does, and reads the array back.  The harness calls the entry points of the already loaded
libvolrend_b200.so through function pointers, so the variant setting, vr_last_error and vr_launch_count are shared
with every other call of the test."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsurface_harness.so")
SYMBOLS = {
    "sh_alloc": (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "sh_free": (C.c_int, [C.c_void_p]),
    "sh_upload": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "sh_download": (C.c_int, [C.c_void_p, C.c_void_p]),
    "sh_render": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "sh_probe": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_float), C.c_int,
                           C.c_void_p]),
    "sh_colour_surface": (C.c_ulonglong, [C.c_void_p]),
}
SENTINEL = 0x5A     # initial byte of the arrays render_surface allocates without rgba_in
_lib = None


def available() -> bool:
    return os.path.exists(LIB_PATH)


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        h = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(h, name)
            fn.restype, fn.argtypes = res, args
        _lib = h
    return _lib


def _cuda(rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError(f"{what}: CUDA error {rc}")


def _entry(name: str) -> int:
    from volrend_b200 import lib as vlib
    return C.cast(getattr(vlib(), name), C.c_void_p).value


def _stream(stream) -> int | None:
    s = int(getattr(stream, "cuda_stream", stream or 0))
    return s or None


class SurfaceFrame:
    """An RGBA8 cudaArray of w x h pixels with its surface object, and with ``depth`` an R32F one."""

    def __init__(self, w: int, h: int, depth: bool = False):
        self.w, self.h = int(w), int(h)
        self.h_ = C.c_void_p()
        _cuda(lib().sh_alloc(self.w, self.h, int(depth), C.byref(self.h_)), "sh_alloc")

    def upload(self, rgba8=None, depth=None) -> None:
        r = None if rgba8 is None else np.ascontiguousarray(rgba8, np.uint8)
        d = None if depth is None else np.ascontiguousarray(depth, np.float32)
        for a in (r, d):
            assert a is None or a.shape[:2] == (self.h, self.w), (a.shape, self.h, self.w)
        _cuda(lib().sh_upload(self.h_, r.ctypes.data if r is not None else None, d.ctypes.data if d is not None else None),
              "sh_upload")

    def download(self) -> np.ndarray:
        out = np.empty((self.h, self.w, 4), np.uint8)
        _cuda(lib().sh_download(self.h_, out.ctypes.data), "sh_download")
        return out

    def surface(self) -> int:
        return lib().sh_colour_surface(self.h_)

    def render_rc(self, tree, cam, opt, composite: bool = False, stream=0) -> int:
        """vr_render_surface into this frame (composite: with the depth surface); its return code."""
        c, o = cam._as_c(), opt._as_c()
        return lib().sh_render(self.h_, _entry("vr_render_surface"), tree._handle, C.byref(c), C.byref(o),
                               int(composite), _stream(stream))

    def render(self, tree, cam, opt, composite: bool = False, stream=0) -> None:
        from volrend_b200 import _capi
        rc = self.render_rc(tree, cam, opt, composite, stream)
        if rc > 0:
            _cuda(rc, "sh_render")
        _capi.check(rc)

    def probe(self, tree, cam, opt, xyz, disp_size: int, stream=0) -> None:
        """The surface form of vr_draw_probe: the disc at world point xyz over this frame."""
        from volrend_b200 import _capi
        c, o = cam._as_c(), opt._as_c()
        arr = (C.c_float * 3)(*[float(v) for v in xyz])
        rc = lib().sh_probe(self.h_, _entry("vr_draw_probe"), tree._handle, C.byref(c), C.byref(o), arr, int(disp_size),
                            _stream(stream))
        if rc > 0:
            _cuda(rc, "sh_probe")
        _capi.check(rc)

    def close(self) -> None:
        if self.h_:
            h, self.h_ = self.h_, C.c_void_p()
            _cuda(lib().sh_free(h), "sh_free")

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def render_surface(tree, cam, opt, rgba_in=None, depth_in=None, array_size=None, probe=None, stream=0) -> np.ndarray:
    """The RGBA8 array after vr_render_surface of ``cam`` (and, with ``probe`` = (world xyz, disp_size), the surface
    disc after it, as launch_renderer draws it) -> uint8 [h, w, 4] of the whole array.

    ``array_size`` (w, h): an array larger than the camera frame (default: the frame's size).  ``rgba_in``: the array's
    initial colour (whole array; default SENTINEL in every byte, so that a pixel the render misses shows).
    ``depth_in``: float32 ray-distance limits of the whole array; given, the render is a composite through the depth
    surface over ``rgba_in``.  ``stream``: a CUDA stream handle or torch stream."""
    w, h = array_size if array_size is not None else (cam.width, cam.height)
    if rgba_in is None:
        rgba_in = np.full((h, w, 4), SENTINEL, np.uint8)
    with SurfaceFrame(w, h, depth=depth_in is not None) as f:
        f.upload(rgba_in, depth_in)
        f.render(tree, cam, opt, composite=depth_in is not None, stream=stream)
        if probe is not None:
            f.probe(tree, cam, opt, probe[0], probe[1], stream=stream)
        return f.download()
