"""ctypes bindings of the lumisphere probe disc's test infrastructure -- TEST INFRASTRUCTURE ONLY.

* ``oracle/libprobe_oracle.so`` (probe_oracle.c): the CPU restatement; :func:`render` marches a frame with the
  march oracle and applies the disc to it.
* ``oracle/_ref/libref_probe.so`` (ref_probe.cu, built by oracle/Makefile.probe from the reference sources): the
  UNMODIFIED reference's launch_renderer with ``enable_probe`` on.  Needs a GPU.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from . import binding as ob

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libprobe_oracle.so")
REF_PATH = os.path.join(_HERE, "_ref", "libref_probe.so")

_lib = None
_ref = None


def build() -> None:
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-pthread",
                           "-o", LIB_PATH, os.path.join(_HERE, "probe_oracle.c"), "-lm"])


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            build()
        h = C.CDLL(LIB_PATH)
        h.orc_probe_overlay.restype = C.c_int
        h.orc_probe_overlay.argtypes = [C.POINTER(ob.orc_tree), C.POINTER(ob.orc_camera), C.POINTER(ob.orc_options),
                                        C.POINTER(C.c_float), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                        C.c_void_p, C.c_void_p, C.c_void_p]
        _lib = h
    return _lib


def overlay(tree: ob.OracleTree, cam: ob.orc_camera, opt: ob.orc_options, probe, disp: int, tile=None,
            f32=None, u8=None) -> np.ndarray:
    """Applies the disc in place to the tile-sized ``f32`` / ``u8`` (either may be None); returns the disc mask
    (bool [h, w])."""
    x0, y0, w, h = tile if tile is not None else (0, 0, cam.width, cam.height)
    mask = np.zeros((h, w), np.uint8)
    xyz = (C.c_float * 3)(*[float(v) for v in probe])
    rc = lib().orc_probe_overlay(C.byref(tree.c), C.byref(cam), C.byref(opt), xyz, int(disp), x0, y0, w, h,
                                 f32.ctypes.data if f32 is not None else None,
                                 u8.ctypes.data if u8 is not None else None, mask.ctypes.data)
    if rc != 0:
        raise RuntimeError(f"orc_probe_overlay failed: {rc}")
    return mask.astype(bool)


def render(tree: ob.OracleTree, cam: ob.orc_camera, opt: ob.orc_options, probe, disp: int, tile=None,
           rgba_in=None, depth_in=None):
    """launch_renderer with enable_probe on the CPU -> (rgba_f32, rgba8, disc mask)."""
    f, u, _ = ob.render(tree, cam, opt, tile=tile, rgba_in=rgba_in, depth_in=depth_in, want_counters=False)
    mask = overlay(tree, cam, opt, probe, disp, tile, f, u)
    return f, u, mask


# ---------------------------------------------------------------- the reference (GPU)
class ref_probe_options(C.Structure):
    _fields_ = [("step_size", C.c_float), ("sigma_thresh", C.c_float), ("stop_thresh", C.c_float),
                ("background_brightness", C.c_float), ("render_bbox", C.c_float * 6),
                ("basis_minmax", C.c_int32 * 2), ("rot_dirs", C.c_float * 3), ("render_depth", C.c_int32),
                ("probe", C.c_float * 3), ("probe_disp_size", C.c_int32)]


def ref_available() -> bool:
    return os.path.exists(REF_PATH)


def ref_lib() -> C.CDLL:
    global _ref
    if _ref is None:
        h = C.CDLL(REF_PATH)
        h.ref_probe_tree_open.restype = C.c_void_p
        h.ref_probe_tree_open.argtypes = [C.c_char_p]
        h.ref_probe_tree_close.restype = None
        h.ref_probe_tree_close.argtypes = [C.c_void_p]
        h.ref_probe_render_u8.restype = C.c_int
        h.ref_probe_render_u8.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float, C.c_void_p,
                                          C.POINTER(ref_probe_options), C.c_void_p, C.c_void_p, C.c_void_p]
        _ref = h
    return _ref


def ref_options(probe, disp: int, **kw) -> ref_probe_options:
    o = ref_probe_options()
    o.step_size, o.sigma_thresh, o.stop_thresh, o.background_brightness = 1e-4, 1e-2, 1e-2, 1.0
    for i, v in enumerate((0, 0, 0, 1, 1, 1)):
        o.render_bbox[i] = v
    o.basis_minmax[0], o.basis_minmax[1] = 0, 24
    for k, v in kw.items():
        if k in ("render_bbox", "rot_dirs", "basis_minmax"):
            arr = getattr(o, k)
            for i, x in enumerate(v):
                arr[i] = x
        else:
            setattr(o, k, v)
    for i in range(3):
        o.probe[i] = float(probe[i])
    o.probe_disp_size = int(disp)
    return o


def ref_render_u8(npz_path: str, w, h, fx, fy, c2w12, opt: ref_probe_options, rgba_in=None, depth_in=None):
    """Bytes of the reference's launch_renderer with the probe on (offscreen, or over rgba_in / depth_in)."""
    t = ref_lib().ref_probe_tree_open(npz_path.encode())
    if not t:
        raise RuntimeError(f"reference loader could not open {npz_path}")
    try:
        out = np.zeros((h, w, 4), np.uint8)
        c = np.ascontiguousarray(c2w12, np.float32)
        rin = None if rgba_in is None else np.ascontiguousarray(rgba_in, np.uint8)
        din = None if depth_in is None else np.ascontiguousarray(depth_in, np.float32)
        rc = ref_lib().ref_probe_render_u8(t, w, h, fx, fy, c.ctypes.data, C.byref(opt),
                                           rin.ctypes.data if rin is not None else None,
                                           din.ctypes.data if din is not None else None, out.ctypes.data)
        if rc:
            raise RuntimeError(f"ref_probe_render_u8 failed {rc}")
        return out
    finally:
        ref_lib().ref_probe_tree_close(t)
