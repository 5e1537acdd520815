"""ctypes binding of oracle/libgrads_oracle.so (orc_leaf_grads) -- TEST INFRASTRUCTURE ONLY.

The CPU restatement of the leaf-gradient pass; trees, cameras and options are those of oracle/binding.py."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from . import binding as ob

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libgrads_oracle.so")
_lib = None


def build() -> None:
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-pthread",
                           "-o", LIB_PATH, os.path.join(_HERE, "grads_oracle.c"), "-lm"])


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            build()
        h = C.CDLL(LIB_PATH)
        h.orc_leaf_grads.restype = C.c_int
        h.orc_leaf_grads.argtypes = [C.POINTER(ob.orc_tree), C.POINTER(ob.orc_camera), C.POINTER(ob.orc_options),
                                     C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_int]
        _lib = h
    return _lib


def leaf_grads(tree: ob.OracleTree, cam: ob.orc_camera, opt: ob.orc_options, dpix, tile=None, grad=None, A=None,
               nthreads=None):
    """-> (grad float64 [capacity * 8, data_dim], A float64 [same], rgba float32 [h, w, 4]).  ``dpix``: float32
    [h, w, 4] dL/d(r, g, b, alpha) of the tile; ``grad`` / ``A`` accumulate in place when given, else start at 0."""
    if tile is None:
        tile = (0, 0, cam.width, cam.height)
    x0, y0, w, h = tile
    shape = (tree.c.capacity * 8, tree.c.data_dim)
    grad = np.zeros(shape) if grad is None else grad
    A = np.zeros(shape) if A is None else A
    for a in (grad, A):
        assert a.dtype == np.float64 and a.shape == shape and a.flags.c_contiguous
    dp = np.ascontiguousarray(dpix, np.float32)
    assert dp.shape == (h, w, 4)
    rgba = np.zeros((h, w, 4), np.float32)
    rc = lib().orc_leaf_grads(C.byref(tree.c), C.byref(cam), C.byref(opt), x0, y0, w, h, dp.ctypes.data,
                              grad.ctypes.data, A.ctypes.data, rgba.ctypes.data, int(nthreads or os.cpu_count() or 1))
    if rc != 0:
        raise RuntimeError(f"orc_leaf_grads failed: {rc}")
    return grad, A, rgba
