"""ctypes binding of oracle/_ref/libref_wire.so -- the UNMODIFIED reference's N3Tree::gen_wireframe (built by
oracle/Makefile.wire).  TEST INFRASTRUCTURE ONLY.  Trees are opened with oracle.ref_binding.RefTree, whose loader
uploads them to the device, so this needs a GPU too."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from oracle import ref_binding as rb

LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libref_wire.so")


def available() -> bool:
    return rb.available() and os.path.exists(LIB_PATH)


_lib = None


def lib():
    global _lib
    if _lib is None:
        rb.lib()                         # the reference library first, so both bindings share one copy
        h = C.CDLL(LIB_PATH)
        h.ref_tree_wireframe.restype = C.c_longlong
        h.ref_tree_wireframe.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_longlong, C.POINTER(C.c_double)]
        _lib = h
    return _lib


def wireframe(tree: "rb.RefTree", max_depth: int) -> np.ndarray:
    """N3Tree::gen_wireframe(max_depth): float32, 9 floats per vertex, 24 vertices per cell."""
    n = lib().ref_tree_wireframe(tree.h, int(max_depth), None, 0, None)
    out = np.zeros(n, np.float32)
    lib().ref_tree_wireframe(tree.h, int(max_depth), out.ctypes.data, n, None)
    return out


def wireframe_ms(tree: "rb.RefTree", max_depth: int) -> float:
    """Host time of one gen_wireframe(max_depth) call."""
    ms = C.c_double()
    lib().ref_tree_wireframe(tree.h, int(max_depth), None, 0, C.byref(ms))
    return float(ms.value)
