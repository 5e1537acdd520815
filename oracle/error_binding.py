"""ctypes binding of oracle/liberror_oracle.so (orc_leaf_error) -- TEST INFRASTRUCTURE ONLY.

The CPU restatement of the leaf-error pass; trees, cameras and options are those of oracle/binding.py."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from . import binding as ob

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "liberror_oracle.so")
_lib = None


def build() -> None:
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-pthread",
                           "-o", LIB_PATH, os.path.join(_HERE, "error_oracle.c"), "-lm"])


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            build()
        h = C.CDLL(LIB_PATH)
        h.orc_leaf_error.restype = C.c_int
        h.orc_leaf_error.argtypes = [C.POINTER(ob.orc_tree), C.POINTER(ob.orc_camera), C.POINTER(ob.orc_options),
                                     C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.POINTER(ob.orc_counters), C.c_int]
        _lib = h
    return _lib


def leaf_error(tree: ob.OracleTree, cam: ob.orc_camera, opt: ob.orc_options, err, tile=None, nthreads=None):
    """-> (score float64 [capacity * 8], absum float64 [capacity * 8], hits uint32 [capacity * 8], counters dict) of
    one view; ``err`` is the tile-sized [h, w] pixel error."""
    if tile is None:
        tile = (0, 0, cam.width, cam.height)
    x0, y0, w, h = tile
    e = np.ascontiguousarray(err, np.float32)
    assert e.size == w * h
    n_slots = tree.c.capacity * 8
    score, absum = np.zeros(n_slots), np.zeros(n_slots)
    hits = np.zeros(n_slots, np.uint32)
    cnt = ob.orc_counters()
    rc = lib().orc_leaf_error(C.byref(tree.c), C.byref(cam), C.byref(opt), x0, y0, w, h, e.ctypes.data,
                              score.ctypes.data, absum.ctypes.data, hits.ctypes.data, C.byref(cnt),
                              int(nthreads or os.cpu_count() or 1))
    if rc != 0:
        raise RuntimeError(f"orc_leaf_error failed: {rc}")
    return score, absum, hits, dict(samples=cnt.samples, child_loads=cnt.child_loads, shaded=cnt.shaded,
                                    rays_hit=cnt.rays_hit)
