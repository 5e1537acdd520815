"""ctypes binding of oracle/libweights_oracle.so (orc_leaf_weights) -- TEST INFRASTRUCTURE ONLY.

The CPU restatement of the leaf-weights pass; trees, cameras and options are those of oracle/binding.py."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from . import binding as ob

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libweights_oracle.so")
_lib = None


def build() -> None:
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-pthread",
                           "-o", LIB_PATH, os.path.join(_HERE, "weights_oracle.c"), "-lm"])


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            build()
        h = C.CDLL(LIB_PATH)
        h.orc_leaf_weights.restype = C.c_int
        h.orc_leaf_weights.argtypes = [C.POINTER(ob.orc_tree), C.POINTER(ob.orc_camera), C.POINTER(ob.orc_options),
                                       C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                       C.POINTER(ob.orc_counters), C.c_int]
        _lib = h
    return _lib


def leaf_weights(tree: ob.OracleTree, cam: ob.orc_camera, opt: ob.orc_options, tile=None, weights=None,
                 want_alpha=True, nthreads=None):
    """-> (weights float32 [capacity * 8], alpha [h, w] | None, counters dict).  ``weights`` (capacity * 8 float32) is
    raised in place when given, else starts at -inf."""
    if tile is None:
        tile = (0, 0, cam.width, cam.height)
    x0, y0, w, h = tile
    n_slots = tree.c.capacity * 8
    if weights is None:
        weights = np.full(n_slots, -np.inf, np.float32)
    assert weights.dtype == np.float32 and weights.size == n_slots and weights.flags.c_contiguous
    alpha = np.zeros((h, w), np.float32) if want_alpha else None
    cnt = ob.orc_counters()
    rc = lib().orc_leaf_weights(C.byref(tree.c), C.byref(cam), C.byref(opt), x0, y0, w, h, weights.ctypes.data,
                                alpha.ctypes.data if alpha is not None else None, C.byref(cnt),
                                int(nthreads or os.cpu_count() or 1))
    if rc != 0:
        raise RuntimeError(f"orc_leaf_weights failed: {rc}")
    return weights, alpha, dict(samples=cnt.samples, child_loads=cnt.child_loads, shaded=cnt.shaded,
                                rays_hit=cnt.rays_hit)
