"""ctypes binding of oracle/_ref/libref_query.so -- the UNMODIFIED reference's query_single_from_root, one thread per
point, on trees opened by the reference's own N3Tree loader (built by oracle/Makefile.query).  TEST INFRASTRUCTURE
ONLY; needs a GPU."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libref_query.so")

_lib = None


def available() -> bool:
    return os.path.exists(LIB_PATH)


def lib():
    global _lib
    if _lib is None:
        h = C.CDLL(LIB_PATH)
        h.ref_query_tree_open.restype = C.c_void_p
        h.ref_query_tree_open.argtypes = [C.c_char_p]
        h.ref_query_tree_close.restype = None
        h.ref_query_tree_close.argtypes = [C.c_void_p]
        h.ref_query_data_dim.restype = C.c_int
        h.ref_query_data_dim.argtypes = [C.c_void_p]
        h.ref_query.restype = C.c_int
        h.ref_query.argtypes = [C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                C.POINTER(C.c_float)]
        _lib = h
    return _lib


class RefQueryTree:
    def __init__(self, npz_path: str):
        self.h = lib().ref_query_tree_open(npz_path.encode())
        if not self.h:
            raise RuntimeError(f"reference loader could not open {npz_path}")
        self.data_dim = lib().ref_query_data_dim(self.h)

    def query(self, xyz: np.ndarray, reps: int = 0, outputs: bool = True):
        """-> (data fp16 [n, data_dim], cube_sz [n], local [n, 3], kernel ms averaged over ``reps`` launches).
        outputs=False times the kernel without copying its outputs back (the three arrays are then None)."""
        x = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
        n = x.shape[0]
        data = np.zeros((n, self.data_dim), np.uint16) if outputs else None
        cube = np.zeros(n, np.float32) if outputs else None
        local = np.zeros((n, 3), np.float32) if outputs else None
        ms = C.c_float()
        ptr = (lambda a: a.ctypes.data if a is not None else None)
        rc = lib().ref_query(self.h, x.ctypes.data, n, ptr(data), ptr(cube), ptr(local), int(reps), C.byref(ms))
        if rc:
            raise RuntimeError(f"ref_query failed: {rc}")
        return (data.view(np.float16) if outputs else None), cube, local, float(ms.value)

    def close(self):
        if self.h:
            lib().ref_query_tree_close(self.h)
            self.h = None

    def __del__(self):
        self.close()
