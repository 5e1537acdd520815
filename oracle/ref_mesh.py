"""ctypes binding of oracle/_ref/libref_mesh.so -- the UNMODIFIED reference's Mesh loaders, presets and transforms
(built by oracle/Makefile.mesh).  TEST INFRASTRUCTURE ONLY.  Needs no GPU.

Every function returns the reference's meshes as dicts with the fields of ``volrend::Mesh``: ``vert`` (float32),
``faces`` (uint32), ``name`` (bytes), ``scale``, ``translation``, ``rotation`` (float32), ``face_size``,
``visible``, ``unlit``."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libref_mesh.so")
_FP = C.POINTER(C.c_float)


def available() -> bool:
    return os.path.exists(LIB_PATH)


_lib = None


def lib():
    global _lib
    if _lib is None:
        h = C.CDLL(LIB_PATH)
        sig = {
            "ref_mesh_open_drawlist_mem": (C.c_void_p, [C.c_char_p, C.c_ulonglong, C.c_int, C.POINTER(C.c_double)]),
            "ref_mesh_load_mem_obj": (C.c_void_p, [C.c_char_p, C.c_ulonglong]),
            "ref_mesh_lattice": (C.c_void_p, [C.c_int, _FP]),
            "ref_mesh_camera_frustum": (C.c_void_p, [C.c_float, C.c_float, C.c_float, C.c_float, _FP]),
            "ref_mesh_from": (C.c_void_p, [C.c_void_p, C.c_longlong, C.c_void_p, C.c_longlong, C.c_int]),
            "ref_mesh_repeat": (None, [C.c_void_p, C.c_int]),
            "ref_mesh_apply_transform": (None, [C.c_void_p, _FP, _FP, C.c_int, C.c_int]),
            "ref_mesh_apply_matrix": (None, [C.c_void_p, _FP, C.c_int, C.c_int]),
            "ref_mesh_count": (C.c_int, [C.c_void_p]),
            "ref_mesh_sizes": (None, [C.c_void_p, C.c_int, C.POINTER(C.c_longlong)]),
            "ref_mesh_get": (None, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_char_p, _FP, C.POINTER(C.c_int)]),
            "ref_mesh_free": (None, [C.c_void_p]),
        }
        for name, (res, args) in sig.items():
            fn = getattr(h, name)
            fn.restype, fn.argtypes = res, args
        _lib = h
    return _lib


def _f3(v):
    v = np.asarray(v, np.float32).reshape(-1)
    return (C.c_float * v.size)(*[float(x) for x in v])


def _take(h) -> list:
    """Copies every mesh out of a handle and frees it."""
    L = lib()
    out = []
    try:
        for i in range(L.ref_mesh_count(h)):
            sz = (C.c_longlong * 3)()
            L.ref_mesh_sizes(h, i, sz)
            vert = np.zeros(sz[0], np.float32)
            faces = np.zeros(sz[1], np.uint32)
            name = C.create_string_buffer(max(sz[2], 1))
            f7, i4 = (C.c_float * 7)(), (C.c_int * 4)()
            L.ref_mesh_get(h, i, vert.ctypes.data, faces.ctypes.data, name, f7, i4)
            f = np.asarray(f7[:], np.float32)
            out.append(dict(vert=vert, faces=faces, name=name.raw[:sz[2]], scale=f[0], translation=f[1:4],
                            rotation=f[4:7], face_size=i4[0], visible=bool(i4[1]), unlit=bool(i4[2])))
    finally:
        L.ref_mesh_free(h)
    return out


def open_drawlist_mem(data: bytes, default_visible: bool = True) -> list:
    return _take(lib().ref_mesh_open_drawlist_mem(data, len(data), int(default_visible), None))


def open_drawlist_mem_ms(data: bytes) -> float:
    """Host time of one Mesh::open_drawlist_mem call on ``data``."""
    ms = C.c_double()
    lib().ref_mesh_free(lib().ref_mesh_open_drawlist_mem(data, len(data), 1, C.byref(ms)))
    return float(ms.value)


def load_mem_obj(text) -> dict:
    b = text.encode("latin-1") if isinstance(text, str) else bytes(text)
    return _take(lib().ref_mesh_load_mem_obj(b, len(b)))[0]


def lattice(reso: int, color) -> dict:
    return _take(lib().ref_mesh_lattice(int(reso), _f3(color)))[0]


def camera_frustum(focal_length, image_width, image_height, z, color) -> dict:
    return _take(lib().ref_mesh_camera_frustum(focal_length, image_width, image_height, z, _f3(color)))[0]


def repeat_transform(vert, faces, face_size: int, n_repeat: int, transforms) -> dict:
    """A mesh of ``vert``/``faces``, then repeat(n_repeat), then each of ``transforms`` in order: (r, t, start, end)
    for apply_transform(r, t, ...) or (M, None, start, end) with M a 4x4 matrix, M[row, col]."""
    vert = np.ascontiguousarray(vert, np.float32)
    faces = np.ascontiguousarray(faces, np.uint32)
    L = lib()
    h = L.ref_mesh_from(vert.ctypes.data, vert.size, faces.ctypes.data, faces.size, int(face_size))
    L.ref_mesh_repeat(h, int(n_repeat))
    for r, t, start, end in transforms:
        if t is None:
            L.ref_mesh_apply_matrix(h, _f3(np.asarray(r, np.float32).T), int(start), int(end))
        else:
            L.ref_mesh_apply_transform(h, _f3(r), _f3(t), int(start), int(end))
    return _take(h)[0]
