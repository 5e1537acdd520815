"""Meshes drawn into the volume render (``include/volrend/mesh.hpp``, ``src/mesh.cpp``), GL-free.

A :class:`Mesh` holds the same fields as the reference's ``volrend::Mesh``; :func:`draw_meshes` rasterizes a
list of them with the CUDA rasterizer behind ``vr_draw_meshes`` (``volrend_b200/csrc/vr_raster.cu``) into an
RGBA8 image and a float32 ray-distance buffer, which ``launch_renderer(..., offscreen=False)`` then composites
the volume into (``VolumeRenderer.render`` does both when it has visible meshes).  Meshes also come from drawlist
``.npz`` files and OBJ files (:meth:`Mesh.open_drawlist`, :meth:`Mesh.load_basic_obj`, in ``mesh_io.py``), whose
normals :func:`estimate_normals` computes with a CUDA kernel (``volrend_b200/csrc/vr_normals.cu``).
"""
from __future__ import annotations

import ctypes as C
import ctypes.util
import math

import numpy as np

from . import _capi
from ._capi import check, lib

VERT_SZ = 9                                   # position, colour, normal (mesh.cpp:26)
DEFAULT_COLOR = (1.0, 0.5, 0.2)               # mesh.hpp:53,57
GREY = (0.5, 0.5, 0.5)                        # mesh.hpp:69-78

_F = np.float32
_libm = C.CDLL(ctypes.util.find_library("m") or "libm.so.6")
_libm.sinf.restype = _libm.cosf.restype = C.c_float
_libm.sinf.argtypes = _libm.cosf.argtypes = [C.c_float]


def _glm_transform(r, t) -> np.ndarray:
    """The 4x4 matrix Mesh::apply_transform(r, t) builds (mesh.cpp:652-663), in float32 with glm's operation
    order: length, the 1e-3 test, angleAxis (sin/cos from the C library's sinf/cosf, as the reference's sincosf)
    and mat4_cast, then translation in column 3.  Row-major indexing M[row, col]."""
    r = np.asarray(r, _F).reshape(3)
    m = np.eye(4, dtype=_F)
    norm = np.sqrt((r[0] * r[0] + r[1] * r[1]) + r[2] * r[2], dtype=_F)
    if float(norm) >= 1e-3:
        ax = r / norm
        half = _F(norm * _F(0.5))
        s, w = _F(_libm.sinf(half)), _F(_libm.cosf(half))
        x, y, z = ax[0] * s, ax[1] * s, ax[2] * s
        xx, yy, zz, xz, xy, yz, wx, wy, wz = x * x, y * y, z * z, x * z, x * y, y * z, w * x, w * y, w * z
        one, two = _F(1), _F(2)
        # glm Result[col][row] -> m[row, col]
        m[0, 0], m[1, 0], m[2, 0] = one - two * (yy + zz), two * (xy + wz), two * (xz - wy)
        m[0, 1], m[1, 1], m[2, 1] = two * (xy - wz), one - two * (xx + zz), two * (yz + wx)
        m[0, 2], m[1, 2], m[2, 2] = two * (xz + wy), two * (yz - wx), one - two * (xx + yy)
    m[:3, 3] = np.asarray(t, _F).reshape(3)
    return m


def model_matrix(rotation, translation, scale) -> np.ndarray:
    """Mesh::draw's model transform (mesh.cpp:368-381): axis-angle rotation (identity below a 1e-3 angle),
    then uniform scale, then translation.  Returns the 4x4 matrix (float32, row-major indexing M[row, col])."""
    r = np.asarray(rotation, np.float64).reshape(3)
    norm = float(np.sqrt(r @ r))
    m = np.eye(4)
    if norm >= 1e-3:
        x, y, z = r / norm
        s, c = math.sin(norm / 2), math.cos(norm / 2)     # glm::angleAxis -> quaternion (w, x, y, z)
        qw, qx, qy, qz = c, x * s, y * s, z * s
        m[:3, :3] = [[1 - 2 * (qy * qy + qz * qz), 2 * (qx * qy - qw * qz), 2 * (qx * qz + qw * qy)],
                     [2 * (qx * qy + qw * qz), 1 - 2 * (qx * qx + qz * qz), 2 * (qy * qz - qw * qx)],
                     [2 * (qx * qz - qw * qy), 2 * (qy * qz + qw * qx), 1 - 2 * (qx * qx + qy * qy)]]
    m[:3, :3] *= float(scale)
    m[:3, 3] = np.asarray(translation, np.float64).reshape(3)
    return m.astype(np.float32)


class Mesh:
    """``volrend::Mesh`` (mesh.hpp:9-92): ``vert`` (n_verts * 9 floats), ``faces`` (uint32, empty = consecutive
    vertices), ``rotation`` (axis-angle), ``translation``, ``scale``, ``face_size`` (3 triangles, 2 lines,
    1 points), ``visible``, ``unlit``, ``name``.  :meth:`update` uploads vert/faces to the device."""

    def __init__(self, n_verts: int = 0, n_faces: int = 0, face_size: int = 3, unlit: bool = False):
        self.vert = np.zeros(n_verts * VERT_SZ, np.float32)
        self.faces = np.zeros(n_faces * face_size, np.uint32)
        self.rotation = np.zeros(3, np.float32)
        self.translation = np.zeros(3, np.float32)
        self.scale = 1.0
        self.face_size = face_size
        self.visible = True
        self.unlit = unlit
        self.name = "Mesh"
        self._vert_dev = None
        self._faces_dev = None

    def update(self) -> None:
        """Mesh::update (mesh.cpp:339-362): copy the current vert/faces to device memory."""
        import torch
        vert = np.ascontiguousarray(self.vert, np.float32).reshape(-1)
        faces = np.ascontiguousarray(self.faces, np.uint32).reshape(-1)
        if vert.size % VERT_SZ:
            raise ValueError(f"Mesh {self.name!r}: vert has {vert.size} floats, not a multiple of {VERT_SZ}")
        self._vert_dev = torch.from_numpy(vert.copy()).cuda()
        self._faces_dev = torch.from_numpy(faces.view(np.int32).copy()).cuda() if faces.size else None

    @classmethod
    def _on_device(cls, vert_dev, face_size: int, unlit: bool) -> "Mesh":
        """A mesh drawn straight from a CUDA float32 tensor of vertices it does not own (no faces, identity model);
        its host ``vert`` stays empty and :meth:`update` is never needed."""
        m = cls(0, 0, face_size, unlit)
        m._vert_dev = vert_dev
        return m

    @property
    def n_verts(self) -> int:
        return int(np.asarray(self.vert).size // VERT_SZ)

    def model_matrix(self) -> np.ndarray:
        return model_matrix(self.rotation, self.translation, self.scale)

    def auto_faces(self) -> None:
        """mesh.cpp:628-631."""
        self.faces = np.arange(self.n_verts, dtype=np.uint32)

    def repeat(self, n: int) -> None:
        """Mesh::repeat (mesh.cpp:633-650): n copies of vert and faces, copy i's indices offset by i * n_verts."""
        if n < 1:
            return
        nv = np.uint32(self.n_verts)
        faces = np.asarray(self.faces, np.uint32)
        self.vert = np.tile(np.asarray(self.vert, np.float32), n)
        self.faces = (np.tile(faces, n) + np.repeat(np.arange(n, dtype=np.uint32) * nv, faces.size)).astype(np.uint32)

    def apply_transform(self, r, t=None, start: int = 0, end: int = -1) -> None:
        """Mesh::apply_transform (mesh.cpp:652-678) on the host vert, positions only, vertices start..end-1 (end -1:
        all).  ``r``, ``t``: axis-angle rotation and translation; or ``r`` a 4x4 matrix (M[row, col]) and no ``t``.
        Bit-exact with glm: each position becomes (M0 x + M1 y) + (M2 z + M3), Mk the matrix's column k."""
        m = np.asarray(r, _F) if t is None else _glm_transform(r, t)
        if m.shape != (4, 4):
            raise ValueError("apply_transform: r must be a 4x4 matrix when t is not given")
        if end == -1:
            end = self.n_verts
        self.vert = np.asarray(self.vert, np.float32)
        v = self.vert.reshape(-1, VERT_SZ)[start:end]
        x, y, z = v[:, 0:1], v[:, 1:2], v[:, 2:3]
        col = [m[:3, k][None, :] for k in range(4)]
        v[:, :3] = (col[0] * x + col[1] * y) + (col[2] * z + col[3] * _F(1))

    def _as_c(self) -> _capi.vr_mesh_desc:
        if self._vert_dev is None:
            self.update()
        d = _capi.vr_mesh_desc()
        n = int(self._vert_dev.numel()) // VERT_SZ
        d.vert_dev = self._vert_dev.data_ptr() if n else None
        d.faces_dev = self._faces_dev.data_ptr() if self._faces_dev is not None else None
        d.n_verts = n
        d.n_faces = int(self._faces_dev.numel()) // self.face_size if self._faces_dev is not None else 0
        d.face_size, d.unlit = int(self.face_size), int(bool(self.unlit))
        col_major = self.model_matrix().T.reshape(16)
        for i in range(16):
            d.model[i] = float(col_major[i])
        return d

    # ---- presets (mesh.cpp:399-626)
    @staticmethod
    def Cube(color=DEFAULT_COLOR) -> "Mesh":
        """Unit cube centred at 0: 36 vertices, 12 triangles, flat normals (mesh.cpp:399-449)."""
        m = Mesh(36, 0, 3)
        # faces in the order -z, +z, -y, +y, -x, +x; each is two triangles with corners (a, b) in units of 0.5,
        # where (a, b) is (x, y) on the z faces, (x, z) on the y faces and (z, y) on the x faces
        corners = [(-1, -1), (1, 1), (1, -1), (1, 1), (-1, -1), (-1, 1)]
        v = []
        for axis, side in [(2, -1), (2, 1), (1, -1), (1, 1), (0, -1), (0, 1)]:
            normal = [0.0, 0.0, 0.0]
            normal[axis] = float(side)
            for a, b in corners:
                p = [0.0, 0.0, 0.0]
                p[axis] = 0.5 * side
                if axis == 2:
                    p[0], p[1] = 0.5 * a, 0.5 * b
                elif axis == 1:
                    p[0], p[2] = 0.5 * a, 0.5 * b
                else:
                    p[1], p[2] = 0.5 * b, 0.5 * a
                v.extend(p + list(color) + normal)
        m.vert = np.asarray(v, np.float32)
        m.name = "Cube"
        return m

    @staticmethod
    def Sphere(rings: int = 15, sectors: int = 30, color=DEFAULT_COLOR) -> "Mesh":
        """UV sphere of radius 1: rings*sectors vertices, (rings-1)*sectors*2 triangles (mesh.cpp:451-491)."""
        m = Mesh(rings * sectors, (rings - 1) * sectors * 2, 3)
        R = float(np.float32(math.pi / float(np.float32(rings - 1))))
        S = float(np.float32(2 * math.pi / float(np.float32(sectors))))
        v = np.zeros((rings, sectors, VERT_SZ), np.float64)
        for r in range(rings):
            rR = float(np.float32(r * R))
            for s in range(sectors):
                sS = float(np.float32(s * S))
                z = math.sin(-0.5 * math.pi + rR)
                x = math.cos(sS) * math.sin(rR)
                y = math.sin(sS) * math.sin(rR)
                v[r, s] = (x, y, z, *color, x, y, z)
        m.vert = v.astype(np.float32).reshape(-1)
        f = []
        for r in range(rings - 1):
            nr = r + 1
            for s in range(sectors):
                ns = (s + 1) % sectors
                f += [r * sectors + ns, r * sectors + s, nr * sectors + s,
                      nr * sectors + s, nr * sectors + ns, r * sectors + ns]
        m.faces = np.asarray(f, np.uint32)
        m.name = "Sphere"
        return m

    @staticmethod
    def Lattice(reso: int = 8, color=GREY) -> "Mesh":
        """reso^3 unlit points at the cell centres of the unit cube, x slowest (mesh.cpp:493-520)."""
        c = (np.arange(reso, dtype=_F) + _F(0.5)) / _F(reso)
        m = Mesh(reso ** 3, 0, 1)
        v = m.vert.reshape(reso, reso, reso, VERT_SZ)
        v[..., 0] = c[:, None, None]
        v[..., 1] = c[None, :, None]
        v[..., 2] = c[None, None, :]
        v[..., 3:6] = np.asarray(color, _F)
        v[..., 6:9] = (1, 0, 0)
        m.name = "Lattice"
        m.unlit = True
        return m

    @staticmethod
    def CameraFrustum(focal_length, image_width, image_height, z=-0.3, color=GREY) -> "Mesh":
        """A camera's frustum as 8 unlit lines from the origin to the z plane (mesh.cpp:522-554), in the reference's
        float operation order, e.g. (z * -halfw) * invf."""
        invf = _F(1) / _F(focal_length)
        hw, hh = _F(image_width) * _F(0.5), _F(image_height) * _F(0.5)
        z = _F(z)
        col = [float(c) for c in np.asarray(color, _F)]
        m = Mesh(5, 8, 2)
        corners = [(-hw, -hh), (-hw, hh), (hw, hh), (hw, -hh)]
        v = [0.0, 0.0, 0.0, *col, 0.0, 0.0, 1.0]
        for a, b in corners:
            v += [(z * a) * invf, (z * b) * invf, z, *col, 0.0, 0.0, 1.0]
        m.vert = np.asarray(v, _F)
        m.faces = np.asarray([0, 1, 0, 2, 0, 3, 0, 4, 1, 2, 2, 3, 3, 4, 4, 1], np.uint32)
        m.name = "CameraFrustum"
        m.unlit = True
        return m

    @staticmethod
    def Line(a, b, color=GREY) -> "Mesh":
        """One unlit segment a -> b (mesh.cpp:556-568)."""
        m = Mesh(2, 1, 2)
        m.vert = np.asarray([*a, *color, 0, 0, 1, *b, *color, 0, 0, 1], np.float32)
        m.faces = np.asarray([0, 1], np.uint32)
        m.name = "Line"
        m.unlit = True
        return m

    @staticmethod
    def Lines(points, color=GREY) -> "Mesh":
        """Polyline through N points (N*3 floats): N-1 unlit segments i -> i+1 (mesh.cpp:570-600)."""
        p = np.asarray(points, np.float32).reshape(-1)
        if p.size % 3:
            print("Lines: Number of elements in points must be divisible by 3")
        n = p.size // 3
        m = Mesh(n, max(n - 1, 0), 2)
        v = m.vert.reshape(n, VERT_SZ)
        v[:, :3] = p[:3 * n].reshape(n, 3)
        v[:, 3:6] = color
        v[:, 6:9] = (0, 0, 1)
        m.faces = np.stack([np.arange(n - 1), np.arange(1, n)], 1).astype(np.uint32).reshape(-1) if n > 1 else \
            np.zeros(0, np.uint32)
        m.name = "Lines"
        m.unlit = True
        return m

    @staticmethod
    def Points(points, color=GREY) -> "Mesh":
        """Point cloud of N points (N*3 floats), unlit, no faces (mesh.cpp:602-626)."""
        p = np.asarray(points, np.float32).reshape(-1)
        if p.size % 3:
            print("Points: Number of elements in points must be divisible by 3")
        n = p.size // 3
        m = Mesh(n, 0, 1)
        v = m.vert.reshape(n, VERT_SZ)
        v[:, :3] = p[:3 * n].reshape(n, 3)
        v[:, 3:6] = color
        v[:, 6:9] = (0, 0, 1)
        m.name = "Points"
        m.unlit = True
        return m


    # ---- loaders (mesh.cpp:680-951; mesh_io.py)
    @staticmethod
    def load_basic_obj(path) -> "Mesh":
        """Mesh::load_basic_obj: triangles, vertex colours and normals of an OBJ file (see mesh_io.py)."""
        from .mesh_io import load_basic_obj
        return load_basic_obj(path)

    @staticmethod
    def load_mem_basic_obj(text) -> "Mesh":
        """Mesh::load_mem_basic_obj: :meth:`load_basic_obj` of OBJ text in memory; the mesh is named "OBJ"."""
        from .mesh_io import load_mem_basic_obj
        return load_mem_basic_obj(text)

    @staticmethod
    def open_drawlist(path, default_visible: bool = True) -> list:
        """Mesh::open_drawlist: the meshes a drawlist .npz file describes, in name order (see mesh_io.py)."""
        from .mesh_io import open_drawlist
        return open_drawlist(path, default_visible)

    @staticmethod
    def open_drawlist_mem(data, default_visible: bool = True) -> list:
        """Mesh::open_drawlist_mem: :meth:`open_drawlist` of the bytes of a drawlist .npz."""
        from .mesh_io import open_drawlist_mem
        return open_drawlist_mem(data, default_visible)


def estimate_normals(mesh: Mesh, stream=None) -> None:
    """estimate_normals (mesh.cpp:63-97) on the GPU: each vertex's normal becomes the normalised sum of the cross
    products of its triangles (``faces`` empty: consecutive vertex triples), byte for byte the reference's.  Uploads
    the mesh, runs ``vr_mesh_estimate_normals`` on its device buffer and copies the vertices back, so the host
    ``vert`` and the device copy both hold the result.  Raises :class:`VolrendError` without a device."""
    import torch
    from .host import _stream_ptr
    faces = np.asarray(mesh.faces, np.uint32).reshape(-1)
    if not torch.cuda.is_available():
        check(lib().vr_mesh_estimate_normals(None, 0, None, 0, None))    # VR_ENODEVICE: no CPU fallback
    mesh.update()
    vd, fd = mesh._vert_dev, mesh._faces_dev
    s = torch.cuda.current_stream() if stream is None else stream
    s.wait_stream(torch.cuda.current_stream())                         # the upload ran on the current stream
    check(lib().vr_mesh_estimate_normals(vd.data_ptr() if vd.numel() else None, vd.numel() // VERT_SZ,
                                         fd.data_ptr() if fd is not None else None, faces.size // 3,
                                         _stream_ptr(s)))
    s.synchronize()
    mesh.vert = vd.cpu().numpy()


def _mesh_table(meshes_per_view):
    """The descriptors of every view's visible meshes, view after view, and the ``mesh_off`` offsets (n_views + 1
    entries) that delimit each view's run of them."""
    per_view = [[m for m in ms if m.visible] for ms in meshes_per_view]
    off = np.zeros(len(per_view) + 1, np.int32)
    off[1:] = np.cumsum([len(v) for v in per_view], dtype=np.int64)
    arr = (_capi.vr_mesh_desc * max(int(off[-1]), 1))()
    i = 0
    for vis in per_view:
        for m in vis:
            arr[i] = m._as_c()
            i += 1
    return arr, (C.c_int32 * len(off))(*[int(v) for v in off])


def draw_meshes_batch(cams, meshes_per_view, images, depth, stream=None) -> None:
    """:func:`draw_meshes` for many views in one call (``vr_draw_meshes_batch``): view i draws the visible meshes of
    ``meshes_per_view[i]`` with ``cams[i]`` over ``images[i]`` (CUDA uint8 [V,H,W,4]) and ``depth[i]`` (CUDA float32
    [V,H,W]), byte for byte what :func:`draw_meshes` would draw.  Every camera has the same size.  A list may hold
    shallow copies (``copy.copy(mesh)``) of one uploaded mesh with their own transform, ``visible`` and ``unlit``:
    they share its device buffers, so nothing is uploaded per view."""
    from .host import _cams_array, _stream_ptr
    if len(meshes_per_view) != len(cams):
        raise ValueError(f"meshes_per_view: expected {len(cams)} lists (one per camera), got {len(meshes_per_view)}")
    arr, off = _mesh_table(meshes_per_view)
    check(lib().vr_draw_meshes_batch(_cams_array(cams), len(cams), arr, off,
                                     images.data_ptr() if images is not None else None,
                                     depth.data_ptr() if depth is not None else None, _stream_ptr(stream)))


def draw_meshes(cam, meshes, image, depth, stream=None) -> None:
    """Draws the visible ``meshes`` in order over ``image`` (CUDA uint8 [H,W,4]) and ``depth`` (CUDA float32
    [H,W], ray distance; GL depth test LESS against it).  Covered pixels receive the mesh colour and the
    fragment's ray distance.  Meshes never uploaded are uploaded first (:meth:`Mesh.update`)."""
    from .host import _stream_ptr
    vis = [m for m in meshes if m.visible]
    arr = (_capi.vr_mesh_desc * max(len(vis), 1))()
    for i, m in enumerate(vis):
        arr[i] = m._as_c()
    c = cam._as_c()
    check(lib().vr_draw_meshes(C.byref(c), arr, len(vis), image.data_ptr() if image is not None else None,
                               depth.data_ptr() if depth is not None else None, _stream_ptr(stream)))
