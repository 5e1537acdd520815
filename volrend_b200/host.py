"""Host-side mirror of volrend's renderer surface, over the C-ABI.

Same names, argument meaning and error behaviour as the reference classes so tests read
like reference usage (paths relative to /root/reference):

* :class:`DataFormat`      ``include/volrend/data_format.hpp``, ``src/n3tree.cpp:55-101``
* :class:`N3Tree`          ``include/volrend/n3tree.hpp``, loader ``src/n3tree.cpp:111-362``;
  ``load_cuda``/``free_cuda`` (``src/cuda/n3tree.cu``) go through ``vr_tree_create``
* :class:`Camera`          ``include/volrend/camera.hpp``, ``src/camera.cpp:26-76``
* :class:`RenderOptions`   ``include/volrend/render_options.hpp:11-53``
* :func:`launch_renderer`  ``include/volrend/cuda/renderer_kernel.hpp:9-12``
* :class:`VolumeRenderer`  ``include/volrend/renderer.hpp:11-42`` with the GL-free offscreen
  Impl that replaces ``src/cuda_renderer.cpp``

PyTorch is used only to own device memory and streams.  The compiled C++ shim
(``volrend_b200/csrc/shim``) offers the same surface to the unchanged reference C++ callers.
"""
from __future__ import annotations

import copy
import ctypes as C
import math
import os
from dataclasses import dataclass, field

import numpy as np

from . import _capi
from ._capi import check, lib

VOLREND_GLOBAL_BASIS_MAX = 25
CAMERA_DEFAULT_FOCAL_LENGTH = 1111.11


# ---------------------------------------------------------------------------- DataFormat
class DataFormat:
    RGBA, SH, SG, ASG = 0, 1, 2, 3
    _NAMES = {0: "RGBA", 1: "SH", 2: "SG", 3: "ASG"}

    def __init__(self, format: int = 0, basis_dim: int = -1):
        self.format = format
        self.basis_dim = basis_dim

    def parse(self, s: str) -> None:
        """'SH16', 'SG25', 'RGBA' ... (src/n3tree.cpp:55-78)."""
        idx = next((i for i, ch in enumerate(s) if not ch.isalpha()), -1)
        if idx >= 0:
            digits = ""
            for ch in s[idx:]:
                if ch.isdigit() or (not digits and ch in "+-"):
                    digits += ch
                else:
                    break
            try:
                self.basis_dim = int(digits)
            except ValueError:
                self.basis_dim = 0          # atoi semantics
            self.format = {"ASG": self.ASG, "SG": self.SG, "SH": self.SH}.get(s[:idx], self.RGBA)
        else:
            self.basis_dim = -1
            self.format = self.RGBA

    def to_string(self) -> str:
        out = self._NAMES.get(self.format, "UNKNOWN")
        if self.basis_dim != -1:
            out += str(self.basis_dim)
        return out


# ---------------------------------------------------------------------------- N3Tree
class N3Tree:
    """Read-only N3Tree: npz loader + device upload (re-layout happens in ``load_cuda``)."""

    def __init__(self, path: str | None = None, gpu_decode: bool = True):
        # gpu_decode: quantised files (quant_colors/quant_map/...) are decoded by the GPU at upload
        # (vr_tree_create_quantized) instead of the reference's CPU loop; ``data_`` then decodes
        # lazily on first access.
        self.gpu_decode = gpu_decode
        self.quant_ = None      # compressed arrays of a quantised file
        self.N = 0
        self.data_dim = 0
        self.data_format = DataFormat()
        self.capacity = 0
        self.scale = np.ones(3, np.float32)
        self.offset = np.zeros(3, np.float32)
        self.use_ndc = False
        self.ndc_width = self.ndc_height = self.ndc_focal = 0.0
        self._data = None       # fp16 [cap,N,N,N,data_dim]  (see the data_ property)
        self.child_ = None      # int32 [cap,N,N,N]
        self.extra_ = None      # f32
        self._handle = None     # vr_tree*
        self._device = None     # CUDA device of the tree (set by load_cuda)
        self._data_loaded = False
        self._cuda_loaded = False
        self._slot_map = False  # loaded with the table entry -> slot map (load_cuda(slot_map=True))
        if path is not None:
            self.open(path)

    @property
    def data_(self):
        """N3Tree::data_ (fp16 [capacity,N,N,N,data_dim]); decoded on demand for quantised files."""
        if self._data is None and self.quant_ is not None:
            self._data = self._decode_quantised()
        return self._data

    @data_.setter
    def data_(self, v):
        self._data = v

    # -- reference surface
    def is_data_loaded(self) -> bool:
        return self._data_loaded

    def is_cuda_loaded(self) -> bool:
        return self._cuda_loaded

    def clear_cpu_memory(self) -> None:
        self._data = None       # n3tree.cpp:441-447 keeps child_

    def open(self, path: str) -> None:
        """src/n3tree.cpp:111-154.  A missing file leaves the tree unloaded, like the reference."""
        self.free_cuda()
        self._data_loaded = False
        assert path.endswith(".npz")
        if not os.path.exists(path):
            print(f"Can't load because file does not exist: {path}")
            return
        with np.load(path) as npz:
            self.load_npz({k: npz[k] for k in npz.files})
        pb = path[:-4] + "_poses_bounds.npy"
        self.use_ndc = os.path.exists(pb)
        if self.use_ndc:
            self._unpack_llff_poses_bounds(np.load(pb))
        self.load_cuda()
        self._data_loaded = True

    def open_arrays(self, *, child, data, offset, invradius3, data_dim, data_format, extra=None) -> None:
        """In-memory equivalent of ``open_mem`` for already-decoded arrays."""
        self.free_cuda()
        npz = dict(child=child, data=data, offset=offset, invradius3=invradius3,
                   data_dim=np.int64(data_dim), data_format=np.array(data_format))
        if extra is not None:
            npz["extra_data"] = extra
        self.load_npz(npz)
        self.use_ndc = False
        self.load_cuda()
        self._data_loaded = True

    @classmethod
    def from_synth(cls, t) -> "N3Tree":
        tree = cls()
        tree.open_arrays(child=t.child, data=t.data, offset=t.offset, invradius3=t.invradius3,
                         data_dim=t.data_dim, data_format=t.data_format, extra=t.extra)
        return tree

    def load_npz(self, npz: dict) -> None:
        """src/n3tree.cpp:228-362 including the quantised-colour decode (:279-340)."""
        self.data_dim = int(np.asarray(npz["data_dim"]).reshape(-1)[0])
        self.data_format = DataFormat()
        if "data_format" in npz:
            self.data_format.parse(str(np.asarray(npz["data_format"]).reshape(-1)[0]))
        elif self.data_dim == 4:
            self.data_format.format = DataFormat.RGBA
        else:
            self.data_format.format = DataFormat.SH
            self.data_format.basis_dim = (self.data_dim - 1) // 3
        if "invradius3" in npz:
            self.scale = np.asarray(npz["invradius3"], np.float32).reshape(3).copy()
        else:
            self.scale = np.full(3, np.float32(np.asarray(npz["invradius"], np.float64).reshape(-1)[0]), np.float32)
        self.offset = np.asarray(npz["offset"], np.float32).reshape(3).copy()
        child = np.asarray(npz["child"])
        if child.dtype != np.int32:
            child = child.astype(np.int32)
        self.child_ = np.ascontiguousarray(child)
        self.N = int(self.child_.shape[1])
        if self.N != 2:
            print("WARNING: N != 2 probably doesn't work.")
        self.quant_ = None
        self._data = None
        if "quant_colors" in npz:
            qc = np.asarray(npz["quant_colors"])
            if qc.dtype.itemsize != 2:
                raise RuntimeError("codebook must be stored in half precision")
            qmap = np.asarray(npz["quant_map"])
            self.capacity = int(qmap.shape[1])
            n_basis = int(qmap.shape[0])
            if qc.shape[0] != n_basis:
                raise RuntimeError("codebook and map basis numbers does not match")
            retained = np.asarray(npz["data_retained"]) if "data_retained" in npz else None
            n_retain = 0 if retained is None else int(retained.shape[0])
            n_child = self.capacity * self.N ** 3
            self.quant_ = dict(
                colors=np.ascontiguousarray(qc.view(np.uint16).reshape(n_basis, 65536, 3)),
                map=np.ascontiguousarray(qmap.astype(np.uint16, copy=False).reshape(n_basis, n_child)),
                sigma=np.ascontiguousarray(np.asarray(npz["sigma"]).view(np.uint16).reshape(n_child)),
                retained=None if retained is None else np.ascontiguousarray(retained.view(np.uint16).reshape(n_retain, n_child, 3)),
                n_quant=n_basis, n_retain=n_retain)
            if not self.gpu_decode:
                self._data = self._decode_quantised()
        else:
            data = np.asarray(npz["data"])
            self.capacity = int(data.shape[0])
            if data.dtype.itemsize != 2:
                raise RuntimeError("data must be stored in half precision")
            self._data = np.ascontiguousarray(data.view(np.float16))
        self.extra_ = np.ascontiguousarray(np.asarray(npz["extra_data"], np.float32)) if "extra_data" in npz else None

    def _decode_quantised(self) -> np.ndarray:
        """Vectorised form of the scalar decode loops of src/n3tree.cpp:309-340."""
        q = self.quant_
        n_basis, n_retain = q["n_quant"], q["n_retain"]
        n_total = n_basis + n_retain
        n_child = self.capacity * self.N ** 3
        data = np.zeros((n_child, self.data_dim), np.uint16)
        for j in range(n_basis):
            cols = q["colors"][j][q["map"][j].astype(np.int64)]      # [n_child,3]
            for k in range(3):
                data[:, j + n_retain + k * n_total] = cols[:, k]
        data[:, self.data_dim - 1] = q["sigma"]
        for j in range(n_retain):
            for k in range(3):
                data[:, j + k * n_total] = q["retained"][j, :, k]
        return data.view(np.float16).reshape(self.capacity, self.N, self.N, self.N, self.data_dim)

    def _unpack_llff_poses_bounds(self, pb: np.ndarray) -> None:
        """src/n3tree.cpp:22-52 (only the fields the ray path uses)."""
        p = np.asarray(pb).reshape(-1)
        self.ndc_height, self.ndc_width, self.ndc_focal = float(p[4]), float(p[9]), float(p[14])

    # -- device side (replaces src/cuda/n3tree.cu)
    def load_cuda(self, slot_map: bool = False) -> None:
        """Uploads the tree (vr_tree_create).  ``slot_map`` keeps the table entry -> slot map on the device
        (VR_TREE_SLOT_MAP, 4 bytes per table entry), which :func:`leaf_weights` needs."""
        self.free_cuda()
        flags = _capi.VR_TREE_SLOT_MAP if slot_map else 0
        use_quant = self.quant_ is not None and self.gpu_decode
        qd = _capi.vr_tree_quant_desc() if use_quant else None
        d = qd.base if use_quant else _capi.vr_tree_desc()
        d.child = self.child_.ctypes.data
        if not use_quant:
            data = np.ascontiguousarray(self.data_)
            d.data = data.ctypes.data
        d.extra = self.extra_.ctypes.data if self.extra_ is not None else None
        d.capacity, d.N, d.data_dim = self.capacity, self.N, self.data_dim
        d.format, d.basis_dim = self.data_format.format, self.data_format.basis_dim
        for i in range(3):
            d.offset[i] = float(self.offset[i])
            d.scale[i] = float(self.scale[i])
        d.use_ndc = int(self.use_ndc)
        d.ndc_width, d.ndc_height, d.ndc_focal = self.ndc_width, self.ndc_height, self.ndc_focal
        h = C.c_void_p()
        if use_quant:
            q = self.quant_
            qd.quant_colors, qd.quant_map, qd.sigma = q["colors"].ctypes.data, q["map"].ctypes.data, q["sigma"].ctypes.data
            qd.data_retained = q["retained"].ctypes.data if q["retained"] is not None else None
            qd.n_quant, qd.n_retain = q["n_quant"], q["n_retain"]
            check(lib().vr_tree_create_quantized_ex(C.byref(qd), flags, C.byref(h)))
        else:
            check(lib().vr_tree_create_ex(C.byref(d), flags, C.byref(h)))
        self._handle = h
        self._cuda_loaded = True
        self._slot_map = bool(slot_map)
        import torch
        self._device = torch.cuda.current_device()     # the device vr_tree_create put the tree on

    def _plain_desc(self):
        """vr_tree_desc over the decoded host arrays (keeps them alive through the returned tuple)."""
        d = _capi.vr_tree_desc()
        data = np.ascontiguousarray(self.data_)
        d.child, d.data = self.child_.ctypes.data, data.ctypes.data
        d.extra = self.extra_.ctypes.data if self.extra_ is not None else None
        d.capacity, d.N, d.data_dim = self.capacity, self.N, self.data_dim
        d.format, d.basis_dim = self.data_format.format, self.data_format.basis_dim
        for i in range(3):
            d.offset[i] = float(self.offset[i])
            d.scale[i] = float(self.scale[i])
        d.use_ndc = int(self.use_ndc)
        d.ndc_width, d.ndc_height, d.ndc_focal = self.ndc_width, self.ndc_height, self.ndc_focal
        return d, data

    def update_data(self, data, stream=None) -> None:
        """Replaces the leaf values on the device (vr_tree_update_data): ``data`` is a CUDA tensor on the tree's device,
        fp16 or fp32 (rounded with ``.half()``), shaped like ``data_``.  The structure does not change.  The host copy
        of the data, and the compressed arrays of a quantised file, are dropped (``clear_cpu_memory``), so this object
        never describes two different trees.  Asynchronous on ``stream``.  The tree must be loaded with
        ``load_cuda(slot_map=True)``."""
        import torch
        dev = _slot_tree(self, "update_data")
        shape = (self.capacity, self.N, self.N, self.N, self.data_dim)
        if (not isinstance(data, torch.Tensor) or data.dtype not in (torch.float16, torch.float32)
                or data.device != dev or tuple(data.shape) != shape):
            raise ValueError(f"data must be a float16 or float32 tensor of shape {shape} on {dev}")
        h = data.half().contiguous()
        check(lib().vr_tree_update_data(self._handle, h.data_ptr(), _stream_ptr(stream)))
        if stream is not None and isinstance(stream, torch.cuda.Stream) and h is not data:
            h.record_stream(stream)     # the temporary is read by the kernel on `stream`
        self.clear_cpu_memory()
        self.quant_ = None

    def free_cuda(self) -> None:
        if self._handle is not None:
            lib().vr_tree_destroy(self._handle)
            self._handle = None
        self._cuda_loaded = False
        self._slot_map = False

    # -- grid wireframe (vr_tree_wireframe)
    def wireframe_vertex_count(self, max_depth: int = 100000) -> int:
        """Vertices of :meth:`gen_wireframe` ``(max_depth)`` (24 per emitted cell), without generating them."""
        if not self.is_cuda_loaded():
            raise RuntimeError("N3Tree is not loaded on the device")
        n = C.c_int64()
        check(lib().vr_tree_wireframe(self._handle, int(max_depth), None, 0, C.byref(n), _stream_ptr(None)))
        return int(n.value)

    def wireframe_device(self, max_depth: int = 100000, stream=None):
        """:meth:`gen_wireframe` into a new CUDA float32 tensor (flat, 9 floats per vertex), stream-ordered."""
        import torch
        n = self.wireframe_vertex_count(max_depth)
        out = torch.empty(n * 9, dtype=torch.float32, device="cuda")
        got = C.c_int64()
        check(lib().vr_tree_wireframe(self._handle, int(max_depth), out.data_ptr(), n, C.byref(got), _stream_ptr(stream)))
        return out

    def gen_wireframe(self, max_depth: int = 100000) -> np.ndarray:
        """N3Tree::gen_wireframe (n3tree.cpp:365-434), byte for byte: the octree cut at ``max_depth`` as line
        segments, 12 per cell = 24 vertices of 9 float32 (position, colour 0, normal 0,0,1).  Generated on the GPU
        from the device tree and copied to the host."""
        return self.wireframe_device(max_depth).cpu().numpy()

    # -- point queries (vr_tree_query / vr_tree_eval)
    def _check_points(self, name: str, pts, n=None) -> bool:
        """Validates a ``[n, 3]`` float32 numpy array or CUDA tensor; True for numpy."""
        import torch
        if self.child_ is None:
            raise RuntimeError("N3Tree has no data: open a tree first")
        is_np = isinstance(pts, np.ndarray)
        if not is_np and not (isinstance(pts, torch.Tensor) and pts.is_cuda):
            raise TypeError(f"{name} must be a float32 numpy array or a CUDA torch tensor")
        if pts.dtype not in (np.float32, torch.float32):
            raise TypeError(f"{name} must be float32, not {pts.dtype}")
        if pts.ndim != 2 or pts.shape[1] != 3 or (n is not None and pts.shape[0] != n):
            raise ValueError(f"{name} must have shape [{'n' if n is None else n}, 3], not {tuple(pts.shape)}")
        return is_np

    def _launch(self, inputs, outputs, stream, call) -> None:
        """Runs ``call(stream_ptr)`` on ``stream`` (None: torch's current stream) on the tree's device, ordered after
        the work of the current stream that produced ``inputs`` and allocated ``outputs``; the tensors are recorded
        on ``stream`` so that the caching allocator does not hand their memory out while the kernel still runs."""
        import torch
        with torch.cuda.device(self._device):
            cur = torch.cuda.current_stream()
            if stream is None:
                s = cur
            elif isinstance(stream, torch.cuda.Stream):
                s = stream
            else:
                s = torch.cuda.ExternalStream(int(stream))
            if s != cur:
                s.wait_stream(cur)
                for t in (*inputs, *outputs):
                    t.record_stream(s)
            call(_stream_ptr(s))
        return s

    def _on_device(self, name: str, pts):
        """Loads the tree onto the GPU if needed; -> contiguous CUDA float32 tensor of ``pts`` on the tree's device."""
        import torch
        if not self.is_cuda_loaded():
            self.load_cuda()
        if isinstance(pts, np.ndarray):
            return torch.from_numpy(np.ascontiguousarray(pts)).to(torch.device("cuda", self._device))
        if pts.device.index != self._device:
            raise ValueError(f"{name} live on {pts.device}, the tree on cuda:{self._device}")
        with torch.cuda.device(self._device):
            return pts.contiguous()

    def query(self, points, *, stream=None):
        """query_single_from_root for world points ``[n, 3]`` float32 -> ``(data, cube_sz, local)``: the leaf's data
        row (float16 ``[n, data_dim]``, sigma last), its cube size N^depth (float32 ``[n]``) and the point's in-cell
        coordinates (float32 ``[n, 3]``).  numpy in, numpy out: the call returns when the results are on the host.  A
        CUDA tensor (on the tree's device) in gives tensors on that device, written on ``stream`` (default: the
        current stream) after the current stream's earlier work, with no host round trip."""
        import torch
        is_np = self._check_points("points", points)
        x = self._on_device("points", points)
        n = x.shape[0]
        data = torch.empty((n, self.data_dim), dtype=torch.float16, device=x.device)
        cube = torch.empty(n, dtype=torch.float32, device=x.device)
        local = torch.empty((n, 3), dtype=torch.float32, device=x.device)
        s = self._launch((x,), (data, cube, local), stream,
                         lambda sp: check(lib().vr_tree_query(self._handle, x.data_ptr(), n, data.data_ptr(),
                                                              cube.data_ptr(), local.data_ptr(), sp)))
        if is_np:
            s.synchronize()
            return data.cpu().numpy(), cube.cpu().numpy(), local.cpu().numpy()
        return data, cube, local

    def eval(self, points, dirs, options=None, *, stream=None):
        """The probe disc's colour of the leaves of world points ``[n, 3]`` seen along ``dirs`` ``[n, 3]`` (used as
        given) -> ``(rgb, sigma)`` float32 ``[n, 3]`` and ``[n]``; of ``options`` (a :class:`RenderOptions`) only
        ``basis_minmax`` is read.  Same input and output types, devices and stream order as :meth:`query`."""
        import torch
        is_np = self._check_points("points", points)
        if self._check_points("dirs", dirs, points.shape[0]) != is_np:
            raise TypeError("points and dirs must both be numpy arrays or both CUDA tensors")
        x, d = self._on_device("points", points), self._on_device("dirs", dirs)
        n = x.shape[0]
        rgb = torch.empty((n, 3), dtype=torch.float32, device=x.device)
        sigma = torch.empty(n, dtype=torch.float32, device=x.device)
        o = (options if options is not None else RenderOptions())._as_c()
        s = self._launch((x, d), (rgb, sigma), stream,
                         lambda sp: check(lib().vr_tree_eval(self._handle, x.data_ptr(), d.data_ptr(), n, C.byref(o),
                                                             rgb.data_ptr(), sigma.data_ptr(), sp)))
        if is_np:
            s.synchronize()
            return rgb.cpu().numpy(), sigma.cpu().numpy()
        return rgb, sigma

    def info(self) -> dict:
        inf = _capi.vr_tree_info()
        check(lib().vr_tree_get_info(self._handle, C.byref(inf)))
        return {k: getattr(inf, k) for k, _ in inf._fields_}

    def __del__(self):
        try:
            self.free_cuda()
        except Exception:
            pass


# ---------------------------------------------------------------------------- Camera
class Camera:
    def __init__(self, width: int = 256, height: int = 256, fx: float = CAMERA_DEFAULT_FOCAL_LENGTH, fy: float = -1.0):
        self.width, self.height = int(width), int(height)
        self.fx = CAMERA_DEFAULT_FOCAL_LENGTH if fx < 0 else float(fx)
        self.fy = self.fx if fy < 0 else float(fy)
        self.center = np.array([-3.55, 0.0, 3.55], np.float32)      # camera.cpp:32-35
        self.v_back = np.array([-0.7071068, 0.0, 0.7071068], np.float32)
        self.v_world_up = np.array([0.0, 0.0, 1.0], np.float32)
        self.origin = np.zeros(3, np.float32)
        self.transform = np.zeros((4, 3), np.float32)               # glm::mat4x3: 4 columns of vec3
        self._update()

    def _update(self, transform_from_vecs: bool = True, copy_cuda: bool = True) -> None:
        """camera.cpp:47-76 (the device copy is unnecessary: c2w travels by value)."""
        if transform_from_vecs:
            self.v_back = (self.v_back / np.linalg.norm(self.v_back)).astype(np.float32)
            r = np.cross(self.v_world_up, self.v_back)
            self.v_right = (r / np.linalg.norm(r)).astype(np.float32)
            self.v_up = np.cross(self.v_back, self.v_right).astype(np.float32)
            self.transform[0], self.transform[1] = self.v_right, self.v_up
            self.transform[2], self.transform[3] = self.v_back, self.center

    def set_c2w(self, c2w) -> None:
        """Row-major 3x4/4x4 camera-to-world, as read by main_headless.cpp:40-63."""
        m = np.asarray(c2w, np.float32)[:3, :4]
        self.transform = np.ascontiguousarray(m.T)

    def _as_c(self) -> _capi.vr_camera:
        c = _capi.vr_camera()
        c.width, c.height, c.fx, c.fy = self.width, self.height, self.fx, self.fy
        flat = np.ascontiguousarray(self.transform, np.float32).reshape(12)
        for i in range(12):
            c.c2w[i] = float(flat[i])
        return c


# ---------------------------------------------------------------------------- RenderOptions
@dataclass
class RenderOptions:
    step_size: float = 1e-4
    sigma_thresh: float = 1e-2
    stop_thresh: float = 1e-2
    background_brightness: float = 1.0
    render_bbox: list = field(default_factory=lambda: [0.0, 0.0, 0.0, 1.0, 1.0, 1.0])
    basis_minmax: list = field(default_factory=lambda: [0, VOLREND_GLOBAL_BASIS_MAX - 1])
    rot_dirs: list = field(default_factory=lambda: [0.0, 0.0, 0.0])
    show_grid: bool = False
    grid_max_depth: int = 4
    render_depth: bool = False
    enable_probe: bool = False
    probe: list = field(default_factory=lambda: [0.0, 0.0, 1.0])
    probe_disp_size: int = 100

    def _as_c(self) -> _capi.vr_options:
        o = _capi.vr_options()
        o.step_size, o.sigma_thresh, o.stop_thresh = self.step_size, self.sigma_thresh, self.stop_thresh
        o.background_brightness = self.background_brightness
        for i in range(6):
            o.render_bbox[i] = float(self.render_bbox[i])
        o.basis_minmax[0], o.basis_minmax[1] = int(self.basis_minmax[0]), int(self.basis_minmax[1])
        for i in range(3):
            o.rot_dirs[i] = float(self.rot_dirs[i])
        o.render_depth = int(self.render_depth)
        return o


def _cams_array(cams) -> "C.Array":
    arr = (_capi.vr_camera * len(cams))()
    for i, cam in enumerate(cams):
        arr[i] = cam._as_c()
    return arr


def _stream_ptr(stream) -> int:
    if stream is None:
        import torch
        return torch.cuda.current_stream().cuda_stream
    return int(getattr(stream, "cuda_stream", stream))


def _rect(tile):
    if tile is None:
        return None
    r = _capi.vr_rect(*[int(v) for v in tile])
    return C.byref(r)


# ---------------------------------------------------------------------------- launch_renderer
def launch_renderer(tree: N3Tree, cam: Camera, options: RenderOptions, image_arr, depth_arr=None,
                    stream=None, offscreen: bool = False, *, float_out=None, counters=None, tile=None) -> None:
    """``launch_renderer`` (renderer_kernel.hpp:9-12).  ``image_arr``: CUDA uint8 tensor
    [H,W,4] written in full (row 0 = top row); ``depth_arr``: float32 [H,W] ray-distance limits,
    required unless ``offscreen``.  Asynchronous on ``stream``.  Extras (keyword-only):
    ``float_out`` float32 [H,W,4] tap of the un-quantised pixel, ``counters`` uint64[5] device
    tensor, ``tile`` (x0,y0,w,h)."""
    if not tree.is_cuda_loaded():
        raise RuntimeError("N3Tree is not loaded on the device")
    c, o = cam._as_c(), options._as_c()
    img = image_arr.data_ptr() if image_arr is not None else None
    fo = float_out.data_ptr() if float_out is not None else None
    s = _stream_ptr(stream)
    if offscreen:
        cn = counters.data_ptr() if counters is not None else None
        check(lib().vr_render(tree._handle, C.byref(c), C.byref(o), _rect(tile), img, fo, cn, s))
    else:
        if depth_arr is None or image_arr is None:
            raise ValueError("offscreen=False needs colour and depth inputs")
        check(lib().vr_render_composite(tree._handle, C.byref(c), C.byref(o), _rect(tile), img,
                                        depth_arr.data_ptr(), fo, s))
    if options.enable_probe:
        _draw_probe(tree, (c,), 1, options, o, tile, img, fo, s)


def _draw_probe(tree: N3Tree, cams, n_views: int, options: RenderOptions, o, tile, img, fo, s) -> None:
    """The ``enable_probe`` disc (volrend.cu:100-134) over the frames just rendered: one vr_draw_probe launch."""
    arr = cams if isinstance(cams, C.Array) else (_capi.vr_camera * n_views)(*cams)
    xyz = (C.c_float * 3)(*[float(v) for v in options.probe])
    check(lib().vr_draw_probe(tree._handle, arr, n_views, C.byref(o), xyz, int(options.probe_disp_size), _rect(tile),
                              img, fo, 0, s))


def render_bands(tree: N3Tree, cam: Camera, options: RenderOptions, band_h: int, n_parts: int, part: int,
                 image, *, float_out=None, stream=None) -> int:
    """Ray-tile sharding: render bands part, part+n_parts, ... (band_h rows each) of the frame into the
    compact ``image`` (uint8 [rows, W, 4]); returns the number of rows this part owns."""
    c, o = cam._as_c(), options._as_c()
    check(lib().vr_render_bands(tree._handle, C.byref(c), C.byref(o), int(band_h), int(n_parts), int(part),
                                image.data_ptr() if image is not None else None,
                                float_out.data_ptr() if float_out is not None else None, _stream_ptr(stream)))
    return lib().vr_band_rows(cam.height, int(band_h), int(n_parts), int(part))


def render_bands_batch(tree: N3Tree, cams, options: RenderOptions, band_h: int, n_parts: int, part: int, images, *,
                       float_out=None, stream=None) -> int:
    """render_bands for several views in ONE launch: ``images`` uint8 [V, rows, W, 4]; returns rows."""
    arr = _cams_array(cams)
    o = options._as_c()
    check(lib().vr_render_bands_batch(tree._handle, arr, len(cams), C.byref(o), int(band_h), int(n_parts), int(part),
                                      images.data_ptr() if images is not None else None,
                                      float_out.data_ptr() if float_out is not None else None, _stream_ptr(stream)))
    return lib().vr_band_rows(cams[0].height, int(band_h), int(n_parts), int(part)) if len(cams) else 0


VR_MG_VIEWS, VR_MG_TILES = 0, 1


class MultiGpuRenderer:
    """One process driving several GPUs (vr_mg_*, volrend_b200/csrc/vr_mg.cu): the tree replicated on
    ``devices``, views or ray tiles sharded over them, frames gathered on ``devices[0]`` by peer copies.
    ``tree`` is a host-loaded N3Tree (its own device copy is not used)."""

    def __init__(self, tree: N3Tree, devices):
        self.devices = [int(d) for d in devices]
        d, keep = tree._plain_desc()
        arr = (C.c_int * len(self.devices))(*self.devices)
        h = C.c_void_p()
        rc = lib().vr_mg_create(C.byref(d), arr, len(self.devices), C.byref(h))
        del keep
        if rc != 0:
            raise _capi.VolrendError(rc, lib().vr_mg_last_error(None).decode("utf-8", "replace"))
        self._h = h

    def render(self, cams, options: RenderOptions, *, mode=VR_MG_VIEWS, band_h=8, batch=0, out_dev0=None, out_host=None) -> float:
        """Renders every view; returns the device time in ms (max over devices).  ``out_dev0``: uint8 CUDA
        tensor [V,H,W,4] on devices[0] (or None: internal buffer); ``out_host``: optional CPU array/tensor."""
        arr = _cams_array(cams)
        o = options._as_c()
        ms = C.c_float(0)
        hp = None
        if out_host is not None:
            hp = out_host.data_ptr() if hasattr(out_host, "data_ptr") else out_host.ctypes.data
        rc = lib().vr_mg_render(self._h, arr, len(cams), C.byref(o), int(mode), int(band_h), int(batch),
                                out_dev0.data_ptr() if out_dev0 is not None else None, hp, C.byref(ms))
        if rc != 0:
            raise _capi.VolrendError(rc, lib().vr_mg_last_error(self._h).decode("utf-8", "replace"))
        return float(ms.value)

    def close(self):
        if self._h is not None:
            lib().vr_mg_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _per_view(cams, options) -> bool:
    """True when ``options`` is a sequence of one RenderOptions per camera, False for one RenderOptions."""
    if isinstance(options, RenderOptions):
        return False
    if len(options) != len(cams) or not all(isinstance(o, RenderOptions) for o in options):
        raise ValueError(f"options: one RenderOptions, or a sequence of {len(cams)} (one per camera)")
    return True


def _options_array(options) -> "C.Array":
    arr = (_capi.vr_options * len(options))()
    for i, o in enumerate(options):
        arr[i] = o._as_c()
    return arr


def render_batch(tree: N3Tree, cams, options, images, *, float_out=None, counters=None,
                 tile=None, stream=None) -> None:
    """The pose loop of main_headless.cpp:208-223 as one call; ``images``: uint8 [V,H,W,4].  ``options`` is one
    RenderOptions for every view, or a sequence of ``len(cams)`` of them: view i is then rendered with options[i]
    (vr_render_batch_opts), and ``enable_probe`` draws each view's disc with that view's probe settings."""
    arr = _cams_array(cams)
    img = images.data_ptr() if images is not None else None
    fo = float_out.data_ptr() if float_out is not None else None
    s = _stream_ptr(stream)
    cn = counters.data_ptr() if counters is not None else None
    if not _per_view(cams, options):
        o = options._as_c()
        check(lib().vr_render_batch(tree._handle, arr, len(cams), C.byref(o), _rect(tile), img, fo, cn, s))
        if options.enable_probe and len(cams):
            _draw_probe(tree, arr, len(cams), options, o, tile, img, fo, s)
        return
    oarr = _options_array(options)
    check(lib().vr_render_batch_opts(tree._handle, arr, len(cams), oarr, _rect(tile), img, fo, cn, s))
    _draw_probe_runs(tree, arr, options, oarr, tile, img, fo, s)


def leaf_weights(tree: N3Tree, cams, options: RenderOptions, out=None, alpha=None, counters=None, stream=None, *,
                 tile=None):
    """Maximum compositing weight of every leaf slot over the views ``cams`` (vr_tree_leaf_weights): a CUDA float32
    tensor ``[capacity, 2, 2, 2]`` (slot = node * 8 + octant) in which every shaded sample of every pixel has raised its
    leaf's entry to at least its weight T * (1 - att).  ``out`` (same shape or ``capacity * 8`` elements, float32, on
    the tree's device) accumulates over calls; without it a new tensor starts at -inf, the value of slots no view
    shades.  ``options`` is one RenderOptions (step, thresholds and bbox act as in rendering).  ``alpha``: optional
    float32 CUDA tensor ``[V, H, W]`` (tile-sized) that receives each ray's alpha; ``counters``: optional int64[5]
    device tensor, accumulated.  Asynchronous on ``stream``.  The tree must be loaded with
    ``load_cuda(slot_map=True)``."""
    import torch
    dev = _slot_tree(tree, "leaf_weights")
    cams, w, h = _march_views(cams, options, tile, "leaf_weights")
    out = _accumulator("out", out, (tree.capacity, tree.N, tree.N, tree.N), float("-inf"), torch.float32, dev)
    if alpha is not None:
        _check_tensor("alpha", alpha, torch.float32, len(cams) * w * h, dev)
    check(lib().vr_tree_leaf_weights(tree._handle, _cams_array(cams), len(cams), C.byref(options._as_c()), _rect(tile),
                                     out.data_ptr(), alpha.data_ptr() if alpha is not None else None,
                                     counters.data_ptr() if counters is not None else None, _stream_ptr(stream)))
    return out


def leaf_error(tree: N3Tree, cams, options: RenderOptions, err, out=None, counters=None, stream=None, *, tile=None):
    """Per-leaf residual error over the views ``cams`` (vr_tree_leaf_error): a CUDA float32 tensor
    ``[capacity, 2, 2, 2]`` (slot = node * 8 + octant) to which every shaded sample of every pixel has added its
    compositing weight T * (1 - att) times the pixel's ``err``, a contiguous float32 CUDA tensor ``[V, H, W]``
    (tile-sized; e.g. the squared colour error of a render).  ``out`` (same shape or ``capacity * 8`` elements, float32,
    on the tree's device) accumulates over calls; without it a new tensor starts at 0.  ``options`` is one
    RenderOptions (the fields that act in :func:`leaf_weights` act here).  ``counters``: optional int64[5] device
    tensor, accumulated.  Asynchronous on ``stream``; the sums are atomic, so they vary in the last bits from run to
    run.  The tree must be loaded with ``load_cuda(slot_map=True)``."""
    import torch
    dev = _slot_tree(tree, "leaf_error")
    cams, w, h = _march_views(cams, options, tile, "leaf_error")
    out = _accumulator("out", out, (tree.capacity, tree.N, tree.N, tree.N), 0.0, torch.float32, dev)
    _check_tensor("err", err, torch.float32, len(cams) * w * h, dev)
    check(lib().vr_tree_leaf_error(tree._handle, _cams_array(cams), len(cams), C.byref(options._as_c()), _rect(tile),
                                   err.data_ptr(), out.data_ptr(), counters.data_ptr() if counters is not None else None,
                                   _stream_ptr(stream)))
    return out


def leaf_grads(tree: N3Tree, cams, options: RenderOptions, dpix, out=None, float_out=None, stream=None, *, tile=None):
    """Gradient of a loss on the float render of the views ``cams`` w.r.t. every leaf's data row (vr_tree_leaf_grads):
    ``dpix`` is dL/d(r, g, b, alpha) of each pixel, a contiguous float32 CUDA tensor ``[V, H, W, 4]`` (tile-sized), and
    the result a float32 tensor ``[capacity, 2, 2, 2, data_dim]`` laid out like ``data_``.  ``out`` (that shape or as
    many elements, on the tree's device) accumulates over calls; without it a new tensor starts at 0.  ``float_out``:
    optional float32 ``[V, H, W, 4]`` that receives the render the gradient is of (``render_batch``'s ``float_out``,
    bit for bit).  ``options`` is one RenderOptions; ``render_depth`` is refused.  Asynchronous on ``stream``; the sums
    are atomic, so they vary in the last bits from run to run.  The tree must be loaded with
    ``load_cuda(slot_map=True)``."""
    import torch
    dev = _slot_tree(tree, "leaf_grads")
    cams, w, h = _march_views(cams, options, tile, "leaf_grads")
    out = _accumulator("out", out, (tree.capacity, tree.N, tree.N, tree.N, tree.data_dim), 0.0, torch.float32, dev)
    _check_tensor("dpix", dpix, torch.float32, len(cams) * w * h * 4, dev)
    if float_out is not None:
        _check_tensor("float_out", float_out, torch.float32, len(cams) * w * h * 4, dev)
    check(lib().vr_tree_leaf_grads(tree._handle, _cams_array(cams), len(cams), C.byref(options._as_c()), _rect(tile),
                                   dpix.data_ptr(), out.data_ptr(), float_out.data_ptr() if float_out is not None else None,
                                   _stream_ptr(stream)))
    return out


def _slot_tree(tree: N3Tree, what: str):
    """The CUDA device of ``tree``, which must be loaded with the slot map that ``what`` needs."""
    import torch
    if not tree.is_cuda_loaded():
        raise RuntimeError("N3Tree is not loaded on the device")
    if not tree._slot_map:
        raise RuntimeError(f"{what} needs the slot map: load the tree with load_cuda(slot_map=True)")
    return torch.device("cuda", tree._device)


def _march_views(cams, options, tile, what: str):
    """(cams, w, h) of a march-based leaf pass: the cameras as a list (one Camera: one view) and the size of the tile,
    or of the views' frame, that the per-pixel tensors cover."""
    if isinstance(cams, Camera):
        cams = [cams]
    if not isinstance(options, RenderOptions):
        raise TypeError(f"{what} takes one RenderOptions for every view")
    w, h = (int(tile[2]), int(tile[3])) if tile is not None else (cams[0].width, cams[0].height) if cams else (0, 0)
    return cams, w, h


def _check_tensor(name: str, t, dtype, n: int, dev) -> None:
    import torch
    if (not isinstance(t, torch.Tensor) or t.dtype != dtype or t.device != dev or not t.is_contiguous()
            or t.numel() != n):
        raise ValueError(f"{name} must be a contiguous {str(dtype).replace('torch.', '')} tensor of {n} elements "
                         f"on {dev}")


def _accumulator(name: str, t, shape, fill: float, dtype, dev):
    """A pass's accumulating output: ``t`` checked to hold as many ``dtype`` elements as ``shape`` on ``dev``, or
    without it a new tensor of ``shape`` that starts at ``fill``."""
    import torch
    if t is None:
        return torch.full(shape, fill, dtype=dtype, device=dev)
    _check_tensor(name, t, dtype, math.prod(shape), dev)
    return t


def leaf_neighbors(tree: N3Tree, out=None, stream=None):
    """Forward neighbour of every leaf slot along x, y and z (vr_tree_leaf_neighbors): a CUDA int32 tensor
    ``[capacity * 8, 3]`` holding, for a reachable leaf slot at depth d with integer cell i, the slot of the leaf whose
    cell holds the point (i + e_a) 2^-d of the tree's unit cube, or -1 where i_a + 1 = 2^d; internal, free and
    unreachable slots hold -1.  ``out``: that many int32 elements on the tree's device, overwritten.  Asynchronous on
    ``stream`` (the first call for a tree counts its cells and synchronises it).  The tree must be loaded with
    ``load_cuda(slot_map=True)``; a structural change (a new ``load_cuda``) needs a new table."""
    import torch
    dev = _slot_tree(tree, "leaf_neighbors")
    n = tree.capacity * tree.N ** 3
    if out is None:
        out = torch.empty((n, 3), dtype=torch.int32, device=dev)
    else:
        _check_tensor("out", out, torch.int32, n * 3, dev)
    check(lib().vr_tree_leaf_neighbors(tree._handle, out.data_ptr(), _stream_ptr(stream)))
    return out


def leaf_tv(tree: N3Tree, nbr, data, lambda_sigma: float, lambda_color: float, out=None, energy=None, stream=None):
    """Total variation between neighbouring leaves (vr_tree_leaf_tv, DESIGN.md section 20) of the float32 rows ``data``
    (``[capacity, 2, 2, 2, data_dim]`` or as many elements, e.g. the fp32 master of :func:`volrend_b200.finetune`):
    ``E = sum_G lambda_G / N_leaf * sum_leaf sum_{c in G} sqrt(1e-8 + sum_a (v[n_a, c] - v[s, c])^2)`` over sigma and
    the colour columns :func:`leaf_grads` writes, ``nbr`` being :func:`leaf_neighbors` of the tree.  dE/d``data`` is
    added to ``out`` (``leaf_grads``' shape; without it a new tensor starts at 0) and E to ``energy`` (a float64 CUDA
    tensor of one element; without it a new one starts at 0).  Returns ``(out, energy)``.  Weights must be finite and
    >= 0; a weight of 0 skips its group.  Asynchronous on ``stream``; the gradient sums are atomic, so they vary in the
    last bits from run to run."""
    import torch
    dev = _slot_tree(tree, "leaf_tv")
    shape = (tree.capacity, tree.N, tree.N, tree.N, tree.data_dim)
    for name, w in (("lambda_sigma", lambda_sigma), ("lambda_color", lambda_color)):
        if not (float(w) >= 0.0) or float(w) == float("inf"):
            raise ValueError(f"{name} {w} must be finite and >= 0")
    _check_tensor("nbr", nbr, torch.int32, math.prod(shape[:4]) * 3, dev)
    _check_tensor("data", data, torch.float32, math.prod(shape), dev)
    out = _accumulator("out", out, shape, 0.0, torch.float32, dev)
    energy = _accumulator("energy", energy, (1,), 0.0, torch.float64, dev)
    check(lib().vr_tree_leaf_tv(tree._handle, nbr.data_ptr(), data.data_ptr(), float(lambda_sigma),
                                float(lambda_color), out.data_ptr(), energy.data_ptr(), _stream_ptr(stream)))
    return out, energy


def _draw_probe_runs(tree: N3Tree, arr, options, oarr, tile, img, fo, s) -> None:
    """The probe discs of a batch rendered with options per view (``arr`` cameras, ``oarr`` their vr_options): one
    vr_draw_probe per run of consecutive views with the same probe settings."""
    n = len(options)
    w, h = (int(tile[2]), int(tile[3])) if tile is not None else (arr[0].width, arr[0].height) if n else (0, 0)
    key = lambda o: (tuple(float(v) for v in o.probe), int(o.probe_disp_size), tuple(int(v) for v in o.basis_minmax))
    v0 = 0
    while v0 < n:
        v1 = v0 + 1
        if options[v0].enable_probe:
            while v1 < n and options[v1].enable_probe and key(options[v1]) == key(options[v0]):
                v1 += 1
            sub = (_capi.vr_camera * (v1 - v0)).from_buffer(arr, v0 * C.sizeof(_capi.vr_camera))
            _draw_probe(tree, sub, v1 - v0, options[v0], oarr[v0], tile,
                        img + 4 * w * h * v0 if img is not None else None,
                        fo + 16 * w * h * v0 if fo is not None else None, s)
        v0 = v1


def render_frames_host(tree: N3Tree, cams, options: RenderOptions, host_images) -> None:
    """main_headless.cpp:208-223 with ``-o``: every frame lands in host memory
    (``host_images``: uint8 CPU tensor / ndarray [V,H,W,4], ideally pinned)."""
    arr = _cams_array(cams)
    o = options._as_c()
    ptr = host_images.data_ptr() if hasattr(host_images, "data_ptr") else host_images.ctypes.data
    check(lib().vr_render_frames_host(tree._handle, arr, len(cams), C.byref(o), ptr))


def write_png_file(filename: str, rgba8, width: int | None = None, height: int | None = None) -> bool:
    """``internal::write_png_file`` (src/imwrite.cpp:14-79) without libpng; ``rgba8``: uint8 [H,W,4]
    host array / CPU tensor."""
    arr = rgba8.numpy() if hasattr(rgba8, "numpy") else np.asarray(rgba8)
    arr = np.ascontiguousarray(arr, np.uint8)
    h, w = (arr.shape[0], arr.shape[1]) if height is None else (height, width)
    return lib().vr_write_png(filename.encode(), arr.ctypes.data, int(w), int(h)) == 0


def render_frames_png(tree: N3Tree, cams, options, paths, n_threads: int = 8) -> None:
    """main_headless.cpp:208-223 with ``-o``: render every pose and write one PNG per pose.  ``options``: one
    RenderOptions, or a sequence of ``len(cams)`` of them (view i rendered with options[i], as render_batch)."""
    arr = _cams_array(cams)
    cp = (C.c_char_p * len(paths))(*[p.encode() for p in paths])
    if _per_view(cams, options):
        check(lib().vr_render_frames_png_opts(tree._handle, arr, len(cams), _options_array(options), cp, int(n_threads)))
        return
    o = options._as_c()
    check(lib().vr_render_frames_png(tree._handle, arr, len(cams), C.byref(o), cp, int(n_threads)))


# ---------------------------------------------------------------------------- VolumeRenderer
VR_MESH_MAX_VERTS = 2 ** 31 - 1    # vr_mesh_desc.n_verts is int32


def _probe_cube():
    """The probe marker of cuda_renderer.cpp:25-38: an unlit black cube whose +-z faces are blue, +-y faces green
    and +-x faces red, at scale 0.05 and hidden."""
    from .mesh import VERT_SZ, Mesh
    m = Mesh.Cube((0.0, 0.0, 0.0))
    v = m.vert.reshape(36, VERT_SZ)
    for i in range(3):
        v[12 * i:12 * (i + 1), 3 + 2 - i] = 1.0
    m.name = "_probe_cube"
    m.visible = False
    m.scale = 0.05
    m.unlit = True
    return m


class VolumeRenderer:
    """GL-free ``VolumeRenderer`` (renderer.hpp:11-42).  ``meshes`` is a list of :class:`volrend_b200.Mesh`;
    visible ones are rasterized by CUDA and the volume is composited over them.  ``options.enable_probe`` draws the
    probe cube at ``options.probe`` after them, and ``options.show_grid`` the octree cut at
    ``options.grid_max_depth`` (:meth:`N3Tree.gen_wireframe`) after that, as the reference does."""

    def __init__(self):
        self.camera = Camera()
        self.options = RenderOptions()
        self.meshes = []            # volrend_b200.mesh.Mesh, drawn in order by render()
        self._tree = None
        self._image = None
        self._depth = None
        self._wire = None           # grid mesh (cuda_renderer.cpp wire_) and the depth it was made for
        self._wire_depth = None     # (last_wire_depth_)
        self._probe = _probe_cube()  # (probe_)
        self.resize(self.camera.width, self.camera.height)

    def get_backend(self) -> str:
        return "CUDA"

    def set(self, tree: N3Tree) -> None:
        self._tree = tree           # cuda_renderer.cpp:171-180
        self.options.basis_minmax = [0, max(tree.data_format.basis_dim - 1, 0)]
        self._probe.scale = float(np.float32(0.02) / np.float32(tree.scale[0]))
        self._wire = self._wire_depth = None

    def clear(self) -> None:
        self._tree = None
        self._wire = self._wire_depth = None

    def _grid_mesh(self, options=None):
        """The grid mesh to draw with ``options`` (default ``self.options``), or None (cuda_renderer.cpp
        maybe_gen_wire): regenerated on the device when ``grid_max_depth`` changed since the last one.  Without a
        loaded tree there is no grid."""
        options = self.options if options is None else options
        if not options.show_grid or self._tree is None or not self._tree.is_cuda_loaded():
            return None
        depth = int(options.grid_max_depth)
        if self._wire is None or self._wire_depth != depth:
            from .mesh import Mesh
            n = self._tree.wireframe_vertex_count(depth)
            if n > VR_MESH_MAX_VERTS:
                raise ValueError(f"grid at depth {depth} has {n} vertices; a mesh holds at most {VR_MESH_MAX_VERTS}")
            self._wire = Mesh._on_device(self._tree.wireframe_device(depth), face_size=2, unlit=True)
            self._wire.name = "Grid"
            self._wire_depth = depth
        return self._wire

    def resize(self, width: int, height: int) -> None:
        import torch
        self.camera.width, self.camera.height = int(width), int(height)
        if torch.cuda.is_available():
            self._image = torch.zeros((height, width, 4), dtype=torch.uint8, device="cuda")
        else:
            self._image = None
        self._depth = None          # ray-distance buffer of the mesh pass, allocated on first use

    def render(self):
        """cuda_renderer.cpp:83-126 into the renderer-owned RGBA8 buffer, which is returned.

        With at least one visible mesh, the probe cube (``enable_probe``) or the grid (``show_grid`` with a loaded
        tree), this follows the reference's three steps: clear colour to the background as GL does
        (round(bg * 255), alpha 255) and the ray-distance buffer to 1e9, draw the meshes, the probe cube and then
        the grid in one call (:func:`volrend_b200.mesh.draw_meshes`; an earlier one wins exact depth ties), then
        composite the volume over them (``launch_renderer(..., offscreen=False)``, which also draws the probe
        disc).  Without any of them it keeps the offscreen march, whose background is ``background_brightness`` in
        float rather than the 8-bit cleared colour, so a renderer without meshes renders exactly as it always
        has."""
        if self._image is None:
            raise RuntimeError("VolumeRenderer needs a CUDA device (no CPU fallback)")
        self.camera._update()
        visible = [m for m in self.meshes if m.visible]
        self._probe.visible = bool(self.options.enable_probe)      # cuda_renderer.cpp:94-95
        self._probe.translation = np.asarray(self.options.probe, np.float32).reshape(3).copy()
        if self._probe.visible:
            visible.append(self._probe)
        wire = self._grid_mesh()
        if wire is not None:
            visible.append(wire)
        if visible:
            import torch
            from .mesh import draw_meshes
            h, w = self._image.shape[:2]
            if self._depth is None or tuple(self._depth.shape) != (h, w):
                self._depth = torch.empty((h, w), dtype=torch.float32, device=self._image.device)
            bg = round(min(max(float(self.options.background_brightness), 0.0), 1.0) * 255)
            self._image[..., :3] = bg
            self._image[..., 3] = 255
            self._depth.fill_(1e9)
            draw_meshes(self.camera, visible, self._image, self._depth)
            if self._tree is not None and self._tree.is_cuda_loaded():
                launch_renderer(self._tree, self.camera, self.options, self._image, self._depth, None, False)
            return self._image
        if self._tree is None or not self._tree.is_cuda_loaded():
            bg = int(self.options.background_brightness * 255)
            self._image[..., :3] = bg
            self._image[..., 3] = 255
            return self._image
        launch_renderer(self._tree, self.camera, self.options, self._image, None, None, True)
        return self._image

    def render_batch(self, cams, options=None, meshes=None, out=None):
        """Renders ``len(cams)`` views and returns them as a CUDA uint8 tensor [V,H,W,4] (``out`` if given).  View i
        is byte for byte what :meth:`render` returns after ``camera = cams[i]``, ``options = options[i]`` and
        ``meshes = meshes[i]``: the cleared background, the meshes, probe cube and grid, the composited volume and the
        probe disc, or the offscreen march for views with none of these.  ``options``: None (``self.options``), one
        :class:`RenderOptions` or one per view; ``meshes``: None (``self.meshes`` for every view) or one list of
        :class:`~volrend_b200.Mesh` per view, which may hold shallow copies (``copy.copy(mesh)``) of one uploaded mesh
        with their own transform, ``visible`` and ``unlit``.  Every camera has the same size; the cameras are not
        modified.  Views are rendered in runs of consecutive views of one kind, a mesh run in one batched draw and
        one batched composite march per chunk of at most ``RENDER_BATCH_CHUNK`` views."""
        import torch
        from .mesh import draw_meshes_batch
        if self._image is None:
            raise RuntimeError("VolumeRenderer needs a CUDA device (no CPU fallback)")
        n = len(cams)
        if options is None:
            options = self.options
        opts = [options] * n if isinstance(options, RenderOptions) else list(options)
        _per_view(cams, opts)
        mlists = [self.meshes] * n if meshes is None else list(meshes)
        if len(mlists) != n:
            raise ValueError(f"meshes: None or a sequence of {n} mesh lists (one per camera)")
        cams = [copy.deepcopy(c) for c in cams]
        for c in cams:
            c._update()
        if n and any((c.width, c.height) != (cams[0].width, cams[0].height) for c in cams):
            raise ValueError("render_batch: every camera must have the same size")
        h, w = (cams[0].height, cams[0].width) if n else (0, 0)
        if out is None:
            out = torch.empty((n, h, w, 4), dtype=torch.uint8, device=self._image.device)
        elif tuple(out.shape) != (n, h, w, 4) or out.dtype != torch.uint8 or not out.is_cuda or not out.is_contiguous():
            raise ValueError(f"out: expected a contiguous CUDA uint8 tensor of shape {(n, h, w, 4)}")
        tree = self._tree if self._tree is not None and self._tree.is_cuda_loaded() else None
        draws, wires = [], {}
        for o, ms in zip(opts, mlists):
            vis = [m for m in ms if m.visible]
            if o.enable_probe:                       # render(): the probe cube at options.probe
                p = copy.copy(self._probe)
                p.visible = True
                p.translation = np.asarray(o.probe, np.float32).reshape(3).copy()
                vis.append(p)
            if o.show_grid and tree is not None:     # one grid per distinct depth in the call
                d = int(o.grid_max_depth)
                if d not in wires:
                    wires[d] = self._grid_mesh(o)
                vis.append(wires[d])
            draws.append(vis)
        s = _stream_ptr(None)
        for mesh_run, v0, v1 in _view_runs([bool(d) for d in draws], RENDER_BATCH_CHUNK):
            img, run_cams, run_opts = out[v0:v1], cams[v0:v1], opts[v0:v1]
            bg = [float(o.background_brightness) for o in run_opts]
            if mesh_run:
                dep = torch.full((v1 - v0, h, w), 1e9, dtype=torch.float32, device=out.device)
                bgv = torch.tensor([round(min(max(b, 0.0), 1.0) * 255) for b in bg], dtype=torch.uint8)
                img[..., :3] = bgv.to(out.device, non_blocking=True).view(-1, 1, 1, 1)
                img[..., 3] = 255
                draw_meshes_batch(run_cams, draws[v0:v1], img, dep)
                if tree is not None:
                    arr, oarr = _cams_array(run_cams), _options_array(run_opts)
                    check(lib().vr_render_composite_batch_opts(tree._handle, arr, v1 - v0, oarr, None, img.data_ptr(),
                                                               dep.data_ptr(), None, s))
                    _draw_probe_runs(tree, arr, run_opts, oarr, None, img.data_ptr(), None, s)
            elif tree is not None:
                render_batch(tree, run_cams, run_opts, img)
            else:                                    # render() without a tree: int(bg * 255), no clamp
                bgv = torch.tensor([int(b * 255) & 0xFF for b in bg], dtype=torch.uint8)
                img[..., :3] = bgv.to(out.device, non_blocking=True).view(-1, 1, 1, 1)
                img[..., 3] = 255
        return out


# Views per batched draw and composite march in VolumeRenderer.render_batch: bounds the ray-distance buffer it
# allocates (4 B per pixel per view, 82 MB at 800x800).
RENDER_BATCH_CHUNK = 32


def _view_runs(has_draw, chunk: int):
    """Splits views into runs of consecutive views of one kind (True: something to draw before the march), each at
    most ``chunk`` long: a list of (kind, v0, v1) in view order."""
    runs, v0 = [], 0
    while v0 < len(has_draw):
        v1 = v0 + 1
        while v1 < len(has_draw) and v1 - v0 < chunk and has_draw[v1] == has_draw[v0]:
            v1 += 1
        runs.append((bool(has_draw[v0]), v0, v1))
        v0 = v1
    return runs
