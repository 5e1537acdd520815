"""Mesh file formats: drawlist ``.npz`` files and basic OBJ files (reference ``src/mesh.cpp:680-951``).

Both loaders return ordinary :class:`~volrend_b200.mesh.Mesh` objects for ``VolumeRenderer.meshes``.  They parse on
the host; the one compute-heavy step, per-vertex normals, runs on the GPU (:func:`~volrend_b200.mesh.estimate_normals`),
so a load that needs normals raises :class:`~volrend_b200.VolrendError` without a device and every other load runs
without one.

The drawlist loader keeps the reference's observable behaviour, which users' files depend on:

* meshes come out sorted by name (bytes), not in file order; draw order decides exact depth ties;
* a key ``<name>__<field>`` is a field, a key without ``__`` is a type entry (so ``cameras_image_width`` is a mesh
  of unsupported type, reported and skipped);
* a type string keeps its first character and lowercases the rest (``"cube"`` works, ``"Cube"`` does not);
* fields are read by element size, not by dtype: a float32 ``rings`` is read as its int32 bits and a float16
  ``color`` as half;
* a ``vert_color`` of the wrong size drops the mesh; other errors are collected and printed after parsing;
* ``mesh`` entries with ``face_size`` 3 get estimated normals before ``vert_color`` is applied.

Where the reference reads past an array (a ``vec3`` field with fewer than 3 values, an empty scalar field, a
camera ``r`` shorter than ``t``) or leaves a value uninitialised (a ``vec3`` of 1-byte elements), this loader prints
the error and uses the default (0 for the missing ``r`` values) instead.
"""
from __future__ import annotations

import io
import math
import re

import numpy as np

from .mesh import DEFAULT_COLOR, VERT_SZ, Mesh, estimate_normals

_F = np.float32
_FLOAT_BY_SIZE = {2: np.float16, 4: np.float32, 8: np.float64}
_INT_BY_SIZE = {1: np.int8, 2: np.int16, 4: np.int32, 8: np.int64}


# ------------------------------------------------------------------------------------------------ drawlist .npz
class _Field:
    """One npz member as the reference sees it: raw little-endian bytes in storage order, element size, shape."""

    def __init__(self, arr: np.ndarray):
        arr = np.asarray(arr)
        self.shape = tuple(arr.shape)
        self.ws = int(arr.dtype.itemsize)
        self.raw = np.ascontiguousarray(arr.ravel(order="K")).view(np.uint8)

    def as_(self, table) -> np.ndarray:
        return self.raw.view(table[self.ws])


def _split_by_2underscore(s: str) -> list:
    """mesh.cpp:166-182: split on '__', dropping empty pieces before each separator.  In a run of three or more
    underscores the reference's unsigned piece length wraps, and the piece becomes the rest of the string."""
    r, j = [], 0
    for i in range(1, len(s)):
        if s[i] == "_" and s[i - 1] == "_":
            if i - 1 != j:
                r.append(s[j:i - 1] if i - 1 > j else s[j:])
            j = i + 1
    if j < len(s):
        r.append(s[j:])
    return r


def _type_string(f: _Field) -> bytes:
    """mesh.cpp:782-786: every 4th byte of the data (the low byte of each UTF-32 unit), all but the first lowercased."""
    b = bytearray(f.raw.tobytes())
    for i in range(4, len(b), 4):
        b[i // 4] = ord(bytes([b[i]]).lower())
    return bytes(b[:len(b) // 4])


def _get_int(fields, key, defval, errs) -> int:
    f = fields.get(key)
    if f is None:
        return int(defval)
    if f.ws not in _INT_BY_SIZE:
        errs.append(f"Invalid word size for int {f.ws}\n")
        return 0
    v = f.as_(_INT_BY_SIZE)
    if v.size < 1:
        errs.append(f"Field '{key}' is empty\n")
        return int(defval)
    return int(v[:1].astype(np.int32)[0])


def _get_float(fields, key, defval, errs) -> np.float32:
    f = fields.get(key)
    if f is None:
        return _F(defval)
    if f.ws not in _FLOAT_BY_SIZE:
        errs.append(f"Invalid word size for float {f.ws}\n")
        return _F(0)
    v = f.as_(_FLOAT_BY_SIZE)
    if v.size < 1:
        errs.append(f"Field '{key}' is empty\n")
        return _F(defval)
    return _F(v[0])


def _get_vec3(fields, key, defval, errs) -> np.ndarray:
    f = fields.get(key)
    if f is None:
        return np.asarray(defval, _F)
    if f.shape != (3,):
        errs.append("Invalid shape for float3, must be (3,)")
    if f.ws not in _FLOAT_BY_SIZE:
        errs.append(f"Invalid word size for float {f.ws}\n")
        return np.asarray(defval, _F)
    v = f.as_(_FLOAT_BY_SIZE)
    if v.size < 3:
        return np.asarray(defval, _F)
    return v[:3].astype(_F)


def _get_floatarr(fields, key, errs) -> np.ndarray:
    f = fields.get(key)
    if f is None:
        return np.zeros(0, _F)
    if f.ws not in _FLOAT_BY_SIZE:
        errs.append(f"Invalid word size for float {f.ws}\n")
        return np.zeros(f.raw.size // f.ws, _F)
    return f.as_(_FLOAT_BY_SIZE).astype(_F)


def _get_intarr(fields, key, errs) -> np.ndarray:
    """As uint32 (the int values the reference copies into its unsigned index vector)."""
    f = fields.get(key)
    if f is None:
        return np.zeros(0, np.uint32)
    if f.ws not in _INT_BY_SIZE:
        errs.append(f"Invalid word size for int {f.ws}\n")
        return np.zeros(f.raw.size // f.ws, np.uint32)
    return f.as_(_INT_BY_SIZE).astype(np.int32).view(np.uint32)


def _camera_frustums(me: Mesh, fields, errs) -> None:
    """mesh.cpp:830-857: one frustum per (r, t) triple, optionally connected centre to centre."""
    t = _get_floatarr(fields, "t", errs)
    r = _get_floatarr(fields, "r", errs)
    if r.size != t.size or r.size % 3:
        errs.append("camerafrustums r, t have different sizes or not multiple of 3\n")
    nv = me.n_verts
    n_reps = t.size // 3
    if r.size < 3 * n_reps:
        r = np.concatenate([r, np.zeros(3 * n_reps - r.size, _F)])
    me.repeat(n_reps)
    for i in range(n_reps):
        me.apply_transform(r[3 * i:3 * i + 3], t[3 * i:3 * i + 3], nv * i, nv * (i + 1))
    if _get_int(fields, "connect", 0, errs) != 0:
        if n_reps == 0:
            raise ValueError("camerafrustum: 'connect' needs at least one camera in 't'")
        links = np.stack([np.arange(n_reps - 1) * nv, np.arange(1, n_reps) * nv], 1).astype(np.uint32)
        me.faces = np.concatenate([np.asarray(me.faces, np.uint32), links.reshape(-1)])


def _build(mesh_type: bytes, fields, errs):
    """The preset or generic mesh of one drawlist entry (mesh.cpp:809-896), or None for an unsupported type."""
    color = _get_vec3(fields, "color", DEFAULT_COLOR, errs)
    if mesh_type == b"cube":
        return Mesh.Cube(color)
    if mesh_type == b"sphere":
        return Mesh.Sphere(_get_int(fields, "rings", 15, errs), _get_int(fields, "sectors", 30, errs), color)
    if mesh_type == b"line":
        return Mesh.Line(_get_vec3(fields, "a", (0, 0, 0), errs), _get_vec3(fields, "b", (0, 0, 1), errs), color)
    if mesh_type == b"camerafrustum":
        me = Mesh.CameraFrustum(_get_float(fields, "focal_length", 1111.0, errs),
                                _get_float(fields, "image_width", 800.0, errs),
                                _get_float(fields, "image_height", 800.0, errs),
                                _get_float(fields, "z", -0.3, errs), color)
        if "t" in fields:
            _camera_frustums(me, fields, errs)
        return me
    if mesh_type == b"lines":
        me = Mesh.Lines(_get_floatarr(fields, "points", errs), color)
        if "segs" in fields:
            me.faces = _get_intarr(fields, "segs", errs)
        return me
    if mesh_type == b"points":
        return Mesh.Points(_get_floatarr(fields, "points", errs), color)
    if mesh_type == b"mesh":
        me = Mesh.Points(_get_floatarr(fields, "points", errs), color)
        me.face_size = _get_int(fields, "face_size", 3, errs)
        if me.face_size <= 0 or me.face_size > 3:
            me.face_size = 3
            errs.append("Mesh face size must be one of 1,2,3\n")
        if "faces" in fields:
            faces = _get_intarr(fields, "faces", errs)
            if faces.size % me.face_size:
                errs.append(f"Faces must have face_size={me.face_size} elements\n")
            me.faces = faces
        if me.face_size == 3:
            estimate_normals(me)
        return me
    return None


def open_drawlist_mem(data, default_visible: bool = True) -> list:
    """The meshes of a drawlist ``.npz`` held in memory (``Mesh::open_drawlist_mem``), sorted by name.

    Each key is ``<name>=<type>`` (a string) or ``<name>__<field>=<value>``.  Types: ``cube``, ``sphere``
    (``rings``, ``sectors``), ``line`` (``a``, ``b``), ``camerafrustum`` (``focal_length``, ``image_width``,
    ``image_height``, ``z``; ``t``/``r`` for one frustum per translation/axis-angle triple, ``connect``),
    ``lines`` (``points``, ``segs``), ``points`` (``points``) and ``mesh`` (``points``, ``face_size``, ``faces``;
    triangles get estimated normals).  Every mesh takes ``color``, ``vert_color``, ``scale``, ``translation``,
    ``rotation``, ``visible`` (default ``default_visible``) and ``unlit`` (default 0)."""
    print("INFO: Loading drawlist npz")
    with np.load(io.BytesIO(bytes(data)), allow_pickle=False) as npz:
        entries = {k: _Field(npz[k]) for k in npz.files}
    parse = {}
    for fullname in sorted(entries, key=lambda k: k.encode("utf-8")):
        spl = _split_by_2underscore(fullname)
        if len(spl) == 1:
            parse.setdefault(spl[0], [b"", {}])[0] = _type_string(entries[fullname])
        elif len(spl) == 2:
            parse.setdefault(spl[0], [b"", {}])[1][spl[1]] = entries[fullname]
        else:
            print(f"Mesh load_npz warning: invalid field '{fullname}', must be of the form <name>=mesh_type or "
                  "<name>__<field>=val")
    meshes, errs = [], []
    for name in sorted(parse, key=lambda k: k.encode("utf-8")):
        mesh_type, fields = parse[name]
        me = _build(mesh_type, fields, errs)
        if me is None:
            errs.append(f"Mesh '{name}' has unsupported type '{mesh_type.decode('latin-1')}'\n")
            continue
        if "vert_color" in fields:
            vc = _get_floatarr(fields, "vert_color", errs)
            if vc.size * VERT_SZ != np.asarray(me.vert).size * 3:
                errs.append(f"Mesh {name} vert_color has invalid size\n")
                continue
            me.vert.reshape(-1, VERT_SZ)[:, 3:6] = vc.reshape(-1, 3)
            if me._vert_dev is not None:
                me.update()
        me.name = name
        me.scale = float(_get_float(fields, "scale", 1.0, errs))
        me.translation = _get_vec3(fields, "translation", (0, 0, 0), errs)
        me.rotation = _get_vec3(fields, "rotation", (0, 0, 0), errs)
        me.visible = _get_int(fields, "visible", int(bool(default_visible)), errs) != 0
        me.unlit = _get_int(fields, "unlit", 0, errs) != 0
        meshes.append(me)
    if errs:
        print("Mesh load_npz encountered errors while parsing:\n" + "".join(errs), end="")
    return meshes


def open_drawlist(path, default_visible: bool = True) -> list:
    """The meshes of a drawlist ``.npz`` file (``Mesh::open_drawlist``); see :func:`open_drawlist_mem`."""
    with open(path, "rb") as f:
        return open_drawlist_mem(f.read(), default_visible)


# ------------------------------------------------------------------------------------------------ OBJ
_POW_LUT = (1.0, 0.1, 0.01, 0.001, 0.0001, 0.00001, 0.000001, 0.0000001)
_ATOI = re.compile(r"[ \t\n\v\f\r]*([+-]?[0-9]*)")


def _is_digit(c: str) -> bool:
    return "0" <= c <= "9"


def _parse_double(s: str):
    """A number at the start of ``s`` as tinyobj reads it (a double built digit by digit: mantissa * 10 + d for the
    integer part, + d * 10^-k for the fraction, then ldexp(m * 5^e, e)); None where tinyobj fails."""
    n = len(s)
    if n == 0:
        return None
    mant, exp, sign, exp_sign, i, lead_dot = 0.0, 0, "+", "+", 0, False
    if s[0] in "+-":
        sign, i = s[0], 1
        lead_dot = i < n and s[i] == "."
    elif s[0] == ".":
        lead_dot = True
    elif not _is_digit(s[0]):
        return None
    if not lead_dot:
        read = 0
        while i < n and _is_digit(s[i]):
            mant = mant * 10
            mant = mant + int(s[i])
            i += 1
            read += 1
        if read == 0:
            return None
    if i < n and s[i] not in ".eE":
        i = n                      # anything else ends the number
    if i < n and s[i] == ".":
        i += 1
        read = 1
        while i < n and _is_digit(s[i]):
            mant = mant + int(s[i]) * (_POW_LUT[read] if read < len(_POW_LUT) else math.pow(10.0, -read))
            read += 1
            i += 1
    if i < n and s[i] in "eE":
        i += 1
        if i < n and s[i] in "+-":
            exp_sign = s[i]
            i += 1
        elif not (i < n and _is_digit(s[i])):
            return None
        read = 0
        while i < n and _is_digit(s[i]):
            if exp > 2147483647 // 10:
                return None
            exp = exp * 10 + int(s[i])
            i += 1
            read += 1
        exp = exp if exp_sign == "+" else -exp
        if read == 0:
            return None
    with np.errstate(all="ignore"):
        v = float(np.ldexp(mant * np.power(5.0, exp), exp)) if exp else mant
    return (1 if sign == "+" else -1) * v


class _Cursor:
    """tinyobj's token pointer over one line."""

    def __init__(self, s: str, i: int = 0):
        self.s, self.i = s, i

    def peek(self) -> str:
        return self.s[self.i] if self.i < len(self.s) else "\0"

    def skip(self, chars: str) -> None:
        while self.i < len(self.s) and self.s[self.i] in chars:
            self.i += 1

    def until(self, chars: str) -> str:
        j = self.i
        while j < len(self.s) and self.s[j] not in chars:
            j += 1
        tok, self.i = self.s[self.i:j], j
        return tok

    def real(self):
        self.skip(" \t")
        return _parse_double(self.until(" \t\r"))

    def atoi(self) -> int:
        m = _ATOI.match(self.s, self.i)
        d = m.group(1)
        return int(d) if d not in ("", "+", "-") else 0


def _fix_index(idx: int, n: int):
    if idx > 0:
        return idx - 1
    if idx == 0:
        return None                # zero is not an OBJ index
    return n + idx


def _parse_triple(c: _Cursor, nv: int, nvn: int, nvt: int):
    """``v``, ``v/vt``, ``v//vn`` or ``v/vt/vn``: the vertex index, or None on a zero index."""
    vi = _fix_index(c.atoi(), nv)
    if vi is None:
        return None
    c.until("/ \t\r")
    if c.peek() != "/":
        return vi
    c.i += 1
    if c.peek() == "/":
        c.i += 1
        if _fix_index(c.atoi(), nvn) is None:
            return None
        c.until("/ \t\r")
        return vi
    if _fix_index(c.atoi(), nvt) is None:
        return None
    c.until("/ \t\r")
    if c.peek() != "/":
        return vi
    c.i += 1
    if _fix_index(c.atoi(), nvn) is None:
        return None
    c.until("/ \t\r")
    return vi


def _triangulate(poly: list, pos: np.ndarray, out: list) -> None:
    """tinyobj's triangulation of one polygon's vertex indices: triangles as they are, quads split along the
    shorter diagonal (fp32 squared lengths), larger polygons fanned from their first vertex, which is what
    tinyobj's ear clipping gives for a convex polygon.  Polygons of fewer than 3 vertices are dropped, and so are
    quads and larger polygons with an index out of range."""
    n, nv = len(poly), pos.shape[0]
    if n < 3:
        return
    if n == 3:
        out.extend(poly)
        return
    if any(i < 0 or i >= nv for i in poly):
        return
    if n == 4:
        p = pos[poly]
        e02, e13 = p[2] - p[0], p[3] - p[1]
        sq02 = (e02[0] * e02[0] + e02[1] * e02[1]) + e02[2] * e02[2]
        sq13 = (e13[0] * e13[0] + e13[1] * e13[1]) + e13[2] * e13[2]
        i0, i1, i2, i3 = poly
        out.extend([i0, i1, i2, i0, i2, i3] if sq02 < sq13 else [i0, i1, i3, i1, i2, i3])
        return
    for k in range(1, n - 1):
        out.extend([poly[0], poly[k], poly[k + 1]])


def _load_obj(text: str, name: str) -> Mesh:
    """mesh.cpp:680-759 over tinyobj configured with triangulation and vertex colours (white where absent)."""
    v, vc, vn, polys = [], [], [], []
    n_vt = 0
    for line_num, line in enumerate(re.split(r"\r\n|\r|\n", text), 1):
        c = _Cursor(line)
        c.skip(" \t")
        t0, t1, t2 = c.peek(), _Cursor(line, c.i + 1).peek(), _Cursor(line, c.i + 2).peek()
        if t0 in "\0#":
            continue
        if t0 == "v" and t1 in " \t":
            c.i += 2
            xyz = [c.real() for _ in range(3)]
            rgb = []
            for _ in range(3):
                x = c.real()
                if x is None:
                    break
                rgb.append(x)
            v.append([0.0 if x is None else x for x in xyz])
            vc.append(rgb if len(rgb) == 3 else [1.0, 1.0, 1.0])
        elif t0 == "v" and t1 == "n" and t2 in " \t":
            c.i += 3
            vn.append([0.0 if x is None else x for x in (c.real(), c.real(), c.real())])
        elif t0 == "v" and t1 == "t" and t2 in " \t":
            n_vt += 1
        elif t0 in "lf" and t1 in " \t":
            c.i += 2
            if t0 == "f":
                c.skip(" \t")
            poly = []
            while c.peek() not in "\r\n\0":
                vi = _parse_triple(c, len(v), len(vn), n_vt)
                if vi is None:
                    print(f"ERROR Failed to load OBJ: Failed parse `{t0}' line(e.g. zero value for "
                          f"{'face' if t0 == 'f' else 'vertex'} index. line {line_num}.)", end="\n")
                    return Mesh()
                poly.append(vi)
                c.skip(" \t\r")
            if t0 == "f":
                polys.append(poly)
    with np.errstate(all="ignore"):
        pos = np.asarray(v, np.float64).reshape(-1, 3).astype(_F)
        col = np.asarray(vc, np.float64).reshape(-1, 3).astype(_F)
        nrm = np.asarray(vn, np.float64).reshape(-1, 3).astype(_F)
    tris = []
    for poly in polys:
        _triangulate(poly, pos, tris)
    nv = pos.shape[0]
    mesh = Mesh(nv, 0, 3)
    vert = mesh.vert.reshape(nv, VERT_SZ)
    vert[:, 0:3] = pos
    vert[:, 3:6] = col
    mesh.faces = np.asarray(tris, np.int64).astype(np.uint32)
    if nrm.shape[0] >= nv:
        vert[:, 6:9] = nrm[:nv]       # by vertex index, as the reference takes them
    else:
        estimate_normals(mesh)
    mesh.face_size = 3
    mesh.name = name
    return mesh


def load_mem_basic_obj(text) -> Mesh:
    """A triangle mesh from OBJ text (``Mesh::load_mem_basic_obj``), named "OBJ"; see :func:`load_basic_obj`."""
    if isinstance(text, (bytes, bytearray)):
        text = bytes(text).decode("latin-1")
    return _load_obj(text, "OBJ")


def load_basic_obj(path) -> Mesh:
    """A triangle mesh from an OBJ file (``Mesh::load_basic_obj``), named by its path.

    Reads ``v x y z [r g b]`` (white without a colour), ``vn``, and ``f`` in the ``v``, ``v/vt``, ``v//vn`` and
    ``v/vt/vn`` forms with negative (relative) indices; ``vt``, ``l``, ``o``, ``g``, ``s``, ``usemtl`` and
    ``mtllib`` are ignored.  Quads are split along the shorter diagonal and larger (convex) polygons fanned.
    Positions stay in vertex order and only the triangles become faces.  Normals are taken by vertex index from the
    ``vn`` list when it has at least as many entries as there are vertices, and estimated on the GPU otherwise.  An
    input that fails to parse (a zero index) gives an empty mesh, after printing the error."""
    try:
        with open(path, "rb") as f:
            text = f.read().decode("latin-1")
    except OSError:
        print(f"ERROR Failed to load OBJ: Cannot open file [{path}]")
        return Mesh()
    return _load_obj(text, str(path))
