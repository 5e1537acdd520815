"""Isosurface extraction without a GPU (DESIGN.md section 23): the generated triangle table, the numpy oracle's topology
and geometry on random and analytic lattices, the OBJ writer's round trip, the command line's argument errors and the
entry point's device check."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import iso_oracle as io
from tools import gen_iso_table as gen

FACES = [(d, s) for d in range(3) for s in range(2)]


# ----------------------------------------------------------------------------------------------------------- table
def _boundary(tris):
    """Directed edges of a triangle list that are not cancelled by their reverse: the loops' segments."""
    directed = [(t[k], t[(k + 1) % 3]) for t in tris for k in range(3)]
    s = set(directed)
    assert len(s) == len(directed), "a directed edge appears twice in one cube"
    return {e for e in s if (e[1], e[0]) not in s}


def _edge_faces(e):
    """The two cube faces (d, s) that contain edge e."""
    d, c = gen.edge_axis(e), gen.corner_xyz(gen.edge_corner(e))
    return {(a, c[a]) for a in range(3) if a != d}


def _segments_on(seg, face):
    return {(a, b) for a, b in seg if face in _edge_faces(a) and face in _edge_faces(b)}


def test_header_is_the_generators_output():
    with open(gen.HEADER) as f:
        assert f.read() == gen.render_header(gen.build_table())


def test_every_entry_is_closed_loops_of_the_face_rule():
    table = gen.build_table()
    for case in range(256):
        ins = lambda c: (case >> c) & 1
        crossing = {e for e in range(12)
                    if ins(gen.edge_corner(e)) != ins(gen.edge_corner(e) + (1 << gen.edge_axis(e)))}
        seg = _boundary(table[case])
        # closed loops through every crossing edge: in- and out-degree 1
        assert sorted(a for a, _ in seg) == sorted(crossing), case
        assert sorted(b for _, b in seg) == sorted(crossing), case
        # no triangle edge other than a segment joins two edges of one face (no cracks, no shared diagonals)
        und = {frozenset((t[k], t[(k + 1) % 3])) for t in table[case] for k in range(3)}
        for pair in und - {frozenset(e) for e in seg}:
            a, b = tuple(pair)
            assert not (_edge_faces(a) & _edge_faces(b)), (case, a, b)
        for face in FACES:
            on = _segments_on(seg, face)
            d, s = face
            corners = [c for c in range(8) if gen.corner_xyz(c)[d] == s]
            inside = [c for c in corners if ins(c)]
            fe = [e for e in crossing if face in _edge_faces(e)]
            assert len(on) == len(fe) // 2, (case, face)
            for a, b in on:
                # a segment cuts off the inside corners on one side: with 2 inside corners on a diagonal, each
                # segment's two edges share their inside corner
                ends = lambda e: {gen.edge_corner(e), gen.edge_corner(e) + (1 << gen.edge_axis(e))}
                if len(inside) == 2 and len(fe) == 4:
                    common = ends(a) & ends(b)
                    assert len(common) == 1 and ins(next(iter(common))), (case, face, a, b)
                else:
                    assert len(fe) == 2


def _face_map(d, s):
    """Edges of face (d, s) keyed by their position on the face (the two in-face corner coordinates of each end)."""
    out = {}
    for e in range(12):
        if (d, s) in _edge_faces(e):
            c0 = gen.corner_xyz(gen.edge_corner(e))
            c1 = gen.corner_xyz(gen.edge_corner(e) + (1 << gen.edge_axis(e)))
            key = frozenset((tuple(v for a, v in enumerate(c0) if a != d), tuple(v for a, v in enumerate(c1) if a != d)))
            out[e] = key
    return out


def test_face_sharing_cubes_agree():
    """All 3 x 256 x 256 pairs of cubes that share a face: where the shared corners agree, the lower cube's directed
    segments on its upper face are the upper cube's on its lower face, reversed (no cracks, one orientation)."""
    table = gen.build_table()
    seg = [_boundary(t) for t in table]
    checked = 0
    for d in range(3):
        hi, lo = _face_map(d, 1), _face_map(d, 0)
        on_hi = [{(hi[a], hi[b]) for a, b in _segments_on(seg[c], (d, 1))} for c in range(256)]
        on_lo = [{(lo[b], lo[a]) for a, b in _segments_on(seg[c], (d, 0))} for c in range(256)]
        bits_hi = [tuple((ca >> c) & 1 for c in range(8) if gen.corner_xyz(c)[d] == 1) for ca in range(256)]
        bits_lo = [tuple((cb >> c) & 1 for c in range(8) if gen.corner_xyz(c)[d] == 0) for cb in range(256)]
        for a in range(256):
            for b in range(256):
                if bits_hi[a] != bits_lo[b]:
                    continue
                assert on_hi[a] == on_lo[b], (d, a, b)
                checked += 1
    assert checked == 3 * 256 * 16


# ---------------------------------------------------------------------------------------------------- topology
def _topology(m):
    """-> Euler characteristic of a closed, oriented 2-manifold mesh (asserted) and its divergence-theorem volume."""
    f = m["faces"].astype(np.int64)
    nv = m["pos"].shape[0]
    assert f.size == 0 or (f.min() >= 0 and f.max() < nv)
    assert len(np.unique(f.reshape(-1))) == nv, "a vertex without a face"
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    key = e[:, 0] * nv + e[:, 1]
    rkey = e[:, 1] * nv + e[:, 0]
    assert len(np.unique(key)) == len(key), "a directed edge appears twice"
    assert np.array_equal(np.sort(key), np.sort(rkey)), "a directed edge without its reverse"
    n_edges = len(key) // 2
    p = m["pos"].astype(np.float64)
    vol = np.einsum("ij,ij->i", p[f[:, 0]], np.cross(p[f[:, 1]], p[f[:, 2]])).sum() / 6.0
    return nv - n_edges + f.shape[0], vol


def _check_values(m, s, level):
    """Every vertex interpolates to `level` on its edge, to float32 rounding (unit offset / scale)."""
    R = s.shape[0] - 2
    g = m["edge"][:, :3] + 1
    d = m["edge"][:, 3]
    e = np.eye(3, dtype=np.int64)[d]
    sa, sb = s[tuple(g.T)].astype(np.float64), s[tuple((g + e).T)].astype(np.float64)
    c = m["pos"][np.arange(len(d)), d].astype(np.float64) * R
    t = c - (m["edge"][np.arange(len(d)), d] + 0.5)
    assert ((t >= 0) & (t <= 1)).all()
    val = sa + t * (sb - sa)
    assert np.allclose(val, level, rtol=0, atol=4e-6 * np.maximum(1.0, np.abs(sb - sa)) * R), np.abs(val - level).max()


def test_random_lattices_are_closed_oriented_manifolds():
    rng = np.random.default_rng(7)
    for trial in range(2000):
        s = np.zeros((10, 10, 10), np.float32)
        if trial % 2:
            s[1:-1, 1:-1, 1:-1] = (rng.random((8, 8, 8)) < rng.uniform(0.1, 0.9)).astype(np.float32)
            level = 0.5
        else:
            s[1:-1, 1:-1, 1:-1] = rng.random((8, 8, 8)).astype(np.float32)
            level = float(rng.uniform(0.05, 0.95))
        m = io.mesh(s, level)
        chi, vol = _topology(m)
        assert chi % 2 == 0
        if m["faces"].shape[0]:
            assert vol > 0, trial
        _check_values(m, s, level)


def _field(kind, L):
    R = 1 << L
    c = (np.arange(R) + 0.5) / R
    x, y, z = np.meshgrid(c, c, c, indexing="ij")
    if kind == "sphere":
        f = 0.3 ** 2 - ((x - 0.5) ** 2 + (y - 0.48) ** 2 + (z - 0.52) ** 2)
    elif kind == "two":
        f = np.maximum(0.15 ** 2 - ((x - 0.3) ** 2 + (y - 0.5) ** 2 + (z - 0.5) ** 2),
                       0.15 ** 2 - ((x - 0.72) ** 2 + (y - 0.5) ** 2 + (z - 0.5) ** 2))
    else:   # torus around z, radii 0.25 / 0.1
        q = np.sqrt((x - 0.5) ** 2 + (y - 0.5) ** 2) - 0.25
        f = 0.1 ** 2 - (q ** 2 + (z - 0.5) ** 2)
    s = np.zeros((R + 2,) * 3, np.float32)
    s[1:-1, 1:-1, 1:-1] = (f * 10 + 1).astype(np.float16).astype(np.float32)
    return s


@pytest.mark.parametrize("kind,chi", [("sphere", 2), ("torus", 0), ("two", 4)])
@pytest.mark.parametrize("L", [4, 5, 6])
def test_analytic_fields(kind, chi, L):
    s = _field(kind, L)
    m = io.mesh(s, 1.0)
    got, vol = _topology(m)
    assert got == chi
    assert vol > 0
    _check_values(m, s, 1.0)


def test_sphere_geometry_level7():
    L, r, x0 = 7, 0.3, np.array([0.5, 0.48, 0.52])
    R = 1 << L
    c = (np.arange(R) + 0.5) / R
    x, y, z = np.meshgrid(c, c, c, indexing="ij")
    s = np.zeros((R + 2,) * 3, np.float32)
    s[1:-1, 1:-1, 1:-1] = (4.0 * (r * r - ((x - x0[0]) ** 2 + (y - x0[1]) ** 2 + (z - x0[2]) ** 2)) + 1.0
                           ).astype(np.float16).astype(np.float32)
    m = io.mesh(s, 1.0)
    chi, vol = _topology(m)
    assert chi == 2
    assert abs(vol / (4 / 3 * np.pi * r ** 3) - 1) < 0.01, vol
    dist = np.linalg.norm(m["pos"].astype(np.float64) - x0, axis=1)
    assert np.abs(dist - r).max() < 1.0 / R


def test_full_tree_is_a_closed_box():
    """sigma > level everywhere: a box whose faces sit t = level / sigma of the way from the padding points to the
    outermost cell centres, through the tree's world transform."""
    child = np.zeros((1, 2, 2, 2), np.int32)
    data = np.full((1, 2, 2, 2, 4), 0.25, np.float16)
    data[..., 3] = 5.0
    off, sc = np.array([0.5, 0.25, 0.5], np.float32), np.array([0.5, 0.25, 0.125], np.float32)
    for L in (1, 3):
        R = 1 << L
        m = io.isosurface(child, data, off, sc, L, 2.0)
        chi, vol = _topology(m)
        assert chi == 2 and vol > 0
        assert m["pos"].shape[0] == 6 * R * R
        d = m["edge"][:, 3]
        lower = m["edge"][np.arange(len(d)), d] == -1
        # from the padding point (sigma 0) up to the outermost centre, and from there down to the padding point
        t_lo = np.float32(2.0) / np.float32(5.0)
        t_hi = (np.float32(2.0) - np.float32(5.0)) / (np.float32(0.0) - np.float32(5.0))
        c = np.where(lower, np.float32(-0.5) + t_lo, np.float32(R - 0.5) + t_hi).astype(np.float32)
        want = ((c / np.float32(R)).astype(np.float32) - off[d]) / sc[d]
        assert np.array_equal(m["pos"][np.arange(len(d)), d], want.astype(np.float32))
        assert np.isclose(t_lo, 0.4) and np.isclose(t_hi, 0.6)


# ------------------------------------------------------------------------------------------------------- OBJ
def _sphere_mesh():
    from volrend_b200.mesh import Mesh
    s = _field("sphere", 4)
    m = io.mesh(s, 1.0, (0.5, 0.5, 0.5), (0.37, 0.41, 0.29))
    rng = np.random.default_rng(3)
    n = m["pos"].shape[0]
    vert = np.zeros((n, 9), np.float32)
    vert[:, :3] = m["pos"]
    vert[:, 3:6] = rng.random((n, 3)).astype(np.float32)
    nrm = rng.standard_normal((n, 3))
    vert[:, 6:9] = (nrm / np.linalg.norm(nrm, axis=1, keepdims=True)).astype(np.float32)
    vert[0, 3:6] = [1e-38, -0.0, 3.4028235e38]                 # denormal-adjacent, signed zero, largest float
    me = Mesh(0, 0, 3)
    me.vert = vert.reshape(-1)
    me.faces = m["faces"].reshape(-1)
    return me


def test_obj_round_trip(tmp_path):
    from volrend_b200.isosurface import write_obj
    from volrend_b200.mesh import Mesh
    me = _sphere_mesh()
    path = str(tmp_path / "s.obj")
    write_obj(me, path)
    back = Mesh.load_basic_obj(path)
    want = me.vert.reshape(-1, 9)
    got = np.asarray(back.vert, np.float32).reshape(-1, 9)
    assert got.shape == want.shape
    diff = np.nonzero((got.view(np.uint32) != want.view(np.uint32)).any(1))[0]
    assert diff.size == 0, [(want[i].tolist(), got[i].tolist()) for i in diff[:5]]
    assert np.array_equal(np.asarray(back.faces, np.uint32), me.faces)


def test_obj_round_trip_reference_loader(tmp_path):
    from oracle import ref_mesh
    if not ref_mesh.available():
        pytest.skip("reference build not present")
    from volrend_b200.isosurface import write_obj
    me = _sphere_mesh()
    path = str(tmp_path / "s.obj")
    write_obj(me, path)
    with open(path) as f:
        r = ref_mesh.load_mem_obj(f.read())
    want = me.vert.reshape(-1, 9)
    got = np.asarray(r["vert"], np.float32).reshape(-1, 9)
    assert got.shape == want.shape
    diff = np.nonzero((got.view(np.uint32) != want.view(np.uint32)).any(1))[0]
    assert diff.size == 0, [(want[i].tolist(), got[i].tolist()) for i in diff[:5]]
    assert np.array_equal(np.asarray(r["faces"], np.uint32).reshape(-1), me.faces)


# ------------------------------------------------------------------------------------------------ CLI, device
@pytest.mark.parametrize("argv", [
    ["t.npz", "o.obj"],                                          # no --level
    ["t.npz", "o.obj", "--level", "0"],
    ["t.npz", "o.obj", "--level", "-1"],
    ["t.npz", "o.obj", "--level", "nan"],
    ["t.npz", "o.obj", "--level", "inf"],
    ["t.npz", "o.obj", "--level", "1", "--depth", "0"],
    ["t.npz", "o.obj", "--level", "1", "--depth", "12"],
    ["t.npy", "o.obj", "--level", "1"],
    ["t.npz", "o.ply", "--level", "1"],
    ["t.npz", "o.obj", "--level", "1", "--no-color", "--basis-minmax", "0", "3"],
    ["missing_tree.npz", "o.obj", "--level", "1"],
])
def test_cli_argument_errors(argv, capsys):
    from volrend_b200 import isosurface
    with pytest.raises(SystemExit) as e:
        isosurface.main(argv)
    assert e.value.code == 2


def test_entry_point_without_a_device(built):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from volrend_b200 import _capi, lib
    L = lib()
    fake = C.create_string_buffer(4096)
    n, m = C.c_int64(-3), C.c_int64(-3)
    args = (C.addressof(fake), 5, C.c_float(1.0), None, 0, None, 0, None, 0, C.byref(n), C.byref(m), None)
    assert L.vr_tree_isosurface(*args) == _capi.VR_ENODEVICE
    assert (n.value, m.value) == (-3, -3)
    assert L.vr_tree_isosurface(C.addressof(fake), 12, C.c_float(1.0), None, 0, None, 0, None, 0, C.byref(n),
                                C.byref(m), None) == _capi.VR_EINVAL
    assert L.vr_tree_isosurface(C.addressof(fake), 5, C.c_float(0.0), None, 0, None, 0, None, 0, C.byref(n),
                                C.byref(m), None) == _capi.VR_EINVAL
    assert L.vr_tree_isosurface(C.addressof(fake), 5, C.c_float(1.0), None, 2, None, 0, None, 0, C.byref(n),
                                C.byref(m), None) == _capi.VR_EINVAL
    from volrend_b200 import N3Tree
    from volrend_b200.isosurface import isosurface_arrays
    with pytest.raises(Exception):
        isosurface_arrays(N3Tree(), 1.0)
