"""The C++ ``volrend::Mesh`` of the shim (volrend_b200/csrc/shim/mesh_b200.cpp) without a device: presets, ``repeat``,
``apply_transform`` and ``auto_faces`` byte for byte against ``volrend_b200.Mesh`` and the reference's own ``mesh.cpp``
(oracle/_ref/libref_mesh.so), and OBJ files that need no normals against the reference's goldens."""
import numpy as np
import pytest

import mesh_io_cases as mc
import shim_mesh_driver as sd
from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)
from oracle import ref_mesh

pytestmark = pytest.mark.skipif(not sd.available(), reason="oracle/_ref/shim_mesh not built (needs the reference)")

GREY = (0.5, 0.5, 0.5)
DEFAULT = (1.0, 0.5, 0.2)


def _cpp(tmp_path, build):
    """Runs ``build(script)``, which adds meshes, and saves every one of them; returns their records."""
    s = sd.Script(tmp_path)
    n = build(s)
    for i in range(n):
        s.save(i)
    meshes, _, out = s.run()
    return meshes, out


def _rec(m):
    return mc.as_record(m)


def _presets(rng):
    """(driver command, product Mesh) pairs."""
    from volrend_b200 import Mesh
    pts7, pts1, pts8f = rng.uniform(-1, 1, 21), rng.uniform(-1, 1, 3), rng.uniform(-1, 1, 8)
    cloud = rng.uniform(-1, 1, 150)
    return [
        (("cube", *DEFAULT), Mesh.Cube()),
        (("cube", 0.1, 0.7, 0.3), Mesh.Cube((0.1, 0.7, 0.3))),
        (("sphere", 15, 30, *DEFAULT), Mesh.Sphere()),
        (("sphere", 9, 12, 0.2, 0.4, 0.9), Mesh.Sphere(9, 12, (0.2, 0.4, 0.9))),
        (("sphere", 4, 5, 1.0, 0.0, 0.0), Mesh.Sphere(4, 5, (1.0, 0.0, 0.0))),
        (("lattice", 8, *GREY), Mesh.Lattice()),
        (("lattice", 3, 0.1, 0.2, 0.3), Mesh.Lattice(3, (0.1, 0.2, 0.3))),
        (("frustum", 1111.0, 800.0, 800.0, -0.3, *GREY), Mesh.CameraFrustum(1111.0, 800.0, 800.0)),
        (("frustum", 500.5, 640.0, 480.0, 0.4, 0.0, 1.0, 1.0), Mesh.CameraFrustum(500.5, 640, 480, 0.4, (0, 1, 1))),
        (("line", 0.1, 0.2, 0.3, -1.0, 2.0, 0.5, *GREY), Mesh.Line((np.float32(0.1), np.float32(0.2), np.float32(0.3)),
                                                                   (-1.0, 2.0, 0.5))),
        (("lines", pts7, 1.0, 0.0, 0.0), Mesh.Lines(pts7, (1.0, 0.0, 0.0))),
        (("lines", pts1, *GREY), Mesh.Lines(pts1)),
        (("lines", pts8f, *GREY), Mesh.Lines(pts8f)),
        (("points", cloud, 0.3, 0.6, 0.9), Mesh.Points(cloud, (0.3, 0.6, 0.9))),
        (("points", np.zeros(0), *GREY), Mesh.Points(np.zeros(0, np.float32))),
        (("empty", 4, 3, 2, 1), Mesh(4, 3, 2, True)),
        (("empty", 0, 0, 3, 0), Mesh()),
    ]


def _add_preset(s, cmd):
    if cmd[0] in ("lines", "points"):
        s.add(cmd[0], s.f32(cmd[1]), *cmd[2:])
    else:
        s.add(*cmd)


def test_presets_match_python(tmp_path):
    cases = _presets(np.random.default_rng(3))

    def build(s):
        for cmd, _ in cases:
            _add_preset(s, cmd)
        return len(cases)

    got, out = _cpp(tmp_path, build)
    want = [_rec(m) for _, m in cases]
    assert mc.mismatches([sd.without_transform(g) for g in got], want) == []
    assert out.count("Lines: Number of elements in points must be divisible by 3") == 1


def _random_mesh(rng, nv, n_idx):
    from volrend_b200 import Mesh
    m = Mesh(0, 0, 3)
    m.vert = rng.uniform(-2, 2, nv * 9).astype(np.float32)
    m.faces = rng.integers(0, nv, n_idx).astype(np.uint32)
    return m


def _transforms(rng, nv):
    """(r, t, start, end) for apply_transform(r, t, ...) and (M, None, start, end) for the matrix form; rotations
    include zero, one below the 1e-3 threshold and one just above it."""
    out = []
    for r in [np.zeros(3), [4e-4, -3e-4, 5e-4], [1e-3, 1e-5, 0.0], rng.normal(size=3) * 2, rng.normal(size=3)]:
        lo = int(rng.integers(0, nv))
        out.append((np.asarray(r, np.float32), rng.normal(size=3).astype(np.float32), lo, int(rng.integers(lo, nv + 1))))
    M = rng.normal(size=(4, 4)).astype(np.float32)
    out.append((M, None, 0, -1))
    out.append((np.eye(4, dtype=np.float32) * np.float32(1.5), None, 2, 5))
    return out


def _add_edits(s, i, n_repeat, transforms):
    s.add("repeat", i, n_repeat)
    for r, t, lo, hi in transforms:
        if t is None:
            s.add("xfm", i, *[np.float32(x) for x in np.asarray(r, np.float32).T.reshape(16)], lo, hi)
        else:
            s.add("xf", i, *[np.float32(x) for x in r], *[np.float32(x) for x in t], lo, hi)


def test_edits_match_python(tmp_path):
    rng = np.random.default_rng(5)
    cases = []
    for nv, n_idx, n_rep in [(7, 9, 3), (5, 0, 1), (12, 30, 0), (1, 3, 4)]:
        m = _random_mesh(rng, nv, n_idx)
        cases.append((m, n_rep, _transforms(rng, nv * max(n_rep, 1))))
    af = _random_mesh(rng, 6, 4)

    def build(s):
        for i, (m, n_rep, tr) in enumerate(cases):
            s.add("from", s.f32(m.vert), s.u32(m.faces), 3)
            _add_edits(s, i, n_rep, tr)
        s.add("from", s.f32(af.vert), s.u32(af.faces), 3)
        s.add("autofaces", len(cases))
        return len(cases) + 1

    got, _ = _cpp(tmp_path, build)
    want = []
    for m, n_rep, tr in cases:
        m.repeat(n_rep)
        for r, t, lo, hi in tr:
            m.apply_transform(r, t, lo, hi)
        want.append(_rec(m))
    af.auto_faces()
    want.append(_rec(af))
    assert mc.mismatches([sd.without_transform(g) for g in got], want) == []


@pytest.mark.skipif(not ref_mesh.available(), reason="oracle/_ref/libref_mesh.so not built (make ref)")
def test_matches_reference_mesh_cpp(tmp_path):
    """Lattice, CameraFrustum, repeat and apply_transform against the reference's own mesh.cpp."""
    rng = np.random.default_rng(9)
    lat = [(8, GREY), (5, (0.1, 0.9, 0.35))]
    fru = [(1111.0, 800.0, 800.0, -0.3, GREY), (300.25, 1000.0, 640.0, 0.7, (1.0, 0.5, 0.0))]
    edits = []
    for nv, n_idx, n_rep in [(9, 12, 4), (4, 6, 2)]:
        m = _random_mesh(rng, nv, n_idx)
        edits.append((m, n_rep, _transforms(rng, nv * n_rep)))

    def build(s):
        for reso, col in lat:
            s.add("lattice", reso, *[float(c) for c in col])
        for f, w, h, z, col in fru:
            s.add("frustum", f, w, h, z, *[float(c) for c in col])
        for i, (m, n_rep, tr) in enumerate(edits):
            s.add("from", s.f32(m.vert), s.u32(m.faces), 3)
            _add_edits(s, len(lat) + len(fru) + i, n_rep, tr)
        return len(lat) + len(fru) + len(edits)

    got, _ = _cpp(tmp_path, build)
    want = [ref_mesh.lattice(reso, col) for reso, col in lat]
    want += [ref_mesh.camera_frustum(f, w, h, z, col) for f, w, h, z, col in fru]
    want += [ref_mesh.repeat_transform(m.vert, m.faces, 3, n_rep, tr) for m, n_rep, tr in edits]
    keys = ("vert", "faces", "face_size", "unlit")
    assert mc.mismatches([{k: g[k] for k in keys + ("name",)} for g in got],
                         [{k: w[k] for k in keys + ("name",)} for w in want]) == []


OBJ_NO_NORMALS = [g for g in mc.golden_files() if g.startswith("mesh_obj_") and not mc.load_golden(g)[3]]


@pytest.mark.parametrize("fname", OBJ_NO_NORMALS)
def test_obj_goldens_without_normals(tmp_path, fname):
    """load_mem_basic_obj and load_basic_obj of every OBJ golden whose file has its own normals (no device)."""
    _, data, _, _, want = mc.load_golden(fname)
    s = sd.Script(tmp_path)
    src = s.file(data, ".obj")
    s.add("objmem", src)
    s.add("obj", src)
    s.save(0)
    s.save(1)
    (mem, path), _, out = s.run()
    assert mc.mismatches([sd.without_transform(mem)], want) == []
    named = [dict(w, name=src.encode() if w["name"] == b"OBJ" else w["name"]) for w in want]
    assert mc.mismatches([sd.without_transform(path)], named) == []
    if fname == "mesh_obj_fail.npz":
        assert out.count("ERROR Failed to load OBJ") == 2 and want[0]["name"] == b"Mesh"


def test_obj_missing_file(tmp_path):
    s = sd.Script(tmp_path)
    s.add("obj", str(tmp_path / "missing.obj"))
    s.save(0)
    (m,), _, out = s.run()
    assert m["vert"].size == 0 and m["faces"].size == 0 and m["name"] == b"Mesh"
    assert "ERROR Failed to load OBJ" in out
