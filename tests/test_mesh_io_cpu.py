"""Drawlist / OBJ loaders, presets and transforms against the reference's goldens, and the numpy restatement of
estimate_normals (oracle/mesh_io_oracle.py).  No GPU: loads that need normals are checked with the oracle's."""
import contextlib
import ctypes as C
import io

import numpy as np
import pytest

import mesh_io_cases as mc
from oracle import mesh_io_oracle as mo
from oracle import ref_mesh
from volrend_b200 import Mesh, mesh_io

GOLDENS = mc.golden_files()
needs_ref = pytest.mark.skipif(not ref_mesh.available(), reason="oracle/_ref/libref_mesh.so not built (make ref)")


def _load(kind, data, vis):
    with contextlib.redirect_stdout(io.StringIO()):
        return Mesh.open_drawlist_mem(data, vis) if kind == "drawlist" else [Mesh.load_mem_basic_obj(data)]


@pytest.fixture
def oracle_normals(monkeypatch):
    monkeypatch.setattr(mesh_io, "estimate_normals", lambda me: setattr(me, "vert", mo.estimate_normals(me.vert, me.faces)))


def test_goldens_present():
    names = {g[len("mesh_"):-len(".npz")] for g in GOLDENS}
    assert {"dl_presets", "dl_quirks", "dl_normals", "dl_cams100", "dl_dtypes", "obj_plain", "obj_forms",
            "obj_numbers", "obj_fail", "obj_legoman", "obj_teapot_tri"} <= names


@pytest.mark.parametrize("fname", [g for g in GOLDENS if not mc.load_golden(g)[3]])
def test_loader_matches_golden_without_normals(fname):
    kind, data, vis, _, want = mc.load_golden(fname)
    got = _load(kind, data, vis)
    assert mc.mismatches([mc.as_record(m) for m in got], want) == []


@pytest.mark.parametrize("fname", GOLDENS)
def test_oracle_normals_match_golden(fname, oracle_normals):
    kind, data, vis, _, want = mc.load_golden(fname)
    got = _load(kind, data, vis)
    assert mc.mismatches([mc.as_record(m) for m in got], want) == []


def test_golden_quirks_are_visible():
    """The drawlist quirks the goldens pin: byte-order names, unsupported types, element-size reads."""
    _, data, vis, _, want = mc.load_golden("mesh_dl_quirks.npz")
    names = [m["name"] for m in want]
    assert names == sorted(names) and b"Zeta" in names and b"alpha" not in names and b"cameras" in names
    assert b"b2" in names and b"bad" not in names and b"_under" not in names and b"cameras_image_width" not in names
    b2 = want[names.index(b"b2")]
    assert b2["vert"].size == 6 * 5 * 9                  # rings from the float32's int32 bits (6), sectors 5
    assert all(m["unlit"] == (m["name"] == b"vis") for m in want)   # unlit defaults to 0 for every type


def test_soup_and_skipped_faces_oracle():
    pts, faces = mc.normals_edge_points()
    v = Mesh.Points(pts.reshape(-1)).vert
    soup = mo.estimate_normals(v, np.zeros(0, np.uint32)).reshape(-1, 9)
    assert (soup[15, 6:9] == 0).all()                      # past the last whole face
    f = np.concatenate([faces, [0, 1, 99]]).astype(np.uint32)
    a = mo.estimate_normals(v, f)
    b = mo.estimate_normals(v, faces.astype(np.uint32))
    assert a.tobytes() == b.tobytes()                      # a face with an index >= n_verts contributes nothing


def test_reads_past_an_array_use_defaults():
    data = mc._npz(False, a="cube", a__color=np.asarray([0.1, 0.2], np.float32), a__scale=np.zeros(0, np.float32),
                   b="camerafrustum", b__t=np.asarray([1.0, 2.0, 3.0, 4.0, 5.0, 6.0]), b__r=np.asarray([0.0, 1.0, 0.0]))
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        a, b = Mesh.open_drawlist_mem(data)
    assert "Invalid shape for float3" in out.getvalue() and "different sizes" in out.getvalue()
    ref = Mesh.Cube()
    assert a.vert.tobytes() == ref.vert.tobytes() and a.scale == 1.0
    two = Mesh.CameraFrustum(1111.0, 800.0, 800.0, color=(1.0, 0.5, 0.2))   # the drawlist default colour
    two.repeat(2)
    two.apply_transform([0, 1, 0], [1, 2, 3], 0, 5)
    two.apply_transform([0, 0, 0], [4, 5, 6], 5, 10)    # the missing r values are 0
    assert b.vert.tobytes() == two.vert.tobytes()


def test_obj_failure_and_missing_file(tmp_path):
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        m = Mesh.load_basic_obj(str(tmp_path / "missing.obj"))
    assert m.n_verts == 0 and m.name == "Mesh" and "ERROR Failed to load OBJ" in out.getvalue()
    p = tmp_path / "t.obj"
    p.write_text("v 0 0 0 1 0 0\nv 1 0 0\nv 0 1 0\nvn 0 0 1\nvn 0 0 1\nvn 0 0 1\nf 1 2 3\n")
    m = Mesh.load_basic_obj(str(p))
    assert m.name == str(p) and m.faces.tolist() == [0, 1, 2]
    assert m.vert.reshape(3, 9)[:, 3:6].tolist() == [[1, 0, 0], [1, 1, 1], [1, 1, 1]]


def test_loads_without_normals_need_no_device(monkeypatch):
    def boom(me):
        raise AssertionError("estimate_normals called")
    monkeypatch.setattr(mesh_io, "estimate_normals", boom)
    _, data, vis, _, want = mc.load_golden("mesh_dl_cams100.npz")
    assert len(_load("drawlist", data, vis)) == len(want)


def test_normals_load_raises_without_device(built):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from volrend_b200 import VolrendError, _capi
    _, data, vis, _, _ = mc.load_golden("mesh_obj_plain.npz")
    with pytest.raises(VolrendError) as e:
        Mesh.load_mem_basic_obj(data)
    assert e.value.code == _capi.VR_ENODEVICE


def test_capi_argument_checks(built):
    import torch
    from volrend_b200 import _capi, lib
    L = lib()
    buf = (C.c_float * 9)()
    assert L.vr_mesh_estimate_normals(buf, -1, None, 0, None) == _capi.VR_EINVAL
    assert L.vr_mesh_estimate_normals(buf, 3, None, -1, None) == _capi.VR_EINVAL
    assert L.vr_mesh_estimate_normals(None, 3, None, 0, None) == _capi.VR_EINVAL
    assert L.vr_mesh_estimate_normals(buf, 2 ** 31, None, 0, None) == _capi.VR_EINVAL
    assert L.vr_mesh_estimate_normals(buf, 3, buf, 2 ** 31 // 3 + 1, None) == _capi.VR_EINVAL
    if torch.cuda.is_available():
        return
    assert L.vr_mesh_estimate_normals(None, 0, None, 0, None) == _capi.VR_ENODEVICE
    assert b"no CPU fallback" in L.vr_last_error()


@needs_ref
def test_presets_and_transforms_against_reference():
    for reso in (1, 2, 8, 13):
        assert mc.mismatches([mc.as_record(Mesh.Lattice(reso, (0.1, 0.2, 0.3)))],
                             [ref_mesh.lattice(reso, (0.1, 0.2, 0.3))]) == []
    for args in [(1111.0, 800, 800, -0.3), (370.7, 1920, 1080, 0.77), (1e-3, 3, 5, -2.5)]:
        assert mc.mismatches([mc.as_record(Mesh.CameraFrustum(*args, color=(1, 0.5, 0)))],
                             [ref_mesh.camera_frustum(*args, (1, 0.5, 0))]) == []
    rng = np.random.default_rng(3)
    tr = [(rng.normal(size=3).astype(np.float32) * rng.choice([1e-4, 1, 3]), rng.normal(size=3).astype(np.float32),
           k * 5 % 63, -1 if k % 3 == 0 else min(252, k * 9)) for k in range(30)]
    tr.append((rng.normal(size=(4, 4)).astype(np.float32), None, 0, -1))
    base = Mesh.Sphere(7, 9)
    want = ref_mesh.repeat_transform(base.vert, base.faces, 3, 4, tr)
    base.repeat(4)
    for r, t, s, e in tr:
        base.apply_transform(r, t, s, e)
    assert base.vert.tobytes() == want["vert"].tobytes() and base.faces.tobytes() == want["faces"].tobytes()


def _random_drawlist(rng):
    arrays = {}
    for i in range(int(rng.integers(3, 9))):
        name = "".join(rng.choice(list("abcXYZ_0"), size=int(rng.integers(1, 5))))
        if "__" in name or name.endswith("_"):     # a trailing "_" turns "<name>__<field>" into a bad key
            continue
        kind = str(rng.choice(["cube", "sphere", "line", "camerafrustum", "lines", "points", "mesh"]))
        arrays[name] = kind
        ft = rng.choice([np.float16, np.float32, np.float64])
        if rng.uniform() < 0.5:
            arrays[name + "__color"] = rng.uniform(0, 1, 3).astype(ft)
        if rng.uniform() < 0.5:
            arrays[name + "__translation"] = rng.normal(size=3).astype(ft)
        if rng.uniform() < 0.5:
            arrays[name + "__rotation"] = rng.normal(size=3).astype(ft)
        if rng.uniform() < 0.3:
            arrays[name + "__visible"] = np.int8(rng.integers(0, 2))
        n = int(rng.integers(3, 40))
        if kind in ("lines", "points", "mesh"):
            arrays[name + "__points"] = rng.normal(size=3 * n).astype(ft)
        if kind == "mesh":
            arrays[name + "__face_size"] = np.int32(rng.integers(1, 4))
            if rng.uniform() < 0.7:
                arrays[name + "__faces"] = rng.integers(0, n, size=3 * int(rng.integers(1, 30))).astype(np.int32)
        if kind == "camerafrustum" and rng.uniform() < 0.7:
            k = int(rng.integers(1, 6))
            arrays[name + "__t"] = rng.normal(size=3 * k)
            arrays[name + "__r"] = rng.normal(size=3 * k)
            arrays[name + "__connect"] = np.int32(rng.integers(0, 2))
        if kind == "sphere":
            arrays[name + "__rings"] = np.int32(rng.integers(2, 12))
    return mc._npz(bool(rng.integers(0, 2)), **arrays)


def _random_obj(rng):
    n = int(rng.integers(4, 30))
    L = []
    for _ in range(n):
        p = " ".join(f"{x:.{int(rng.integers(1, 9))}g}" for x in rng.normal(size=3))
        L.append("v " + p + (" 0.25 0.5 1" if rng.uniform() < 0.5 else ""))
    if rng.uniform() < 0.5:
        L += ["vn 0 0 1"] * n
    for _ in range(int(rng.integers(1, 20))):
        k = int(rng.choice([3, 3, 4]))
        idx = rng.choice(n, size=k, replace=False) + 1
        L.append("f " + " ".join(str(int(i)) if rng.uniform() < 0.7 else str(int(i) - n - 1) for i in idx))
    return "\n".join(L) + "\n"


@needs_ref
def test_live_reference_on_random_inputs(oracle_normals):
    rng = np.random.default_rng(11)
    for _ in range(25):
        data = _random_drawlist(rng)
        with contextlib.redirect_stdout(io.StringIO()):
            want = ref_mesh.open_drawlist_mem(data)
        assert mc.mismatches([mc.as_record(m) for m in _load("drawlist", data, True)], want) == []
        text = _random_obj(rng)
        with contextlib.redirect_stdout(io.StringIO()):
            want = [ref_mesh.load_mem_obj(text)]
        assert mc.mismatches([mc.as_record(m) for m in _load("obj", text.encode(), True)], want) == []
