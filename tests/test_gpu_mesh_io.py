"""`-m gpu`: vr_mesh_estimate_normals (volrend_b200/csrc/vr_normals.cu) and the loaders that use it, against the
reference's goldens, the live reference harness, and the numpy oracle (oracle/mesh_io_oracle.py); loaded meshes
drawn by VolumeRenderer against the mesh and march oracles."""
import contextlib
import io

import numpy as np
import pytest

import mesh_io_cases as mc
from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)
from oracle import mesh_io_oracle as mo
from oracle import ref_mesh

pytestmark = pytest.mark.gpu
GOLDENS = mc.golden_files()


def _load(kind, data, vis=True):
    from volrend_b200 import Mesh
    with contextlib.redirect_stdout(io.StringIO()):
        return Mesh.open_drawlist_mem(data, vis) if kind == "drawlist" else [Mesh.load_mem_basic_obj(data)]


def _gpu_normals(vert, faces, stream=None):
    from volrend_b200 import Mesh, estimate_normals
    m = Mesh(0, 0, 3)
    m.vert, m.faces = np.asarray(vert, np.float32).reshape(-1), np.asarray(faces, np.uint32).reshape(-1)
    estimate_normals(m, stream)
    return np.asarray(m.vert, np.float32), m


@pytest.mark.parametrize("fname", GOLDENS)
def test_loader_matches_golden(built, fname):
    kind, data, vis, _, want = mc.load_golden(fname)
    got = _load(kind, data, vis)
    assert mc.mismatches([mc.as_record(m) for m in got], want) == []


@pytest.mark.skipif(not ref_mesh.available(), reason="oracle/_ref/libref_mesh.so not built (make ref)")
def test_live_reference_on_random_inputs(built):
    from test_mesh_io_cpu import _random_drawlist, _random_obj
    rng = np.random.default_rng(29)
    for _ in range(20):
        data = _random_drawlist(rng)
        with contextlib.redirect_stdout(io.StringIO()):
            want = ref_mesh.open_drawlist_mem(data)
        assert mc.mismatches([mc.as_record(m) for m in _load("drawlist", data)], want) == []
        text = _random_obj(rng)
        with contextlib.redirect_stdout(io.StringIO()):
            want = [ref_mesh.load_mem_obj(text)]
        assert mc.mismatches([mc.as_record(m) for m in _load("obj", text.encode())], want) == []


def _random_mesh(rng, nv, nf, hub=False):
    v = np.zeros((nv, 9), np.float32)
    v[:, :3] = rng.normal(size=(nv, 3))
    v[:, 3:6] = rng.uniform(size=(nv, 3))
    v[:, 6:9] = 7.0                                  # overwritten
    f = rng.integers(0, nv, size=(nf, 3)).astype(np.uint32)
    if hub:
        f[::3, 0] = 0                                # one vertex shared by a third of the faces: a long serial chain
    return v.reshape(-1), f.reshape(-1)


@pytest.mark.parametrize("nv,nf", [(1, 0), (5, 1), (1000, 3000), (1_900_000, 1_000_000), (400_000, 4_000_000)])
def test_normals_match_oracle(built, nv, nf):
    rng = np.random.default_rng(nv + nf)
    v, f = _random_mesh(rng, nv, nf, hub=nf >= 3000)
    if nf == 0:
        f = np.zeros(0, np.uint32)
        f_idx = np.asarray([0, 0, 0], np.uint32)    # a degenerate face on the only vertex
        got, _ = _gpu_normals(v, f_idx)
        assert got.tobytes() == mo.estimate_normals(v, f_idx).tobytes()
        return
    got, _ = _gpu_normals(v, f)
    want = mo.estimate_normals(v, f)
    assert got.tobytes() == want.tobytes()
    g, w = got.reshape(-1, 9), v.reshape(-1, 9)
    assert g[:, :6].tobytes() == w[:, :6].tobytes()          # only floats 6..8 change


def test_triangle_soup(built):
    rng = np.random.default_rng(5)
    for nv in (3, 4, 5, 3 * 1000 + 2, 6_000_000):
        v = rng.choice(np.asarray([-1, -0.0, 0.0, 1, 0.5], np.float32), size=(nv, 9)).reshape(-1)
        got, _ = _gpu_normals(v, np.zeros(0, np.uint32))
        assert got.tobytes() == mo.estimate_normals(v, np.zeros(0, np.uint32)).tobytes()


def test_out_of_range_faces_are_skipped(built):
    rng = np.random.default_rng(6)
    v, f = _random_mesh(rng, 300, 900)
    bad = f.copy().reshape(-1, 3)
    bad[::7, int(rng.integers(0, 3))] = 300 + rng.integers(0, 2 ** 31, size=len(bad[::7]))
    keep = (bad < 300).all(1)
    got, _ = _gpu_normals(v, bad)
    assert got.tobytes() == _gpu_normals(v, bad[keep])[0].tobytes()
    assert got.tobytes() == mo.estimate_normals(v, bad).tobytes()


def test_repeatable_across_runs_and_streams(built):
    import torch
    rng = np.random.default_rng(8)
    v, f = _random_mesh(rng, 200_000, 600_000, hub=True)
    a, _ = _gpu_normals(v, f)
    b, _ = _gpu_normals(v, f)
    s = torch.cuda.Stream()
    c, m = _gpu_normals(v, f, s)
    assert a.tobytes() == b.tobytes() == c.tobytes()
    assert m._vert_dev.cpu().numpy().tobytes() == a.tobytes()       # the device copy is current


def test_launches(built):
    from volrend_b200 import lib
    for fname in GOLDENS:
        kind, data, vis, needs, _ = mc.load_golden(fname)
        n0 = lib().vr_launch_count()
        _load(kind, data, vis)
        if not needs:
            assert lib().vr_launch_count() == n0, fname
        else:
            assert lib().vr_launch_count() > n0, fname
    rng = np.random.default_rng(9)
    v, f = _random_mesh(rng, 100, 50)
    n0 = lib().vr_launch_count()
    _gpu_normals(v, np.zeros(0, np.uint32))
    assert lib().vr_launch_count() - n0 == 1                       # soup: one kernel
    n0 = lib().vr_launch_count()
    _gpu_normals(v, f)
    assert lib().vr_launch_count() - n0 == 4                       # corners, sort, scan, per-vertex sum


@pytest.fixture(scope="module")
def sh4(small_trees):
    from volrend_b200 import N3Tree
    st = small_trees["sh4_d5"]
    return st, N3Tree.from_synth(st)


def _scene_drawlist():
    rng = np.random.default_rng(12)
    n = 6
    ang = np.linspace(0, 2 * np.pi, n, endpoint=False)
    t = np.stack([0.9 * np.cos(ang), 0.9 * np.sin(ang), np.full(n, 0.3)], 1)
    r = rng.normal(size=(n, 3)) * 0.5
    pts = rng.uniform(-0.6, 0.6, size=(200, 3))
    sph = __import__("volrend_b200").Mesh.Sphere(8, 12)
    sp = np.asarray(sph.vert).reshape(-1, 9)[:, :3] * 0.3
    return mc._npz(True, cams="camerafrustum", cams__t=t, cams__r=r, cams__connect=np.int32(1), cams__z=-0.2,
                   cams__focal_length=np.float32(400), cloud="points", cloud__points=pts.reshape(-1),
                   cloud__color=np.asarray([1.0, 0.2, 0.2]), blob="mesh", blob__points=sp.reshape(-1),
                   blob__faces=np.asarray(sph.faces, np.int32), blob__color=np.asarray([0.3, 0.8, 0.4]),
                   blob__translation=np.asarray([0.1, -0.1, 0.0]))


@pytest.mark.parametrize("which", ["drawlist", "obj"])
def test_volume_renderer_with_loaded_meshes(built, sh4, which):
    from test_gpu_mesh import _gpu_chain, _oracle_chain, _renderer
    st, tree = sh4
    if which == "drawlist":
        meshes = _load("drawlist", _scene_drawlist())
        assert [m.name for m in meshes] == ["blob", "cams", "cloud"] and not meshes[0].unlit
    else:
        _, data, _, _, _ = mc.load_golden("mesh_obj_teapot_tri.npz")
        (m,) = _load("obj", data)
        m.scale = 1.0
        m.rotation[:] = (1.2, 0.0, 0.0)
        meshes = [m]
    eye = (2.6, -1.9, 1.2)
    vr = _renderer(st, tree, 80, 60, eye, 1.0, meshes)
    u, u_chain, f = _gpu_chain(vr)
    fo, uo, _, _, win = _oracle_chain(st, vr, meshes)
    assert (win > 0).sum() > 50
    assert np.array_equal(u, u_chain)
    assert np.abs(f - fo).max() <= 1e-4
    assert (u != uo).any(-1).sum() <= 3
