"""Isosurface extraction on an H100 (vr_tree_isosurface, volrend_b200.isosurface; DESIGN.md section 23): bit identity
with the numpy oracle on every test tree under both table parities, normals and colours against the library's own
passes, determinism across slab sizes, topology at lattice sizes the oracle cannot reach, the mesh in the renderer and
the refusals."""
import ctypes as C
import functools

import numpy as np
import pytest

import edge_cases as ec
import golden_cases as gc
import layout_cases as lc
from oracle import iso_oracle as io
from volrend_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(params=["0", "1"])
def parity(request, monkeypatch):
    monkeypatch.setenv("VR_WIDE_PARITY", request.param)
    return int(request.param)


def _tree(st):
    from volrend_b200 import N3Tree
    return N3Tree.from_synth(st)


def _level(st):
    s = np.asarray(st.data, np.float16)[..., -1].astype(np.float32).reshape(-1)
    s = s[np.isfinite(s) & (s > 0)]
    return float(np.float32(np.quantile(s, 0.5))) if s.size else 1.0


def _gpu(tree, level, L, color=False, options=None):
    from volrend_b200.isosurface import isosurface_arrays
    v, f = isosurface_arrays(tree, level, depth=L, color=color, options=options)
    return v.cpu().numpy(), f.cpu().numpy().view(np.uint32)


def _normals(vert, faces):
    """vr_mesh_estimate_normals on the positions and faces."""
    import torch
    from volrend_b200 import lib
    from volrend_b200._capi import check
    v = torch.from_numpy(vert.copy()).cuda()
    v[:, 6:] = 0
    f = torch.from_numpy(faces.view(np.int32).copy()).cuda()
    check(lib().vr_mesh_estimate_normals(v.data_ptr() if v.numel() else None, v.shape[0],
                                         f.data_ptr() if f.numel() else None, f.shape[0], None))
    return v.cpu().numpy()[:, 6:]


def _same_as_oracle(st, tree, L, level, child=None, data=None):
    want = io.isosurface(st.child if child is None else child, st.data if data is None else data,
                         st.offset, st.invradius3, L, level)
    vert, faces = _gpu(tree, level, L)
    assert vert.shape[0] == want["pos"].shape[0] and faces.shape[0] == want["faces"].shape[0], (vert.shape, faces.shape)
    assert np.array_equal(vert[:, :3].view(np.uint32), want["pos"].view(np.uint32))
    assert np.array_equal(faces, want["faces"])
    assert (vert[:, 3:6] == 1).all()
    assert np.array_equal(vert[:, 6:].view(np.uint32), _normals(vert, faces).view(np.uint32))
    return want


GOLDEN = [n for n in gc.CASES if not n.endswith("_ndc")]


@pytest.mark.parametrize("name", GOLDEN)
def test_golden_trees(built, parity, name):
    st = gc.build_case(name)[0]
    L = min(max(int(_tree(st).info()["max_depth"]), 1), 6)
    _same_as_oracle(st, _tree(st), L, _level(st))


EDGE = [n for n in ec.TREES if n not in ec.NDC and n not in ec.REFUSED]


@pytest.mark.parametrize("name", EDGE)
def test_edge_trees(built, parity, name):
    st, npz = ec.edge_tree(name)
    from volrend_b200 import N3Tree
    if npz is not None:
        tree = N3Tree()
        tree.load_npz(npz)
        tree.load_cuda()
    else:
        tree = _tree(st)
    for L in (3, 6):
        _same_as_oracle(st, tree, L, 1.0 if name == "sigma_bits" else _level(st))


@pytest.mark.parametrize("layout", lc.LAYOUTS)
def test_relaid_trees(built, parity, layout):
    st = ec.mixed_tree(6, 9, "SH", 111)
    r = lc.relayout(st, layout, seed=5)
    _same_as_oracle(r.st, _tree(r.st), 5, _level(st))


def _analytic(kind, level_cells=5, fmt="SH9", seed=0):
    """A tree built on the GPU from a dense level-`level_cells` grid of an analytic sigma (1 at the surface), colour
    coefficients random; world box [-1, 1]^3 (dyadic offset and scale)."""
    from volrend_b200 import build
    R = 1 << level_cells
    c = (np.arange(R) + 0.5) / R
    x, y, z = np.meshgrid(c, c, c, indexing="ij")
    if kind == "sphere":
        f = 0.3 ** 2 - ((x - 0.5) ** 2 + (y - 0.48) ** 2 + (z - 0.52) ** 2)
    else:
        q = np.sqrt((x - 0.5) ** 2 + (y - 0.5) ** 2) - 0.25
        f = 0.1 ** 2 - (q ** 2 + (z - 0.5) ** 2)
    dd = 4 if fmt == "RGBA" else 3 * int(fmt[2:]) + 1
    grid = np.random.default_rng(seed).standard_normal((R, R, R, dd)).astype(np.float32) * 0.5
    grid[..., -1] = f * 10 + 1
    cells, rows = build.grid_cells(grid, sigma_thresh=0.0)
    npz = build.build_npz(cells, rows, data_format=fmt)
    st = synth.SynthTree(child=npz["child"], data=npz["data"], offset=npz["offset"], invradius3=npz["invradius3"],
                         data_dim=int(npz["data_dim"]), data_format=str(npz["data_format"]), depth=level_cells, extra=None)
    return st


def test_analytic_trees_every_depth(built, parity):
    for kind in ("sphere", "torus"):
        st = _analytic(kind)
        tree = _tree(st)
        for L in range(1, 8):
            _same_as_oracle(st, tree, L, 1.0)


def _inside_world(st, inside, L):
    R = np.float32(1 << L)
    u = (inside.astype(np.float32) + np.float32(0.5)) / R
    return ((u - st.offset[None]) / st.invradius3[None]).astype(np.float32)


@pytest.mark.parametrize("fmt", ["SH9", "SH16", "RGBA", "SH1"])
def test_colours_are_eval_at_the_inside_endpoint(built, parity, fmt):
    from volrend_b200 import RenderOptions
    st = _analytic("sphere", 5, fmt, seed=3)
    tree = _tree(st)
    L = 6
    want = io.isosurface(st.child, st.data, st.offset, st.invradius3, L, 1.0)
    for bmm in (None, [1, 3]):
        opt = None
        if bmm is not None:
            opt = RenderOptions()
            opt.basis_minmax = bmm
        vert, faces = _gpu(tree, 1.0, L, color=True, options=opt)
        plain, _ = _gpu(tree, 1.0, L)
        assert np.array_equal(vert[:, [0, 1, 2, 6, 7, 8]].view(np.uint32), plain[:, [0, 1, 2, 6, 7, 8]].view(np.uint32))
        rgb, _ = tree.eval(_inside_world(st, want["inside"], L), np.ascontiguousarray(-vert[:, 6:9]), opt)
        assert np.array_equal(vert[:, 3:6].view(np.uint32), rgb.view(np.uint32)), bmm


def test_determinism_and_slabs(built, monkeypatch):
    import torch
    from volrend_b200 import lib, _capi
    st = _analytic("torus", 6, seed=1)
    tree = _tree(st)
    L = 7
    base = _gpu(tree, 1.0, L, color=True)
    again = _gpu(tree, 1.0, L, color=True)
    assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(base, again))
    for planes in ("2", "3", "5", "64"):
        monkeypatch.setenv("VR_ISO_SLAB_PLANES", planes)
        got = _gpu(tree, 1.0, L, color=True)
        assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(base, got)), planes
    monkeypatch.delenv("VR_ISO_SLAB_PLANES")
    nv, nf = C.c_int64(), C.c_int64()
    assert lib().vr_tree_isosurface(tree._handle, L, C.c_float(1.0), None, _capi.VR_ISO_COLOR, None, 0, None, 0,
                                    C.byref(nv), C.byref(nf), None) == 0
    assert (nv.value, nf.value) == (base[0].shape[0], base[1].shape[0])
    torch.cuda.synchronize()


def _topology(vert, faces):
    f = faces.astype(np.int64)
    nv = vert.shape[0]
    assert len(np.unique(f.reshape(-1))) == nv
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    key = np.sort(e[:, 0] * nv + e[:, 1])
    assert (np.diff(key) > 0).all(), "a directed edge appears twice"
    assert np.array_equal(key, np.sort(e[:, 1] * nv + e[:, 0])), "a directed edge without its reverse"
    p = vert[:, :3].astype(np.float64)
    vol = np.einsum("ij,ij->i", p[f[:, 0]], np.cross(p[f[:, 1]], p[f[:, 2]])).sum() / 6.0
    return nv - len(key) // 2 + f.shape[0], vol


@functools.lru_cache(maxsize=1)
def _bench_tree():
    return synth.make_tree("lego", depth=10, basis_dim=16, seed=0)   # the stand-in tree of bench.py


@pytest.mark.parametrize("L", [9, 10])
def test_large_lattices(built, L):
    for kind, chi in (("sphere", 2), ("torus", 0)):
        st = _analytic(kind, 7)
        vert, faces = _gpu(_tree(st), 1.0, L)
        got, vol = _topology(vert, faces)
        assert got == chi and vol > 0, (kind, got, vol)
    st = _bench_tree()
    vert, faces = _gpu(_tree(st), _level(st), L, color=True)
    _, vol = _topology(vert, faces)
    assert vol > 0 and np.isfinite(vert).all()


def test_mesh_in_the_renderer(built):
    import torch
    from volrend_b200 import Camera, VolumeRenderer, render_batch, RenderOptions
    from volrend_b200.isosurface import extract_mesh
    st = _analytic("sphere", 7)
    tree = _tree(st)
    L = 7
    m = extract_mesh(tree, 1.0, depth=L)
    assert m.name == "isosurface" and m.face_size == 3
    centre = np.array([0.5, 0.48, 0.52]) * 2 - 1              # world: unit * 2 - 1
    r_world = 0.3 * 2
    W = H = 64
    cam = Camera(W, H, synth.focal_for(W), synth.focal_for(W))
    cam.center = (centre + np.array([0, 0, 3.0])).astype(np.float32)     # looking down -z at the sphere's centre
    cam.v_back = np.array([0, 0, 1], np.float32)
    cam.v_world_up = np.array([0, 1, 0], np.float32)
    r = VolumeRenderer()
    r.camera = cam
    r.resize(W, H)
    r.meshes.append(m)
    img = r.render()
    torch.cuda.synchronize()
    depth = r._depth.cpu().numpy()
    d = depth[H // 2 - 1:H // 2 + 1, W // 2 - 1:W // 2 + 1]
    assert np.abs(d - (3.0 - r_world)).max() < 2.0 / (1 << L), d
    assert (img.cpu().numpy()[H // 2, W // 2, :3] != round(RenderOptions().background_brightness * 255)).any()
    # with the tree, through the batch path
    r.set(tree)
    one = r.render().cpu().numpy().copy()
    batch = r.render_batch([cam])
    batch = (batch if not isinstance(batch, (tuple, list)) else batch[0])
    assert np.asarray(batch.cpu().numpy()).reshape(-1, H, W, 4).shape[0] == 1
    r.meshes.clear()
    bare = r.render().cpu().numpy()
    assert (one != bare).any()


def _pool_used():
    import torch
    cu = C.CDLL("libcuda.so.1")
    dev, pool, v = C.c_int(), C.c_void_p(), C.c_uint64()
    assert cu.cuDeviceGet(C.byref(dev), torch.cuda.current_device()) == 0
    assert cu.cuDeviceGetDefaultMemPool(C.byref(pool), dev) == 0
    assert cu.cuMemPoolGetAttribute(pool, 7, C.byref(v)) == 0          # CU_MEMPOOL_ATTR_USED_MEM_CURRENT
    return v.value


def test_refusals(built):
    import torch
    from volrend_b200 import lib, _capi, N3Tree
    Lb = lib()
    st = _analytic("sphere", 4)
    tree = _tree(st)
    h = tree._handle
    nv, nf = C.c_int64(), C.c_int64()
    assert Lb.vr_tree_isosurface(h, 5, C.c_float(1.0), None, 0, None, 0, None, 0, C.byref(nv), C.byref(nf), None) == 0
    n_v, n_f = nv.value, nf.value
    assert n_v > 0 and n_f > 0
    vert = torch.full((n_v + 4, 9), 7.5, dtype=torch.float32, device="cuda")
    faces = torch.full((n_f + 4, 3), -9, dtype=torch.int32, device="cuda")
    host = (C.c_float * 16)()
    E, U = _capi.VR_EINVAL, _capi.VR_EUNSUPPORTED
    vp, fp = vert.data_ptr(), faces.data_ptr()
    cases = [
        ("depth 0", (h, 0, 1.0, 0, vp, n_v, fp, n_f), E, False),
        ("depth 12", (h, 12, 1.0, 0, vp, n_v, fp, n_f), E, False),
        ("level 0", (h, 5, 0.0, 0, vp, n_v, fp, n_f), E, False),
        ("level < 0", (h, 5, -1.0, 0, vp, n_v, fp, n_f), E, False),
        ("level nan", (h, 5, float("nan"), 0, vp, n_v, fp, n_f), E, False),
        ("level inf", (h, 5, float("inf"), 0, vp, n_v, fp, n_f), E, False),
        ("flags", (h, 5, 1.0, 2, vp, n_v, fp, n_f), E, False),
        ("one output", (h, 5, 1.0, 0, vp, n_v, None, n_f), E, False),
        ("other output", (h, 5, 1.0, 0, None, n_v, fp, n_f), E, False),
        ("small vert", (h, 5, 1.0, 0, vp, n_v - 1, fp, n_f), E, True),
        ("small faces", (h, 5, 1.0, 0, vp, n_v, fp, n_f - 1), E, True),
        ("host vert", (h, 5, 1.0, 0, C.addressof(host), n_v, fp, n_f), E, False),
    ]
    for what, (t, L, lv, fl, v, mv, f, mf), code, counted in cases:
        v0, f0 = vert.clone(), faces.clone()
        torch.cuda.synchronize()
        used0, alloc0 = _pool_used(), torch.cuda.memory_allocated()
        nv.value, nf.value = -7, -7
        rc = Lb.vr_tree_isosurface(t, L, C.c_float(lv), None, fl, v, mv, f, mf, C.byref(nv), C.byref(nf), None)
        torch.cuda.synchronize()
        assert rc == code, (what, rc, Lb.vr_last_error())
        assert (nv.value, nf.value) == ((n_v, n_f) if counted else (-7, -7)), what
        assert torch.equal(vert, v0) and torch.equal(faces, f0), what
        assert _pool_used() == used0 and torch.cuda.memory_allocated() == alloc0, what
    assert Lb.vr_tree_isosurface(h, 5, C.c_float(1.0), None, 0, None, 0, None, 0, None, C.byref(nf), None) == E
    assert Lb.vr_tree_isosurface(h, 5, C.c_float(1.0), None, 0, None, 0, None, 0, C.byref(nv), None, None) == E
    assert Lb.vr_tree_isosurface(None, 5, C.c_float(1.0), None, 0, None, 0, None, 0, C.byref(nv), C.byref(nf),
                                 None) == E
    # NDC trees; colours of a basis the device keeps only coefficient 0 of
    st_ndc, *_rest = gc.build_case("lego_sh16_ndc")
    ndc = gc.build_case("lego_sh16_ndc")[5]
    t_ndc = N3Tree()
    t_ndc.load_npz(st_ndc.npz_dict())
    t_ndc.use_ndc = True
    t_ndc.ndc_width, t_ndc.ndc_height, t_ndc.ndc_focal = ndc
    t_ndc.load_cuda()
    assert Lb.vr_tree_isosurface(t_ndc._handle, 5, C.c_float(1.0), None, 0, None, 0, None, 0, C.byref(nv),
                                 C.byref(nf), None) == U
    sg7 = synth.make_tree("lego", depth=5, basis_dim=7, fmt="SG", seed=8)
    t7 = _tree(sg7)
    assert Lb.vr_tree_isosurface(t7._handle, 5, C.c_float(1.0), None, _capi.VR_ISO_COLOR, None, 0, None, 0,
                                 C.byref(nv), C.byref(nf), None) == U
    assert Lb.vr_tree_isosurface(t7._handle, 5, C.c_float(1.0), None, 0, None, 0, None, 0, C.byref(nv),
                                 C.byref(nf), None) == 0
    with pytest.raises(ValueError):
        from volrend_b200.isosurface import isosurface_arrays
        isosurface_arrays(tree, 0.0)


def test_cli(built, tmp_path):
    from volrend_b200 import isosurface, Mesh
    st = _analytic("sphere", 5)
    path = str(tmp_path / "t.npz")
    np.savez(path, **st.npz_dict())
    out = str(tmp_path / "s.obj")
    assert isosurface.main([path, out, "--level", "1.0", "--depth", "6", "--basis-minmax", "0", "3"]) == 0
    m = Mesh.load_basic_obj(out)
    from volrend_b200 import RenderOptions
    opt = RenderOptions()
    opt.basis_minmax = [0, 3]
    want = isosurface.extract_mesh(_tree(st), 1.0, depth=6, options=opt)
    assert np.array_equal(np.asarray(m.vert, np.float32).view(np.uint32), want.vert.view(np.uint32))
    assert np.array_equal(np.asarray(m.faces, np.uint32), want.faces)
