"""`-m gpu`: the octree grid.  vr_tree_wireframe / N3Tree.gen_wireframe against the reference's stored
gen_wireframe output and oracle/wire_oracle.py (both table parities), its buffer contract, and VolumeRenderer's
show_grid against wire_oracle -> mesh_oracle -> the CPU march oracle."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import ROOT
from oracle import mesh_oracle as mo
from oracle import wire_oracle as wo
from wire_cases import WIRE_DEPTHS, golden_name, matches, wire_tree

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref")


def _load(monkeypatch, name, parity):
    from volrend_b200 import N3Tree
    st = wire_tree(name)
    monkeypatch.setenv("VR_WIDE_PARITY", str(parity))
    tree = N3Tree.from_synth(st)
    monkeypatch.delenv("VR_WIDE_PARITY")
    assert tree.info()["wide_parity"] == parity
    return st, tree


@pytest.mark.parametrize("parity", [0, 1])
@pytest.mark.parametrize("name", sorted(WIRE_DEPTHS))
def test_wireframe_matches_reference_and_oracle(built, monkeypatch, name, parity):
    st, tree = _load(monkeypatch, name, parity)
    for d in WIRE_DEPTHS[name]:
        v = tree.gen_wireframe(d)
        rec = np.load(os.path.join(GOLDEN, golden_name(name, d) + ".npz"))
        assert matches(rec, v), (name, d, v.size, int(rec["n_floats"]))
        o = wo.wireframe(st.child, st.offset, st.invradius3, d)
        assert np.array_equal(v.view(np.uint32), o.view(np.uint32)), (name, d)
        assert tree.wireframe_vertex_count(d) * 9 == v.size


def test_reference_harness_matches_goldens(built):
    from oracle import ref_binding as rb
    from oracle import ref_wire
    if not ref_wire.available():
        pytest.skip("reference build (oracle/_ref) not present")
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        for name in ("sh4_d5", "chain"):
            path = os.path.join(tmp, name + ".npz")
            wire_tree(name).save_npz(path)
            rt = rb.RefTree(path)
            for d in WIRE_DEPTHS[name]:
                rec = np.load(os.path.join(GOLDEN, golden_name(name, d) + ".npz"))
                assert matches(rec, ref_wire.wireframe(rt, d)), (name, d)
            rt.close()


def test_count_only_and_short_buffer(built, monkeypatch):
    import torch
    from volrend_b200 import _capi, lib
    st, tree = _load(monkeypatch, "sh16_d6", 0)
    guard = 4096
    for d in (0, 3, 9):
        n = C.c_int64(-1)
        assert lib().vr_tree_wireframe(tree._handle, d, None, 0, C.byref(n), None) == 0
        nv = n.value
        buf = torch.full((nv * 9 + guard,), -3.25, dtype=torch.float32, device="cuda")
        rc = lib().vr_tree_wireframe(tree._handle, d, buf.data_ptr(), nv - 1, C.byref(n), None)
        assert rc == _capi.VR_EINVAL and b"buffer" in lib().vr_last_error()
        torch.cuda.synchronize()
        assert bool((buf == -3.25).all())
        assert lib().vr_tree_wireframe(tree._handle, d, buf.data_ptr(), nv, C.byref(n), None) == 0
        torch.cuda.synchronize()
        out = buf.cpu().numpy()
        assert n.value == nv and np.all(out[nv * 9:] == -3.25)
        o = wo.wireframe(st.child, st.offset, st.invradius3, d)
        assert np.array_equal(out[:nv * 9].view(np.uint32), o.view(np.uint32))


def test_unloaded_tree_raises(built):
    from volrend_b200 import N3Tree
    with pytest.raises(RuntimeError, match="not loaded"):
        N3Tree().gen_wireframe(2)


# ---------------------------------------------------------------------------------------------- VolumeRenderer
W, H = 64, 48
EYE = (3.2, -2.0, 1.4)


def _renderer(tree, meshes=(), depth=2, bg=1.0):
    from volrend_b200 import VolumeRenderer, synth
    vr = VolumeRenderer()
    vr.resize(W, H)
    vr.camera.fx = vr.camera.fy = synth.focal_for(W)
    vr.camera.center = np.asarray(EYE, np.float32)
    vr.camera.v_back = np.asarray(EYE, np.float32) / np.linalg.norm(EYE)
    vr.options.background_brightness = bg
    vr.set(tree)
    vr.meshes = list(meshes)
    vr.options.show_grid = True
    vr.options.grid_max_depth = depth
    return vr


def _c12(cam):
    return np.ascontiguousarray(cam.transform, np.float32).reshape(12)


def _spec(m):
    faces = np.asarray(m.faces, np.uint32)
    return dict(vert=np.asarray(m.vert, np.float32), faces=faces if faces.size else None, face_size=m.face_size,
                unlit=int(m.unlit), model=m.model_matrix().T.reshape(16))


def _wire_spec(st, depth):
    return dict(vert=wo.wireframe(st.child, st.offset, st.invradius3, depth), faces=None, face_size=2, unlit=1,
                model=np.eye(4, dtype=np.float32).reshape(16))


def _oracle_chain(st, vr, meshes):
    from oracle import binding as ob
    cam = vr.camera
    bgb = round(min(max(vr.options.background_brightness, 0.0), 1.0) * 255)
    rgba0 = np.zeros((H, W, 4), np.uint8)
    rgba0[..., :3], rgba0[..., 3] = bgb, 255
    d0 = np.full((H, W), 1e9, np.float32)
    specs = [_spec(m) for m in meshes] + [_wire_spec(st, vr.options.grid_max_depth)]
    rgba, depth, win = mo.draw_meshes(W, H, cam.fx, cam.fy, _c12(cam), specs, rgba0, d0)
    t = ob.OracleTree.from_synth(st)
    oc = ob.make_camera(W, H, cam.fx, cam.fy, _c12(cam))
    opt = ob.make_options(background_brightness=vr.options.background_brightness, basis_minmax=vr.options.basis_minmax)
    f, u, _ = ob.render(t, oc, opt, rgba_in=rgba, depth_in=depth)
    return f, u, win


def _gpu_chain(vr):
    """vr.render(), and the same clear -> draw -> composite chain with the float tap of the composite march."""
    import torch
    from volrend_b200 import draw_meshes, launch_renderer
    u = vr.render().cpu().numpy()
    cam = vr.camera
    img = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    bgb = round(min(max(vr.options.background_brightness, 0.0), 1.0) * 255)
    img[..., :3], img[..., 3] = bgb, 255
    dep = torch.full((H, W), 1e9, dtype=torch.float32, device="cuda")
    draw_meshes(cam, [m for m in vr.meshes if m.visible] + [vr._wire], img, dep)
    fo = torch.zeros((H, W, 4), dtype=torch.float32, device="cuda")
    launch_renderer(vr._tree, cam, vr.options, img, dep, None, False, float_out=fo)
    torch.cuda.synchronize()
    return u, img.cpu().numpy(), fo.cpu().numpy(), dep.cpu().numpy()


@pytest.fixture(scope="module")
def sh4(small_trees):
    from volrend_b200 import N3Tree
    st = small_trees["sh4_d5"]
    return st, N3Tree.from_synth(st)


@pytest.mark.parametrize("with_cube", [False, True])
@pytest.mark.parametrize("depth", [0, 2])
def test_volume_renderer_grid_vs_oracle(built, sh4, with_cube, depth):
    from volrend_b200 import Mesh
    st, tree = sh4
    meshes = []
    if with_cube:
        cube = Mesh.Cube((0.2, 0.9, 0.4))
        cube.scale = 0.5
        cube.rotation[:] = (0.3, 0.2, 0.5)
        meshes = [cube]
    vr = _renderer(tree, meshes, depth=depth, bg=0.5)
    u, u_chain, f, dep = _gpu_chain(vr)
    fo, uo, win = _oracle_chain(st, vr, meshes)
    assert (win > 0).sum() > 50
    assert np.array_equal(dep != 1e9, win > 0)
    assert np.array_equal(u, u_chain)
    assert np.abs(f - fo).max() <= 1e-4
    assert (u != uo).any(-1).sum() <= 2


def test_user_line_on_grid_edge_wins_tie(built, sh4):
    import torch
    from volrend_b200 import Mesh, draw_meshes
    st, tree = sh4
    v = wo.wireframe(st.child, st.offset, st.invradius3, 0).reshape(-1, 9)
    # the last edge of the first root cell: the z-parallel edge through the volume's centre, which three more
    # root cells repeat
    line = Mesh.Line(v[22, :3], v[23, :3], (1.0, 0.0, 0.0))
    vr = _renderer(tree, [line], depth=0)
    vr.render()
    cam = vr.camera

    def draw(meshes):
        img = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
        img[..., 1] = 200
        dep = torch.full((H, W), 1e9, dtype=torch.float32, device="cuda")
        draw_meshes(cam, meshes, img, dep)
        torch.cuda.synchronize()
        return img.cpu().numpy()

    own = draw([line])
    cov = own[..., 0] == 255
    assert cov.sum() > 10
    # other grid edges may pass in front of the line at a few pixels (near the corners it shares)
    both = draw([line, vr._wire])
    assert (both[cov][:, :3] == (255, 0, 0)).all(1).mean() > 0.9
    grid_first = draw([vr._wire, line])                           # the tie is real: drawn first, the grid wins
    assert (grid_first[cov][:, :3] == (0, 0, 0)).all(1).mean() > 0.9


def test_grid_regenerates_only_when_depth_changes(built, sh4):
    from volrend_b200 import lib
    st, tree = sh4
    vr = _renderer(tree, depth=2)

    def launches():
        n0 = lib().vr_launch_count()
        vr.render()
        return lib().vr_launch_count() - n0

    first = launches()
    wire = vr._wire
    again = launches()
    assert vr._wire is wire and again < first
    vr.options.grid_max_depth = 3
    assert launches() > again and vr._wire is not wire
    assert int(vr._wire._vert_dev.numel()) == tree.wireframe_vertex_count(3) * 9
    assert launches() == again
    vr.set(tree)
    vr.options.show_grid, vr.options.grid_max_depth = True, 3
    assert launches() > again


def test_show_grid_off_and_no_tree(built, sh4):
    import torch
    from volrend_b200 import VolumeRenderer, launch_renderer
    st, tree = sh4
    for bg in (1.0, 0.3):
        vr = _renderer(tree, depth=3, bg=bg)
        vr.options.show_grid = False
        u = vr.render().cpu().numpy()
        ref = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
        launch_renderer(tree, vr.camera, vr.options, ref, None, None, True)
        torch.cuda.synchronize()
        assert np.array_equal(u, ref.cpu().numpy()) and vr._wire is None
    empty = VolumeRenderer()
    empty.resize(W, H)
    empty.options.show_grid = True
    u = empty.render().cpu().numpy()
    assert np.all(u[..., :3] == 255) and np.all(u[..., 3] == 255)
