"""GPU: the lumisphere probe (``enable_probe``) -- the disc drawn by vr_draw_probe after the march, against the
reference's own launch_renderer (goldens and, where oracle/_ref is built, the live harness) and the CPU oracle; the
probe cube of VolumeRenderer against mesh_oracle and the march oracle."""
import os
import subprocess
import tempfile
import zlib

import numpy as np
import pytest

from conftest import ROOT
from oracle import binding as ob
from oracle import mesh_oracle as mo
from oracle import probe_oracle as po
from probe_cases import PROBE_CASES, H, W, focal, golden_path, probe_case

pytestmark = pytest.mark.gpu

VARIANTS = [3 + 16 * 193, 7]      # the two product kernels: inline shading, shading queue


def _opts(optkw, probe, disp, enable=True):
    from volrend_b200 import RenderOptions
    o = RenderOptions(**{k: v for k, v in optkw.items()})
    o.enable_probe, o.probe, o.probe_disp_size = enable, [float(v) for v in probe], int(disp)
    return o


def _camera(pose, w=W, h=H):
    from volrend_b200 import Camera
    cam = Camera(w, h, focal(), focal())
    cam.set_c2w(pose)
    return cam


def _render(tree, cam, opts, comp=None, tile=None, float_out=False):
    """launch_renderer (offscreen, or over the composite inputs) -> (bytes, float tap or None)."""
    import torch
    from volrend_b200 import launch_renderer
    x0, y0, w, h = tile if tile is not None else (0, 0, cam.width, cam.height)
    img = torch.zeros((h, w, 4), dtype=torch.uint8, device="cuda")
    fo = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda") if float_out else None
    if comp is None:
        launch_renderer(tree, cam, opts, img, None, None, True, float_out=fo, tile=tile)
    else:
        rgba, depth = comp
        img.copy_(torch.from_numpy(rgba[y0:y0 + h, x0:x0 + w].copy()))
        dep = torch.from_numpy(depth[y0:y0 + h, x0:x0 + w].copy()).cuda()
        launch_renderer(tree, cam, opts, img, dep, None, False, float_out=fo, tile=tile)
    torch.cuda.synchronize()
    return img.cpu().numpy(), (fo.cpu().numpy() if fo is not None else None)


@pytest.fixture(scope="module")
def trees():
    from volrend_b200 import N3Tree
    cache = {}

    def get(name):
        if name not in cache:
            st, *_ = probe_case(name)
            cache[name] = (st, N3Tree.from_synth(st))
        return cache[name]
    return get


@pytest.mark.parametrize("v", VARIANTS)
@pytest.mark.parametrize("name", list(PROBE_CASES))
def test_probe_matches_reference_golden(built, trees, name, v):
    from volrend_b200 import lib
    z = np.load(golden_path(name), allow_pickle=False)
    st, tree = trees(name)
    _, pose, optkw, probe, disp, comp = probe_case(name)
    kbd = tree.info()["kernel_basis"]
    if not lib().vr_variant_supported(kbd, v):
        pytest.skip(f"variant {v} is not built for kernel basis {kbd}")
    assert lib().vr_set_variant(v) == 0
    try:
        u, _ = _render(tree, _camera(pose), _opts(optkw, probe, disp), comp)
        off, _ = _render(tree, _camera(pose), _opts(optkw, probe, disp, enable=False), comp)
    finally:
        lib().vr_set_variant(0)
    assert np.array_equal(off, z["ref_u8_off"]), (name, int((off != z["ref_u8_off"]).any(-1).sum()))
    bad = (u != z["ref_u8"]).any(-1)
    assert not bad.any(), (name, int(bad.sum()), np.argwhere(bad)[:5].tolist())


@pytest.mark.skipif(not po.ref_available(), reason="oracle/_ref/libref_probe.so not built")
@pytest.mark.parametrize("name", ["sh16_centre", "rgba", "sg9_rot", "asg4", "sh25_bbox"])
def test_probe_matches_live_reference_random_poses(built, trees, name):
    from volrend_b200 import synth
    st, tree = trees(name)
    _, _, optkw, probe, _, _ = probe_case(name)
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    poses = synth.nerf_synthetic_test_poses(40)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "t.npz")
        st.save_npz(path)
        for k in range(3):
            pose = poses[int(rng.integers(0, 40))]
            disp = int(rng.integers(5, 140))
            ref = po.ref_render_u8(path, W, H, focal(), focal(), synth.c2w_to_colmajor12(pose),
                                   po.ref_options(probe, disp, **optkw))
            u, _ = _render(tree, _camera(pose), _opts(optkw, probe, disp))
            assert np.array_equal(u, ref), (name, k, disp, int((u != ref).any(-1).sum()))


@pytest.mark.parametrize("name", ["sh16_centre", "sh16_d37", "rgba", "sg9_rot", "asg4", "sh9_composite",
                                  "sh16_minmax13"])
def test_float_tap_disc_against_oracle(built, trees, name):
    st, tree = trees(name)
    _, pose, optkw, probe, disp, comp = probe_case(name)
    u, f = _render(tree, _camera(pose), _opts(optkw, probe, disp), comp, float_out=True)
    _, f_off = _render(tree, _camera(pose), _opts(optkw, probe, disp, enable=False), comp, float_out=True)
    t = ob.OracleTree.from_synth(st)
    oc = ob.make_camera(W, H, focal(), focal(), _c12_pose(pose))
    fo = np.zeros((H, W, 4), np.float32)
    mask = po.overlay(t, oc, ob.make_options(**optkw), probe, disp, None, fo, None)
    assert mask.sum() > 100
    changed = (f != f_off).any(-1)
    assert not (changed & ~mask).any()                        # only disc pixels are touched
    assert (f[mask][:, 3] == 1.0).all()
    assert np.abs(f[mask] - fo[mask]).max() <= 2e-6
    assert np.array_equal(f[~mask], f_off[~mask])


def _c12_pose(pose):
    from volrend_b200 import synth
    return synth.c2w_to_colmajor12(pose)


@pytest.mark.parametrize("tile", [(100, 0, 60, 50), (90, 10, 33, 70), (0, 0, 80, 120), (130, 100, 30, 20)])
def test_tile_equals_crop(built, trees, tile):
    for name in ("sh16_centre", "sh9_composite"):
        st, tree = trees(name)
        _, pose, optkw, probe, disp, comp = probe_case(name)
        full, ff = _render(tree, _camera(pose), _opts(optkw, probe, disp), comp, float_out=True)
        x0, y0, w, h = tile
        u, f = _render(tree, _camera(pose), _opts(optkw, probe, disp), comp, tile=tile, float_out=True)
        assert np.array_equal(u, full[y0:y0 + h, x0:x0 + w]), (name, tile)
        assert np.array_equal(f, ff[y0:y0 + h, x0:x0 + w]), (name, tile)


def test_render_batch_equals_per_view(built, trees):
    import torch
    from volrend_b200 import lib, render_batch, synth
    st, tree = trees("sh16_centre")
    _, _, optkw, probe, disp, _ = probe_case("sh16_centre")
    poses = synth.nerf_synthetic_test_poses(8)
    cams = [_camera(p) for p in poses[:5]]
    opts = _opts(optkw, probe, disp)
    imgs = torch.zeros((5, H, W, 4), dtype=torch.uint8, device="cuda")
    fo = torch.zeros((5, H, W, 4), dtype=torch.float32, device="cuda")
    n0 = lib().vr_launch_count()
    render_batch(tree, cams, opts, imgs, float_out=fo)
    torch.cuda.synchronize()
    assert lib().vr_launch_count() - n0 == 2                   # one march, one overlay for all views
    for i, cam in enumerate(cams):
        u, f = _render(tree, cam, opts, float_out=True)
        assert np.array_equal(imgs[i].cpu().numpy(), u), i
        assert np.array_equal(fo[i].cpu().numpy(), f), i


@pytest.mark.skipif(not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "shim_probe")),
                    reason="oracle/_ref/shim_probe not built")
@pytest.mark.parametrize("name", ["sh16_centre", "rgba", "sh16_minmax13"])
def test_surface_path_through_shim(built, trees, name):
    st, tree = trees(name)
    _, pose, optkw, probe, disp, _ = probe_case(name)
    u, _ = _render(tree, _camera(pose), _opts(optkw, probe, disp))
    bmm = optkw.get("basis_minmax", [0, 24])
    m = np.asarray(pose, np.float32)[:3, :4]
    with tempfile.TemporaryDirectory() as d:
        path, pf, out = os.path.join(d, "t.npz"), os.path.join(d, "pose.txt"), os.path.join(d, "out.rgba")
        st.save_npz(path)
        np.savetxt(pf, m, fmt="%.9g")
        subprocess.check_call([os.path.join(ROOT, "oracle", "_ref", "shim_probe"), path, pf, str(W), str(H),
                               repr(focal()), *[repr(float(v)) for v in probe], str(disp), str(bmm[0]), str(bmm[1]), out])
        got = np.fromfile(out, np.uint8).reshape(H, W, 4)
    assert np.array_equal(got, u), int((got != u).any(-1).sum())


def test_probe_off_is_unchanged(built, trees):
    from volrend_b200 import RenderOptions, lib
    st, tree = trees("sh16_centre")
    _, pose, _, probe, disp, _ = probe_case("sh16_centre")
    cam = _camera(pose)
    n0 = lib().vr_launch_count()
    base, fb = _render(tree, cam, RenderOptions(), float_out=True)
    n1 = lib().vr_launch_count()
    off = RenderOptions(probe=[float(v) for v in probe], probe_disp_size=37)
    u, f = _render(tree, cam, off, float_out=True)
    n2 = lib().vr_launch_count()
    assert n1 - n0 == n2 - n1 == 1
    assert np.array_equal(u, base) and np.array_equal(f, fb)
    on = RenderOptions(enable_probe=True, probe=[float(v) for v in probe], probe_disp_size=0)
    u0, _ = _render(tree, cam, on)                                  # disp 0: nothing drawn, nothing launched
    assert lib().vr_launch_count() - n2 == 1 and np.array_equal(u0, base)


def test_back_to_back_leaves_last_frame(built, trees):
    import torch
    from volrend_b200 import launch_renderer
    st, tree = trees("sh16_centre")
    _, pose, optkw, probe, disp, _ = probe_case("sh16_centre")
    cam = _camera(pose)
    want_on, _ = _render(tree, cam, _opts(optkw, probe, disp))
    want_off, _ = _render(tree, cam, _opts(optkw, probe, disp, enable=False))
    img = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    seq = [True, False, True, True, False, False, True]
    for on in seq:
        launch_renderer(tree, cam, _opts(optkw, probe, disp, enable=on), img, None, None, True)
    torch.cuda.synchronize()
    assert np.array_equal(img.cpu().numpy(), want_on)
    launch_renderer(tree, cam, _opts(optkw, probe, disp, enable=False), img, None, None, True)
    torch.cuda.synchronize()
    assert np.array_equal(img.cpu().numpy(), want_off)


def test_unsupported_tree_raises_only_with_probe(built, small_trees):
    import torch
    from volrend_b200 import N3Tree, RenderOptions, VolrendError, launch_renderer, synth
    tree = N3Tree.from_synth(small_trees["sg7_d5"])       # basis 7: only coefficient 0 is resident
    cam = _camera(synth.nerf_synthetic_test_poses(8)[2])
    img = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    launch_renderer(tree, cam, RenderOptions(), img, None, None, True)
    with pytest.raises(VolrendError):
        launch_renderer(tree, cam, RenderOptions(enable_probe=True), img, None, None, True)
    torch.cuda.synchronize()


# ---------------------------------------------------------------- VolumeRenderer
EYE = (3.2, -2.0, 1.4)


def _renderer(tree=None, meshes=()):
    from volrend_b200 import VolumeRenderer, synth
    vr = VolumeRenderer()
    vr.resize(W, H)
    vr.camera.fx = vr.camera.fy = synth.focal_for(W)
    vr.camera.center = np.asarray(EYE, np.float32)
    vr.camera.v_back = np.asarray(EYE, np.float32) / np.linalg.norm(EYE)
    if tree is not None:
        vr.set(tree)
    vr.meshes = list(meshes)
    vr.options.enable_probe = True
    return vr


def _spec(m):
    faces = np.asarray(m.faces, np.uint32)
    return dict(vert=np.asarray(m.vert, np.float32), faces=faces if faces.size else None, face_size=m.face_size,
                unlit=int(m.unlit), model=m.model_matrix().T.reshape(16))


def test_volume_renderer_probe_scale(built, small_trees):
    from volrend_b200 import N3Tree
    st = small_trees["sh4_d5"]
    vr = _renderer()
    assert vr._probe.scale == pytest.approx(0.05) and not vr._probe.visible
    vr.set(N3Tree.from_synth(st))
    assert vr._probe.scale == float(np.float32(0.02) / np.float32(st.invradius3[0]))
    vr.render()
    assert vr._probe.visible
    assert np.array_equal(vr._probe.translation, np.asarray(vr.options.probe, np.float32))


@pytest.mark.parametrize("with_tree", [False, True])
def test_volume_renderer_probe_vs_oracle(built, small_trees, with_tree):
    from volrend_b200 import Mesh, N3Tree
    st = small_trees["sh4_d5"]
    user = Mesh.Cube((0.2, 0.9, 0.4))
    user.scale = 0.3
    user.translation[:] = (0.6, 0.0, 0.0)
    vr = _renderer(N3Tree.from_synth(st) if with_tree else None, [user])
    vr.options.probe = [0.0, 0.1, 0.2]
    if with_tree:
        vr._probe.scale = 0.3     # the set() scale leaves the cube a few pixels wide; make it easy to see
    vr.options.probe_disp_size = 40
    u = vr.render().cpu().numpy()
    cam = vr.camera
    c12 = np.ascontiguousarray(cam.transform, np.float32).reshape(12)
    bgb = round(min(max(vr.options.background_brightness, 0.0), 1.0) * 255)
    rgba0 = np.zeros((H, W, 4), np.uint8)
    rgba0[..., :3], rgba0[..., 3] = bgb, 255
    d0 = np.full((H, W), 1e9, np.float32)
    rgba, depth, win = mo.draw_meshes(W, H, cam.fx, cam.fy, c12, [_spec(user), _spec(vr._probe)], rgba0, d0)
    assert (win > 0).sum() > 50
    if not with_tree:
        cube_px = win > 0
        assert np.array_equal((u != rgba0).any(-1), cube_px)
        assert np.abs(u.astype(int) - rgba.astype(int)).max() <= 1
        return
    t = ob.OracleTree.from_synth(st)
    oc = ob.make_camera(W, H, cam.fx, cam.fy, c12)
    opt = ob.make_options(background_brightness=vr.options.background_brightness, basis_minmax=vr.options.basis_minmax)
    fo, uo, mask = po.render(t, oc, opt, vr.options.probe, vr.options.probe_disp_size, rgba_in=rgba, depth_in=depth)
    assert mask.sum() > 100
    assert (u != uo).any(-1).sum() <= 2
    assert np.abs(u.astype(int) - uo.astype(int)).max() <= 1


def test_volume_renderer_draw_order(built, small_trees, monkeypatch):
    import volrend_b200.mesh as vm
    from volrend_b200 import Mesh, N3Tree
    st = small_trees["sh4_d5"]
    vr = _renderer(N3Tree.from_synth(st), [Mesh.Cube()])
    vr.options.show_grid = True
    vr.options.grid_max_depth = 1
    seen = []
    real = vm.draw_meshes
    monkeypatch.setattr(vm, "draw_meshes", lambda cam, meshes, *a, **k: (seen.append(list(meshes)), real(cam, meshes, *a, **k)))
    vr.render()
    assert [m.name for m in seen[0]] == ["Cube", "_probe_cube", "Grid"]


def test_user_mesh_wins_tie_with_probe_cube(built, small_trees):
    import torch
    from volrend_b200 import Mesh, N3Tree, draw_meshes
    vr = _renderer(N3Tree.from_synth(small_trees["sh4_d5"]))
    vr.options.probe = [0.0, 0.0, 0.0]
    vr.render()
    vr._probe.scale = 0.5
    twin = Mesh.Cube((1.0, 1.0, 0.0))     # the probe cube's geometry in another colour: every depth ties exactly
    twin.unlit, twin.scale = True, 0.5
    twin.translation[:] = vr._probe.translation

    def draw(meshes):
        img = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
        dep = torch.full((H, W), 1e9, dtype=torch.float32, device="cuda")
        draw_meshes(vr.camera, meshes, img, dep)
        torch.cuda.synchronize()
        return img.cpu().numpy()

    cov = draw([twin])[..., 3] == 255
    assert cov.sum() > 50
    assert (draw([twin, vr._probe])[cov][:, :3] == (255, 255, 0)).all()       # drawn first, the user mesh wins
    assert not (draw([vr._probe, twin])[cov][:, :3] == (255, 255, 0)).all(1).any()
