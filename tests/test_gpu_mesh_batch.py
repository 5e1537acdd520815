"""`-m gpu`: batched mesh rendering.  vr_draw_meshes_batch against per-view vr_draw_meshes (bit for bit) and
oracle/mesh_oracle.py, vr_render_composite_batch(_opts) against per-view vr_render_composite, VolumeRenderer.render_batch
against VolumeRenderer.render(), launch counts, and render_animation's batched frames against the per-frame path."""
import contextlib
import copy
import ctypes as C
import io

import numpy as np
import pytest

from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)
from oracle import mesh_oracle as mo

pytestmark = pytest.mark.gpu
QUEUE, INLINE = 7, 3 + 16 * 193


def _cam(W, H, eye, target=(0.0, 0.0, 0.0), f=1.4):
    from volrend_b200 import Camera, synth
    c = Camera(W, H, synth.focal_for(W) * f, synth.focal_for(W) * f * 0.95)
    c.set_c2w(synth.look_at_c2w(eye, target))
    return c


def _orbit(W, H, n, r=3.2):
    return [_cam(W, H, (r * np.cos(0.7 * i), r * np.sin(0.7 * i), 1.5 * np.sin(0.3 * i) + 0.4)) for i in range(n)]


def _golden_meshes(name):
    from volrend_b200 import Mesh
    z = np.load(f"{ROOT}/tests/golden/ref/{name}.npz")
    data = bytes(z["input"])
    with contextlib.redirect_stdout(io.StringIO()):
        return Mesh.open_drawlist_mem(data) if str(z["kind"]) == "drawlist" else [Mesh.load_mem_basic_obj(data)]


@pytest.fixture(scope="module")
def sh16():
    from volrend_b200 import N3Tree, synth
    return N3Tree.from_synth(synth.make_tree("lego", depth=6, basis_dim=16, seed=1))


@pytest.fixture(scope="module")
def scenes(sh16):
    """name -> mesh list: the section 8 scenes, the legoman OBJ, a 100-camera drawlist and a depth-3 grid."""
    from volrend_b200 import Mesh
    rng = np.random.default_rng(5)
    cube = Mesh.Cube((0.9, 0.6, 0.3))
    cube.rotation[:] = (0.4, -0.3, 0.8)
    sph = Mesh.Sphere(9, 14, (0.3, 0.7, 0.9))
    sph.translation[:] = (0.6, 0.5, 0.3)
    sph.scale = 0.7
    helix = np.stack([np.cos(np.linspace(0, 9, 40)), np.sin(np.linspace(0, 9, 40)), np.linspace(-1, 1, 40)], 1)
    lines = Mesh.Lines(helix.reshape(-1), (1.0, 0.2, 0.2))
    pts = Mesh.Points(rng.uniform(-1.2, 1.2, (60, 3)).reshape(-1), (0.1, 0.1, 1.0))
    quad = Mesh(4, 2, 3)                     # runs under and behind most cameras: clipped at the near plane
    v = quad.vert.reshape(-1, 9)
    v[:, :3] = [(-6, -6, -0.2), (6, -6, -0.2), (6, 6, -0.2), (-6, 6, -0.2)]
    v[:, 3:6] = (0.8, 0.8, 0.2)
    v[:, 6:9] = (0, 0, 1)
    quad.faces[:] = (0, 1, 2, 0, 2, 3)
    big = Mesh(3, 0, 3, unlit=True)         # fills every frame: the large-primitive path
    big.vert.reshape(-1, 9)[:, :3] = [(-40, -40, 0.05), (40, -40, 0.05), (0, 60, 0.05)]
    big.vert.reshape(-1, 9)[:, 3:6] = 0.4
    tie_a, tie_b = Mesh.Cube((1.0, 0.0, 0.0)), Mesh.Cube((0.0, 0.0, 1.0))   # exact ties: the earlier one wins
    grid = Mesh._on_device(sh16.wireframe_device(3), face_size=2, unlit=True)
    return dict(cube=[cube], sphere=[sph], lines=[lines], points=[pts], straddler=[quad], filling=[big],
                ties=[tie_a, tie_b], legoman=_golden_meshes("mesh_obj_legoman"),
                frustums=_golden_meshes("mesh_dl_cams100"), grid=[grid])


def _view_lists(scenes, n, seed=0):
    """Per-view mesh lists: shallow copies with per-view model transforms (one per scene, so the tie scene keeps its
    ties), cycling through the scenes, with a view without meshes and a view whose meshes are all invisible every five
    views."""
    rng = np.random.default_rng(seed)
    names = sorted(scenes)
    out = []
    for i in range(n):
        ms = []
        for name in (names[i % len(names)], names[(3 * i + 1) % len(names)]):
            dr, dt, ds = rng.uniform(-0.3, 0.3, 3), rng.uniform(-0.2, 0.2, 3), float(rng.uniform(0.8, 1.2))
            for m in scenes[name]:
                c = copy.copy(m)
                if name != "grid":
                    c.rotation = (np.asarray(m.rotation, np.float32) + dr).astype(np.float32)
                    c.translation = (np.asarray(m.translation, np.float32) + dt).astype(np.float32)
                    c.scale = float(m.scale) * ds
                ms.append(c)
        if i % 5 == 3:
            ms = []
        elif i % 5 == 4:
            for c in ms:
                c.visible = False
        out.append(ms)
    return out


def _inputs(n, H, W, seed=1):
    import torch
    rng = np.random.default_rng(seed)
    img = torch.from_numpy(rng.integers(0, 256, (n, H, W, 4), dtype=np.uint8)).cuda()
    dep = np.where(rng.uniform(size=(n, H, W)) < 0.3, rng.uniform(1.0, 5.0, (n, H, W)), 1e9).astype(np.float32)
    return img, torch.from_numpy(dep).cuda()


def _singles(cams, lists, img0, dep0):
    import torch
    from volrend_b200 import draw_meshes
    img, dep = img0.clone(), dep0.clone()
    for i, (c, ms) in enumerate(zip(cams, lists)):
        draw_meshes(c, ms, img[i], dep[i])
    torch.cuda.synchronize()
    return img.cpu().numpy(), dep.cpu().numpy()


def _batch(cams, lists, img0, dep0):
    import torch
    from volrend_b200 import draw_meshes_batch, lib
    img, dep = img0.clone(), dep0.clone()
    n0 = lib().vr_launch_count()
    draw_meshes_batch(cams, lists, img, dep)
    torch.cuda.synchronize()
    return img.cpu().numpy(), dep.cpu().numpy(), lib().vr_launch_count() - n0


@pytest.mark.parametrize("n", [1, 2, 7, 64])
def test_draw_batch_equals_single_draws(built, scenes, n):
    W, H = 96, 72
    cams = _orbit(W, H, n)
    lists = _view_lists(scenes, n, seed=n)
    # the grid was generated on the current stream: nothing else to wait for
    img0, dep0 = _inputs(n, H, W, seed=n)
    u1, d1 = _singles(cams, lists, img0, dep0)
    u2, d2, launches = _batch(cams, lists, img0, dep0)
    assert np.array_equal(u1, u2) and np.array_equal(d1.view(np.uint32), d2.view(np.uint32))
    drawn = (d1 != dep0.cpu().numpy()).reshape(n, -1).any(1)
    assert drawn.sum() >= min(n, 2)
    assert launches == 4          # one launch group at this size, whatever the number of views
    for i in range(n):
        if i % 5 in (3, 4):
            assert not drawn[i] and np.array_equal(u2[i], img0[i].cpu().numpy())


def test_draw_batch_matches_oracle(built, scenes):
    W, H = 64, 48
    cams = _orbit(W, H, 5)
    lists = [[copy.copy(m) for m in scenes[k]] for k in ("cube", "sphere", "lines", "points", "ties")]
    lists[1][0].rotation = np.array([0.0, 0.5, 0.2], np.float32)
    img0, dep0 = _inputs(5, H, W, seed=9)
    u, d, _ = _batch(cams, lists, img0, dep0)
    for i, (cam, ms) in enumerate(zip(cams, lists)):
        specs = []
        for m in ms:
            f = np.asarray(m.faces, np.uint32)
            specs.append(dict(vert=np.asarray(m.vert, np.float32), faces=f if f.size else None, face_size=m.face_size,
                              unlit=int(m.unlit), model=m.model_matrix().T.reshape(16)))
        c12 = np.ascontiguousarray(cam.transform, np.float32).reshape(12)
        r0, z0 = img0[i].cpu().numpy(), dep0[i].cpu().numpy()
        uo, do, win = mo.draw_meshes(W, H, cam.fx, cam.fy, c12, specs, r0, z0)
        cov = d[i] != z0
        assert np.array_equal(cov, win > 0), (i, cov.sum(), (win > 0).sum())
        assert np.all(np.abs(d[i] - do) <= 1e-5 * np.abs(do))
        assert np.abs(u[i].astype(int) - uo.astype(int)).max() <= 1
        assert cov.sum() > 10


def test_draw_batch_split_into_launch_groups(built, scenes):
    """64 views at 800x800 need 328 MB of z-buffer: more than one launch group, same bytes as single draws."""
    W, H, n = 800, 800, 64
    cams = _orbit(W, H, n)
    lists = [[copy.copy(m) for m in scenes["filling"] + scenes["sphere"] + scenes["grid"]] for _ in range(n)]
    for i, ms in enumerate(lists):
        ms[1].translation = np.array([0.1 * np.sin(i), 0.0, 0.2], np.float32)
    img0, dep0 = _inputs(n, H, W, seed=3)
    u1, d1 = _singles(cams, lists, img0, dep0)
    u2, d2, launches = _batch(cams, lists, img0, dep0)
    assert np.array_equal(u1, u2) and np.array_equal(d1.view(np.uint32), d2.view(np.uint32))
    assert launches % 4 == 0 and 8 <= launches <= 16


def test_draw_batch_errors(built, scenes):
    from volrend_b200 import _capi, draw_meshes_batch, lib
    from volrend_b200._capi import VolrendError
    import torch
    cams = _orbit(32, 24, 3)
    img = torch.zeros((3, 24, 32, 4), dtype=torch.uint8, device="cuda")
    dep = torch.full((3, 24, 32), 1e9, dtype=torch.float32, device="cuda")
    cams[1].width = 40
    with pytest.raises(VolrendError) as e:
        draw_meshes_batch(cams, [scenes["cube"]] * 3, img, dep)
    assert e.value.code == _capi.VR_EINVAL
    cams[1].width = 32
    with pytest.raises(ValueError):
        draw_meshes_batch(cams, [scenes["cube"]] * 2, img, dep)
    arr = (_capi.vr_camera * 3)(*[c._as_c() for c in cams])
    for off in ([1, 1, 1, 1], [0, 1, 0, 1]):
        o = (C.c_int32 * 4)(*off)
        assert lib().vr_draw_meshes_batch(arr, 3, None, o, img.data_ptr(), dep.data_ptr(), None) == _capi.VR_EINVAL
    assert lib().vr_draw_meshes_batch(arr, 3, None, None, img.data_ptr(), dep.data_ptr(), None) == _capi.VR_EINVAL
    assert lib().vr_draw_meshes_batch(arr, -1, None, None, img.data_ptr(), dep.data_ptr(), None) == _capi.VR_EINVAL
    n0 = lib().vr_launch_count()
    o = (C.c_int32 * 4)(0, 0, 0, 0)
    assert lib().vr_draw_meshes_batch(arr, 3, None, o, img.data_ptr(), dep.data_ptr(), None) == _capi.VR_OK
    assert lib().vr_draw_meshes_batch(arr, 0, None, None, None, None, None) == _capi.VR_OK
    assert lib().vr_launch_count() == n0


# ------------------------------------------------------------------------------------------- composite batches
@pytest.fixture(scope="module")
def trees(small_trees):
    from volrend_b200 import N3Tree
    return {k: N3Tree.from_synth(small_trees[k]) for k in ("sh16_d6", "sh25_d5", "rgba_d5", "sg9_d5")}


def _composite(tree, cams, opts, img0, dep0, tile, batch, per_view):
    import torch
    from volrend_b200 import _capi, lib
    from volrend_b200.host import _cams_array, _options_array, _rect
    img = img0.clone()
    fo = torch.zeros(img.shape, dtype=torch.float32, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    n, px = len(cams), img[0].numel()
    if batch:
        oarr = _options_array(opts if per_view else opts[:1])
        fn = lib().vr_render_composite_batch_opts if per_view else lib().vr_render_composite_batch
        _capi.check(fn(tree._handle, _cams_array(cams), n, oarr, _rect(tile), img.data_ptr(), dep0.data_ptr(),
                       fo.data_ptr(), s))
    else:
        for i in range(n):
            c, o = cams[i]._as_c(), (opts[i] if per_view else opts[0])._as_c()
            _capi.check(lib().vr_render_composite(tree._handle, C.byref(c), C.byref(o), _rect(tile),
                                                  img.data_ptr() + i * px, dep0.data_ptr() + 4 * (px // 4) * i,
                                                  fo.data_ptr() + 4 * px * i, s))
    torch.cuda.synchronize()
    return img.cpu().numpy(), fo.cpu().numpy()


@pytest.mark.parametrize("variant", [INLINE, QUEUE])
@pytest.mark.parametrize("name", ["sh16_d6", "sh25_d5", "rgba_d5", "sg9_d5"])
def test_composite_batch_equals_single(built, trees, name, variant):
    from volrend_b200 import RenderOptions, lib
    if name == "rgba_d5" and variant == QUEUE:
        pytest.skip("RGBA trees have no shading-queue kernel")
    tree = trees[name]
    bmax = max(tree.data_format.basis_dim - 1, 0)
    W, H, n = 80, 64, 6
    cams = _orbit(W, H, n, r=3.8)
    opts = [RenderOptions(step_size=1e-4 * (1 + i), background_brightness=0.15 * i, basis_minmax=[0, bmax],
                          sigma_thresh=[1e-2, 0.5][i % 2]) for i in range(n)]
    old = lib().vr_get_variant()
    lib().vr_set_variant(variant)
    try:
        for tile in (None, (8, 4, 48, 40)):
            w, h = (W, H) if tile is None else tile[2:]
            img0, dep0 = _inputs(n, h, w, seed=7)
            for per_view in (False, True):
                a = _composite(tree, cams, opts, img0, dep0, tile, False, per_view)
                b = _composite(tree, cams, opts, img0, dep0, tile, True, per_view)
                assert np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))
                assert not np.array_equal(a[0], img0.cpu().numpy())
    finally:
        lib().vr_set_variant(old)


def test_composite_batch_beyond_camera_ring(built, trees):
    from volrend_b200 import RenderOptions
    tree = trees["sh16_d6"]
    n, W, H = 8192 + 37, 8, 8
    cams = [_orbit(W, H, 8, r=3.8)[i % 8] for i in range(n)]
    opts = [RenderOptions(background_brightness=(i % 11) / 10, basis_minmax=[0, 15]) for i in range(n)]
    img0, dep0 = _inputs(n, H, W, seed=2)
    for per_view in (False, True):
        a = _composite(tree, cams, opts, img0, dep0, None, False, per_view)
        b = _composite(tree, cams, opts, img0, dep0, None, True, per_view)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))


def test_composite_batch_variants_and_errors(built, trees):
    import torch
    from volrend_b200 import RenderOptions, _capi, lib
    from volrend_b200.host import _cams_array, _options_array
    tree = trees["sh16_d6"]
    cams = _orbit(16, 16, 2)
    img = torch.zeros((2, 16, 16, 4), dtype=torch.uint8, device="cuda")
    dep = torch.full((2, 16, 16), 1e9, dtype=torch.float32, device="cuda")
    oarr = _options_array([RenderOptions(), RenderOptions()])
    for fn in (lib().vr_render_composite_batch, lib().vr_render_composite_batch_opts):
        assert fn(tree._handle, _cams_array(cams), 2, oarr, None, img.data_ptr(), None, None, None) == _capi.VR_EINVAL
        assert fn(tree._handle, _cams_array(cams), -1, oarr, None, img.data_ptr(), dep.data_ptr(), None,
                  None) == _capi.VR_EINVAL
        cams[1].width = 17
        assert fn(tree._handle, _cams_array(cams), 2, oarr, None, img.data_ptr(), dep.data_ptr(), None,
                  None) == _capi.VR_EINVAL
        cams[1].width = 16


# ------------------------------------------------------------------------------------- VolumeRenderer.render_batch
def _renderer(tree, W, H):
    from volrend_b200 import VolumeRenderer
    rend = VolumeRenderer()
    rend.resize(W, H)
    if tree is not None:
        rend.set(tree)
    return rend


@pytest.mark.parametrize("with_tree", [True, False])
def test_render_batch_equals_render(built, sh16, scenes, with_tree):
    from volrend_b200 import RenderOptions, lib
    W, H, n = 96, 72, 12
    rend = _renderer(sh16 if with_tree else None, W, H)
    cams = []
    for i in range(n):
        c = copy.deepcopy(rend.camera)
        c.center = np.array([3.3 * np.cos(0.6 * i), 3.3 * np.sin(0.6 * i), 1.2 + 0.1 * i], np.float32)
        c.v_back = (c.center / np.linalg.norm(c.center)).astype(np.float32)
        c.fx = c.fy = 110.0 + i
        cams.append(c)
    box, ball = scenes["cube"][0], scenes["sphere"][0]
    opts, lists = [], []
    for i in range(n):
        o = RenderOptions(background_brightness=[0.0, 0.3, 0.55, 1.0, 0.8][i % 5], basis_minmax=[0, 15],
                          step_size=1e-4 * (1 + i % 3))
        o.enable_probe = i % 4 == 1
        o.probe = [0.1 * (i % 3), 0.2, 0.1]
        o.show_grid = i % 3 == 2
        o.grid_max_depth = 2 + i % 2
        ms = []
        if i % 6 in (0, 1, 4):
            b, s = copy.copy(box), copy.copy(ball)
            b.rotation = np.array([0.1 * i, 0.2, 0.0], np.float32)
            s.translation = np.array([0.5, 0.05 * i, 0.2], np.float32)
            s.unlit = i % 2 == 1
            ms = [b, s]
        if i == 4:
            ms[0].visible = ms[1].visible = False
        opts.append(o)
        lists.append(ms)
    n0 = lib().vr_launch_count()
    got = rend.render_batch(cams, opts, lists).cpu().numpy()
    assert lib().vr_launch_count() - n0 < 16 * n
    kinds = set()
    for i in range(n):
        rend.camera, rend.options, rend.meshes = copy.deepcopy(cams[i]), opts[i], lists[i]
        want = rend.render().cpu().numpy()
        assert np.array_equal(got[i], want), i
        kinds.add((bool([m for m in lists[i] if m.visible]), opts[i].enable_probe, opts[i].show_grid))
    assert len(kinds) >= 5
    # one RenderOptions for every view, and self.meshes
    rend.meshes = [box]
    rend.options = opts[1]
    got = rend.render_batch(cams[:3]).cpu().numpy()
    for i in range(3):
        rend.camera = copy.deepcopy(cams[i])
        assert np.array_equal(got[i], rend.render().cpu().numpy()), i


def test_render_batch_launches_do_not_grow_with_views(built, sh16, scenes):
    from volrend_b200 import RenderOptions, lib
    rend = _renderer(sh16, 64, 48)
    o = RenderOptions(basis_minmax=[0, 15])
    counts = []
    for n in (8, 32):
        cams = [copy.deepcopy(rend.camera) for _ in range(n)]
        for i, c in enumerate(cams):
            c.center = np.array([3.0 * np.cos(i), 3.0 * np.sin(i), 1.5], np.float32)
            c.v_back = (c.center / np.linalg.norm(c.center)).astype(np.float32)
        rend.render_batch(cams, o, [scenes["cube"]] * n)      # warm (grid, rings)
        n0 = lib().vr_launch_count()
        rend.render_batch(cams, o, [scenes["cube"]] * n)
        counts.append(lib().vr_launch_count() - n0)
    assert counts[0] == counts[1] == 5                       # 4 raster launches and one composite march


# ---------------------------------------------------------------------------------------------------- animator
def test_render_animation_batched_frames(built, sh16, tmp_path):
    """A 40-frame orbit with a drawlist mesh, the probe and the grid: the same PNG bytes as rendering and writing
    each frame with VolumeRenderer.render(), in O(chunks) launches."""
    from volrend_b200 import Camera, Mesh, RenderOptions, lib, write_png_file
    from volrend_b200.anim import ANIM_CHUNK, AnimKF, MeshState, animation_frames, render_animation
    kfs = []
    for c in ([-3.5, 0.0, 3.0], [3.5, 0.2, 2.5]):
        k = AnimKF(t_max=1.0, fx=80.0, fy=80.0)
        k.center = np.array(c, np.float32)
        k.v_back = (k.center / np.linalg.norm(k.center)).astype(np.float32)
        k.opt = RenderOptions(basis_minmax=[0, 15], enable_probe=True, probe=[0.0, 0.0, 0.0], show_grid=True,
                              grid_max_depth=3, background_brightness=0.4)
        kfs.append(k)
    kfs[0].mesh_state = {"box": MeshState(np.zeros(3, np.float32), np.array([0.4, 0.5, 0.6], np.float32), 0.2)}
    kfs[1].mesh_state = {"box": MeshState(np.array([0.3, 0.1, 0.2], np.float32), np.array([0.5, 0.5, 0.4], np.float32),
                                          0.3)}
    dl = str(tmp_path / "dl.npz")
    np.savez(dl, box="cube", box__color=np.asarray([0.1, 0.7, 0.3], np.float32))
    W, H, fps = 64, 48, 40.0
    rend = _renderer(sh16, W, H)
    rend.meshes = Mesh.open_drawlist(dl)
    rend.render()                      # warm: grid, rings, pool
    n0 = lib().vr_launch_count()
    paths = render_animation(sh16, kfs, fps, str(tmp_path / "new"), width=W, height=H, meshes=Mesh.open_drawlist(dl))
    launches = lib().vr_launch_count() - n0
    states = list(animation_frames(kfs, fps, (0, 0, 1), Camera(W, H)))
    assert len(paths) == len(states) >= 40
    chunks = -(-len(paths) // ANIM_CHUNK)
    assert launches <= 12 * chunks, launches
    for (state, _), p in zip(states, paths):
        state.to_renderer(rend)
        ref = str(tmp_path / "ref.png")
        assert write_png_file(ref, rend.render().cpu().numpy())
        assert open(p, "rb").read() == open(ref, "rb").read(), p
