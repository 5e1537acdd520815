"""`-m gpu`: the CUDA mesh rasterizer (vr_draw_meshes) against oracle/mesh_oracle.py, and VolumeRenderer's
mesh + volume composite against the oracle raster followed by the CPU march oracle."""
import math

import numpy as np
import pytest

from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)
from oracle import mesh_oracle as mo

pytestmark = pytest.mark.gpu
W, H = 96, 72


def _cam(W, H, eye, target=(0.0, 0.0, 0.0)):
    from volrend_b200 import Camera, synth
    c = Camera(W, H, synth.focal_for(W) * 1.4, synth.focal_for(W) * 1.3)
    c.set_c2w(synth.look_at_c2w(eye, target))
    return c


def _spec(m):
    faces = np.asarray(m.faces, np.uint32)
    return dict(vert=np.asarray(m.vert, np.float32), faces=faces if faces.size else None, face_size=m.face_size,
                unlit=int(m.unlit), model=m.model_matrix().T.reshape(16))


def _c12(cam):
    return np.ascontiguousarray(cam.transform, np.float32).reshape(12)


def gpu_draw(cam, meshes, rgba0, depth0):
    import torch
    from volrend_b200 import draw_meshes
    img = torch.from_numpy(rgba0.copy()).cuda()
    dep = torch.from_numpy(depth0.copy()).cuda()
    draw_meshes(cam, meshes, img, dep)
    torch.cuda.synchronize()
    return img.cpu().numpy(), dep.cpu().numpy()


def oracle_draw(cam, meshes, rgba0, depth0):
    return mo.draw_meshes(cam.width, cam.height, cam.fx, cam.fy, _c12(cam), [_spec(m) for m in meshes if m.visible],
                          rgba0, depth0)


def check_vs_oracle(cam, meshes, rgba0=None, depth0=None):
    h, w = cam.height, cam.width
    rgba0 = np.full((h, w, 4), 7, np.uint8) if rgba0 is None else rgba0
    depth0 = np.full((h, w), 1e9, np.float32) if depth0 is None else depth0
    u, d = gpu_draw(cam, meshes, rgba0, depth0)
    uo, do, win = oracle_draw(cam, meshes, rgba0, depth0)
    cov = d != depth0
    assert np.array_equal(cov, win > 0), (cov.sum(), (win > 0).sum())
    assert np.all(np.abs(d - do) <= 1e-5 * np.abs(do))
    assert np.abs(u.astype(int) - uo.astype(int)).max() <= 1
    assert np.array_equal(u[~cov], rgba0[~cov])
    return u, d, cov


def _random_tris(rng, n, lit=True):
    from volrend_b200 import Mesh
    m = Mesh(3 * n, 0, 3, unlit=not lit)
    v = m.vert.reshape(-1, 9)
    ctr = rng.uniform(-1, 1, (n, 1, 3))
    v[:, :3] = (ctr + rng.uniform(-0.4, 0.4, (n, 3, 3))).reshape(-1, 3)
    v[:, 3:6] = rng.uniform(0, 1, (3 * n, 3))
    nn = rng.standard_normal((3 * n, 3))
    v[:, 6:9] = nn / np.linalg.norm(nn, axis=1, keepdims=True)
    return m


def _scenes():
    from volrend_b200 import Mesh
    rng = np.random.default_rng(5)
    cube = Mesh.Cube((0.9, 0.6, 0.3))
    cube.rotation[:] = (0.4, -0.3, 0.8)
    cube.scale = 1.3
    cube.translation[:] = (0.2, -0.1, 0.1)
    sph = Mesh.Sphere(9, 14, (0.3, 0.7, 0.9))
    sph.translation[:] = (0.6, 0.5, 0.3)
    sph.scale = 0.7
    helix = np.stack([np.cos(np.linspace(0, 9, 40)), np.sin(np.linspace(0, 9, 40)), np.linspace(-1, 1, 40)], 1)
    lines = Mesh.Lines(helix.reshape(-1), (1.0, 0.2, 0.2))
    line = Mesh.Line((-1.5, 0.3, -0.6), (1.4, -0.2, 0.9), (0.2, 1.0, 0.2))
    pts = Mesh.Points(rng.uniform(-1.2, 1.2, (60, 3)).reshape(-1), (0.1, 0.1, 1.0))
    tris = _random_tris(rng, 25)
    unlit = _random_tris(rng, 10, lit=False)
    # non-indexed lines and points with a model transform
    seg = Mesh(8, 0, 2, unlit=True)
    seg.vert.reshape(-1, 9)[:, :3] = rng.uniform(-1, 1, (8, 3))
    seg.vert.reshape(-1, 9)[:, 3:6] = 0.5
    seg.rotation[:] = (0, 0, 1.0)
    seg.translation[:] = (0.1, 0.2, 0.0)
    # degenerate (collinear), off-screen, empty, out-of-range indices
    degen = Mesh(3, 1, 3)
    degen.vert.reshape(-1, 9)[:, :3] = [(0, 0, 0), (0.5, 0.5, 0.5), (1, 1, 1)]
    degen.faces[:] = (0, 1, 2)
    off = Mesh.Cube()
    off.translation[:] = (0, 0, -40.0)
    empty = Mesh(0, 0, 3)
    bad = Mesh.Sphere(5, 6)
    f = bad.faces.copy()
    f[::7] = 10_000_000
    f[5] = bad.n_verts
    bad.faces = f
    return dict(cube=[cube], sphere=[sph], lines=[lines, line], points=[pts], tris=[tris], unlit=[unlit],
                nonindexed=[seg], degenerate=[degen, off, empty, bad],
                all=[cube, sph, lines, line, pts, tris, unlit, seg, degen, off, empty, bad])


@pytest.mark.parametrize("scene", ["cube", "sphere", "lines", "points", "tris", "unlit", "nonindexed", "degenerate",
                                   "all"])
def test_raster_vs_oracle(built, scene):
    meshes = _scenes()[scene]
    for eye in [(3.0, -2.2, 1.6), (-2.0, 2.8, -1.2)]:
        u, d, cov = check_vs_oracle(_cam(W, H, eye), meshes)
        if scene not in ("degenerate",):
            assert cov.sum() > 10
    if scene == "degenerate":
        # only the valid faces of the sphere with out-of-range indices draw
        assert cov.sum() > 0


def test_near_plane_straddler_and_depth_input(built):
    """A ground quad running under and behind the camera is clipped at the near plane; an existing depth
    buffer occludes fragments behind it (LESS), and a tie with it keeps the old pixel."""
    from volrend_b200 import Mesh
    cam = _cam(W, H, (0.0, -2.0, 0.5), target=(0.0, 0.0, 0.2))
    quad = Mesh(4, 2, 3)
    v = quad.vert.reshape(-1, 9)
    v[:, :3] = [(-3, -6, 0), (3, -6, 0), (3, 4, 0), (-3, 4, 0)]
    v[:, 3:6] = (0.8, 0.8, 0.2)
    v[:, 6:9] = (0, 0, 1)
    quad.faces[:] = (0, 1, 2, 0, 2, 3)
    u, d, cov = check_vs_oracle(cam, [quad])
    assert cov[-1].all() and not cov[0].any()        # reaches the bottom edge, stays below the horizon
    rng = np.random.default_rng(3)
    depth0 = rng.uniform(0.5, 4.0, (H, W)).astype(np.float32)
    depth0[::5] = d[::5]                            # exact ties: the old value must stay (LESS)
    u2, d2, cov2 = check_vs_oracle(cam, [quad], depth0=depth0)
    assert not cov2[::5].any() and cov2.sum() > 0


def test_ties_first_drawn_wins_and_determinism(built):
    from volrend_b200 import Mesh
    cam = _cam(W, H, (2.5, -2.0, 1.5))
    a, b = Mesh.Cube((1.0, 0.0, 0.0)), Mesh.Cube((0.0, 1.0, 0.0))
    a.unlit = b.unlit = True
    rgba0 = np.zeros((H, W, 4), np.uint8)
    d0 = np.full((H, W), 1e9, np.float32)
    u, d = gpu_draw(cam, [a, b], rgba0, d0)
    cov = d != d0
    assert cov.sum() > 100 and np.all(u[cov][:, :3] == (255, 0, 0))
    u_ba, _ = gpu_draw(cam, [b, a], rgba0, d0)
    assert np.all(u_ba[cov][:, :3] == (0, 255, 0))
    # a frame-filling triangle pair (raster_big path) plus many small ones: bit-identical on a second run
    big = Mesh(4, 2, 3)
    big.vert.reshape(-1, 9)[:, :3] = [(-30, -30, -0.2), (30, -30, -0.2), (30, 30, -0.2), (-30, 30, -0.2)]
    big.vert.reshape(-1, 9)[:, 3:9] = (0.5, 0.5, 0.5, 0, 0, 1)
    big.faces[:] = (0, 1, 2, 0, 2, 3)
    scene = [big, Mesh.Sphere(40, 60), a, b]
    r1 = gpu_draw(cam, scene, rgba0, d0)
    r2 = gpu_draw(cam, scene, rgba0, d0)
    assert np.array_equal(r1[0], r2[0]) and np.array_equal(r1[1].view(np.uint32), r2[1].view(np.uint32))
    assert (r1[1] != d0).all()
    check_vs_oracle(cam, [big, a])


def _renderer(st, tree, W, H, eye, bg, meshes):
    from volrend_b200 import VolumeRenderer, synth
    vr = VolumeRenderer()
    vr.resize(W, H)
    vr.camera.fx = vr.camera.fy = synth.focal_for(W)
    vr.camera.center = np.asarray(eye, np.float32)
    vr.camera.v_back = np.asarray(eye, np.float32) / np.linalg.norm(eye)
    vr.options.background_brightness = bg
    vr.set(tree)
    vr.meshes = meshes
    return vr


def _oracle_chain(st, vr, meshes, f_only=False):
    from oracle import binding as ob
    cam = vr.camera
    h, w = cam.height, cam.width
    bgb = round(min(max(vr.options.background_brightness, 0.0), 1.0) * 255)
    rgba0 = np.zeros((h, w, 4), np.uint8)
    rgba0[..., :3], rgba0[..., 3] = bgb, 255
    d0 = np.full((h, w), 1e9, np.float32)
    rgba, depth, win = oracle_draw(cam, meshes, rgba0, d0)
    t = ob.OracleTree.from_synth(st)
    oc = ob.make_camera(w, h, cam.fx, cam.fy, _c12(cam))
    opt = ob.make_options(background_brightness=vr.options.background_brightness,
                          basis_minmax=vr.options.basis_minmax)
    f, u, _ = ob.render(t, oc, opt, rgba_in=rgba, depth_in=depth)
    return f, u, rgba, depth, win


def _gpu_chain(vr):
    import torch
    from volrend_b200 import launch_renderer
    u = vr.render().cpu().numpy()
    # the same chain with the float tap of the composite march
    cam = vr.camera
    img = torch.zeros((cam.height, cam.width, 4), dtype=torch.uint8, device="cuda")
    bgb = round(min(max(vr.options.background_brightness, 0.0), 1.0) * 255)
    img[..., :3], img[..., 3] = bgb, 255
    dep = torch.full((cam.height, cam.width), 1e9, dtype=torch.float32, device="cuda")
    from volrend_b200 import draw_meshes
    draw_meshes(cam, vr.meshes, img, dep)
    fo = torch.zeros((cam.height, cam.width, 4), dtype=torch.float32, device="cuda")
    launch_renderer(vr._tree, cam, vr.options, img, dep, None, False, float_out=fo)
    torch.cuda.synchronize()
    return u, img.cpu().numpy(), fo.cpu().numpy()


@pytest.fixture(scope="module")
def sh4(small_trees):
    from volrend_b200 import N3Tree
    st = small_trees["sh4_d5"]
    return st, N3Tree.from_synth(st)


@pytest.mark.parametrize("bg", [1.0, 0.5])
def test_volume_renderer_cube_inside_volume(built, sh4, bg):
    from volrend_b200 import Mesh
    st, tree = sh4
    cube = Mesh.Cube((0.2, 0.9, 0.4))
    cube.scale = 0.5
    cube.rotation[:] = (0.3, 0.2, 0.5)
    eye = (3.2, -2.0, 1.4)
    vr = _renderer(st, tree, 64, 48, eye, bg, [cube])
    u, u_chain, f = _gpu_chain(vr)
    fo, uo, _, _, win = _oracle_chain(st, vr, [cube])
    assert (win > 0).sum() > 50
    assert np.array_equal(u, u_chain)
    assert np.abs(f - fo).max() <= 1e-4
    assert (u != uo).any(-1).sum() <= 2


@pytest.mark.parametrize("where", ["front", "behind"])
def test_volume_renderer_occlusion(built, sh4, where):
    from volrend_b200 import Mesh
    st, tree = sh4
    eye = np.array([2.8, -2.6, 1.5], np.float32)
    dirn = eye / np.linalg.norm(eye)
    quad = Mesh(4, 2, 3)
    v = quad.vert.reshape(-1, 9)
    v[:, :3] = [(-1, -1, 0), (1, -1, 0), (1, 1, 0), (-1, 1, 0)]
    v[:, 3:6] = (0.9, 0.3, 0.1)
    v[:, 6:9] = (0, 0, 1)
    quad.faces[:] = (0, 1, 2, 0, 2, 3)
    # turn the quad's +z towards the camera
    axis = np.cross((0, 0, 1), dirn)
    quad.rotation[:] = axis / np.linalg.norm(axis) * math.acos(float(dirn[2]))
    if where == "front":
        quad.translation[:] = dirn * 2.6
        quad.scale = 2.0
    else:
        quad.translation[:] = -dirn * 2.5
        quad.scale = 8.0
    vr = _renderer(st, tree, 56, 40, eye, 1.0, [quad])
    u, u_chain, f = _gpu_chain(vr)
    fo, uo, rgba, depth, win = _oracle_chain(st, vr, [quad])
    assert np.array_equal(u, u_chain)
    assert np.abs(f - fo).max() <= 2e-6
    assert (u != uo).any(-1).sum() <= 2
    if where == "front":
        assert (win > 0).all() and np.array_equal(u[..., :3], rgba[..., :3])   # the quad hides the volume
    else:
        assert (win > 0).all() and not np.array_equal(u[..., :3], rgba[..., :3])


def test_no_visible_mesh_keeps_offscreen_path(built, sh4):
    import torch
    from volrend_b200 import Mesh, launch_renderer
    st, tree = sh4
    for meshes in ([], [Mesh.Cube()]):
        for m in meshes:
            m.visible = False
        for bg in (1.0, 0.5, 0.3):
            vr = _renderer(st, tree, 40, 32, (3.0, -2.5, 1.2), bg, meshes)
            u = vr.render().cpu().numpy()
            ref = torch.zeros((32, 40, 4), dtype=torch.uint8, device="cuda")
            launch_renderer(tree, vr.camera, vr.options, ref, None, None, True)
            torch.cuda.synchronize()
            assert np.array_equal(u, ref.cpu().numpy())


def test_meshes_without_tree_and_resize(built):
    from volrend_b200 import Mesh, VolumeRenderer
    vr = VolumeRenderer()
    vr.resize(40, 30)
    vr.meshes = [Mesh.Cube()]
    u = vr.render().cpu().numpy()
    assert (u[..., :3] != 255).any(-1).sum() > 20 and np.all(u[..., 3] >= 76)
    vr.resize(24, 20)
    assert vr.render().shape == (20, 24, 4)


def test_invalid_arguments_report_einval(built):
    import torch
    from volrend_b200 import Mesh, VolrendError, _capi, draw_meshes
    cam = _cam(16, 12, (3, 0, 0))
    img = torch.zeros((12, 16, 4), dtype=torch.uint8, device="cuda")
    dep = torch.full((12, 16), 1e9, dtype=torch.float32, device="cuda")
    m = Mesh.Cube()
    m.face_size = 4
    with pytest.raises(VolrendError) as e:
        draw_meshes(cam, [m], img, dep)
    assert e.value.code == _capi.VR_EINVAL and "face_size" in str(e.value)
    with pytest.raises(VolrendError) as e:
        draw_meshes(cam, [Mesh.Cube()], None, dep)
    assert e.value.code == _capi.VR_EINVAL
    cam.width = 0
    with pytest.raises(VolrendError) as e:
        draw_meshes(cam, [Mesh.Cube()], img, dep)
    assert e.value.code == _capi.VR_EINVAL and "zero-size" in str(e.value)
