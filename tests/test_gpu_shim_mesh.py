"""`-m gpu`: the C++ shim's ``volrend::Mesh`` loaders and ``VolumeRenderer::render()`` with meshes, the probe cube and
the grid (volrend_b200/csrc/shim/mesh_b200.cpp, volrend_backend.cu), driven by oracle/_ref/shim_mesh: loaded meshes
byte for byte against the reference's goldens, and frames byte for byte against Python's ``VolumeRenderer.render()``
with the same tree, camera, options and meshes."""
import copy

import numpy as np
import pytest

import mesh_io_cases as mc
import shim_mesh_driver as sd
from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not sd.available(), reason="oracle/_ref/shim_mesh not built (needs the reference)")]

W, H = 96, 72


def test_loaders_match_goldens(built, tmp_path):
    """Every drawlist golden and every OBJ golden that needs normals (estimated on the device), from memory; one
    drawlist also from its file."""
    cases = []
    s = sd.Script(tmp_path)
    n = 0
    for fname in mc.golden_files():
        kind, data, vis, needs, want = mc.load_golden(fname)
        if kind != "drawlist" and not needs:
            continue
        src = s.file(data, ".npz" if kind == "drawlist" else ".obj")
        if kind == "drawlist":
            s.add("drawlistmem", src, int(vis))
        else:
            s.add("objmem", src)
        for i in range(len(want)):
            s.save(n + i)
        cases.append((fname, want))
        n += len(want)
    _, data, vis, _, dl_want = mc.load_golden("mesh_dl_presets.npz")
    s.add("drawlist", s.file(data, ".npz"), int(vis))
    for i in range(len(dl_want)):
        s.save(n + i)
    cases.append(("mesh_dl_presets.npz (file)", dl_want))
    got, _, _ = s.run()
    k = 0
    for fname, want in cases:
        assert mc.mismatches([sd.without_transform(g) for g in got[k:k + len(want)]], want) == [], fname
        k += len(want)


@pytest.fixture(scope="module")
def scene(small_trees, tmp_path_factory):
    """The SH16 depth-6 stand-in written as tree.npz, and a pose file of a NeRF-synthetic orbit view."""
    from volrend_b200 import synth
    d = tmp_path_factory.mktemp("shim_mesh_scene")
    path = str(d / "tree.npz")
    small_trees["sh16_d6"].save_npz(path)
    poses = synth.nerf_synthetic_test_poses(8)
    return path, synth.write_pose_files(poses, str(d), synth.focal_for(W))[2], float(synth.focal_for(W))


class Twin:
    """The same scene built twice: as driver commands and as Python objects."""

    def __init__(self, tmp_path, scene):
        from volrend_b200 import N3Tree, VolumeRenderer
        self.s = sd.Script(tmp_path)
        self.tree_path, pose, fx = scene
        self.s.add("renderer")
        self.s.add("tree", self.tree_path)
        self.s.add("set")
        self.s.add("size", W, H)
        self.s.add("fx", np.float32(fx))
        self.s.add("pose", pose)
        self.r = VolumeRenderer()
        self.tree = N3Tree(self.tree_path)
        self.r.set(self.tree)
        self.r.resize(W, H)
        self.r.camera.fx = self.r.camera.fy = float(np.float32(fx))
        self.r.camera._update = lambda *a, **k: None   # the pose comes from the driver's Camera::_update
        self.expected = []                             # Python frames, one per driver render

    def mesh(self, cmd, py_mesh):
        self.s.add(*cmd)
        self.r.meshes.append(py_mesh)
        return len(self.r.meshes) - 1

    def edit(self, i, field, *vals):
        self.s.add(field, i, *[np.float32(v) for v in vals])
        setattr(self.r.meshes[i], field, np.asarray(vals, np.float32) if len(vals) == 3 else float(np.float32(vals[0])))

    def render(self):
        """Queues a driver render; the Python frame is rendered after the driver ran, with its camera pose."""
        self.s.render()
        self.expected.append(self._snapshot())

    def _snapshot(self):
        """The Python state a driver render sees: meshes (uploaded now, so later host edits without update() do
        not reach them), options, size and tree."""
        for m in self.r.meshes:
            if m._vert_dev is None:
                m.update()
        meshes = [copy.copy(m) for m in self.r.meshes]
        opts = copy.deepcopy(self.r.options)
        size = (self.r.camera.width, self.r.camera.height)
        tree = self.r._tree
        return meshes, opts, size, tree

    def run(self):
        got, frames, out = self.s.run()
        return got, frames, out


def _python_frames(twin, frames):
    from volrend_b200 import VolumeRenderer
    out = []
    r = VolumeRenderer()
    r.camera._update = lambda *a, **k: None
    r.set(twin.tree)
    for (meshes, opts, (w, h), tree), (_, c2w) in zip(twin.expected, frames):
        r.resize(w, h)
        r.camera.fx, r.camera.fy = twin.r.camera.fx, twin.r.camera.fy
        r.camera.transform = np.ascontiguousarray(c2w, np.float32)
        if tree is None:
            r.clear()
        else:
            r.set(tree)
        r.options = opts
        r.meshes = meshes
        out.append(r.render().cpu().numpy().copy())
    return out


def _assert_frames(frames, want, labels):
    for k, ((got, _), w, label) in enumerate(zip(frames, want, labels)):
        g = got.reshape(w.shape)
        bad = int((g != w).any(-1).sum())
        assert bad == 0, f"frame {k} ({label}): {bad} pixels differ"


def test_renderer_matches_python(built, scene, tmp_path):
    from volrend_b200 import Mesh
    rng = np.random.default_rng(17)
    tw = Twin(tmp_path, scene)
    s = tw.s
    s.add("bg", np.float32(0.6))
    tw.r.options.background_brightness = float(np.float32(0.6))
    # drawlist cameras (sorted by name: cameras, one, traj), then lines, points, a rotated Cube and an unlit Sphere
    _, dl, _, _, _ = mc.load_golden("mesh_dl_cams100.npz")
    s.add("drawlistmem", s.file(dl, ".npz"), 1)
    tw.r.meshes.extend(Mesh.open_drawlist_mem(dl, True))
    pts = rng.uniform(-0.6, 0.6, 3 * 9).astype(np.float32)
    cloud = rng.uniform(-0.5, 0.5, 3 * 40).astype(np.float32)
    li = tw.mesh(("lines", s.f32(pts), 1.0, 0.2, 0.1), Mesh.Lines(pts, (1.0, 0.2, 0.1)))
    tw.mesh(("points", s.f32(cloud), 0.1, 0.9, 0.2), Mesh.Points(cloud, (0.1, 0.9, 0.2)))
    cube = tw.mesh(("cube", 0.8, 0.3, 0.9), Mesh.Cube((0.8, 0.3, 0.9)))
    tw.edit(cube, "rotation", 0.4, -0.9, 0.3)
    tw.edit(cube, "translation", 0.1, -0.2, 0.05)
    tw.edit(cube, "scale", 0.45)
    sph = tw.mesh(("sphere", 12, 20, 0.2, 0.6, 1.0), Mesh.Sphere(12, 20, (0.2, 0.6, 1.0)))
    tw.s.add("unlit", sph, 1)
    tw.r.meshes[sph].unlit = True
    tw.edit(sph, "translation", 0.35, 0.3, 0.2)
    tw.edit(sph, "scale", 0.2)
    tw.edit(sph, "rotation", 1e-4, 0.0, 2e-4)                    # below the 1e-3 threshold: identity rotation
    for i in (li, li + 1, cube, sph):
        s.add("update", i)                                        # the caller uploads presets, as in GL
    labels = ["meshes"]
    tw.render()
    # the probe cube (and its disc) with the probe in view
    s.add("probe", 1, np.float32(0.0), np.float32(0.0), np.float32(0.3))
    tw.r.options.enable_probe, tw.r.options.probe = True, [0.0, 0.0, float(np.float32(0.3))]
    tw.render()
    labels.append("probe")
    s.add("probe", 0, np.float32(0.0), np.float32(0.0), np.float32(0.3))
    tw.r.options.enable_probe = False
    # the grid at depths 2 -> 4 -> 2 (the cached grid is regenerated each time)
    for d in (2, 4, 2):
        s.add("grid", 1, d)
        tw.r.options.show_grid, tw.r.options.grid_max_depth = True, d
        tw.render()
        labels.append(f"grid {d}")
    s.add("grid", 0, 2)
    tw.r.options.show_grid = False
    # a vertex edit without update(): the upload is drawn, unchanged; then with update()
    k = 9 * 3 + 2                                                 # z of the Lines mesh's fourth vertex
    s.add("vert", li, k, np.float32(0.9))
    tw.r.meshes[li].vert[k] = np.float32(0.9)                     # the Python mesh keeps its device copy too
    tw.render()
    labels.append("edit, no update")
    s.add("update", li)
    tw.r.meshes[li] = copy.copy(tw.r.meshes[li])
    tw.r.meshes[li].update()
    tw.render()
    labels.append("edit, update")
    # a copy of the cube with its own transform, sharing the upload
    s.add("copy", cube)
    c = copy.copy(tw.r.meshes[cube])
    tw.r.meshes.append(c)
    cc = len(tw.r.meshes) - 1
    tw.edit(cc, "rotation", -0.2, 0.5, 1.4)
    tw.edit(cc, "translation", -0.35, 0.25, -0.1)
    tw.edit(cc, "scale", 0.25)
    tw.render()
    labels.append("copy")
    # resize between renders
    s.add("size", 64, 48)
    tw.r.resize(64, 48)
    tw.render()
    labels.append("resize")
    s.add("size", W, H)
    tw.r.resize(W, H)
    # meshes without a tree
    s.add("clear")
    tw.r.clear()
    tw.render()
    labels.append("clear")
    # only invisible meshes: the offscreen march
    s.add("set")
    tw.r.set(tw.tree)
    for i in range(len(tw.r.meshes)):
        s.add("visible", i, 0)
    drawn = [(i, copy.copy(m)) for i, m in enumerate(tw.r.meshes)]
    for i in range(len(tw.r.meshes)):
        tw.r.meshes[i] = copy.copy(tw.r.meshes[i])
        tw.r.meshes[i].visible = False
    tw.render()
    labels.append("invisible")
    saved = [s.save(i) for i, _ in drawn]
    got, frames, _ = tw.run()

    # 1. the model matrices first, so that a frame mismatch is localised
    for (i, m), j in zip(drawn, saved):
        assert got[j]["transform"].tobytes() == m.model_matrix().T.reshape(16).tobytes(), (i, m.name)
    # 2. the frames
    want = _python_frames(tw, frames)
    _assert_frames(frames, want, labels)
    # the probe, the grid, the vertex edit, the copy and hiding every mesh each change the frame
    f = [x[0].tobytes() for x in frames]
    for a, b in [(0, 1), (0, 2), (2, 3), (0, 6), (6, 7), (7, 10)]:
        assert f[a] != f[b], (labels[a], labels[b])
    assert f[5] == f[0] and f[4] == f[2]            # no update(): the frame is unchanged; grid 2 regenerated


def test_invisible_meshes_give_the_offscreen_frame(built, scene, tmp_path):
    """Only invisible meshes: the offscreen march, byte for byte the shim's launch_renderer frame."""
    from volrend_b200 import Camera, RenderOptions, launch_renderer
    import torch
    tw = Twin(tmp_path, scene)
    tw.s.add("cube", 1.0, 0.5, 0.2)
    tw.s.add("update", 0)
    tw.s.add("visible", 0, 0)
    tw.s.render()
    _, frames, _ = tw.run()
    rgba, c2w = frames[0]
    cam = Camera(W, H, tw.r.camera.fx, tw.r.camera.fy)
    cam.transform = np.ascontiguousarray(c2w, np.float32)
    opts = RenderOptions()
    opts.basis_minmax = [0, 15]
    img = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    launch_renderer(tw.tree, cam, opts, img, None, None, True)
    torch.cuda.synchronize()
    assert rgba.tobytes() == img.cpu().numpy().tobytes()
