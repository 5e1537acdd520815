"""`-m "not gpu"`: Mesh presets and model matrix against the reference's definitions (src/mesh.cpp:366-626),
the mesh oracle's fill rule and near-plane clipping, and the C-ABI's argument checks."""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import mesh_oracle as mo


def _cam_c2w(center, target, up=(0.0, 0.0, 1.0)):
    """Column-major 3x4 c2w looking from center at target (camera looks down its -z axis)."""
    c, t, u = (np.asarray(v, np.float64) for v in (center, target, up))
    back = c - t
    back /= np.linalg.norm(back)
    right = np.cross(u, back)
    right /= np.linalg.norm(right)
    upv = np.cross(back, right)
    return np.concatenate([right, upv, back, c]).astype(np.float32)


def _identity16():
    return np.eye(4, dtype=np.float32).T.reshape(16)


def test_cube_preset():
    from volrend_b200 import Mesh
    m = Mesh.Cube((0.1, 0.2, 0.3))
    v = m.vert.reshape(-1, 9)
    assert v.shape == (36, 9) and m.faces.size == 0 and m.face_size == 3 and not m.unlit and m.name == "Cube"
    assert np.allclose(v[:, 3:6], (0.1, 0.2, 0.3))
    # mesh.cpp:403-443: six faces of two triangles, in the order -z, +z, -y, +y, -x, +x; every vertex lies on
    # its face's plane and carries that face's outward normal
    normals = [(0, 0, -1), (0, 0, 1), (0, -1, 0), (0, 1, 0), (-1, 0, 0), (1, 0, 0)]
    for f, n in enumerate(normals):
        blk = v[6 * f:6 * f + 6]
        assert np.all(blk[:, 6:9] == n)
        axis = int(np.nonzero(n)[0][0])
        assert np.all(blk[:, axis] == 0.5 * n[axis])
        assert np.all(np.abs(blk[:, :3]) == 0.5)
    # first vertices of the reference's table
    assert list(v[0, :3]) == [-0.5, -0.5, -0.5] and list(v[1, :3]) == [0.5, 0.5, -0.5]
    assert list(v[25, :3]) == [-0.5, 0.5, 0.5] and list(v[35, :3]) == [0.5, 0.5, -0.5]


@pytest.mark.parametrize("rings,sectors", [(15, 30), (4, 7), (50, 64)])
def test_sphere_preset(rings, sectors):
    from volrend_b200 import Mesh
    m = Mesh.Sphere(rings, sectors)
    v = m.vert.reshape(-1, 9)
    assert v.shape[0] == rings * sectors and m.faces.size == (rings - 1) * sectors * 2 * 3
    assert np.allclose(np.linalg.norm(v[:, :3], axis=1), 1.0, atol=1e-6)
    assert np.array_equal(v[:, :3], v[:, 6:9])          # normal = position on the unit sphere
    assert np.allclose(v[:, 3:6], (1.0, 0.5, 0.2))
    # vertex (r, s) at polar angle r*pi/(rings-1) from the south pole, azimuth s*2pi/sectors
    r, s = rings // 2, sectors // 3
    th, ph = r * math.pi / (rings - 1), s * 2 * math.pi / sectors
    assert np.allclose(v[r * sectors + s, :3], (math.cos(ph) * math.sin(th), math.sin(ph) * math.sin(th),
                                                 -math.cos(th)), atol=1e-6)
    f = m.faces.reshape(-1, 3)
    assert f.max() < rings * sectors
    assert list(f[0]) == [1, 0, sectors] and list(f[1]) == [sectors, sectors + 1, 1]


def test_line_lines_points_presets():
    from volrend_b200 import Mesh
    ln = Mesh.Line((0, 0, 0), (1, 2, 3))
    assert ln.vert.size == 18 and list(ln.faces) == [0, 1] and ln.face_size == 2 and ln.unlit
    assert np.allclose(ln.vert.reshape(2, 9)[:, 3:], [[0.5, 0.5, 0.5, 0, 0, 1]] * 2)
    pts = np.arange(12, dtype=np.float32)
    ls = Mesh.Lines(pts)
    assert ls.vert.size == 36 and list(ls.faces) == [0, 1, 1, 2, 2, 3] and ls.face_size == 2 and ls.unlit
    assert np.array_equal(ls.vert.reshape(4, 9)[:, :3], pts.reshape(4, 3))
    p = Mesh.Points(pts, color=(1, 0, 0))
    assert p.vert.size == 36 and p.faces.size == 0 and p.face_size == 1 and p.unlit and p.name == "Points"
    assert np.allclose(p.vert.reshape(4, 9)[:, 3:], [[1, 0, 0, 0, 0, 1]] * 4)


@pytest.mark.parametrize("rot,scale,trans", [((0.3, -1.2, 0.7), 2.5, (1, -2, 3)), ((0, 0, 2.0), 0.5, (0, 0, 0)),
                                              ((-3.0, 0.1, 0.1), 1.0, (0.25, 0.5, -0.75))])
def test_model_matrix_matches_scipy(rot, scale, trans):
    from scipy.spatial.transform import Rotation
    from volrend_b200.mesh import model_matrix
    M = model_matrix(rot, trans, scale)
    want = np.eye(4)
    want[:3, :3] = Rotation.from_rotvec(rot).as_matrix() * scale
    want[:3, 3] = trans
    assert M.dtype == np.float32 and np.allclose(M, want, atol=1e-6)


def test_model_matrix_small_rotation_is_identity():
    from volrend_b200.mesh import model_matrix
    M = model_matrix((5e-4, 0, 0), (0, 0, 0), 2.0)          # mesh.cpp:369: angles below 1e-3 are ignored
    assert np.array_equal(M, np.diag([2, 2, 2, 1]).astype(np.float32))


def test_shared_edge_covered_exactly_once():
    """Top-left rule: two triangles sharing an edge (a quad, in several placements, with edges through
    pixel centres) cover every pixel of the quad exactly once."""
    W, H, f = 64, 48, 40.0
    c2w = _cam_c2w((0, 0, 5), (0, 0, 0), up=(0, 1, 0))
    rng = np.random.default_rng(1)
    for trial in range(12):
        if trial < 4:
            # axis-aligned in window space with corners exactly on pixel centres / edges
            x0, x1 = [(v - W / 2) * 5 / f for v in sorted(rng.integers(0, W, 2) + (0.5 if trial % 2 else 0.0))]
            y0, y1 = [(H / 2 - v) * 5 / f for v in sorted(rng.integers(0, H, 2) + (0.5 if trial % 2 else 0.0))]
            quad = [(x0, y0), (x1, y0), (x1, y1), (x0, y1)]
        else:
            ang = np.sort(rng.uniform(0, 2 * math.pi, 4))   # points on an ellipse in angle order: convex
            cx, cy, rx, ry = rng.uniform(-1, 1), rng.uniform(-1, 1), rng.uniform(0.5, 2.5), rng.uniform(0.5, 2)
            quad = [(cx + rx * math.cos(a), cy + ry * math.sin(a)) for a in ang]
        v = np.zeros((4, 9), np.float32)
        v[:, 0:2] = quad
        v[:, 3:6] = 1
        v[:, 8] = 1
        mesh = dict(vert=v.reshape(-1), faces=np.array([0, 1, 2, 0, 2, 3], np.uint32), face_size=3, unlit=1,
                    model=_identity16())
        cnt = mo.coverage(W, H, f, f, c2w, mesh)
        assert cnt.max() <= 1, trial
        # no gaps: every pixel inside the quad proper is covered, via the union of the two halves
        t1 = dict(mesh, faces=np.array([0, 1, 2], np.uint32))
        t2 = dict(mesh, faces=np.array([0, 2, 3], np.uint32))
        c1, c2 = mo.coverage(W, H, f, f, c2w, t1), mo.coverage(W, H, f, f, c2w, t2)
        assert np.array_equal(c1 + c2, cnt) and not (c1 & c2).any()


def test_near_plane_straddler_keeps_visible_part():
    """A triangle with one vertex behind the camera is clipped at d = 1e-3, not dropped or wrapped."""
    W, H, f = 64, 48, 40.0
    c2w = _cam_c2w((0, 0, 0), (0, 0, -1), up=(0, 1, 0))     # camera at the origin looking down -z
    v = np.zeros((3, 9), np.float32)
    v[:, :3] = [(-1.0, -0.5, -2.0), (1.0, -0.5, -2.0), (0.0, -0.5, 1.0)]   # third vertex behind the camera
    v[:, 3:6] = (0.2, 0.4, 0.6)
    v[:, 8] = 1
    mesh = dict(vert=v.reshape(-1), faces=None, face_size=3, unlit=1, model=_identity16())
    rgba0 = np.zeros((H, W, 4), np.uint8)
    d0 = np.full((H, W), 1e9, np.float32)
    rgba, depth, win = mo.draw_meshes(W, H, f, f, c2w, [mesh], rgba0, d0)
    cov = win > 0
    # a floor below the camera, widening towards the bottom of the frame; the top half stays empty
    assert cov[-1, 8:-8].all() and cov[-1].sum() > cov[36].sum() and not cov[: H // 2].any()
    # the far edge at z = -2 projects to row H/2 + 0.5*f/2 = 34: rows beyond it covered near the centre column
    assert cov[36:, W // 2].all() and not cov[:33, W // 2].any()
    # the clipped triangle is fanned into two sub-triangles (sequence numbers 1 and 2)
    assert set(np.unique(win[cov])) <= {1, 2} and len(np.unique(win[cov])) == 2
    assert np.all(depth[cov] < 1e9) and np.all(depth[cov] > 0.5)
    assert np.all(rgba[cov][:, :3] == np.rint(np.array([0.2, 0.4, 0.6]) * 255).astype(np.uint8))


def test_capi_rejects_invalid_arguments(built):
    from volrend_b200 import _capi, lib
    l = lib()
    cam = _capi.vr_camera(16, 8, 10.0, 10.0)
    for i, val in enumerate(_cam_c2w((0, 0, 3), (0, 0, 0), up=(0, 1, 0))):
        cam.c2w[i] = float(val)
    dummy = C.c_void_p(16)           # never dereferenced: validation happens before any device work

    def desc(**kw):
        d = _capi.vr_mesh_desc()
        d.vert_dev, d.faces_dev, d.n_verts, d.n_faces, d.face_size = 16, None, 3, 1, 3
        for k, v in kw.items():
            setattr(d, k, v)
        return d

    def call(meshes, n=None, c=cam, img=dummy, dep=dummy):
        arr = (_capi.vr_mesh_desc * max(len(meshes), 1))(*meshes)
        return l.vr_draw_meshes(C.byref(c) if c is not None else None, arr, len(meshes) if n is None else n,
                                img, dep, None)

    for d, word in [(desc(face_size=4), b"face_size"), (desc(face_size=0), b"face_size"),
                    (desc(n_verts=-1), b"negative"), (desc(n_faces=-2), b"negative"),
                    (desc(vert_dev=None), b"vert_dev")]:
        assert call([d]) == _capi.VR_EINVAL and word in l.vr_last_error()
    assert call([desc()], n=-1) == _capi.VR_EINVAL and b"negative" in l.vr_last_error()
    assert call([desc()], c=_capi.vr_camera(0, 8, 10.0, 10.0)) == _capi.VR_EINVAL and b"zero-size" in l.vr_last_error()
    assert call([desc()], c=_capi.vr_camera(16, 0, 10.0, 10.0)) == _capi.VR_EINVAL
    assert call([desc()], c=None) == _capi.VR_EINVAL
    assert call([desc()], img=None) == _capi.VR_EINVAL
    # a NULL vert_dev is fine when there are no vertices
    import torch
    if not torch.cuda.is_available():
        assert call([desc(vert_dev=None, n_verts=0)]) == _capi.VR_ENODEVICE
