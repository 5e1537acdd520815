"""`-m "not gpu"`: the float64 ray-cast reference of the mesh pass (oracle/raster_ref64.py) against analytic
answers and exact fill-rule ownership, and oracle/mesh_oracle.py (which the rasterizer matches bit for bit) against
the reference on every scene of tests/raster_ref64_cases.py.  The oracle repeats the kernel's float operations, so a
mistake in what the kernel computes is shared by both; the reference is written from the GL pipeline instead."""
import numpy as np
import pytest

from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)
from oracle import mesh_oracle as mo
from oracle import raster_ref64 as rr
import raster_ref64_cases as rc


def _oracle(s):
    rgba, depth, win = mo.draw_meshes(s.W, s.H, s.fx, s.fy, s.c2w, [rc.oracle_spec(m) for m in s.meshes],
                                      s.rgba0, s.depth0)
    return rgba, depth, np.where(win > 0, (win - 1) >> 3, -1)


def test_rectangle_covers_predicted_block():
    """A fronto-parallel unlit rectangle from window (10.3, 5.7) to (40.6, 30.2) covers pixels 10..40 x 6..29."""
    W, H, f, D = 64, 48, 50.0, 3.0
    a, b = (10.3, 5.7), (40.6, 30.2)
    quad = [(a[0], a[1]), (b[0], a[1]), (b[0], b[1]), (a[0], b[1])]
    prims = [rc.win_xyz([quad[k][0] for k in t], [quad[k][1] for k in t], D, f, W, H) for t in ((0, 1, 2), (0, 2, 3))]
    m = rc.soup(prims, colours=[(0.2, 0.4, 0.6)] * 6)
    s = rc.Scene(W, H, f, f, rc.IDENT, [m])
    ref = rc.reference(s)
    want = np.zeros((H, W), bool)
    want[6:30, 10:41] = True
    # the shared diagonal passes within the band of one pixel centre, which is then ambiguous
    assert np.array_equal(ref["covered"] | ref["ambiguous"], want) and ref["ambiguous"].sum() == 1
    assert np.allclose(ref["rgba"][ref["covered"]], (0.2, 0.4, 0.6, 1.0), atol=1e-7)


def test_head_on_plane_depth():
    """A plane z = -k seen head-on: the ray distance is k * |dir| / |dir_z| at every pixel."""
    W, H, fx, fy, k = 40, 30, 35.0, 22.0, 2.5
    quad = np.array([(-50, -50, -k), (50, -50, -k), (50, 50, -k), (-50, 50, -k)], np.float64)
    m = rc.soup([quad[[0, 1, 2]], quad[[0, 2, 3]]])
    s = rc.Scene(W, H, fx, fy, rc.IDENT, [m])
    ref = rc.reference(s)
    y, x = np.mgrid[0:H, 0:W] + 0.5
    d = np.stack([(x - W / 2) / fx, (H / 2 - y) / fy, -np.ones_like(x)], -1)
    want = k * np.linalg.norm(d, axis=-1)
    un = ~ref["ambiguous"]
    assert ref["covered"].all() and un.mean() > 0.95
    assert np.allclose(ref["depth"][un], want[un], rtol=1e-13)


def test_camera_position_of_scaled_rotation():
    """camPos = -transpose(mat3(V)) * V[3] is t / s^2 for a rotation scaled by s (mesh.cpp:376)."""
    c2w = rc.c2w_look((3.0, -2.0, 1.5), (0, 0, 0), scale=1.25)
    _, cam_pos = rr.camera_f64(c2w)
    assert np.allclose(cam_pos, np.asarray(c2w[9:12], np.float64) / 1.25 ** 2, rtol=1e-6)
    _, cam_pos = rr.camera_f64(rc.c2w_look((3.0, -2.0, 1.5), (0, 0, 0)))
    assert np.allclose(cam_pos, (3.0, -2.0, 1.5), rtol=1e-6)


def test_model_matrix_matches_mesh_model():
    from volrend_b200.mesh import model_matrix
    for rot, t, s in [((0.3, -1.2, 0.7), (1, -2, 3), 2.5), ((0.99e-3, 0, 0), (0, 0, 0), 0.5),
                      ((1.01e-3, 0, 0), (0.1, 0.2, 0.3), 1.0)]:
        assert np.allclose(rr.model_f64(rot, t, s), model_matrix(rot, t, s), atol=1e-6)
    assert np.array_equal(rr.model_f64((0.99e-3, 0, 0), (0, 0, 0), 1.0), np.eye(4))


@pytest.mark.parametrize("name", sorted(rc.EXACT))
def test_exact_ownership(name):
    """Window coordinates are exact here: the reference's unambiguous pixels, and every pixel of the oracle, follow
    the fill, line and point rules computed with fractions."""
    s = rc.EXACT[name](True)
    own = rc.exact_owner(s)
    assert (own >= 0).sum() > 50
    _, _, win = _oracle(s)
    assert np.array_equal(win, own)
    ref = rc.reference(s)
    un = ~ref["ambiguous"]
    assert np.array_equal(ref["covered"][un], own[un] >= 0)


@pytest.mark.parametrize("name", list(rc.SCENES))
def test_oracle_matches_reference(name):
    s = rc.scene(name, small=True)
    ref = rc.reference(s)
    rgba, depth, win = _oracle(s)
    frac = rc.compare(s, ref, rgba, depth, winner=win)
    print(f"{name}: ambiguous {frac:.4f} of {int((ref['covered'] | ref['ambiguous']).sum())} pixels")
    assert frac <= (s.amb_max if name in rc.ADVERSARIAL else 0.03)
    if name == "depth_zero":
        assert not ref["covered"].any() and np.array_equal(rgba, s.rgba0)
    elif name != "collinear":
        assert ref["covered"].sum() > 0
    if name == "invalid_vertices":
        bad = np.isin(win, s.extra["invalid"])
        assert not bad.any() and ref["covered"].sum() > 100
