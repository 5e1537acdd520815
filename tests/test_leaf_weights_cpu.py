"""`-m "not gpu"`: the CPU restatement of the leaf-weights pass (oracle/weights_oracle.c, orc_leaf_weights) on one-ray
cases worked out by hand, and its alpha against orc_render's on every edge-case frame."""
import math

import numpy as np
import pytest

import edge_cases as ec
from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)


def _root_tree(sigmas):
    """Root-only SH1 tree, unit box ([0,1]^3 in world = tree coordinates): leaf o has sigma sigmas[o]."""
    from oracle import binding as ob
    child = np.zeros((1, 2, 2, 2), np.int32)
    data = np.zeros((1, 2, 2, 2, 4), np.float16)
    data.reshape(8, 4)[:, 3] = np.asarray(sigmas, np.float16)
    return ob.OracleTree(child, data, [0, 0, 0], [1, 1, 1], 4, "SH1")


AXIS = (1, 1, 1, 1)   # pixel (1, 1) of a 2x2 frame: screen2worlddir gives it the direction -back exactly


def _ray_along_x(y, z):
    """A 2x2 camera at x = -1 with back = -x, centred on (., y, z): pixel (1, 1)'s ray runs along +x."""
    from oracle import binding as ob
    c2w = [0, 0, -1, 0, 1, 0, -1, 0, 0, -1.0, y, z]   # right, up, back, centre (column-major)
    return ob.make_camera(2, 2, 1.0, 1.0, c2w)


def _run(tree, cam, **kw):
    from oracle import binding as ob
    from oracle import weights_binding as wb
    opt = ob.make_options(**kw)
    w, a, cnt = wb.leaf_weights(tree, cam, opt, tile=AXIS)
    f, _, c2 = ob.render(tree, cam, opt, tile=AXIS)
    assert cnt == c2
    assert np.array_equal(a.view(np.uint32), np.ascontiguousarray(f[..., 3]).view(np.uint32))
    return w, a[0, 0], cnt


def test_one_ray_two_leaves():
    # the ray y = z = 0.25 crosses octants 0 (x < 1/2) and 4 (x >= 1/2): two samples, each ~1/2 long
    s0, s1 = 2.0, 3.0
    tree = _root_tree([s0, 0, 0, 0, s1, 0, 0, 0])
    w, alpha, cnt = _run(tree, _ray_along_x(0.25, 0.25), step_size=0.0, stop_thresh=0.0)
    assert cnt["samples"] == 2 and cnt["shaded"] == 2
    # sample 1 at t ~ 1 + 1e-6 (x ~ 1e-6), exit at x = 1/2; sample 2 at x = 1/2, exit at x = 1 - 1e-6 (bbox)
    a0, a1 = math.exp(-0.5 * s0), math.exp(-0.5 * s1)
    assert w[0] == pytest.approx(1 - a0, rel=1e-5)
    assert w[4] == pytest.approx(a0 * (1 - a1), rel=1e-5)
    assert np.isneginf(np.delete(w, [0, 4])).all()
    assert alpha == pytest.approx(1 - a0 * a1, rel=1e-5)


def test_one_ray_thresholds_and_stop():
    tree = _root_tree([0.005, 0, 0, 0, 50.0, 0, 0, 0])
    cam = _ray_along_x(0.25, 0.25)
    w, alpha, _ = _run(tree, cam, step_size=0.0)                          # sigma 0.005 <= 1e-2: not shaded
    assert np.isneginf(w[0]) and w[4] == pytest.approx(1 - math.exp(-25.0), rel=1e-5)
    assert alpha == 1.0                                                   # T < stop_thresh: early stop
    w, _, _ = _run(tree, cam, step_size=0.0, sigma_thresh=0.0)
    assert w[0] == pytest.approx(1 - math.exp(-0.5 * float(np.float16(0.005))), rel=1e-4)   # sigma is stored as fp16
    # sigma_thresh < 0 shades sigma 0 leaves: weight T * (1 - exp(0)) = +0; and sigma < 0 gives negative weights
    tree = _root_tree([-1.0, 0, 0, 0, 0.0, 0, 0, 0])
    w, _, _ = _run(tree, cam, step_size=0.0, sigma_thresh=-2.0)
    assert w[0] == pytest.approx(1 - math.exp(0.5), rel=1e-5) and w[0] < 0
    assert w[4] == 0.0 and not np.signbit(w[4])


def test_one_ray_stops_before_the_second_leaf():
    tree = _root_tree([40.0, 0, 0, 0, 3.0, 0, 0, 0])
    w, alpha, cnt = _run(tree, _ray_along_x(0.25, 0.25), step_size=0.0)
    assert cnt["shaded"] == 1 and alpha == 1.0
    assert w[0] == pytest.approx(1 - math.exp(-20.0), rel=1e-6) and np.isneginf(w[4])


def test_accumulates_into_the_callers_buffer():
    from oracle import binding as ob
    from oracle import weights_binding as wb
    tree = _root_tree([2.0, 0, 0, 0, 3.0, 0, 0, 0])
    opt = ob.make_options(step_size=0.0, stop_thresh=0.0)
    buf = np.full(8, 0.5, np.float32)
    wb.leaf_weights(tree, _ray_along_x(0.25, 0.25), opt, tile=AXIS, weights=buf)
    assert buf[0] == pytest.approx(1 - math.exp(-1.0), rel=1e-5)          # 0.63 > 0.5
    assert buf[4] == 0.5                                                  # exp(-1) * (1 - exp(-1.5)) = 0.28 < 0.5


@pytest.mark.parametrize("tree_name", ec.TREES)
def test_alpha_equals_render_alpha_on_edge_frames(tree_name):
    from oracle import binding as ob
    from oracle import weights_binding as wb
    from volrend_b200 import synth
    st, _ = ec.edge_tree(tree_name)
    for fr in ec.frames_of(tree_name):
        t, W, H, fx, fy, pose, kw, comp = ec.frame(fr, st)
        if comp is not None:
            continue
        ot = ob.OracleTree.from_synth(st, ndc=ec.NDC.get(t))
        cam = ob.make_camera(W, H, fx, fy, synth.c2w_to_colmajor12(pose))
        opt = ob.make_options(**kw)
        w, a, cnt = wb.leaf_weights(ot, cam, opt)
        f, _, c2 = ob.render(ot, cam, ob.make_options(**dict(kw, render_depth=0)))
        assert np.array_equal(a.view(np.uint32), np.ascontiguousarray(f[..., 3]).view(np.uint32)), fr
        assert cnt == c2, fr
        leaf = st.child.reshape(-1) == 0
        assert not (~leaf & ~np.isneginf(w)).any(), fr                   # only leaf slots are shaded
        assert (np.isneginf(w).sum() < w.size) == (cnt["shaded"] > 0), fr
