"""The references and helpers of tests/test_gpu_fit_shapes.py, checked without a GPU.

- The gradient and error references run on a window of the frame equal, bit for bit, the references run on the whole
  frame with dpix / err zero outside the window: the windowed references stand for the whole batch.
- On every node layout of tests/layout_cases.py the references' sums, mapped back through the slot map, are the
  canonical tree's bit for bit; free nodes, internal slots and the wide layout's extra columns get nothing.
- block_mode restates set_work's decision: checked against counts worked by hand.

The references run single-threaded here: each thread keeps its own sums, so only then is the order of every slot's
additions that of the pixels."""
import numpy as np
import pytest

import edge_cases as ec
import fit_shape_cases as fc
import golden_cases as gc
import layout_cases as lc
from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)


def _cams(views):
    from volrend_b200 import Camera
    out = []
    for W, H, fx, fy, pose in views:
        c = Camera(W, H, fx, fy)
        c.set_c2w(pose)
        out.append(c)
    return out


def _edge_views(name, st, which=("px", "inside")):
    return [ec.view(v, name, st)[:5] for v in which]


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


WINDOWED = ["mixed_sh9", "mixed_rgba", "lego_sh16"]


@pytest.mark.parametrize("name", WINDOWED)
def test_windowed_references_equal_full_frame(built, name):
    from oracle import binding as ob
    if name in gc.CASES:
        st, W, H, pose, _, _ = gc.build_case(name)
        from volrend_b200 import synth
        f = synth.focal_for(W)
        cams = _cams([(W, H, f, f, pose), (W, H, f, f, synth.nerf_synthetic_test_poses(8)[5])])
    else:
        st, _ = ec.edge_tree(name)
        cams = _cams(_edge_views(name, st))
    W, H = cams[0].width, cams[0].height
    ot = ob.OracleTree.from_synth(st)
    ocams = fc.oracle_cams(cams)
    wins = [(W // 2 - 7, H // 2 - 3, 11, 7), (W - 9, H - 6, 9, 6)]
    dpix = fc.windowed(2, W, H, wins, 4, -1.0, 1.0, seed=1)
    err = fc.windowed(2, W, H, wins, 0, 0.25, 2.0, seed=2)
    g_w, a_w = fc.oracle_grads(ot, ocams, {}, dpix, wins, nthreads=1)
    g_f, a_f = fc.oracle_grads(ot, ocams, {}, dpix, None, nthreads=1)
    assert np.array_equal(_bits(g_w), _bits(g_f)) and np.array_equal(_bits(a_w), _bits(a_f))
    assert (a_w > 0).any()
    s_w, b_w, _ = fc.oracle_error(ot, ocams, {}, err, wins, nthreads=1)
    s_f, b_f, _ = fc.oracle_error(ot, ocams, {}, err, None, nthreads=1)
    assert np.array_equal(_bits(s_w), _bits(s_f)) and np.array_equal(_bits(b_w), _bits(b_f))
    assert s_w.max() > 0


RELAID = [(t, lay) for t in ("mixed_sh9", "mixed_rgba", "root_mixed", "quant_mixed") for lay in lc.LAYOUTS]


def _to_canonical(r, canon_shape, a, cols):
    """Sums of the relaid tree ``a`` [new slots, columns] in the canonical tree's slots and columns."""
    out = np.zeros(canon_shape)
    m = r.slot_map
    out[m[m >= 0]] = a[m >= 0][:, cols] if a.ndim == 2 else a[m >= 0]
    return out


@pytest.mark.parametrize("name,layout", RELAID, ids=[f"{t}-{lay}" for t, lay in RELAID])
def test_relaid_references_equal_canonical(built, name, layout):
    """quant_mixed is relaid as its decoded tree (the references read decoded data): the wide layout needs that."""
    from oracle import binding as ob
    st, _ = ec.edge_tree(name)
    r = lc.relayout(st, layout, None, seed=7)
    cams = _cams(_edge_views(name, st))
    ocams = fc.oracle_cams(cams)
    W, H = cams[0].width, cams[0].height
    dpix = np.random.default_rng(3).uniform(-1, 1, (len(cams), H, W, 4)).astype(np.float32)
    err = np.random.default_rng(4).uniform(0.25, 2.0, (len(cams), H, W)).astype(np.float32)
    oc, orl = ob.OracleTree.from_synth(st), ob.OracleTree.from_synth(r.st)
    dd, ddr = st.data_dim, r.st.data_dim
    cols = list(range(dd - 1)) + [ddr - 1]            # the canonical columns in the relaid row
    g0, a0 = fc.oracle_grads(oc, ocams, {}, dpix, nthreads=1)
    g1, a1 = fc.oracle_grads(orl, ocams, {}, dpix, nthreads=1)
    assert np.abs(g0).max() > 0
    for x0, x1 in ((g0, g1), (a0, a1)):
        assert np.array_equal(_bits(_to_canonical(r, x0.shape, x1, cols)), _bits(x0)), layout
        assert not x1[r.slot_map < 0].any()                        # free and trailing nodes
        assert not x1[r.st.child.reshape(-1) != 0].any()           # internal slots
        assert not x1[:, [c for c in range(ddr) if c not in cols]].any()      # the wide layout's extra columns
    s0, b0, h0 = fc.oracle_error(oc, ocams, {}, err, nthreads=1)
    s1, b1, h1 = fc.oracle_error(orl, ocams, {}, err, nthreads=1)
    assert s0.max() > 0
    for x0, x1 in ((s0, s1), (b0, b1), (h0, h1)):
        assert np.array_equal(_to_canonical(r, x0.shape, x1, None), x0), layout
        assert not x1[r.slot_map < 0].any() and not x1[r.st.child.reshape(-1) != 0].any()


def test_block_mode_counts():
    # the finetune bench's step: 8 views of 800x800, SH16, 132 SMs: 200 x 100 tiles -> 50 x 25 blocks per group of
    # 4 views, 2 groups: 2 500 blocks >= 16 * 132 = 2 112
    assert fc.block_mode(8, 800, 800, 16, 132) == (True, 2500)
    # the refine CLI's default batch: 16 views, 4 groups
    assert fc.block_mode(16, 800, 800, 16, 132) == (True, 5000)
    # SH25: one view per block of 8 x 8 tiles: 25 x 13 (100 / 8 rounded up) blocks per view
    assert fc.block_mode(8, 800, 800, 25, 132) == (True, 2600)
    assert fc.block_mode(6, 800, 800, 25, 132) == (False, 1950)
    # tests/test_gpu_finetune.py's batches: 6 views of 48x40 (SH9): 12 x 5 tiles -> 3 x 2 blocks, 2 groups: 12 blocks;
    # 4 views of 64x64: 16 x 8 tiles -> 4 x 2 blocks, 1 group
    assert fc.block_mode(6, 48, 40, 9, 132) == (False, 12)
    assert fc.block_mode(4, 64, 64, 9, 132) == (False, 8)
    # tests/test_gpu_refine.py's orbit: 24 views of 64x48, SH16: 16 x 6 tiles -> 4 x 2 blocks, 6 groups
    assert fc.block_mode(24, 64, 48, 16, 132) == (False, 48)
    # RGBA / SH1 trees block like SH16; a single view never does; fewer views than a group does not
    assert fc.block_mode(8, 800, 800, -1, 132) == (True, 2500)
    assert fc.block_mode(1, 8000, 8000, 16, 132)[0] is False
    assert fc.block_mode(3, 4000, 4000, 16, 132)[0] is False
    assert fc.block_mode(1, 8000, 8000, 25, 132)[0] is False


@pytest.mark.parametrize("kbd", [16, 25, -1])
@pytest.mark.parametrize("num_sms", [132, 114, 78])
def test_block_batch_and_windows(kbd, num_sms):
    W, H = 150, 110
    n, small = fc.block_batch(kbd, num_sms, W, H)
    assert n % 4 and fc.block_mode(n, W, H, kbd, num_sms)[0]
    assert not any(fc.block_mode(m, W, H, kbd, num_sms)[0] for m in range(5, n) if m % 4)
    assert small >= 4 and not fc.block_mode(small, W, H, kbd, num_sms)[0]
    bpw, bph = fc.block_pixels(kbd)
    wins = fc.windows(n, W, H, kbd, seed=kbd + 1)
    for v, (x0, y0, w, h) in enumerate(wins):
        assert 0 <= x0 and x0 + w <= W and 0 <= y0 and y0 + h <= H
        if v % 5 == 4:
            assert (x0 + w, y0 + h) == (W, H)
        else:                                           # a block edge strictly inside the window in x and in y
            assert (x0 + w - 1) // bpw > x0 // bpw and (y0 + h - 1) // bph > y0 // bph, (v, x0, y0)
    assert len({w[:2] for w in wins}) > n // 3
    d = fc.windowed(n, W, H, wins, 4, -1, 1, seed=0)
    for v, (x0, y0, w, h) in enumerate(wins):
        inside = np.zeros((H, W), bool)
        inside[y0:y0 + h, x0:x0 + w] = True
        assert not d[v][~inside].any() and (d[v][inside] != 0).all()


def test_compact_tree_keeps_what_the_window_rays_meet(built):
    """The frustum cut of a tree renders the window pixels bit for bit as the whole tree (march oracle), and the
    gradient reference on it, mapped back, is the whole tree's."""
    from oracle import binding as ob
    from volrend_b200 import synth
    st = synth.make_tree("lego", depth=7, basis_dim=4, seed=9)
    W = H = 200
    f = synth.focal_for(W)
    cams = _cams([(W, H, f, f, p) for p in synth.nerf_synthetic_test_poses(8)[1:3]])
    wins = [(90, 95, 9, 7), (101, 87, 9, 7)]
    keep = fc.frustum_nodes(st, list(zip(cams, wins)))
    assert 1 < keep.sum() < st.capacity // 2
    small, slots = fc.compact(st, keep)
    ocams = fc.oracle_cams(cams)
    dpix = fc.windowed(2, W, H, wins, 4, -1, 1, seed=5)
    g0, a0 = fc.oracle_grads(ob.OracleTree.from_synth(st), ocams, {}, dpix, wins, nthreads=1)
    g1, a1 = fc.oracle_grads(ob.OracleTree.from_synth(small), ocams, {}, dpix, wins, nthreads=1)
    assert (a0 > 0).any()
    full = np.zeros_like(g0)
    full[slots] = g1
    assert np.array_equal(full, g0)
    for oc, win in zip(ocams, wins):
        f0, _, _ = ob.render(ob.OracleTree.from_synth(st), oc, ob.make_options(), tile=win, nthreads=1)
        f1, _, _ = ob.render(ob.OracleTree.from_synth(small), oc, ob.make_options(), tile=win, nthreads=1)
        assert np.array_equal(f0.view(np.uint32), f1.view(np.uint32))
