"""`-m "not gpu"`: leaf splitting (volrend_b200/refine.py) against its plain restatement (oracle/refine_oracle.py), the
field and the render of refined trees under the query and march oracles, the CPU restatement of the leaf-error pass
(oracle/error_oracle.c, orc_leaf_error) on one-ray cases worked out by hand and against orc_leaf_weights, and the
file handling and CLI argument errors of refinement."""
import ctypes as C
import math

import numpy as np
import pytest

import edge_cases as ec
import golden_cases as gc
import layout_cases as lc
from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)
from oracle import refine_oracle as ro
from volrend_b200 import prune

# Largest |refined - original| of the march oracle's float RGBA over the golden cases, when splitting a quarter or all
# of the leaves (measured: at most 0.0059 with the default step of 1e-4 tree units, 0.021 for lego_sh4_stop0's step of
# 1e-3; mean at most 4.1e-4).  Each new cell face is one more exit at which the march overshoots by step_size.
RENDER_TOL = {"default": 0.01, "lego_sh4_stop0": 0.04}
RENDER_MEAN_TOL = 1e-3


def _check_plan(child, scores, fraction, max_depth=23, what=""):
    from volrend_b200 import refine_plan
    c2, src = refine_plan(child, scores, fraction, max_depth)
    oc, osrc = ro.refine(child, scores, fraction, max_depth)
    assert np.array_equal(np.asarray(c2, np.int64), oc.astype(np.int64)), what
    assert np.array_equal(src, np.asarray(osrc, np.int64)), what
    return c2, src


def _scores(cap, rng, special=True):
    s = rng.standard_normal(cap * 8).astype(np.float32)
    s[rng.random(cap * 8) < 0.2] = 0.5                                  # ties
    if special:
        k = rng.choice(cap * 8, size=min(cap * 8, 6), replace=False)
        s[k] = [np.nan, np.inf, -np.inf, 0.0, -0.0, -1.0][:k.size]
    return s


# ------------------------------------------------------------------------------------------- refine_plan vs oracle
@pytest.mark.parametrize("name", ec.TREES)
def test_plan_matches_oracle_on_edge_trees(name):
    st, _ = ec.edge_tree(name)
    rng = np.random.default_rng(hash(name) % 2**32)
    for frac in (0.0, 0.3, 1.0):
        for md in (1, 3, 23, 40):
            _check_plan(st.child, _scores(st.capacity, rng), frac, md, f"{name} {frac} {md}")


LAYOUT_CASES = [(t, lay) for t in ("mixed_sh9", "mixed_rgba", "root_mixed", "chain22") for lay in lc.LAYOUTS]


@pytest.mark.parametrize("name,layout", LAYOUT_CASES, ids=[f"{t}-{lay}" for t, lay in LAYOUT_CASES])
def test_plan_matches_oracle_on_layouts(name, layout):
    st, npz = ec.edge_tree(name)
    r = lc.relayout(st, layout, npz, seed=7)
    rng = np.random.default_rng(5)
    cap = r.st.capacity
    for frac in (0.1, 0.5, 1.0):
        c2, src = _check_plan(r.st.child, _scores(cap, rng), frac, 23, f"{name}-{layout} {frac}")
        # existing nodes (free ones of the dirty layout included) are untouched
        assert np.array_equal(np.asarray(c2)[:cap][np.asarray(r.st.child) != 0], r.st.child[r.st.child != 0])
        assert np.array_equal(src[:cap * 8], np.arange(cap * 8))
    if layout == "dirty":
        levels, _ = prune._structure(r.st.child)
        free = np.setdiff1d(np.arange(cap), np.concatenate(levels))
        c2, _ = _check_plan(r.st.child, np.ones(cap * 8, np.float32), 1.0)
        assert np.array_equal(np.asarray(c2)[free], r.st.child[free])


@pytest.mark.parametrize("seed", range(12))
def test_plan_matches_oracle_on_random_trees(seed):
    rng = np.random.default_rng(seed)
    st = ec.mixed_tree(int(rng.integers(2, 7)), 1, "SH", seed, p_refine=float(rng.uniform(0.1, 0.5)))
    s = _scores(st.capacity, rng)
    s[rng.random(s.size) < 0.3] = s[0] if np.isfinite(s[0]) and s[0] > 0 else 1.0     # many ties
    for frac in (0.0, float(rng.random()), 1 / 3, 1.0):
        for md in (2, int(rng.integers(1, 8)), 23):
            _check_plan(st.child, s, frac, md, f"seed {seed} {frac} {md}")


def test_plan_rules_directly():
    from volrend_b200 import refine_plan
    child = np.zeros((1, 2, 2, 2), np.int32)
    s = np.array([3, 1, 5, 5, 0, np.nan, -2, 4], np.float32)
    c2, src = refine_plan(child, s, 0.5)                      # candidates 0, 1, 2, 3, 7: ceil(2.5) = 3 -> 2, 3, 7
    assert c2.shape == (4, 2, 2, 2)
    assert c2.reshape(-1)[:8].tolist() == [0, 0, 1, 2, 0, 0, 0, 3]
    assert src.tolist() == list(range(8)) + [2] * 8 + [3] * 8 + [7] * 8
    same, ident = refine_plan(child, s, 0.0)                  # nothing chosen: the input itself
    assert same is child and np.array_equal(ident, np.arange(8))
    c1, _ = refine_plan(child, s, 0.01)                       # ceil(0.05) = 1: the highest, 5 at slot 2 before slot 3
    assert c1.reshape(-1)[:8].tolist() == [0, 0, 1, 0, 0, 0, 0, 0]
    for bad in (float("nan"), -0.1, 1.5):
        with pytest.raises(ValueError, match="fraction"):
            refine_plan(child, s, bad)
    with pytest.raises(ValueError, match="scores"):
        refine_plan(child, s[:7], 0.5)
    with pytest.raises(ValueError, match="max_depth"):
        refine_plan(child, s, 0.5, 0)
    assert refine_plan(child, s, 1.0, 1)[0] is child          # root slots are depth 1: none below max_depth 1


def test_plan_refuses_malformed_trees():
    from volrend_b200 import refine_plan
    st = ec.edge_tree("mixed_sh9")[0]
    for name, (bad, msg) in lc.malformed(st).items():
        with pytest.raises(ValueError, match=msg):
            refine_plan(bad.child, np.ones(bad.capacity * 8, np.float32), 0.5)


def test_chains_at_the_depth_cap():
    from volrend_b200 import refine_plan
    for levels in (22, 23):
        st = ec.varied_chain(levels)
        s = np.ones(levels * 8, np.float32)
        slots, depth, _ = lc.leaf_centres(st)
        for md in (23, 24, 100):
            c2, src = _check_plan(st.child, s, 1.0, md, f"chain{levels} {md}")
            split = np.unique(src[levels * 8:])
            assert np.array_equal(split, np.sort(slots[depth < 23]))    # the deepest leaves (level 23) never split
            _, d2, _ = lc.leaf_centres(_tree(st, c2, src))
            assert d2.max() == 23
        c2, src = refine_plan(st.child, s, 1.0, 22)
        assert lc.leaf_centres(_tree(st, c2, src))[1].max() == max(22, depth.max())


def test_capacity_refused():
    from volrend_b200 import refine
    refine.check_capacity(0xFFFFFFFF // 8)
    with pytest.raises(ValueError, match="slot map"):
        refine.check_capacity(0xFFFFFFFF // 8 + 1)


def test_capacity_refused_by_the_plan(monkeypatch):
    from volrend_b200 import refine, refine_plan
    st = ec.edge_tree("mixed_sh9")[0]
    monkeypatch.setattr(refine, "MAX_NODES", st.capacity + 2)
    refine_plan(st.child, np.ones(st.capacity * 8, np.float32), 1e-9)                  # one split: fits
    with pytest.raises(ValueError, match="slot map"):
        refine_plan(st.child, np.ones(st.capacity * 8, np.float32), 1.0)


# ------------------------------------------------------------------------------------------- the refined field
def _tree(st, child, src):
    from volrend_b200 import synth
    dd = st.data_dim
    return synth.SynthTree(child=np.asarray(child), data=st.data.reshape(-1, dd)[src].reshape(-1, 2, 2, 2, dd),
                           offset=st.offset, invradius3=st.invradius3, data_dim=dd, data_format=st.data_format,
                           depth=st.depth, extra=st.extra)


@pytest.mark.parametrize("name", ["mixed_sh16", "mixed_rgba", "root_only", "aniso", "chain22", "sigma_bits"])
def test_field_unchanged_at_every_new_leaf_centre(name):
    from oracle import query_oracle as qo
    from volrend_b200 import refine_plan
    st, _ = ec.edge_tree(name)
    rng = np.random.default_rng(3)
    c2, src = refine_plan(st.child, rng.random(st.capacity * 8).astype(np.float32), 0.5)
    r = _tree(st, c2, src)
    slots, depth, centres = lc.leaf_centres(r)
    pts = lc.centre_points(r, centres, depth)
    rows, _, _ = qo.query(st.child, st.data, st.offset, st.invradius3, pts)
    want = r.data.reshape(-1, st.data_dim)[slots]
    assert np.array_equal(rows.view(np.uint16), want.view(np.uint16))
    assert (src[slots] != slots).any()                                  # new leaves were queried


@pytest.mark.parametrize("name", [c for c in gc.CASES if c != "lego_sh9_composite"])
def test_render_close_to_the_original(name):
    from oracle import binding as ob
    from volrend_b200 import refine_plan, synth
    st, W, H, pose, kw, ndc = gc.build_case(name)
    cam = ob.make_camera(W, H, synth.focal_for(W), synth.focal_for(W), synth.c2w_to_colmajor12(pose))
    opt = ob.make_options(**kw)
    f0, _, c0 = ob.render(ob.OracleTree.from_synth(st, ndc=ndc), cam, opt)
    rng = np.random.default_rng(0)
    c2, src = refine_plan(st.child, rng.random(st.capacity * 8).astype(np.float32), 0.25)
    r = _tree(st, c2, src)
    f1, _, c1 = ob.render(ob.OracleTree.from_synth(r, ndc=ndc), cam, opt)
    d = np.abs(f1 - f0)
    assert d.max() <= RENDER_TOL.get(name, RENDER_TOL["default"]), (name, float(d.max()))
    assert d.mean() <= RENDER_MEAN_TOL, (name, float(d.mean()))
    assert c1["samples"] > c0["samples"]                                # the new cells are marched


# ------------------------------------------------------------------------------------------- orc_leaf_error
def _root_tree(sigmas):
    from oracle import binding as ob
    child = np.zeros((1, 2, 2, 2), np.int32)
    data = np.zeros((1, 2, 2, 2, 4), np.float16)
    data.reshape(8, 4)[:, 3] = np.asarray(sigmas, np.float16)
    return ob.OracleTree(child, data, [0, 0, 0], [1, 1, 1], 4, "SH1")


AXIS = (1, 1, 1, 1)   # pixel (1, 1) of a 2x2 frame: its ray runs along +x (test_leaf_weights_cpu.py)


def _ray_along_x(y, z):
    from oracle import binding as ob
    return ob.make_camera(2, 2, 1.0, 1.0, [0, 0, -1, 0, 1, 0, -1, 0, 0, -1.0, y, z])


def _err(tree, cam, e, **kw):
    from oracle import binding as ob
    from oracle import error_binding as eb
    return eb.leaf_error(tree, cam, ob.make_options(**kw), np.full((1, 1), e, np.float32), tile=AXIS)


def test_error_one_ray_two_leaves():
    s0, s1 = 2.0, 3.0
    tree = _root_tree([s0, 0, 0, 0, s1, 0, 0, 0])
    score, absum, hits, cnt = _err(tree, _ray_along_x(0.25, 0.25), 0.75, step_size=0.0, stop_thresh=0.0)
    a0, a1 = math.exp(-0.5 * s0), math.exp(-0.5 * s1)
    assert score[0] == pytest.approx(0.75 * (1 - a0), rel=1e-5)
    assert score[4] == pytest.approx(0.75 * a0 * (1 - a1), rel=1e-5)
    assert hits.tolist() == [1, 0, 0, 0, 1, 0, 0, 0] and not np.delete(score, [0, 4]).any()
    assert np.array_equal(absum, np.abs(score)) and cnt["shaded"] == 2
    neg, nabs, _, _ = _err(tree, _ray_along_x(0.25, 0.25), -2.0, step_size=0.0, stop_thresh=0.0)
    assert np.allclose(neg, score * (-2.0 / 0.75), rtol=1e-6) and np.allclose(nabs, -neg)


def test_error_thresholds_stop_and_zero():
    tree = _root_tree([40.0, 0, 0, 0, 3.0, 0, 0, 0])
    score, _, hits, _ = _err(tree, _ray_along_x(0.25, 0.25), 2.0, step_size=0.0)
    assert hits.tolist() == [1, 0, 0, 0, 0, 0, 0, 0]                   # stopped before the second leaf
    assert score[0] == pytest.approx(2.0 * (1 - math.exp(-20.0)), rel=1e-6)
    score, _, hits, cnt = _err(tree, _ray_along_x(0.25, 0.25), 0.0, step_size=0.0)
    assert hits[0] == 1 and score[0] == 0.0 and cnt["shaded"] == 1   # err 0: a term of 0, the same samples
    tree = _root_tree([0.005, 0, 0, 0, 0.0, 0, 0, 0])
    score, _, hits, _ = _err(tree, _ray_along_x(0.25, 0.25), 1.0, step_size=0.0)
    assert not hits.any()                                               # nothing above sigma_thresh 1e-2
    score, _, hits, _ = _err(tree, _ray_along_x(0.25, 0.25), 1.0, step_size=0.0, sigma_thresh=-1.0)
    assert hits[0] == 1 and hits[4] == 1 and score[4] == 0.0            # sigma 0: weight 0


@pytest.mark.parametrize("tree_name", ec.TREES)
def test_unit_error_is_the_sum_of_the_weights(tree_name):
    from oracle import binding as ob
    from oracle import error_binding as eb
    from oracle import weights_binding as wb
    from volrend_b200 import synth
    st, _ = ec.edge_tree(tree_name)
    for fr in ec.frames_of(tree_name)[:4]:
        t, W, H, fx, fy, pose, kw, comp = ec.frame(fr, st)
        if comp is not None:
            continue
        ot = ob.OracleTree.from_synth(st, ndc=ec.NDC.get(t))
        cam = ob.make_camera(W, H, fx, fy, synth.c2w_to_colmajor12(pose))
        opt = ob.make_options(**kw)
        w, _, wc = wb.leaf_weights(ot, cam, opt, want_alpha=False)
        score, absum, hits, ec_ = eb.leaf_error(ot, cam, opt, np.ones((H, W), np.float32))
        assert ec_ == wc, fr
        assert np.array_equal(hits > 0, ~np.isneginf(w)), fr            # the same slots
        f = hits > 0
        assert (score[f] >= w[f].astype(np.float64) - 1e-6 * np.maximum(1.0, absum[f])).all(), fr   # sum >= max
        assert not score[~f].any() and not absum[~f].any(), fr


# ------------------------------------------------------------------------------------------- npz and CLI
def _files(tmp_path):
    from volrend_b200 import synth
    st = ec.mixed_tree(3, 4, "SG", 5)
    src = str(tmp_path / "t.npz")
    d = st.npz_dict()
    d["parent_depth"] = np.zeros(3, np.int32)
    np.savez(src, **d)
    qsrc = str(tmp_path / "q.npz")
    np.savez(qsrc, **synth.quantise_tree(ec.mixed_tree(3, 4, "SH", 5), n_retain=1, seed=3))
    pose = str(tmp_path / "p.txt")
    np.savetxt(pose, np.vstack([np.eye(4), np.eye(4)]))
    return st, src, qsrc, pose


def test_refine_npz_keys_and_dtype(tmp_path):
    from volrend_b200 import refine_npz, refine_plan, synth
    st, src, qsrc, _ = _files(tmp_path)
    scores = np.random.default_rng(1).random(st.capacity * 8).astype(np.float32)
    with np.load(src) as z:
        out = refine_npz(z, scores, 0.5)
        assert set(out) == set(z.files) - {"parent_depth"} and "extra_data" in out
        for k in out:
            if k not in ("child", "data"):
                assert np.array_equal(out[k], z[k]), k
        c2, s2 = refine_plan(z["child"], scores, 0.5)
        assert np.array_equal(out["child"], c2) and out["child"].dtype == np.int32
        assert out["data"].dtype == np.float16
        assert np.array_equal(out["data"].reshape(-1, st.data_dim), st.data.reshape(-1, st.data_dim)[s2])
        none = refine_npz(z, scores, 0.0)
        assert np.array_equal(none["child"], z["child"]) and np.array_equal(none["data"], z["data"])
    d32 = dict(st.npz_dict(), data=st.data.astype(np.float32))
    assert refine_npz(d32, scores, 1.0)["data"].dtype == np.float32
    with np.load(qsrc) as q, pytest.raises(ValueError, match="compressed"):
        refine_npz(q, scores, 0.5)


def test_finetune_npz_with_a_refined_structure(tmp_path):
    from volrend_b200 import finetune_npz, refine_plan
    st, src, _, _ = _files(tmp_path)
    c2, s2 = refine_plan(st.child, np.ones(st.capacity * 8, np.float32), 0.5)
    new = st.data.reshape(-1, st.data_dim)[s2].reshape(-1, 2, 2, 2, st.data_dim).astype(np.float32)
    with np.load(src) as z:
        out = finetune_npz(z, new, child=c2)
        assert np.array_equal(out["child"], c2) and np.array_equal(out["data"], new.astype(np.float16))
        with pytest.raises(ValueError, match="shape"):
            finetune_npz(z, new)
        with pytest.raises(ValueError, match="shape"):
            finetune_npz(z, st.data, child=c2)


def test_cli_argument_errors(tmp_path, capsys):
    import importlib
    refine = importlib.import_module("volrend_b200.refine")
    finetune = importlib.import_module("volrend_b200.finetune")
    st, src, qsrc, pose = _files(tmp_path)
    out = str(tmp_path / "o.npz")
    npy = str(tmp_path / "t.npy")
    np.save(npy, np.zeros((2, 8, 6, 3), np.uint8))
    size = ["--width", "6", "--height", "8"]
    base = [src, out, pose, "--targets", npy] + size
    cases = [
        (refine, [src, out, pose, "--fraction", "0.5"] + size, "--targets"),
        (refine, base, "--fraction"),
        (refine, base + ["--fraction", "nan"], "--fraction"),
        (refine, base + ["--fraction", "1.5"], "--fraction"),
        (refine, base + ["--fraction", "-0.5"], "--fraction"),
        (refine, base + ["--fraction", "0.5", "--max-depth", "0"], "--max-depth"),
        (refine, base + ["--fraction", "0.5", "--batch", "0"], "--batch"),
        (refine, [src, src, pose, "--targets", npy, "--fraction", "0.5"] + size, "overwrite the input"),
        (refine, [src, out, pose, "--targets", str(tmp_path / "no.npy"), "--fraction", "0.5"] + size,
         "does not exist"),
        (refine, [src, out, pose, "--targets", npy, "--fraction", "0.5", "--width", "0"], "image size"),
        (refine, [src, out, pose, "--targets", npy, "--fraction", "0.5", "--width", "8", "--height", "6"],
         "the views 8x6"),
        (refine, [qsrc, out, pose, "--targets", npy, "--fraction", "0.5"] + size, "compressed"),
        (finetune, base + ["--refine-every", "-1"], "--refine-every"),
        (finetune, base + ["--refine-fraction", "nan"], "--refine-fraction"),
        (finetune, base + ["--refine-fraction", "2"], "--refine-fraction"),
        (finetune, base + ["--max-depth", "0"], "--max-depth"),
    ]
    for mod, argv, msg in cases:
        with pytest.raises(SystemExit) as e:
            mod.main(argv)
        assert e.value.code == 2, argv
        assert msg in capsys.readouterr().err, argv
    assert not (tmp_path / "o.npz").exists()


def test_leaf_error_without_a_device(built):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from volrend_b200 import _capi, lib
    L = lib()
    fake = C.create_string_buffer(4096)
    cam = _capi.vr_camera(8, 8, 10.0, 10.0)
    o = _capi.vr_options()
    L.vr_default_options(C.byref(o))
    buf = C.c_void_p(0x1000)
    t = C.addressof(fake)
    assert L.vr_tree_leaf_error(t, C.byref(cam), 1, C.byref(o), None, buf, buf, None, None) == _capi.VR_ENODEVICE
    assert b"no CPU fallback" in L.vr_last_error()
    assert L.vr_tree_leaf_error(t, C.byref(cam), 1, C.byref(o), None, None, buf, None, None) == _capi.VR_EINVAL
    assert L.vr_tree_leaf_error(t, C.byref(cam), 1, C.byref(o), None, buf, None, None, None) == _capi.VR_EINVAL
    assert L.vr_tree_leaf_error(t, C.byref(cam), -1, C.byref(o), None, buf, buf, None, None) == _capi.VR_EINVAL
    assert L.vr_tree_leaf_error(None, None, 0, None, None, None, None, None, None) == _capi.VR_OK
