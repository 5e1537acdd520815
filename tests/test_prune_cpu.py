"""`-m "not gpu"`: pruning by weight (volrend_b200/prune.py) against the recursive restatement (oracle/prune_oracle.py)
on the edge-case trees and seeded random trees, hand cases, the npz key handling and the CLI's argument errors."""
import ctypes as C

import numpy as np
import pytest

import edge_cases as ec
from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)

THRESHS = [-np.inf, 0.0, 1e-3, 0.3]


def _weights(cap, seed, nan=True):
    rng = np.random.default_rng(seed)
    w = rng.uniform(-0.1, 1.0, cap * 8).astype(np.float32)
    w[rng.random(cap * 8) < 0.35] = -np.inf                   # never shaded
    w[rng.random(cap * 8) < 0.05] = 0.0
    w[rng.random(cap * 8) < 0.05] = -0.0
    if nan:
        w[rng.random(cap * 8) < 0.03] = np.nan
    return w


def _same(a, b):
    assert a[0].dtype == np.int32 and np.array_equal(a[0], b[0])
    assert np.array_equal(a[1].view(np.uint16), b[1].view(np.uint16))


def _random_tree(seed, depth=6):
    from volrend_b200 import synth
    return ec.mixed_tree(depth, 4, "SH", 500 + seed, p_refine=0.35)


@pytest.mark.parametrize("name", [n for n in ec.TREES if n != "quant_mixed"] + ["quant_mixed"])
def test_matches_recursive_oracle_on_edge_trees(name):
    from oracle import prune_oracle as po
    from volrend_b200 import prune_arrays
    st, _ = ec.edge_tree(name)
    w = _weights(st.capacity, hash(name) % 1000)
    for th in THRESHS:
        for col in (True, False):
            _same(prune_arrays(st.child, st.data, w, th, col), po.prune(st.child, st.data, w, th, col))


@pytest.mark.parametrize("seed", range(6))
def test_matches_recursive_oracle_on_random_trees(seed):
    from oracle import prune_oracle as po
    from volrend_b200 import prune_arrays
    st = _random_tree(seed)
    # weights concentrated on some subtrees, so that whole subtrees collapse
    w = _weights(st.capacity, seed)
    w[: st.capacity * 4] = -np.inf
    for th in THRESHS:
        for col in (True, False):
            _same(prune_arrays(st.child, st.data, w, th, col), po.prune(st.child, st.data, w, th, col))


def test_nothing_dropped_returns_identical_arrays():
    from volrend_b200 import prune_arrays
    st = _random_tree(1)
    w = np.ones(st.capacity * 8, np.float32)
    for col in (True, False):
        c, d = prune_arrays(st.child, st.data, w, 0.5, col)
        assert np.array_equal(c, st.child) and np.array_equal(d.view(np.uint16), st.data.view(np.uint16))


def test_everything_dropped_leaves_only_the_root():
    from volrend_b200 import prune_arrays
    st = _random_tree(2)
    c, d = prune_arrays(st.child, st.data, np.full(st.capacity * 8, -np.inf, np.float32), 0.0, True)
    assert c.shape == (1, 2, 2, 2) and not c.any()
    assert d.shape == (1, 2, 2, 2, st.data_dim) and not d.view(np.uint16).any()   # +0 everywhere
    c, d = prune_arrays(st.child, st.data, np.full(st.capacity * 8, np.nan, np.float32), 0.0, False)
    assert c.shape == st.child.shape and np.array_equal(c, st.child)               # no collapse: structure stays
    assert not d.view(np.uint16).reshape(-1, st.data_dim)[st.child.reshape(-1) == 0].any()


def test_dropped_chain_collapses_to_root():
    from volrend_b200 import prune_arrays
    st, _ = ec.edge_tree("chain22")
    w = np.full(st.capacity * 8, -np.inf, np.float32)
    c, d = prune_arrays(st.child, st.data, w, 1e-3, True)
    assert c.shape == (1, 2, 2, 2) and not c.any() and not d.view(np.uint16).any()
    # one kept leaf at the bottom keeps the whole chain
    leaves = np.nonzero(st.child.reshape(-1) == 0)[0]
    w[leaves[-1]] = 0.5
    c, _ = prune_arrays(st.child, st.data, w, 1e-3, True)
    assert c.shape[0] == st.capacity


def test_mixed_depths_and_order():
    """Root with leaves and subtrees of several depths: survivors keep their order, links are rewritten."""
    from oracle import prune_oracle as po
    from volrend_b200 import prune_arrays
    st, _ = ec.edge_tree("root_mixed")
    cap = st.capacity
    w = np.full(cap * 8, -np.inf, np.float32)
    # keep the leaves of every third node: whole subtrees in between go
    for n in range(0, cap, 3):
        w[n * 8:(n + 1) * 8] = 1.0
    c, d = prune_arrays(st.child, st.data, w, 0.5, True)
    _same((c, d), po.prune(st.child, st.data, w, 0.5, True))
    assert 1 < c.shape[0] < cap
    # every link points forward inside the array and every node but the root is linked exactly once
    flat = c.reshape(c.shape[0], 8)
    tgt = (np.arange(c.shape[0])[:, None] + flat)[flat != 0]
    assert (tgt > 0).all() and (tgt < c.shape[0]).all()
    assert np.array_equal(np.sort(tgt), np.arange(1, c.shape[0]))


def test_weight_rules():
    """weight < thresh and NaN drop a leaf; -0 counts as 0 against thresh 0."""
    from volrend_b200 import prune_arrays
    st, _ = ec.edge_tree("root_only")
    w = np.array([0.0, -0.0, np.nan, -np.inf, 1e-3, 9.99e-4, np.inf, -1.0], np.float32)
    _, d = prune_arrays(st.child, st.data, w, 0.0, False)
    zero = ~d.view(np.uint16).reshape(8, -1).any(axis=1)
    assert zero.tolist() == [False, False, True, True, False, False, False, True]
    _, d = prune_arrays(st.child, st.data, w, 1e-3, False)
    zero = ~d.view(np.uint16).reshape(8, -1).any(axis=1)
    assert zero.tolist() == [True, True, True, True, False, True, False, True]
    with pytest.raises(ValueError, match="NaN"):
        prune_arrays(st.child, st.data, w, np.nan)
    with pytest.raises(ValueError, match="weights"):
        prune_arrays(st.child, st.data, w[:7], 0.0)


def test_npz_keys_and_compressed_input():
    from volrend_b200 import prune_npz, synth
    st = _random_tree(3)
    z = st.npz_dict()
    z.update(parent_depth=np.zeros(3), geom_resize_fact=np.float32(1), n_free=np.int64(0), n_internal=np.int64(1),
             depth_limit=np.int64(6), custom=np.arange(4))
    out = prune_npz(z, _weights(st.capacity, 3), 1e-3)
    assert set(out) == {"child", "data", "data_dim", "data_format", "invradius3", "offset", "custom"}
    assert out["custom"] is z["custom"] and out["data"].dtype == np.float16 and out["child"].dtype == np.int32
    q = synth.quantise_tree(st, n_retain=1, seed=3)
    with pytest.raises(ValueError, match="prune .*first, then compress"):
        prune_npz(q, _weights(st.capacity, 3), 1e-3)


def test_cli_argument_errors(tmp_path, capsys):
    from volrend_b200 import prune, synth
    st = _random_tree(4)
    src = str(tmp_path / "t.npz")
    np.savez(src, **st.npz_dict())
    qsrc = str(tmp_path / "q.npz")
    np.savez(qsrc, **synth.quantise_tree(st, n_retain=1, seed=3))
    pose = str(tmp_path / "p.txt")
    np.savetxt(pose, np.eye(4))
    out = str(tmp_path / "o.npz")
    cases = [
        ([src, out], "required"),
        ([src, out, pose, "--thresh", "nan"], "NaN"),
        ([src, out, pose, "--width", "0"], "image size"),
        ([src, src, pose], "overwrite the input"),
        ([src, out, str(tmp_path / "missing.txt")], "does not exist"),
        ([qsrc, out, pose], "already compressed"),
        ([src, out, pose, "--batch", "0"], "--batch"),
    ]
    for argv, msg in cases:
        with pytest.raises(SystemExit) as e:
            prune.main(argv)
        assert e.value.code == 2, argv
        assert msg in capsys.readouterr().err, argv
    assert not (tmp_path / "o.npz").exists()


def test_pose_and_intrinsics_files(tmp_path):
    from volrend_b200 import prune
    p = tmp_path / "two.txt"
    m = np.arange(32, dtype=np.float32).reshape(2, 4, 4)
    p.write_text("\n".join(" ".join(str(v) for v in r) for r in m.reshape(8, 4)))
    got = prune.read_poses(str(p))
    assert len(got) == 2 and np.array_equal(np.stack(got), m)
    k = tmp_path / "k.txt"
    k.write_text("500 0 400 0\n0 510 400 0\n0 0 1 0\n0 0 0 1\n")
    assert prune.read_intrinsics(str(k)) == (500.0, 510.0)


def test_new_entry_points_without_a_device(built):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from volrend_b200 import _capi, lib
    L = lib()
    fake = C.create_string_buffer(4096)
    cam = _capi.vr_camera(8, 8, 10.0, 10.0)
    o = _capi.vr_options()
    L.vr_default_options(C.byref(o))
    d, qd, h = _capi.vr_tree_desc(), _capi.vr_tree_quant_desc(), C.c_void_p()
    buf = C.c_void_p(0x1000)
    assert L.vr_tree_create_ex(C.byref(d), 1, C.byref(h)) == _capi.VR_ENODEVICE
    assert b"no CPU fallback" in L.vr_last_error()
    assert L.vr_tree_create_ex(C.byref(d), 4, C.byref(h)) == _capi.VR_EINVAL
    assert L.vr_tree_create_quantized_ex(C.byref(qd), 1, C.byref(h)) == _capi.VR_ENODEVICE
    assert L.vr_tree_create_quantized_ex(None, 1, C.byref(h)) == _capi.VR_EINVAL
    t = C.addressof(fake)
    assert L.vr_tree_leaf_weights(t, C.byref(cam), 1, C.byref(o), None, buf, None, None, None) == _capi.VR_ENODEVICE
    assert L.vr_tree_leaf_weights(t, C.byref(cam), 1, C.byref(o), None, None, None, None, None) == _capi.VR_EINVAL
    assert L.vr_tree_leaf_weights(t, C.byref(cam), -1, C.byref(o), None, buf, None, None, None) == _capi.VR_EINVAL
    assert L.vr_tree_leaf_weights(None, None, 0, None, None, None, None, None, None) == _capi.VR_OK
    assert L.vr_tree_leaf_weights(None, C.byref(cam), 1, C.byref(o), None, buf, None, None, None) == _capi.VR_EINVAL
