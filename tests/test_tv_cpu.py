"""`-m "not gpu"`: the restatement of the total-variation prior between neighbouring leaves (oracle/tv_oracle.py,
DESIGN.md 20) on trees worked out by hand, its gradient against central differences of its energy, its neighbour
tables on the edge-case trees, their relayouts and refined trees, and the argument errors of the fitting CLI and of the
two C entry points without a device."""
import ctypes as C
import math

import numpy as np
import pytest

import edge_cases as ec
import layout_cases as lc
from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)
from oracle import tv_oracle as tvo


def _child(cap, links):
    """child [cap, 2, 2, 2] with the given {(node, octant): target node} links."""
    c = np.zeros((cap, 8), np.int32)
    for (n, o), t in links.items():
        c[n, o] = t - n
    return c.reshape(cap, 2, 2, 2)


def _fmt(st):
    fmt = st.data_format.rstrip("0123456789")
    return fmt, int(st.data_format[len(fmt):]) if fmt != "RGBA" else -1


def _check_definition(child, nbr):
    """Every entry is the leaf holding the forward corner; every other slot -1."""
    cells = {s: (d, i) for s, d, i in tvo.leaves(child)}
    cap = np.asarray(child).shape[0]
    for s in range(cap * 8):
        if s not in cells:
            assert (nbr[s] == -1).all(), s
            continue
        d, i = cells[s]
        for a in range(3):
            if i[a] + 1 == 1 << d:
                assert nbr[s, a] == -1, (s, a)
                continue
            n = int(nbr[s, a])
            assert n in cells, (s, a, n)
            dn, j = cells[n]
            p = list(i)
            p[a] += 1
            # the neighbour's cell holds the corner (i + e_a) 2^-d
            for b in range(3):
                lo = j[b] * 2.0 ** -dn
                assert lo <= p[b] * 2.0 ** -d < lo + 2.0 ** -dn, (s, a, n)


# ------------------------------------------------------------------------------------------- worked by hand
def test_two_levels_by_hand():
    child = _child(2, {(0, 7): 1})                      # the root's (1, 1, 1) octant split
    nbr = tvo.neighbors(child)
    assert nbr[0].tolist() == [4, 2, 1]                 # equal neighbours
    assert nbr[4].tolist() == [-1, 6, 5]                # +x face of the cube
    assert nbr[3].tolist() == [8, -1, -1]               # finer: the min-corner octant of node 1
    assert nbr[6].tolist() == [-1, -1, 8]
    assert nbr[5].tolist() == [-1, 8, -1]
    assert (nbr[7] == -1).all()                         # internal
    assert nbr[8].tolist() == [12, 10, 9]               # inside node 1
    assert nbr[12].tolist() == [-1, 14, 13]
    assert (nbr[15] == -1).all()                        # the (+x, +y, +z) corner leaf
    _check_definition(child, nbr)


def test_three_levels_by_hand():
    child = _child(3, {(0, 7): 1, (1, 0): 2})           # (1,1,1) of the root, then its (0,0,0)
    nbr = tvo.neighbors(child)
    assert nbr[3].tolist() == [16, -1, -1]              # finer by two levels: node 2's min-corner octant
    assert nbr[20].tolist() == [12, 22, 21]             # node 2's (1,0,0): coarser +x neighbour, node 1's (1,0,0)
    assert nbr[23].tolist() == [12, 10, 9]              # node 2's (1,1,1): three coarser neighbours
    assert nbr[0].tolist() == [4, 2, 1]
    assert (nbr[8] == -1).all()                         # node 1's (0,0,0) is internal now
    _check_definition(child, nbr)


def test_energy_by_hand():
    child = _child(1, {})
    v = np.zeros((8, 4))
    v[4, 3] = 2.0                                        # sigma of (1,0,0)
    cols, sig = tvo.columns(4, "RGBA", -1)
    E, g, A = tvo.tv(child, v, 0.5, 0.0, cols, sig)
    # slot 0: sqrt(eps + 4); slot 4: its +y, +z neighbours hold 0 -> sqrt(eps + 8); five other leaves sqrt(eps)
    want = 0.5 / 8 * (math.sqrt(1e-8 + 4) + math.sqrt(1e-8 + 8) + 6 * math.sqrt(1e-8))
    assert E == pytest.approx(want, rel=1e-12)
    assert g[:, :3].sum() == 0 and A[:, :3].sum() == 0   # colour weight 0: nothing
    # slot 0's term: +D / r to slot 4, -D / r to slot 0
    assert g[0, 3] == pytest.approx(-0.5 / 8 * 2 / math.sqrt(1e-8 + 4), rel=1e-12)


@pytest.mark.parametrize("seed", range(3))
def test_gradient_against_central_differences(seed):
    rng = np.random.default_rng(seed)
    st = ec.mixed_tree(3, 4, "SH", seed, p_refine=0.4)
    dd = st.data_dim
    v = rng.standard_normal((st.capacity * 8, dd))
    cols, sig = tvo.columns(dd, "SH", 4)
    nbr = tvo.neighbors(st.child)
    E, g, _ = tvo.tv(st.child, v, 0.7, 1.3, cols, sig, nbr)
    slots = [s for s, _, _ in tvo.leaves(st.child)]
    h = 1e-6
    for s in rng.choice(slots, 6, replace=False):
        for c in (sig, cols[0], cols[-1], 1):           # column 1: coefficient 1 of red, in the colour group
            vp, vm = v.copy(), v.copy()
            vp[s, c] += h
            vm[s, c] -= h
            num = (tvo.tv(st.child, vp, 0.7, 1.3, cols, sig, nbr)[0] - tvo.tv(st.child, vm, 0.7, 1.3, cols, sig, nbr)[0]) / (2 * h)
            assert g[s, c] == pytest.approx(num, rel=1e-5, abs=1e-8), (s, c)
    assert np.abs(g).max() > 0 and E > 0


def test_columns():
    assert tvo.columns(4, "RGBA", -1) == ([0, 1, 2], 3)
    assert tvo.columns(13, "SH", 4) == ([0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11], 12)
    assert tvo.columns(22, "SH", 7) == ([0, 7, 14], 21)                   # no kernel of its own: coefficient 0 only
    assert tvo.columns(16, "SH", 4) == (list(range(12)), 15)               # wider rows: sigma stays last


# ------------------------------------------------------------------------------------------- neighbour tables
@pytest.mark.parametrize("name", ec.TREES)
def test_neighbors_on_edge_trees(name):
    st, _ = ec.edge_tree(name)
    nbr = tvo.neighbors(st.child)
    _check_definition(st.child, nbr)
    assert np.array_equal(tvo.neighbors_levels(st.child), nbr)


LAYOUT_CASES = [(t, lay) for t in ("mixed_sh9", "mixed_rgba", "root_mixed", "chain22", "quant_mixed") for lay in lc.LAYOUTS
                if not (t == "quant_mixed" and lay == "wide")]


@pytest.mark.parametrize("name,layout", LAYOUT_CASES, ids=[f"{t}-{lay}" for t, lay in LAYOUT_CASES])
def test_neighbors_invariant_under_relayout(name, layout):
    st, npz = ec.edge_tree(name)
    r = lc.relayout(st, layout, npz, seed=11)
    base = tvo.neighbors(st.child)
    nbr = tvo.neighbors(r.st.child)
    assert np.array_equal(tvo.neighbors_levels(r.st.child), nbr)
    m = r.slot_map
    free = m < 0
    assert (nbr[free] == -1).all()                       # free nodes of the dirty layout
    mapped = np.where(nbr[~free] >= 0, m[np.maximum(nbr[~free], 0)], -1)
    assert np.array_equal(mapped, base[m[~free]])
    if layout in ("shuffle", "dirty", "wide"):
        fmt, basis = _fmt(st)
        cols, sig = tvo.columns(r.st.data_dim, fmt, basis)
        cols0, sig0 = tvo.columns(st.data_dim, fmt, basis)
        v = r.st.data.reshape(-1, r.st.data_dim).astype(np.float64)
        v0 = st.data.reshape(-1, st.data_dim).astype(np.float64)
        E, g, _ = tvo.tv(r.st.child, v, 1.0, 0.5, cols, sig, nbr)
        E0, g0, _ = tvo.tv(st.child, v0, 1.0, 0.5, cols0, sig0, base)
        assert E == pytest.approx(E0, rel=1e-12)
        assert np.allclose(g[~free][:, cols + [sig]], g0[m[~free]][:, cols0 + [sig0]], rtol=1e-12, atol=0)
        assert not g[free].any()


@pytest.mark.parametrize("levels", [22, 23])
def test_neighbors_on_deep_chains(levels):
    st = ec.varied_chain(levels)
    nbr = tvo.neighbors(st.child)
    _check_definition(st.child, nbr)
    assert max(d for _, d, _ in tvo.leaves(st.child)) == levels
    assert np.array_equal(tvo.neighbors_levels(st.child), nbr)


@pytest.mark.parametrize("seed", range(4))
def test_neighbors_on_refined_trees(seed):
    from volrend_b200 import refine_plan
    rng = np.random.default_rng(seed)
    st = ec.mixed_tree(4, 1, "SH", seed, p_refine=0.3)
    c2, _ = refine_plan(st.child, rng.random(st.capacity * 8).astype(np.float32), 0.4)
    nbr = tvo.neighbors(c2)
    _check_definition(c2, nbr)
    assert np.array_equal(tvo.neighbors_levels(c2), nbr)


# ------------------------------------------------------------------------------------------- CLI and C-ABI
def test_cli_argument_errors(tmp_path, capsys):
    import importlib
    finetune = importlib.import_module("volrend_b200.finetune")
    st = ec.mixed_tree(3, 4, "SH", 5)
    src = str(tmp_path / "t.npz")
    np.savez(src, **st.npz_dict())
    pose = str(tmp_path / "p.txt")
    np.savetxt(pose, np.vstack([np.eye(4), np.eye(4)]))
    npy = str(tmp_path / "t.npy")
    np.save(npy, np.zeros((2, 8, 6, 3), np.uint8))
    base = [src, str(tmp_path / "o.npz"), pose, "--targets", npy, "--width", "6", "--height", "8"]
    for flag in ("--tv-sigma", "--tv-color"):
        for bad in ("-1", "nan", "inf", "-0.001"):
            with pytest.raises(SystemExit) as e:
                finetune.main(base + [flag, bad])
            assert e.value.code == 2
            assert flag in capsys.readouterr().err
    assert not (tmp_path / "o.npz").exists()


def test_finetune_refuses_bad_weights():
    from volrend_b200 import finetune
    for kw in ({"tv_sigma": -1.0}, {"tv_color": float("nan")}, {"tv_color": float("inf")}):
        with pytest.raises(ValueError, match="tv_"):
            finetune(None, [None], [None], None, steps=1, lr=1e-2, batch=1, seed=0, **kw)


def test_entry_points_without_a_device(built):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from volrend_b200 import _capi, lib
    L = lib()
    fake = C.create_string_buffer(4096)
    t = C.addressof(fake)
    buf = C.c_void_p(0x1000)
    assert L.vr_tree_leaf_neighbors(t, buf, None) == _capi.VR_ENODEVICE
    assert b"no CPU fallback" in L.vr_last_error()
    assert L.vr_tree_leaf_tv(t, buf, buf, 1.0, 1.0, buf, buf, None) == _capi.VR_ENODEVICE
    assert b"no CPU fallback" in L.vr_last_error()
    assert L.vr_tree_leaf_neighbors(None, buf, None) == _capi.VR_EINVAL
    assert L.vr_tree_leaf_tv(None, buf, buf, 1.0, 1.0, buf, buf, None) == _capi.VR_EINVAL
