"""Tree construction from voxel cells on the CPU: the host oracle on hand-worked trees, the oracle against the
canonical trees the generators write, ``leaf_cells`` on every layout, ``build_npz`` / ``grid_cells`` and the CLI's
argument errors (DESIGN.md section 21)."""
import ctypes as C

import numpy as np
import pytest

import edge_cases as ec
import golden_cases as gc
import layout_cases as lc
from oracle import build_oracle as bo
from volrend_b200 import synth
from volrend_b200.build import build_npz, grid_cells, leaf_cells, main

DD = 4


def _rows(*vals, dd=DD):
    return np.array([[v] * dd for v in vals], np.float16)


def _zero_tree(n, dd=DD):
    return np.zeros((n, 8), np.int32), np.zeros((n, 8, dd), np.float16)


def _check(cells, rows, child, data, merge=False):
    c, d = bo.build(cells, rows, merge)
    assert np.array_equal(c.reshape(-1, 8), child)
    assert np.array_equal(d.reshape(-1, 8, d.shape[-1]).view(np.uint16), data.view(np.uint16))


def test_empty_list_is_the_root_alone():
    for merge in (False, True):
        child, data = _zero_tree(1)
        _check(np.zeros((0, 4), np.int32), np.zeros((0, DD), np.float16), child, data, merge)


def test_one_cell_at_level_one_and_two():
    child, data = _zero_tree(1)
    data[0, 5] = 1.0                                     # (x, y, z) = (1, 0, 1): octant 4 + 1
    _check([[1, 1, 0, 1]], _rows(1.0), child, data)
    child, data = _zero_tree(2)                          # (2, 3, 0, 1) lies in level-1 cell (1, 0, 0): octant 4
    child[0, 4] = 1
    data[1, 5] = 2.0                                     # (3, 0, 1) & 1 = (1, 0, 1)
    _check([[2, 3, 0, 1]], _rows(2.0), child, data)


def test_mixed_levels_three_deep():
    cells = [[3, 7, 7, 7], [1, 0, 0, 0], [2, 2, 2, 2]]
    child, data = _zero_tree(3)
    child[0, 7] = 1                                      # level-1 cell (1, 1, 1)
    child[1, 7] = 1                                      # level-2 cell (3, 3, 3): node 2
    data[0, 0] = 1.0
    data[1, 0] = 2.0                                     # (2, 2, 2) is octant 0 of (1, 1, 1)
    data[2, 7] = 3.0
    _check(cells, _rows(3.0, 1.0, 2.0), child, data)


def test_breadth_first_morton_numbering():
    # level-2 cells under root octants 6 and 0: nodes 1 (octant 0) and 2 (octant 6), whatever the input order
    cells = [[2, 2, 3, 0], [2, 0, 1, 1]]
    child, data = _zero_tree(3)
    child[0, 0], child[0, 6] = 1, 2
    data[1, 3] = 5.0                                     # (0, 1, 1)
    data[2, 2] = 4.0                                     # (2, 3, 0) & 1 = (0, 1, 0)
    _check(cells, _rows(4.0, 5.0), child, data)
    _check(cells[::-1], _rows(5.0, 4.0), child, data)


def test_merge_cascade():
    # every level-2 cell with one row: the level-1 nodes collapse, the root stays
    g = np.stack(np.meshgrid(*[np.arange(4)] * 3, indexing="ij"), -1).reshape(-1, 3)
    cells = np.concatenate([np.full((64, 1), 2), g], 1)
    child, data = _zero_tree(1)
    data[:] = 1.5
    _check(cells, _rows(*[1.5] * 64), child, data, merge=True)
    # three levels: level-3 cells fill level-2 cell (0, 0, 0), whose 7 siblings are listed, all one row: level-1 cell
    # (0, 0, 0) becomes a leaf of the root with that row; without merge the tree keeps its 3 nodes
    sub = np.concatenate([np.full((8, 1), 3), np.array([[(o >> 2) & 1, (o >> 1) & 1, o & 1] for o in range(8)])], 1)
    sib = np.concatenate([np.full((7, 1), 2), np.array([[(o >> 2) & 1, (o >> 1) & 1, o & 1] for o in range(1, 8)])], 1)
    cells = np.concatenate([sub, sib])
    child, data = _zero_tree(1)
    data[0, 0] = -2.0
    _check(cells, _rows(*[-2.0] * 15), child, data, merge=True)
    c, _ = bo.build(cells, _rows(*[-2.0] * 15))
    assert c.shape[0] == 3
    # one different row stops the cascade at its node
    rows = _rows(*[-2.0] * 15)
    rows[3, 1] = 7.0
    c, _ = bo.build(cells, rows, merge=True)
    assert c.shape[0] == 3


def test_merge_compares_bits():
    cells = np.concatenate([np.full((8, 1), 2), np.array([[(o >> 2) & 1, (o >> 1) & 1, o & 1] for o in range(8)])], 1)
    neg0 = np.full((8, DD), 0x8000, np.uint16)
    c, d = bo.build(cells, neg0.view(np.float16), merge=True)      # eight -0 rows merge into a -0 leaf
    assert c.shape[0] == 1 and (d.view(np.uint16)[0, 0, 0, 0] == 0x8000).all()
    mixed = neg0.copy()
    mixed[5] = 0                                                   # -0 != +0
    c, _ = bo.build(cells, mixed.view(np.float16), merge=True)
    assert c.shape[0] == 2
    nan = np.full((8, DD), 0x7E00, np.uint16)
    c, _ = bo.build(cells, nan.view(np.float16), merge=True)        # NaNs compare as bits
    assert c.shape[0] == 1
    nan[2, 0] = 0x7E01
    c, _ = bo.build(cells, nan.view(np.float16), merge=True)
    assert c.shape[0] == 2


def test_merge_listed_zero_rows_equal_unlisted():
    cells = np.array([[3, 0, 0, 0], [3, 5, 1, 2], [2, 3, 3, 3], [1, 0, 1, 1]])
    rows = _rows(0.0, 2.0, 0.0, 0.0)
    a = bo.build(cells, rows, merge=True)
    keep = rows[:, 0] != 0
    b = bo.build(cells[keep], rows[keep], merge=True)
    assert all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(a, b))


@pytest.mark.parametrize("cells", [
    [[1, 0, 0, 0], [1, 0, 0, 0]],                 # duplicate
    [[1, 1, 1, 1], [3, 7, 6, 5]],                 # containment, coarse first
    [[3, 7, 6, 5], [1, 1, 1, 1]],                 # containment, fine first
    [[2, 0, 0, 0], [2, 1, 1, 1], [3, 0, 0, 1]],
    [[0, 0, 0, 0]], [[24, 0, 0, 0]], [[2, 4, 0, 0]], [[2, 0, -1, 0]], [[23, 0, 0, 1 << 23]],
])
def test_oracle_refusals(cells):
    with pytest.raises(ValueError):
        bo.build(cells, np.ones((len(cells), DD), np.float16))


def _is_canonical(st) -> bool:
    order = np.concatenate(lc.bfs_levels(st.child))
    internal = st.child.reshape(-1) != 0
    return (np.array_equal(order, np.arange(st.capacity)) and
            not st.data.reshape(st.capacity * 8, -1).view(np.uint16)[internal].any())


def canonical_trees():
    out = {f"edge_{n}": ec.edge_tree(n)[0] for n in ec.TREES if n != "quant_mixed"}
    out.update({f"golden_{n}": gc.build_case(n)[0] for n in gc.CASES})
    out["synth_lego_d4_rgba"] = synth.make_tree("lego", depth=4, fmt="RGBA", seed=3)
    out["synth_shell_full_d3"] = synth.make_tree("shell", depth=3, basis_dim=4, full=True, seed=2)
    return out


@pytest.mark.parametrize("name", sorted(canonical_trees()))
def test_oracle_rebuilds_canonical_trees(name):
    st = canonical_trees()[name]
    assert _is_canonical(st), name
    cells, rows = leaf_cells(st.child, st.data)
    rng = np.random.default_rng(7)
    perm = rng.permutation(cells.shape[0])
    child, data = bo.build(cells[perm], rows[perm])
    assert np.array_equal(child, st.child)
    assert np.array_equal(data.view(np.uint16), st.data.view(np.uint16))


@pytest.mark.parametrize("layout", lc.LAYOUTS)
def test_leaf_cells_of_relaid_trees(layout):
    st = ec.edge_tree("mixed_sh9")[0]
    r = lc.relayout(st, layout, seed=5)
    cells, rows = leaf_cells(r.st.child, r.st.data)
    child, data = bo.build(cells, rows)
    assert np.array_equal(child, st.child)
    if layout == "wide":   # the extra columns travel with the rows; internal slots read +0
        want = r.st.data.reshape(-1, r.st.data_dim).view(np.uint16).copy()
        want[st.child.reshape(-1) != 0] = 0
        assert np.array_equal(data.view(np.uint16).reshape(want.shape), want)
    else:
        assert np.array_equal(data.view(np.uint16), st.data.view(np.uint16))


def test_leaf_cells_refuses_what_prune_refuses():
    st = ec.edge_tree("mixed_sh9")[0]
    for bad, _ in lc.malformed(st).values():
        with pytest.raises(ValueError):
            leaf_cells(bad.child, bad.data)
    with pytest.raises(ValueError):
        leaf_cells(st.child, st.data.astype(np.float32))


def _oracle_backend(cells, rows, merge):
    return bo.build(np.asarray(cells), np.asarray(rows, np.float16), merge)


def test_build_npz_keys_and_dtypes():
    st = ec.edge_tree("mixed_sg9")[0]
    cells, rows = leaf_cells(st.child, st.data)
    d = build_npz(cells, rows, data_format="SG9", center=(0.5, -1.0, 2.0), radius=(2.0, 1.0, 4.0), extra=st.extra,
                  backend=_oracle_backend)
    assert sorted(d) == ["child", "data", "data_dim", "data_format", "extra_data", "invradius3", "offset"]
    ref = st.npz_dict()
    for k in ("child", "data", "data_dim", "data_format", "extra_data"):
        assert d[k].dtype == ref[k].dtype and d[k].shape == ref[k].shape, k
    assert np.array_equal(d["child"], st.child) and str(d["data_format"]) == "SG9"
    inv = np.array([0.25, 0.5, 0.125], np.float32)
    assert np.array_equal(d["invradius3"], inv)
    assert np.array_equal(d["offset"], (0.5 - np.array([0.5, -1.0, 2.0]) * inv).astype(np.float32))
    d = build_npz(cells[:0], np.zeros((0, 28), np.float16), data_format="SH9", backend=_oracle_backend)
    assert "extra_data" not in d and d["child"].shape == (1, 2, 2, 2)
    assert np.array_equal(d["offset"], np.full(3, 0.5, np.float32))
    assert np.array_equal(d["invradius3"], np.full(3, 0.5, np.float32))
    for kw in (dict(data_format="SG9"), dict(data_format="SH16"), dict(data_format="XY9"),
               dict(data_format="SH9", radius=0.0), dict(data_format="SH9", extra=st.extra),
               dict(data_format="SG9", extra=st.extra[:4])):
        kw.setdefault("extra", None)
        with pytest.raises(ValueError):
            build_npz(cells, rows, backend=_oracle_backend, **kw)


def test_grid_cells_small_grids():
    import torch
    rng = np.random.default_rng(3)
    g = rng.standard_normal((4, 4, 4, 5)).astype(np.float32)
    cells, rows = grid_cells(torch.from_numpy(g))
    assert cells.dtype == torch.int32 and rows.dtype == torch.float16 and cells.shape == (64, 4)
    c = cells.numpy()
    assert (c[:, 0] == 2).all()
    assert np.array_equal(rows.numpy().view(np.uint16), g[c[:, 1], c[:, 2], c[:, 3]].astype(np.float16).view(np.uint16))
    cells, rows = grid_cells(torch.from_numpy(g), sigma_thresh=0.25)
    keep = g[..., -1].astype(np.float16).astype(np.float32) > np.float32(0.25)
    assert cells.shape[0] == keep.sum() and (rows.numpy()[:, -1].astype(np.float32) > 0.25).all()
    child, data = bo.build(cells.numpy(), rows.numpy())
    assert child.shape[0] == 1 + len({tuple(v) for v in (cells.numpy()[:, 1:] >> 1).tolist()})
    for bad in (np.zeros((3, 3, 3, 2), np.float32), np.zeros((1, 1, 1, 2), np.float32), np.zeros((4, 4, 2, 2)),
                np.zeros((4, 4, 4, 0), np.float32)):
        with pytest.raises(ValueError):
            grid_cells(torch.from_numpy(bad))


@pytest.mark.parametrize("argv", [
    ["out.npz", "--format", "SH9"],                                       # no IN
    ["a.npy", "out.npz", "--format", "SH9", "--uniform", "3"],             # IN with --uniform
    ["out.npz", "--format", "SH9", "--uniform", "0"],
    ["out.npz", "--format", "SH9", "--uniform", "11"],
    ["out.npz", "--format", "SH9", "--uniform", "3", "--merge"],
    ["out.npz", "--format", "SH9", "--uniform", "3", "--sigma-thresh", "1"],
    ["a.npy", "out.npz", "--format", "SH9", "--init-sigma", "1"],
    ["a.npy", "out.npz", "--format", "XYZ"],
    ["a.npy", "out.npz", "--format", "SH0"],
    ["a.npy", "out.npz", "--format", "SH9", "--radius", "0"],
    ["a.npy", "out.npz", "--format", "SH9", "--radius", "nan"],
    ["a.npy", "out.npz", "--format", "SH9", "--center", "0", "inf", "0"],
    ["a.npy", "out.npz", "--format", "SH9", "--sigma-thresh", "nan"],
    ["a.npy", "out.txt", "--format", "SH9"],
    ["a.txt", "out.npz", "--format", "SH9"],
    ["a.npy", "out.npz"],                                                  # no --format
])
def test_cli_argument_errors(argv, tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    np.save("a.npy", np.zeros((2, 2, 2, 28), np.float32))
    with pytest.raises(SystemExit) as e:
        main(argv)
    assert e.value.code == 2
    assert not (tmp_path / "out.npz").exists()


def test_cli_npz_without_cells(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    np.savez("in.npz", rows=np.zeros((1, 4), np.float16))
    with pytest.raises(SystemExit) as e:
        main(["in.npz", "out.npz", "--format", "RGBA"])
    assert e.value.code == 2
    with pytest.raises(SystemExit):
        main(["in.npz", "out.npz", "--format", "RGBA", "--sigma-thresh", "1"])


def test_entry_point_without_a_device(built):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from volrend_b200 import _capi, lib
    L = lib()
    n = C.c_int64(-7)
    buf = C.create_string_buffer(64)
    assert L.vr_tree_build(None, None, 0, 4, 0, None, None, 0, C.byref(n), None) == _capi.VR_ENODEVICE
    assert L.vr_tree_build(buf, buf, 1, 4, 1, None, None, 0, C.byref(n), None) == _capi.VR_ENODEVICE
    # argument checks come first
    assert L.vr_tree_build(None, None, -1, 4, 0, None, None, 0, C.byref(n), None) == _capi.VR_EINVAL
    assert L.vr_tree_build(None, None, 0, 0, 0, None, None, 0, C.byref(n), None) == _capi.VR_EINVAL
    assert L.vr_tree_build(None, None, 1, 4, 0, None, None, 0, C.byref(n), None) == _capi.VR_EINVAL
    assert L.vr_tree_build(None, None, 0, 4, 2, None, None, 0, C.byref(n), None) == _capi.VR_EINVAL
    assert L.vr_tree_build(None, None, 0, 4, 0, buf, None, 8, C.byref(n), None) == _capi.VR_EINVAL
    assert L.vr_tree_build(None, None, 0, 4, 0, None, None, 0, None, None) == _capi.VR_EINVAL
    assert n.value == -7
