"""Tree construction from voxel cells on an H100 (vr_tree_build, volrend_b200.build; DESIGN.md section 21): bit parity
with the host oracle, order independence, round trips of every test tree, the merge, dense grids and the refusals."""
import ctypes as C
import os

import numpy as np
import pytest

import edge_cases as ec
import golden_cases as gc
import layout_cases as lc
from oracle import build_oracle as bo
from volrend_b200 import synth

pytestmark = pytest.mark.gpu

OCT = np.array([[(o >> 2) & 1, (o >> 1) & 1, o & 1] for o in range(8)], np.int64)
SPECIALS = np.array([0x7E00, 0xFE01, 0x7C00, 0xFC00, 0x8000, 0x0001, 0x7BFF], np.uint16)


def _gpu(cells, rows, merge=False):
    from volrend_b200 import build_arrays
    c, d = build_arrays(cells, rows, merge=merge)
    return c.cpu().numpy(), d.cpu().numpy()


def _same(a, b, what=""):
    (c0, d0), (c1, d1) = a, b
    assert c0.shape == c1.shape and np.array_equal(c0, c1), what
    assert d0.shape == d1.shape and np.array_equal(d0.view(np.uint16), d1.view(np.uint16)), what


def _random_cells(level, k, rng):
    """k distinct cells of one level, in groups of siblings, so that merges happen."""
    parents = rng.choice(8 ** (level - 1), size=max(1, k // 8), replace=False) if level > 1 else np.zeros(1, np.int64)
    pc = np.stack([_demorton(p, level - 1) for p in parents]) if level > 1 else np.zeros((1, 3), np.int64)
    xyz = (pc[:, None, :] * 2 + OCT[None]).reshape(-1, 3)
    keep = rng.random(xyz.shape[0]) < 0.9
    xyz = xyz[keep]
    return np.concatenate([np.full((xyz.shape[0], 1), level), xyz], 1).astype(np.int32)


def _demorton(p, level):
    x = y = z = 0
    for b in range(level):
        o = (int(p) >> (3 * b)) & 7
        x |= ((o >> 2) & 1) << b
        y |= ((o >> 1) & 1) << b
        z |= (o & 1) << b
    return np.array([x, y, z], np.int64)


def _rows_for(cells, dd, rng, specials=False):
    """Rows from a small palette (with +0 and -0), constant over a cell's parent in half of the parents."""
    palette = rng.standard_normal((5, dd)).astype(np.float16)
    palette[0] = 0
    palette[1] = -0.0
    if specials:
        palette[2] = SPECIALS[rng.integers(0, len(SPECIALS), dd)].view(np.float16)
    parent = cells[:, 1:] >> 1
    h = (parent[:, 0] * 73856093 ^ parent[:, 1] * 19349663 ^ parent[:, 2] * 83492791) & 0xffff
    pick = np.where(h % 2 == 0, h % 5, rng.integers(0, 5, cells.shape[0]))
    return palette[pick]


def parity_cases():
    rng = np.random.default_rng(11)
    out = {}
    for L in range(1, 11):
        cells = _random_cells(L, min(8 ** L, 400), rng)
        out[f"level{L}"] = (cells, _rows_for(cells, 28, rng))
    for i, name in enumerate(("mixed_sh9", "mixed_rgba", "root_mixed")):
        st = ec.edge_tree(name)[0]
        cells, rows = _leaf_cells(st)
        keep = rng.random(cells.shape[0]) < 0.7
        out[f"mixed_{name}"] = (cells[keep], rows[keep])
    g = np.stack(np.meshgrid(*[np.arange(8)] * 3, indexing="ij"), -1).reshape(-1, 3)
    cells = np.concatenate([np.full((512, 1), 3), g], 1).astype(np.int32)
    out["dense8"] = (cells, _rows_for(cells, 4, rng))
    out["empty"] = (np.zeros((0, 4), np.int32), np.zeros((0, 28), np.float16))
    out["one_level23"] = (np.array([[23, 8388607, 12345, 4000000]], np.int32), rng.standard_normal((1, 4)).astype(np.float16))
    for name in ("chain22", "chain23"):
        out[name] = _leaf_cells(ec.edge_tree(name)[0])
    for dd in (4, 28, 49, 76, 31):           # 31: a padded SH9 row
        cells = _random_cells(5, 300, rng)
        out[f"dd{dd}"] = (cells, _rows_for(cells, dd, rng))
    cells = _random_cells(4, 300, rng)
    out["specials"] = (cells, _rows_for(cells, 13, rng, specials=True))
    return out


def _leaf_cells(st):
    from volrend_b200 import leaf_cells
    return leaf_cells(st.child, st.data)


CASES = sorted(parity_cases())


@pytest.fixture(scope="module")
def cases():
    return parity_cases()


@pytest.mark.parametrize("merge", [False, True])
@pytest.mark.parametrize("name", CASES)
def test_oracle_parity(built, cases, name, merge):
    cells, rows = cases[name]
    _same(_gpu(cells, rows, merge), bo.build(cells, rows, merge), (name, merge))


@pytest.mark.parametrize("merge", [False, True])
def test_order_independence_and_repeats(built, cases, merge):
    rng = np.random.default_rng(5)
    for name in ("level8", "mixed_mixed_sh9", "dense8", "specials"):
        cells, rows = cases[name]
        ref = _gpu(cells, rows, merge)
        p = rng.permutation(cells.shape[0])
        _same(_gpu(cells[p], rows[p], merge), ref, name)
        for _ in range(2):
            _same(_gpu(cells, rows, merge), ref, name)


# ------------------------------------------------------------------------------------------------------ round trip
def round_trip_trees():
    """name -> (tree to read the leaves from, its canonical form, NDC (width, height, focal) or None)."""
    out = {}
    for n in gc.CASES:
        st, _, _, _, _, ndc = gc.build_case(n)
        out[f"golden_{n}"] = (st, st, ndc)
    for n in ec.TREES:
        st, npz = ec.edge_tree(n)
        canon = _zero_internal(st)
        out[f"edge_{n}"] = (st, canon, ec.NDC.get(n))
    base = ec.edge_tree("mixed_sh16")[0]
    for layout in lc.LAYOUTS:
        r = lc.relayout(base, layout, seed=3)
        canon = _zero_internal(r.st) if layout == "wide" else base
        out[f"relaid_{layout}"] = (r.st, canon, None)
    st, npz = gc.ref_frame_tree("quant16")
    from volrend_b200 import N3Tree
    host = N3Tree(gpu_decode=False)
    host.load_npz(npz)
    dec = synth.SynthTree(child=st.child, data=host.data_.copy(), offset=st.offset, invradius3=st.invradius3,
                          data_dim=st.data_dim, data_format=st.data_format, depth=st.depth)
    out["quant16_decoded"] = (dec, _zero_internal(dec), None)
    return out


def _zero_internal(st):
    from dataclasses import replace
    d = st.data.reshape(st.capacity * 8, -1).view(np.uint16).copy()
    d[st.child.reshape(-1) != 0] = 0
    return replace(st, data=d.view(np.float16).reshape(st.data.shape), meta={})


ROUND = sorted(round_trip_trees())


def _render(st, child, data, ndc, parity, W=64, H=48):
    import torch
    from volrend_b200 import Camera, N3Tree, RenderOptions, launch_renderer
    t = N3Tree()
    t.load_npz(dict(child=child, data=data, offset=st.offset, invradius3=st.invradius3,
                    data_dim=np.int64(data.shape[-1]), data_format=np.array(st.data_format),
                    **({"extra_data": st.extra} if st.extra is not None else {})))
    if ndc is not None:
        t.use_ndc = True
        t.ndc_width, t.ndc_height, t.ndc_focal = ndc
    os.environ["VR_WIDE_PARITY"] = str(parity)
    try:
        t.load_cuda()
    finally:
        os.environ.pop("VR_WIDE_PARITY", None)
    assert t.info()["wide_parity"] == parity
    cam = Camera(W, H, synth.focal_for(W), synth.focal_for(W))
    cam.set_c2w(synth.nerf_synthetic_test_poses(8)[3] if ndc is None else np.eye(4, dtype=np.float32))
    img = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    fo = torch.zeros((H, W, 4), dtype=torch.float32, device="cuda")
    launch_renderer(t, cam, RenderOptions(), img, None, None, True, float_out=fo)
    torch.cuda.synchronize()
    return img.cpu().numpy(), fo.cpu().numpy()


@pytest.mark.parametrize("name", ROUND)
def test_round_trip(built, name):
    src, canon, ndc = round_trip_trees()[name]
    cells, rows = _leaf_cells(src)
    got = _gpu(cells, rows)
    _same(got, (canon.child, canon.data), name)
    for parity in (0, 1):
        a = _render(canon, canon.child, canon.data, ndc, parity)
        b = _render(canon, got[0], got[1], ndc, parity)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32)), (name, parity)


def test_round_trip_bench_tree(built):
    st = synth.make_tree("lego", depth=10, basis_dim=16, seed=0)
    cells, rows = _leaf_cells(st)
    _same(_gpu(cells, rows), (st.child, st.data), "bench tree")


@pytest.mark.parametrize("name", ["golden_lego_sh16", "golden_lego_rgba", "golden_lego_sg9_rot", "golden_lego_asg4"])
def test_written_npz_renders_through_every_loader(built, tmp_path, name):
    """The CLI's npz, written from the tree's leaf cells, opens in N3Tree and (where oracle/_ref is built) in the
    reference loader, and both render it exactly as the source tree renders."""
    import torch
    from oracle import ref_binding as rb
    from volrend_b200 import Camera, N3Tree, RenderOptions, launch_renderer
    from volrend_b200.build import main
    st = round_trip_trees()[name][1]
    cells, rows = _leaf_cells(st)
    np.savez(tmp_path / "cells.npz", cells=cells, rows=rows)
    inv = st.invradius3.astype(np.float64)
    radius, center = 0.5 / inv, (0.5 - st.offset.astype(np.float64)) / inv
    argv = [str(tmp_path / "cells.npz"), str(tmp_path / "tree.npz"), "--format", st.data_format,
            "--radius", repr(float(radius[0])), "--center", *[repr(float(c)) for c in center]]
    if st.extra is not None:
        np.save(tmp_path / "extra.npy", st.extra)
        argv += ["--extra", str(tmp_path / "extra.npy")]
    assert main(argv) == 0
    path = str(tmp_path / "tree.npz")
    with np.load(path) as z:
        assert np.array_equal(z["offset"], st.offset) and np.array_equal(z["invradius3"], st.invradius3)
    frames = []
    for tree in (N3Tree.from_synth(st), N3Tree(path)):
        f = []
        for i in (0, 37):
            cam = Camera(96, 72, synth.focal_for(96), synth.focal_for(96))
            cam.set_c2w(synth.nerf_synthetic_test_poses(200)[i])
            img = torch.zeros((72, 96, 4), dtype=torch.uint8, device="cuda")
            fo = torch.zeros((72, 96, 4), dtype=torch.float32, device="cuda")
            launch_renderer(tree, cam, RenderOptions(), img, None, None, True, float_out=fo)
            torch.cuda.synchronize()
            f.append((cam, fo.cpu().numpy(), img.cpu().numpy()))
        frames.append(f)
        tree.free_cuda()
    assert any(fo.any() for _, fo, _ in frames[0])
    for (_, f0, u0), (_, f1, u1) in zip(*frames):
        assert np.array_equal(f0.view(np.uint32), f1.view(np.uint32)) and np.array_equal(u0, u1), name
    if rb.available():
        rt = rb.RefTree(path)
        try:
            for cam, f, u in frames[1]:
                c12 = np.ascontiguousarray(cam.transform, np.float32).reshape(12)
                assert np.array_equal(f, rt.render_f32(cam.width, cam.height, cam.fx, cam.fy, c12, rb.make_options()))
                assert np.array_equal(u, rt.render_u8(cam.width, cam.height, cam.fx, cam.fy, c12, rb.make_options()))
        finally:
            rt.close()


# ----------------------------------------------------------------------------------------------------------- merge
def _assert_no_mergeable_node(child, data):
    c = child.reshape(-1, 8)
    d = data.reshape(c.shape[0], 8, -1).view(np.uint16)
    for i in range(1, c.shape[0]):
        if (c[i] == 0).all():
            assert not (d[i] == d[i, :1]).all(), i


@pytest.mark.parametrize("name", ["edge_mixed_sh9", "edge_root_mixed", "golden_cfg1_sh1", "relaid_dfs"])
def test_merge_of_a_refined_tree(built, name):
    from volrend_b200 import refine_plan
    st = round_trip_trees()[name][1]
    child, src = refine_plan(st.child, np.ones(st.capacity * 8, np.float32), 1.0)
    data = st.data.reshape(st.capacity * 8, -1)[src].reshape(child.shape + (st.data_dim,))
    a = _gpu(*_leaf_cells(st), merge=True)
    b = _gpu(*_leaf_cells(synth.SynthTree(child=child, data=data, offset=st.offset, invradius3=st.invradius3,
                                           data_dim=st.data_dim, data_format=st.data_format, depth=st.depth + 1)),
             merge=True)
    _same(a, b, name)
    _assert_no_mergeable_node(*a)


def test_merge_listed_zero_rows_equal_unlisted(built, cases):
    for name in ("level6", "dense8", "mixed_mixed_sh9", "dd49"):
        cells, rows = cases[name]
        nz = rows.view(np.uint16).any(1)
        got = _gpu(cells, rows, merge=True)
        _same(got, _gpu(cells[nz], rows[nz], merge=True), name)
        _assert_no_mergeable_node(*got)


# ----------------------------------------------------------------------------------------------------------- grids
def test_grid_query_at_every_cell_centre(built):
    import torch
    from volrend_b200 import N3Tree, build_npz, grid_cells
    rng = np.random.default_rng(2)
    R, dd = 16, 28
    grid = rng.standard_normal((R, R, R, dd)).astype(np.float32)
    grid[..., -1] = rng.uniform(-1.0, 3.0, (R, R, R))
    center, radius = np.array([0.3, -1.2, 2.5]), np.array([1.7, 0.9, 2.2])
    for thresh in (None, 0.5):
        cells, rows = grid_cells(torch.from_numpy(grid).cuda(), sigma_thresh=thresh)
        d = build_npz(cells, rows, data_format="SH9", center=center, radius=radius)
        t = N3Tree()
        t.load_npz(d)
        t.load_cuda()
        g = np.stack(np.meshgrid(*[np.arange(R)] * 3, indexing="ij"), -1).reshape(-1, 3)
        ctr = (g + 0.5) / R
        st = synth.SynthTree(child=d["child"], data=d["data"], offset=d["offset"], invradius3=d["invradius3"],
                             data_dim=dd, data_format="SH9", depth=4)
        pts = lc.centre_points(st, ctr, np.full(g.shape[0], 4))
        got, _, _ = t.query(pts)
        want = grid.reshape(-1, dd).astype(np.float16)
        if thresh is not None:
            want[~(want[:, -1].astype(np.float32) > np.float32(thresh))] = 0
        assert np.array_equal(got.view(np.uint16), want.view(np.uint16)), thresh


def test_uniform_tree_fits_with_refinement(built, tmp_path):
    import torch
    from volrend_b200 import Camera, N3Tree, RenderOptions, finetune, render_batch
    from volrend_b200.build import main
    assert main([str(tmp_path / "u.npz"), "--uniform", "3", "--format", "SH9", "--radius", "1.5"]) == 0
    fine = synth.make_tree("lego", depth=5, basis_dim=9, seed=7)
    W = H = 48
    f = synth.focal_for(W)
    cams = []
    for p in synth.nerf_synthetic_test_poses(16):
        c = Camera(W, H, f, f)
        c.set_c2w(p)
        cams.append(c)
    opt = RenderOptions()
    ref = N3Tree.from_synth(fine)
    fo = torch.empty((len(cams), H, W, 4), dtype=torch.float32, device="cuda")
    render_batch(ref, cams, opt, None, float_out=fo)
    targets = fo[..., :3].cpu().clone()
    tree = N3Tree()
    with np.load(tmp_path / "u.npz") as z:
        d = {k: z[k] for k in z.files}
    assert d["child"].shape[0] == 1 + 8 + 64 and np.array_equal(d["invradius3"], np.full(3, 1 / 3, np.float32))
    tree.load_npz(d)
    tree.load_cuda(slot_map=True)
    _, losses = finetune(tree, cams, targets, opt, steps=60, lr=5e-2, batch=4, seed=0, refine_every=20,
                         refine_fraction=0.3)
    assert tree.capacity > 73
    first, last = float(np.mean(losses[:4])), float(np.mean(losses[-4:]))
    print(f"uniform level-3 start: nodes 73 -> {tree.capacity}, loss {first:.6g} -> {last:.6g}")
    # first H100 run: 73 -> 342 nodes, loss 0.0486 -> 0.0076 (x 0.16); the gradients' float atomics vary the last bits
    assert last < 0.3 * first


# -------------------------------------------------------------------------------------------------------- refusals
def _pool_used():
    """Bytes in use in the current device's default stream-ordered pool (driver API)."""
    import torch
    cu = C.CDLL("libcuda.so.1")
    dev, pool, v = C.c_int(), C.c_void_p(), C.c_uint64()
    assert cu.cuDeviceGet(C.byref(dev), torch.cuda.current_device()) == 0
    assert cu.cuDeviceGetDefaultMemPool(C.byref(pool), dev) == 0
    assert cu.cuMemPoolGetAttribute(pool, 7, C.byref(v)) == 0          # CU_MEMPOOL_ATTR_USED_MEM_CURRENT
    return v.value


def test_refusals(built):
    import torch
    from volrend_b200 import _capi, lib
    L = lib()
    dd = 4
    dev = torch.device("cuda")
    good = torch.tensor([[2, 1, 2, 3], [1, 1, 1, 1]], dtype=torch.int32, device=dev)
    rows = torch.ones((2, dd), dtype=torch.float16, device=dev)
    child = torch.full((64, 8), -12345, dtype=torch.int32, device=dev)
    data = torch.full((64, 8, dd), 0x5555, dtype=torch.int16, device=dev)
    n = C.c_int64()
    s = torch.cuda.current_stream().cuda_stream
    assert L.vr_tree_build(good.data_ptr(), rows.data_ptr(), 2, dd, 0, None, None, 0, C.byref(n), s) == 0
    assert n.value == 2                                   # the root and level-1 cell (0, 1, 1)
    host_cells = (C.c_int32 * 8)(2, 1, 2, 3, 1, 0, 0, 0)

    def cells(*rowsv):
        return torch.tensor(rowsv, dtype=torch.int32, device=dev)

    cases = [
        ("level 0", cells([0, 0, 0, 0]), 1, dd, 0, 64),
        ("level 24", cells([24, 0, 0, 0]), 1, dd, 0, 64),
        ("x >= 2^L", cells([3, 8, 0, 0]), 1, dd, 0, 64),
        ("y < 0", cells([3, 0, -1, 0]), 1, dd, 0, 64),
        ("z at 2^23", cells([23, 0, 0, 1 << 23]), 1, dd, 0, 64),
        ("duplicate", cells([3, 1, 2, 3], [3, 1, 2, 3]), 2, dd, 1, 64),
        ("overlap", cells([3, 1, 6, 7], [1, 0, 1, 1]), 2, dd, 0, 64),
        ("overlap level 23", cells([23, 5, 5, 5], [22, 2, 2, 2]), 2, dd, 1, 64),
        ("n < 0", good, -1, dd, 0, 64),
        ("n > INT32_MAX", good, 1 << 31, dd, 0, 64),
        ("data_dim 0", good, 2, 0, 0, 64),
        ("capacity", good, 2, dd, 0, 1),
        ("flags", good, 2, dd, 4, 64),
    ]
    for what, c, nn, d_, fl, cap in cases:
        for merge_flag in (fl, fl | 1) if fl != 4 else (fl,):
            ch0, da0 = child.clone(), data.clone()
            r = torch.ones((max(c.shape[0], 1), max(d_, 1)), dtype=torch.float16, device=dev)
            torch.cuda.synchronize()
            used0, alloc0 = _pool_used(), torch.cuda.memory_allocated()
            n.value = -7
            rc = L.vr_tree_build(c.data_ptr(), r.data_ptr(), nn, d_, merge_flag, child.data_ptr(), data.data_ptr(),
                                 cap, C.byref(n), s)
            torch.cuda.synchronize()
            assert rc == _capi.VR_EINVAL, (what, rc, L.vr_last_error())
            assert n.value == -7, what
            assert torch.equal(child, ch0) and torch.equal(data, da0), what
            assert _pool_used() == used0 and torch.cuda.memory_allocated() == alloc0, what
    # NULL inputs with n > 0, host memory, one output NULL, NULL count
    for args in ((None, rows.data_ptr(), 2), (good.data_ptr(), None, 2), (C.addressof(host_cells), rows.data_ptr(), 2)):
        assert L.vr_tree_build(*args, dd, 0, child.data_ptr(), data.data_ptr(), 64, C.byref(n), s) == _capi.VR_EINVAL
    assert L.vr_tree_build(good.data_ptr(), rows.data_ptr(), 2, dd, 0, child.data_ptr(), None, 64, C.byref(n), s) == \
        _capi.VR_EINVAL
    assert L.vr_tree_build(good.data_ptr(), rows.data_ptr(), 2, dd, 0, None, None, 0, None, s) == _capi.VR_EINVAL
    # more nodes than the int32 links and the u32 slot map address: 48 M random level-23 cells start nodes at every
    # level below 23, about 48 M per level from level 9 on; the count call refuses it
    from volrend_b200 import build_arrays
    big = torch.randint(0, 1 << 23, (48 << 20, 4), dtype=torch.int32, device=dev)
    big[:, 0] = 23
    with pytest.raises(ValueError, match="nodes"):
        build_arrays(big, torch.ones((big.shape[0], 1), dtype=torch.float16, device=dev))
