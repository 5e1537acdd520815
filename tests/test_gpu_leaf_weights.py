"""`-m gpu`: the leaf-weights pass (vr_tree_leaf_weights) and pruning by weight on an H100.

The weights are compared with the CPU restatement (oracle/weights_oracle.c, orc_leaf_weights): the same slots are
shaded (every other slot keeps -inf) and the values agree within 2e-6, the tolerance of the march's colours, because
the oracle's expf is glibc's; the work counters agree exactly.  Between GPU calls (batch shapes, splits, view order)
and against the render kernels (alpha, counters), the comparisons are bit for bit."""
import ctypes as C
import os

import numpy as np
import pytest

import edge_cases as ec
import golden_cases as gc
from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)

pytestmark = pytest.mark.gpu
TOL = 2e-6


def _same_bits(a, b, what=""):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    assert a.shape == b.shape, what
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), what


def _close_to_oracle(g, o, what):
    g, o = np.asarray(g, np.float32).reshape(-1), np.asarray(o, np.float32).reshape(-1)
    assert np.array_equal(np.isneginf(g), np.isneginf(o)), (what, "shaded slots differ",
                                                            int((np.isneginf(g) != np.isneginf(o)).sum()))
    f = ~np.isneginf(g)
    assert np.isfinite(g[f]).all(), what
    d = np.abs(g[f].astype(np.float64) - o[f])
    assert d.size == 0 or d.max() <= TOL, (what, float(d.max()))


def _device_tree(st, npz=None, ndc=None, parity=None, slot_map=True):
    from volrend_b200 import N3Tree
    t = N3Tree()
    t.load_npz(npz if npz is not None else st.npz_dict())
    if ndc is not None:
        t.use_ndc = True
        t.ndc_width, t.ndc_height, t.ndc_focal = ndc
    if parity is not None:
        os.environ["VR_WIDE_PARITY"] = str(parity)
    try:
        t.load_cuda(slot_map=slot_map)
    finally:
        os.environ.pop("VR_WIDE_PARITY", None)
    if parity is not None:
        assert t.info()["wide_parity"] == parity
    return t


def _cam(W, H, fx, fy, pose):
    from volrend_b200 import Camera
    c = Camera(W, H, fx, fy)
    c.set_c2w(pose)
    return c


def _gpu(tree, cams, opt, tile=None, out=None, with_alpha=True):
    import torch
    from volrend_b200 import leaf_weights
    cams = cams if isinstance(cams, list) else [cams]
    w, h = (tile[2], tile[3]) if tile is not None else (cams[0].width, cams[0].height)
    alpha = torch.full((len(cams), h, w), float("nan"), dtype=torch.float32, device="cuda") if with_alpha else None
    cnt = torch.zeros(5, dtype=torch.int64, device="cuda")
    out = leaf_weights(tree, cams, opt, out=out, alpha=alpha, counters=cnt, tile=tile)
    torch.cuda.synchronize()
    return out.cpu().numpy().reshape(-1), (alpha.cpu().numpy() if with_alpha else None), cnt.cpu().tolist()


def _oracle(st, W, H, fx, fy, pose, kw, ndc=None, tile=None):
    from oracle import binding as ob
    from oracle import weights_binding as wb
    from volrend_b200 import synth
    ot = ob.OracleTree.from_synth(st, ndc=ndc)
    cam = ob.make_camera(W, H, fx, fy, synth.c2w_to_colmajor12(pose))
    return wb.leaf_weights(ot, cam, ob.make_options(**kw), tile=tile)


def _check_view(tree, st, W, H, fx, fy, pose, kw, ndc=None, what=""):
    from volrend_b200 import RenderOptions
    g, ga, gc_ = _gpu(tree, _cam(W, H, fx, fy, pose), RenderOptions(**kw))
    o, oa, oc = _oracle(st, W, H, fx, fy, pose, kw, ndc)
    _close_to_oracle(g, o, what)
    assert gc_[:4] == [oc["samples"], oc["child_loads"], oc["shaded"], oc["rays_hit"]], (what, gc_, oc)
    assert np.abs(ga[0] - oa).max() <= TOL, what


@pytest.mark.parametrize("name", gc.CASES)
def test_golden_trees_match_oracle(built, name):
    from volrend_b200 import synth
    st, W, H, pose, kw, ndc = gc.build_case(name)
    tree = _device_tree(st, ndc=ndc)
    f = synth.focal_for(W)
    _check_view(tree, st, W, H, f, f, pose, kw, ndc, name)


EDGE = [(n, p) for n in ec.TREES for p in (0, 1)]


@pytest.mark.parametrize("name,parity", EDGE, ids=[f"{n}-{p}" for n, p in EDGE])
def test_edge_trees_match_oracle(built, name, parity):
    st, npz = ec.edge_tree(name)
    ndc = ec.NDC.get(name)
    tree = _device_tree(st, npz, ndc, parity)
    for v in ec.views_for(name):
        if v == "composite":
            continue
        W, H, fx, fy, pose, kw, _ = ec.view(v, name, st)
        for s in (1e-2, 0.0, -1.0):
            _check_view(tree, st, W, H, fx, fy, pose, dict(kw, sigma_thresh=s), ndc, f"{name}.{v} sigma_thresh {s}")


@pytest.fixture(scope="module")
def orbit():
    from volrend_b200 import RenderOptions, synth
    st, _, _, _, _, _ = gc.build_case("lego_sh16")
    tree = _device_tree(st)
    cams = [_cam(64, 48, synth.focal_for(64), synth.focal_for(64), p) for p in synth.nerf_synthetic_test_poses(24)]
    return st, tree, cams, RenderOptions()


def test_batch_shapes_agree(built, orbit):
    import torch
    st, tree, cams, opt = orbit
    many, _, _ = _gpu(tree, cams, opt)
    one = np.full_like(many, -np.inf)
    for c in cams:
        w1, _, _ = _gpu(tree, c, opt)
        one = _max(one, w1)
    _close_to_oracle(w1, _oracle(st, 64, 48, c.fx, c.fy, c.transform.T, {})[0], "last view")
    _same_bits(many, one, "one call over all views vs the maximum of single-view calls")
    split = torch.full((st.capacity, 2, 2, 2), float("-inf"), dtype=torch.float32, device="cuda")
    _gpu(tree, cams[:10], opt, out=split)
    s, _, _ = _gpu(tree, cams[10:], opt, out=split)
    _same_bits(many, s, "views split over two calls")
    r, _, _ = _gpu(tree, cams[::-1], opt)
    _same_bits(many, r, "views in reverse order")


def _max(a, b):
    """Element-wise maximum in the order of the weights pass (-0 < +0; no NaN)."""
    def key(x):
        u = np.ascontiguousarray(x, np.float32).view(np.uint32)
        return np.where(u & 0x80000000, ~u, u | 0x80000000)
    return np.where(key(b) > key(a), b, a)


def test_tile_matches_oracle(built, orbit):
    st, tree, cams, opt = orbit
    c = cams[5]
    tile = (9, 7, 33, 26)
    g, ga, _ = _gpu(tree, c, opt, tile=tile)
    o, oa, _ = _oracle(st, 64, 48, c.fx, c.fy, c.transform.T, {}, tile=tile)
    _close_to_oracle(g, o, "tile")
    assert np.abs(ga[0] - oa).max() <= TOL


def test_large_batch_equals_chunks(built, orbit):
    """Enough views for the SM-local tile blocks of the persistent queue."""
    import torch
    from volrend_b200 import synth
    st, tree, _, opt = orbit
    cams = [_cam(64, 48, synth.focal_for(64), synth.focal_for(64), p) for p in synth.nerf_synthetic_test_poses(4224)]
    big, _, _ = _gpu(tree, cams, opt, with_alpha=False)
    acc = torch.full((st.capacity, 2, 2, 2), float("-inf"), dtype=torch.float32, device="cuda")
    for v0 in range(0, len(cams), 500):
        small, _, _ = _gpu(tree, cams[v0:v0 + 500], opt, out=acc, with_alpha=False)
    _same_bits(big, small, "4224 views in one call vs in chunks of 500")


def test_alpha_and_counters_equal_render(built, orbit):
    import torch
    from volrend_b200 import render_batch
    st, tree, cams, opt = orbit
    _, ga, gcnt = _gpu(tree, cams, opt)
    img = torch.zeros((len(cams), 48, 64, 4), dtype=torch.uint8, device="cuda")
    fo = torch.zeros((len(cams), 48, 64, 4), dtype=torch.float32, device="cuda")
    cnt = torch.zeros(5, dtype=torch.int64, device="cuda")
    render_batch(tree, cams, opt, img, float_out=fo)
    render_batch(tree, cams, opt, img, counters=cnt)
    torch.cuda.synchronize()
    _same_bits(ga, fo.cpu().numpy()[..., 3], "alpha vs the float output's alpha")
    assert gcnt == cnt.cpu().tolist()


def test_slot_map_flag(built):
    import torch
    from volrend_b200 import RenderOptions, VolrendError, _capi, leaf_weights, lib
    st, _, _, _, _, _ = gc.build_case("lego_sh16")
    plain, mapped = _device_tree(st, slot_map=False), _device_tree(st, slot_map=True)
    a, b = plain.info(), mapped.info()
    assert b["device_bytes"] - a["device_bytes"] == 4 * 64 * a["n_tables"]
    assert a["device_bytes"] == a["kernel_bytes"] and b["kernel_bytes"] == a["kernel_bytes"]
    with pytest.raises(RuntimeError, match="slot map"):
        leaf_weights(plain, _cam(8, 8, 10.0, 10.0, np.eye(4)), RenderOptions())
    w = torch.zeros(st.capacity * 8, dtype=torch.float32, device="cuda")
    c = _cam(8, 8, 10.0, 10.0, np.eye(4))._as_c()
    o = RenderOptions()._as_c()
    assert lib().vr_tree_leaf_weights(plain._handle, C.byref(c), 1, C.byref(o), None, w.data_ptr(), None, None,
                                      None) == _capi.VR_EUNSUPPORTED
    assert b"slot map" in lib().vr_last_error()
    # host memory in any of the buffers is refused before a launch: the device buffer stays as it was
    host, cnt = np.zeros(st.capacity * 8, np.float32), np.zeros(5, np.int64)
    for name, bufs in ((b"weight_dev", (host.ctypes.data, None, None)),
                       (b"alpha_dev", (w.data_ptr(), host.ctypes.data, None)),
                       (b"counters_dev", (w.data_ptr(), None, cnt.ctypes.data))):
        assert lib().vr_tree_leaf_weights(mapped._handle, C.byref(c), 1, C.byref(o), None, *bufs,
                                          None) == _capi.VR_EINVAL
        assert name in lib().vr_last_error()
    torch.cuda.synchronize()
    assert not w.any() and not host.any()
    h = C.c_void_p()
    d, keep = plain._plain_desc()
    assert lib().vr_tree_create_ex(C.byref(d), 2, C.byref(h)) == _capi.VR_EINVAL and not h.value
    del keep


def _render_pair(a, b, cams, opt):
    import torch
    from volrend_b200 import render_batch
    out = []
    for t in (a, b):
        img = torch.zeros((len(cams), cams[0].height, cams[0].width, 4), dtype=torch.uint8, device="cuda")
        fo = torch.zeros((len(cams), cams[0].height, cams[0].width, 4), dtype=torch.float32, device="cuda")
        render_batch(t, cams, opt, img, float_out=fo)
        torch.cuda.synchronize()
        out.append((img.cpu().numpy(), fo.cpu().numpy()))
    return out


@pytest.mark.parametrize("sigma_thresh", [1e-2, 0.0])
def test_thresh0_no_collapse_renders_identically(built, orbit, sigma_thresh):
    from volrend_b200 import N3Tree, RenderOptions, prune_npz
    st, _, cams, _ = orbit
    opt = RenderOptions(sigma_thresh=sigma_thresh)
    tree = _device_tree(st)
    w, _, _ = _gpu(tree, cams, opt, with_alpha=False)
    p = prune_npz(st.npz_dict(), w, 0.0, collapse=False)
    assert (p["data"].reshape(-1, st.data_dim)[:, -1] == 0).sum() > (st.data.reshape(-1, st.data_dim)[:, -1] == 0).sum()
    pruned = N3Tree()
    pruned.load_npz(p)
    pruned.load_cuda()
    (ua, fa), (ub, fb) = _render_pair(tree, pruned, cams, opt)
    assert np.array_equal(ua, ub)
    _same_bits(fa, fb, "float frames of the pruned tree")


def test_collapsed_file_loads_and_renders(built, orbit, tmp_path):
    from oracle import binding as ob
    from oracle import ref_binding as rb
    from volrend_b200 import N3Tree, RenderOptions, prune_npz, synth
    from volrend_b200.compress import _write_npz
    st, tree, cams, opt = orbit
    w, _, _ = _gpu(tree, cams, opt, with_alpha=False)
    p = prune_npz(st.npz_dict(), w, 1e-3, collapse=True)
    assert p["child"].shape[0] < st.capacity
    path = str(tmp_path / "pruned.npz")
    _write_npz(path, p)
    loaded = N3Tree(path)
    ot = ob.OracleTree(p["child"], p["data"], p["offset"], p["invradius3"], int(p["data_dim"]), str(p["data_format"]))
    ref = rb.RefTree(path) if rb.available() else None
    try:
        for c in cams[:6]:
            img, fo = _render_pair(loaded, loaded, [c], opt)[0]
            oc = ob.make_camera(c.width, c.height, c.fx, c.fy, c.transform.reshape(12))
            f, u, _ = ob.render(ot, oc, ob.make_options())
            assert np.abs(fo[0] - f).max() <= TOL
            if ref is not None:
                rf = ref.render_f32(c.width, c.height, c.fx, c.fy, c.transform.reshape(12), rb.make_options())
                _same_bits(fo[0], rf, "our kernel vs the reference kernel on the pruned file")
                assert np.abs(rf - f).max() <= TOL
    finally:
        if ref is not None:
            ref.close()
