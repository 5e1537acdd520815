"""`-m gpu`: the gradient, weights and error passes (vr_tree_leaf_grads, vr_tree_leaf_weights, vr_tree_leaf_error) on
an H100 against the float64 autograd reference of tests/axis_ray_cases.py, entry by entry, under both table parities;
and the render that follows an in-place leaf update on the same stream."""
import os

import numpy as np
import pytest

import axis_ray_cases as ac
from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)

pytestmark = pytest.mark.gpu
RTOL, ATOL = 1e-4, 1e-7          # gradients: |g - g64| <= RTOL * A + ATOL (test_gpu_finetune.py's tolerance)
SIGN = 1e-3                      # entries with |g64| > SIGN * A + ATOL have the reference's sign (below ATOL, a term
                                 # that cancels to 0 exactly leaves float64 rounding noise of either sign)
PIX_TOL = 1e-5
W_RTOL, W_ATOL = 1e-6, 1e-7
E_RTOL, E_ATOL = 1e-5, 1e-7


def _device_tree(st, parity, slot_map=True):
    from volrend_b200 import N3Tree
    t = N3Tree()
    t.load_npz(st.npz_dict())
    os.environ["VR_WIDE_PARITY"] = str(parity)
    try:
        t.load_cuda(slot_map=slot_map)
    finally:
        os.environ.pop("VR_WIDE_PARITY", None)
    assert t.info()["wide_parity"] == parity
    return t


def _cams(case):
    from volrend_b200 import Camera
    cams = []
    for v in case.views:
        c = Camera(2, 2, 1.0, 1.0)
        c.set_c2w(v.pose)
        cams.append(c)
    return cams


CASES = [(n, p) for n in ac.CASES for p in (0, 1)]


@pytest.mark.parametrize("name,parity", CASES, ids=[f"{n}-{p}" for n, p in CASES])
def test_passes_match_reference(built, name, parity):
    import torch
    from volrend_b200 import RenderOptions, leaf_error, leaf_grads, leaf_weights, render_batch
    case = ac.CASES[name]
    ref = ac.reference(case)
    tree = _device_tree(case.st, parity)
    cams = _cams(case)
    opt = RenderOptions(**case.options())
    V = len(cams)
    dpix = torch.from_numpy(case.dpix().reshape(V, 1, 1, 4)).cuda()
    fo = torch.full((V, 1, 1, 4), float("nan"), dtype=torch.float32, device="cuda")
    g = leaf_grads(tree, cams, opt, dpix, float_out=fo, tile=ac.TILE)
    rf = torch.full((V, 1, 1, 4), float("nan"), dtype=torch.float32, device="cuda")
    img = torch.empty((V, 1, 1, 4), dtype=torch.uint8, device="cuda")
    render_batch(tree, cams, opt, img, float_out=rf, tile=ac.TILE)
    cnt = torch.zeros(5, dtype=torch.int64, device="cuda")
    w = leaf_weights(tree, cams, opt, counters=cnt, tile=ac.TILE)
    ecnt = torch.zeros(5, dtype=torch.int64, device="cuda")
    e = leaf_error(tree, cams, opt, torch.from_numpy(case.err().reshape(V, 1, 1)).cuda(), counters=ecnt, tile=ac.TILE)
    torch.cuda.synchronize()

    fo, rf = fo.cpu().numpy(), rf.cpu().numpy()
    assert np.array_equal(fo.view(np.uint32), rf.view(np.uint32)), "gradient replay != vr_render_batch"
    np.testing.assert_allclose(fo.reshape(V, 4), ref.pix, rtol=0, atol=PIX_TOL)

    g = g.cpu().numpy().reshape(ref.grad.shape).astype(np.float64)
    d = np.abs(g - ref.grad)
    bad = d > RTOL * ref.A + ATOL
    assert not bad.any(), (int(bad.sum()), float(d.max()), np.argwhere(bad)[:5].tolist())
    big = np.abs(ref.grad) > SIGN * ref.A + ATOL
    assert big.any()
    assert (np.sign(g[big]) == np.sign(ref.grad[big])).all()
    assert not g[ref.unreached].any(), np.argwhere((g != 0) & ref.unreached)[:5].tolist()

    w = w.cpu().numpy().reshape(-1).astype(np.float64)
    touched = np.isfinite(ref.wmax)
    assert np.array_equal(np.isfinite(w), touched)
    assert (w[~touched] == -np.inf).all()
    np.testing.assert_allclose(w[touched], ref.wmax[touched], rtol=W_RTOL, atol=W_ATOL)

    e = e.cpu().numpy().reshape(-1).astype(np.float64)
    assert (np.abs(e - ref.err) <= E_RTOL * ref.err_abs + E_ATOL).all(), float(np.abs(e - ref.err).max())
    assert not e[~touched].any()
    for c in (cnt, ecnt):
        c = c.cpu().tolist()
        assert [c[0], c[2], c[3]] == [ref.counters["samples"], ref.counters["shaded"], ref.counters["rays_hit"]], c


@pytest.mark.parametrize("parity", [0, 1])
def test_render_right_after_update_on_the_same_stream(built, parity):
    """``update_data`` on a side stream, then at once, with no synchronisation, a single-view render and a one-view
    ``render_batch`` on that stream: both equal, byte for byte, the renders of a tree created from the new data.  The
    single-view march kernels read the tree before they wait for their predecessor, so this checks that the first
    launch after an update is ordered behind it in full.  It checks the contract; it cannot force the race."""
    import torch
    import edge_cases as ec
    from volrend_b200 import Camera, RenderOptions, launch_renderer, render_batch, synth
    st = ec.mixed_tree(6, 16, "SH", 77)
    new = ec.mixed_tree(6, 16, "SH", 77)            # same structure, other values
    rng = np.random.default_rng(78)
    new.data = (new.data.astype(np.float32) * rng.uniform(0.5, 1.5, new.data.shape)).astype(np.float16)
    tree = _device_tree(st, parity)
    fresh = _device_tree(new, parity, slot_map=False)
    cam = Camera(96, 80, 70.0, 70.0)
    cam.set_c2w(synth.nerf_synthetic_test_poses(8)[2])
    opt = RenderOptions()
    data = torch.from_numpy(np.ascontiguousarray(new.data)).cuda()
    old = torch.from_numpy(np.ascontiguousarray(st.data)).cuda()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())

    def frames():
        a = torch.zeros((80, 96, 4), dtype=torch.uint8, device="cuda")
        af = torch.zeros((80, 96, 4), dtype=torch.float32, device="cuda")
        b = torch.zeros((1, 80, 96, 4), dtype=torch.uint8, device="cuda")
        bf = torch.zeros((1, 80, 96, 4), dtype=torch.float32, device="cuda")
        return a, af, b, bf

    outs = frames()
    want = frames()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        tree.update_data(data, stream=side)
        launch_renderer(tree, cam, opt, outs[0], None, side, True, float_out=outs[1])
    tree.update_data(old)
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        tree.update_data(data, stream=side)
        render_batch(tree, [cam], opt, outs[2], float_out=outs[3], stream=side)
    launch_renderer(fresh, cam, opt, want[0], None, None, True, float_out=want[1])
    render_batch(fresh, [cam], opt, want[2], float_out=want[3])
    torch.cuda.synchronize()
    for o, w_ in zip(outs, want):
        assert np.array_equal(o.cpu().numpy().view(np.uint8), w_.cpu().numpy().view(np.uint8))
