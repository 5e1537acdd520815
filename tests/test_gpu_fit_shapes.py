"""`-m gpu`: the gradient pass (vr_tree_leaf_grads) and the error pass (vr_tree_leaf_error) at the launch shapes the
fitting loop uses, and on relaid trees, against the CPU references (oracle/grads_oracle.c, oracle/error_oracle.c).

- Batches big enough that set_work hands their tiles out in SM-local blocks (fit_shape_cases.block_mode says so for
  the device the test runs on), with view counts that are not a multiple of 4 and images that end inside a block; the
  same views in batches below block mode give the same sums.
- One call of 8 192 + 5 views, which march() launches in two chunks of the camera ring.
- Gradient sub-rectangles, options and dpix that are alpha-only or colour-only.
- Every node layout of tests/layout_cases.py: the sums mapped through the slot map are the canonical tree's, and free
  nodes, internal slots and the wide layout's extra columns stay exactly 0; vr_tree_update_data on relaid trees.
- The fitting loop's real steps on the bench tree: 8 views of 800x800 (gradients) and 16 (error).

Big batches give each view a dpix / err that is random in a small window and 0 elsewhere, and the references run on
the windows (fit_shape_cases.py).  Every gradient call's float output is compared with vr_render_batch's, bit for bit.
Tolerances are those of tests/test_gpu_finetune.py and tests/test_gpu_refine.py."""
import ctypes as C
import os
from dataclasses import replace

import numpy as np
import pytest

import edge_cases as ec
import fit_shape_cases as fc
import golden_cases as gc
import layout_cases as lc
from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)

pytestmark = pytest.mark.gpu
SEED = 7


def _load(arrays, parity=None, ndc=None, slot_map=True):
    from volrend_b200 import N3Tree
    t = N3Tree()
    t.load_npz(arrays)
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


def _num_sms():
    import torch
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _render(tree, cams, opt, tile=None):
    """vr_render_batch's float output of the views (tile-sized), on the device."""
    import torch
    from volrend_b200 import render_batch
    w, h = (tile[2], tile[3]) if tile else (cams[0].width, cams[0].height)
    fo = torch.full((len(cams), h, w, 4), float("nan"), dtype=torch.float32, device="cuda")
    render_batch(tree, cams, opt, None, float_out=fo, tile=tile)
    torch.cuda.synchronize()
    return fo


def _grads(tree, cams, opt, dpix, out=None, tile=None):
    """-> (gradient tensor, float output) of one leaf_grads call; the float output must equal vr_render_batch's."""
    import torch
    from volrend_b200 import leaf_grads
    fo = torch.full(tuple(dpix.shape), float("nan"), dtype=torch.float32, device="cuda")
    out = leaf_grads(tree, cams, opt, dpix, out=out, float_out=fo, tile=tile)
    torch.cuda.synchronize()
    assert torch.equal(fo.view(torch.int32), _render(tree, cams, opt, tile).view(torch.int32)), \
        "gradient pass float output != vr_render_batch"
    return out, fo


def _error(tree, cams, opt, err, out=None):
    """-> score tensor of one leaf_error call; a new buffer starts at -0."""
    import torch
    from volrend_b200 import leaf_error
    if out is None:
        out = torch.full((tree.capacity * 8,), -0.0, dtype=torch.float32, device="cuda")
    leaf_error(tree, cams, opt, err, out=out)
    torch.cuda.synchronize()
    return out


def _touched(score):
    return score.cpu().numpy().reshape(-1).view(np.uint32) != fc.NEG0


def _assert_cut_grads(g, slots, og, oA, what):
    """Gradient rows g [slots of the whole tree, data_dim] against the reference of the cut tree (fc.cut_oracle_tree):
    close on the cut tree's slots, exactly 0 on all others."""
    fc.assert_grads_close(g[slots], og, oA, what)
    assert not np.delete(g, slots, 0).any(), (what, "a gradient outside the windows' rays")


# ------------------------------------------------------------------------------------------------ tile blocks
BLOCK_TREES = {"sh16": dict(depth=6, basis_dim=16, seed=1), "sh25": dict(depth=5, basis_dim=25, seed=4)}
BLOCKS = [(t, p) for t in BLOCK_TREES for p in (0, 1)]
BW, BH = 150, 110           # 37.5 x 13.75 tiles: the last tile column, tile row and block of every view are cut


@pytest.fixture(scope="module")
def block_trees():
    from volrend_b200 import synth
    return {k: synth.make_tree("lego", **kw) for k, kw in BLOCK_TREES.items()}


def _block_batch(st, parity):
    """(device tree, kbd, batch views, small batch size, windows) of a batch in block mode on this device."""
    from volrend_b200 import synth
    tree = _load(st.npz_dict(), parity)
    kbd = tree.info()["kernel_basis"]
    sms = _num_sms()
    n, small = fc.block_batch(kbd, sms, BW, BH)
    assert fc.block_mode(n, BW, BH, kbd, sms)[0] and n % 4
    assert not fc.block_mode(small, BW, BH, kbd, sms)[0]
    f = synth.focal_for(BW)
    cams = [_cam(BW, BH, f, f, p) for p in synth.nerf_synthetic_test_poses(n)]
    return tree, kbd, cams, small, fc.windows(n, BW, BH, kbd, seed=n + parity, centre=True)


@pytest.mark.parametrize("name,parity", BLOCKS, ids=[f"{t}-{p}" for t, p in BLOCKS])
def test_grads_in_tile_blocks(built, block_trees, name, parity):
    from volrend_b200 import RenderOptions
    st = block_trees[name]
    tree, kbd, cams, small, wins = _block_batch(st, parity)
    n, opt = len(cams), RenderOptions()
    dpix = fc.windowed(n, BW, BH, wins, 4, -1.0, 1.0, seed=parity)
    g, _ = _grads(tree, cams, opt, _dev(dpix))
    ot, slots = fc.cut_oracle_tree(st, cams, wins)
    og, oA = fc.oracle_grads(ot, fc.oracle_cams(cams), {}, dpix, wins)
    g = g.cpu().numpy().reshape(-1, st.data_dim)
    _assert_cut_grads(g, slots, og, oA, (name, parity, n, "block mode"))
    split = None
    for v0 in range(0, n, small):
        part = cams[v0:v0 + small]
        assert not fc.block_mode(len(part), BW, BH, kbd, _num_sms())[0]
        split, _ = _grads(tree, part, opt, _dev(dpix[v0:v0 + small]), out=split)
    split = split.cpu().numpy().reshape(g.shape)
    d = np.abs(split[slots].astype(np.float64) - g[slots])
    assert (d <= 2 * (fc.RTOL * oA + fc.ATOL)).all(), float(d.max())
    assert not np.delete(split, slots, 0).any()


@pytest.mark.parametrize("name,parity", BLOCKS, ids=[f"{t}-{p}" for t, p in BLOCKS])
def test_error_in_tile_blocks(built, block_trees, name, parity):
    from volrend_b200 import RenderOptions
    st = block_trees[name]
    tree, kbd, cams, small, wins = _block_batch(st, parity)
    n, opt = len(cams), RenderOptions()
    err = fc.windowed(n, BW, BH, wins, 0, 0.25, 2.0, seed=10 + parity)
    s = _error(tree, cams, opt, _dev(err))
    ot, slots = fc.cut_oracle_tree(st, cams, wins)
    score, absum, hits = fc.oracle_error(ot, fc.oracle_cams(cams), {}, err, wins)
    sn = s.cpu().numpy()
    fc.assert_error_close(sn[slots], score, absum, hits, float(err.max()), (name, parity, n), exact_set=False)
    assert not np.delete(sn, slots).any(), "an error term outside the windows' rays"
    split = None
    for v0 in range(0, n, small):
        part = cams[v0:v0 + small]
        assert not fc.block_mode(len(part), BW, BH, kbd, _num_sms())[0]
        split = _error(tree, part, opt, _dev(err[v0:v0 + small]), out=split)
    assert np.array_equal(_touched(split), _touched(s)), "the batches below block mode shade other slots"
    d = np.abs(split.cpu().numpy()[slots].astype(np.float64) - sn[slots])
    tol = fc.RTOL * absum + fc.ATOL + fc.WEIGHT_TOL * float(err.max()) * hits
    assert (d <= 2 * tol).all(), float(d.max())


# ------------------------------------------------------------------------------------------------ camera ring
RING_VIEWS = 8192 + 5       # kCamRing (vr_api.cu) + 5: two chunks


def _ring_views():
    """12x10 views: 8 192 around the orbit, then 5 from below, which see cells the others do not."""
    from volrend_b200 import synth
    W, H = 12, 10
    f = synth.focal_for(W)
    poses = np.concatenate([synth.nerf_synthetic_test_poses(8192), synth.nerf_synthetic_test_poses(5, elev_deg=-40.0)])
    return [_cam(W, H, f, f, p) for p in poses]


@pytest.fixture(scope="module")
def ring():
    from volrend_b200 import synth
    st = synth.make_tree("lego", depth=4, basis_dim=4, seed=3)
    return st, _load(st.npz_dict()), _ring_views()


def test_grads_over_camera_ring_chunks(built, ring):
    from oracle import binding as ob
    from volrend_b200 import RenderOptions
    st, tree, cams = ring
    opt = RenderOptions()
    dpix = np.random.default_rng(1).uniform(-1, 1, (RING_VIEWS, 10, 12, 4)).astype(np.float32)
    _grads(tree, cams[:3], opt, _dev(dpix[:3]))      # the ring's position is inside a batch: the next one wraps
    g, _ = _grads(tree, cams, opt, _dev(dpix))
    og, oA = fc.oracle_grads(ob.OracleTree.from_synth(st), fc.oracle_cams(cams), {}, dpix, nthreads=1)
    fc.assert_grads_close(g.cpu().numpy(), og, oA, "8 197 views")


def test_error_over_camera_ring_chunks(built, ring):
    from oracle import binding as ob
    from volrend_b200 import RenderOptions
    st, tree, cams = ring
    opt = RenderOptions()
    err = np.random.default_rng(2).uniform(0.25, 2.0, (RING_VIEWS, 10, 12)).astype(np.float32)
    _error(tree, cams[:3], opt, _dev(err[:3]))
    s = _error(tree, cams, opt, _dev(err))
    score, absum, hits = fc.oracle_error(ob.OracleTree.from_synth(st), fc.oracle_cams(cams), {}, err, nthreads=1)
    fc.assert_error_close(s.cpu().numpy(), score, absum, hits, float(err.max()), "8 197 views")


# ------------------------------------------------------------------------------------------------ sub-rectangles
@pytest.mark.parametrize("parity", [0, 1])
def test_grads_of_sub_rectangles(built, parity):
    import torch
    from oracle import binding as ob
    from oracle import grads_binding as gb
    from volrend_b200 import RenderOptions, _capi, lib, synth
    from volrend_b200.host import _cams_array, _rect
    st, W, H, pose, kw, _ = gc.build_case("lego_sh16")
    tree = _load(st.npz_dict(), parity)
    f = synth.focal_for(W)
    poses = [pose] + list(synth.nerf_synthetic_test_poses(8)[5:7])
    cams = [_cam(W, H, f, f, p) for p in poses]
    kw = dict(kw, sigma_thresh=-1.0)               # every sample shades: the corner pixel's too
    ot, ocams, opt = ob.OracleTree.from_synth(st), fc.oracle_cams(cams), RenderOptions(**kw)
    rng = np.random.default_rng(parity)
    # a rectangle across tile edges, the corner pixel, a bottom strip lower than a warp tile, a thin strip inside
    cases = [((9, 7, 33, 26), 1), ((W - 1, H - 1, 1, 1), 1), ((0, H - 5, W, 5), 1), ((13, H - 3, 50, 3), 1),
             ((9, 7, 33, 26), 3)]
    for tile, nv in cases:
        x0, y0, w, h = tile
        dpix = rng.uniform(-1, 1, (nv, h, w, 4)).astype(np.float32)
        g, _ = _grads(tree, cams[:nv], opt, _dev(dpix), tile=tile)
        og = oA = None
        for v in range(nv):
            og, oA, _ = gb.leaf_grads(ot, ocams[v], ob.make_options(**kw), dpix[v], tile=tile, grad=og, A=oA)
        fc.assert_grads_close(g.cpu().numpy(), og, oA, (tile, nv))
    # a zero-area rectangle: VR_OK, and neither buffer is written
    L = lib()
    arr = _cams_array(cams[:2])
    o = opt._as_c()
    dpix = _dev(rng.uniform(-1, 1, (2, 8, 8, 4)).astype(np.float32))
    out = torch.full((st.capacity * 8 * st.data_dim,), 3.0, dtype=torch.float32, device="cuda")
    fo = torch.full((2 * 8 * 8 * 4,), 5.0, dtype=torch.float32, device="cuda")
    for tile in ((4, 4, 0, 8), (4, 4, 8, 0), (W, H, 0, 0)):
        assert L.vr_tree_leaf_grads(tree._handle, arr, 2, C.byref(o), _rect(tile), dpix.data_ptr(), out.data_ptr(),
                                    fo.data_ptr(), None) == _capi.VR_OK, tile
    torch.cuda.synchronize()
    assert bool((out == 3.0).all()) and bool((fo == 5.0).all())


# ------------------------------------------------------------------------------------------------ options
OPTION_TREES = ["mixed_sh9", "mixed_rgba", "mixed_asg4", "lego_sh16"]
OPTIONS = {"sigma_thresh_0": dict(sigma_thresh=0.0), "sigma_thresh_neg": dict(sigma_thresh=-1.0),
           "stop_0": dict(stop_thresh=0.0), "stop_0.5": dict(stop_thresh=0.5), "stop_0.99": dict(stop_thresh=0.99),
           "bg_0": dict(background_brightness=0.0), "bg_2.5": dict(background_brightness=2.5),
           "step_1e-5": dict(step_size=1e-5), "step_2e-2": dict(step_size=2e-2),
           "minmax_0_0": dict(basis_minmax=[0, 0]), "minmax_2_5": dict(basis_minmax=[2, 5]),
           "rot_dirs": dict(rot_dirs=[0.3, -0.2, 0.5])}
OPTION_CASES = [(t, o) for t in OPTION_TREES for o in OPTIONS]


def _option_views(name):
    """(SynthTree, ndc, cameras) of two views of the tree."""
    from volrend_b200 import synth
    if name in gc.CASES:
        st, W, H, pose, _, ndc = gc.build_case(name)
        f = synth.focal_for(W)
        return st, ndc, [_cam(W, H, f, f, p) for p in (pose, synth.nerf_synthetic_test_poses(8)[5])]
    st, _ = ec.edge_tree(name)
    return st, ec.NDC.get(name), [_cam(*ec.view(v, name, st)[:5]) for v in ("px", "inside")]


@pytest.mark.parametrize("name,option", OPTION_CASES, ids=[f"{t}-{o}" for t, o in OPTION_CASES])
def test_grads_under_options_and_dpix_shapes(built, name, option):
    """Random dpix, alpha-only and colour-only dpix (the two halves of the sigma term), and zero dpix (no gradient at
    all, the full render still)."""
    from oracle import binding as ob
    from volrend_b200 import RenderOptions
    st, ndc, cams = _option_views(name)
    kw = OPTIONS[option]
    tree = _load(st.npz_dict(), ndc=ndc)
    ot, ocams, opt = ob.OracleTree.from_synth(st, ndc=ndc), fc.oracle_cams(cams), RenderOptions(**kw)
    n, H, W = len(cams), cams[0].height, cams[0].width
    rnd = np.random.default_rng(len(option)).uniform(-1, 1, (n, H, W, 4)).astype(np.float32)
    shapes = {"random": rnd, "alpha": rnd * np.array([0, 0, 0, 1], np.float32),
              "colour": rnd * np.array([1, 1, 1, 0], np.float32)}
    for what, dpix in shapes.items():
        g, fo = _grads(tree, cams, opt, _dev(dpix))
        og, oA = fc.oracle_grads(ot, ocams, kw, dpix)
        # stop_thresh 0.99: a stopped ray's alpha is 1 whatever sigma, and on the edge trees every ray that meets the
        # tree stops: an alpha-only dpix may have no gradient at all
        fc.assert_grads_close(g.cpu().numpy(), og, oA, (name, option, what),
                              terms=not (what == "alpha" and option == "stop_0.99"))
    if option == "stop_0.99":                       # most rays that meet the tree stop early
        a = fo[..., 3].cpu().numpy()
        assert (a == 1.0).sum() > 0.5 * (a > 0).sum(), "too few rays take the stopped branch"
    import torch
    g, _ = _grads(tree, cams, opt, torch.zeros((n, H, W, 4), dtype=torch.float32, device="cuda"))
    assert not g.any(), "a zero dpix gave a gradient"


# ------------------------------------------------------------------------------------------------ relaid trees
RELAID_TREES = ["mixed_sh16", "mixed_rgba", "chain23", "quant_mixed"]
# quant_mixed is created from its quantised arrays, which have no wide layout (data_dim is 3 * basis_dim + 1)
RELAID = [(t, lay, p) for t in RELAID_TREES for lay in lc.LAYOUTS for p in (0, 1)
          if not (t == "quant_mixed" and lay == "wide")]
_CANON = {}


def _canonical(name):
    """(SynthTree, npz, cameras, dpix, err, oracle grad, A, score, absum, hits) of the tree's canonical layout."""
    if name not in _CANON:
        from oracle import binding as ob
        st, npz = ec.edge_tree(name)
        views = ["px", "inside", "face"] + (["deep"] if name.startswith("chain") else [])
        cams = [_cam(*ec.view(v, name, st)[:5]) for v in views]
        n, H, W = len(cams), cams[0].height, cams[0].width
        dpix = np.random.default_rng(5).uniform(-1, 1, (n, H, W, 4)).astype(np.float32)
        err = np.random.default_rng(6).uniform(0.25, 2.0, (n, H, W)).astype(np.float32)
        ot, ocams = ob.OracleTree.from_synth(st), fc.oracle_cams(cams)
        _CANON[name] = (st, npz, cams, dpix, err) + fc.oracle_grads(ot, ocams, {}, dpix) + \
            fc.oracle_error(ot, ocams, {}, err)
    return _CANON[name]


@pytest.mark.parametrize("name,layout,parity", RELAID, ids=[f"{t}-{lay}-{p}" for t, lay, p in RELAID])
def test_relaid_trees_follow_the_slot_map(built, name, layout, parity):
    from volrend_b200 import RenderOptions
    st, npz, cams, dpix, err, og, oA, score, absum, hits = _canonical(name)
    r = lc.relayout(st, layout, npz, seed=SEED)
    tree = _load(r.arrays(), parity)
    opt = RenderOptions()
    m, inner = r.slot_map, r.st.child.reshape(-1) != 0
    dd, ddr = st.data_dim, r.st.data_dim
    cols = list(range(dd - 1)) + [ddr - 1]
    extra = [c for c in range(ddr) if c not in cols]
    g, _ = _grads(tree, cams, opt, _dev(dpix))
    g = g.cpu().numpy().reshape(-1, ddr)
    mapped = np.zeros(og.shape)
    mapped[m[m >= 0]] = g[m >= 0][:, cols]
    fc.assert_grads_close(mapped, og, oA, (name, layout, parity))
    assert not g[m < 0].any() and not g[inner].any() and not g[:, extra].any(), (name, layout, parity)
    s = _error(tree, cams, opt, _dev(err)).cpu().numpy()
    touched = s.view(np.uint32) != fc.NEG0
    assert not touched[m < 0].any() and not touched[inner].any()
    mapped = np.full(score.shape, -0.0, np.float32)
    mapped[m[m >= 0]] = s[m >= 0]
    fc.assert_error_close(mapped, score, absum, hits, float(err.max()), (name, layout, parity))


# ------------------------------------------------------------------------------------------------ update_data
def _query_state(tree, st):
    """Everything besides the march that reads leaf values: vr_tree_query's rows, vr_tree_eval, the probe."""
    import torch
    from volrend_b200 import RenderOptions, VolrendError, lib
    rng = np.random.default_rng(3)
    lo = -st.offset / st.invradius3
    pts = (lo + rng.uniform(0, 1, (257, 3)) / st.invradius3).astype(np.float32)
    dirs = rng.normal(size=(257, 3)).astype(np.float32)
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    out = {}
    try:
        out["query"] = tree.query(pts)[0].view(np.uint16)
    except VolrendError:
        pass
    rgb, sig = tree.eval(pts, dirs, RenderOptions())
    out["eval"] = np.concatenate([rgb, sig[:, None]], 1).view(np.uint32)
    probe = torch.full((75,), float("nan"), dtype=torch.float32, device="cuda")
    xyz = (C.c_float * 3)(*[float(v) for v in pts[0]])
    assert lib().vr_probe_lumisphere(tree._handle, xyz, probe.data_ptr(), None) == 0
    torch.cuda.synchronize()
    out["probe"] = probe.cpu().numpy().view(np.uint32)
    return out


UPDATE = [(lay, p) for lay in ("dirty", "reverse", "wide") for p in (0, 1)]


@pytest.mark.parametrize("layout,parity", UPDATE, ids=[f"{lay}-{p}" for lay, p in UPDATE])
def test_update_data_on_relaid_trees(built, layout, parity):
    """New leaf rows, and garbage (NaN, +-Inf, -0 among random bits) in free nodes and internal slots: the updated
    tree renders, queries, evaluates and probes as a tree created from the same arrays."""
    import torch
    from volrend_b200 import RenderOptions
    name = "mixed_sh16"
    st, _ = ec.edge_tree(name)
    r = lc.relayout(st, layout, None, seed=SEED)
    tree = _load(r.st.npz_dict(), parity)
    info0 = tree.info()
    rng = np.random.default_rng(20 + parity)
    shape = r.st.data.shape
    new = rng.normal(0, 0.5, shape).astype(np.float16)
    new[..., -1] = (np.abs(new[..., -1]) * rng.choice([0.0, 1.0, 30.0], shape[:4])).astype(np.float16)
    bits = new.view(np.uint16).reshape(-1, shape[-1])
    junk = (r.slot_map < 0) | (r.st.child.reshape(-1) != 0)
    noise = rng.integers(0, 1 << 16, (int(junk.sum()), shape[-1]), dtype=np.uint16)
    special = lc.SPECIAL_BITS[rng.integers(0, len(lc.SPECIAL_BITS), noise.shape)]
    bits[junk] = np.where(rng.random(noise.shape) < 0.3, special, noise)
    assert junk.any()
    tree.update_data(torch.from_numpy(new).cuda())
    torch.cuda.synchronize()
    assert tree.info() == info0
    fresh_st = replace(r.st, data=new, meta={})
    fresh = _load(fresh_st.npz_dict(), parity)
    for v in ("px", "inside", "face", "odd"):
        W, H, fx, fy, pose, kw, _ = ec.view(v, name, st)
        c = _cam(W, H, fx, fy, pose)
        a, b = _render(tree, [c], RenderOptions(**kw)), _render(fresh, [c], RenderOptions(**kw))
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), (layout, v)
        assert (a[..., 3] > 0).any()
    q1, q2 = _query_state(tree, fresh_st), _query_state(fresh, fresh_st)
    assert set(q1) == set(q2) and "eval" in q1
    for k in q1:
        assert np.array_equal(q1[k], q2[k]), (layout, k)


# ------------------------------------------------------------------------------------------------ the real steps
@pytest.fixture(scope="module")
def bench():
    """The bench tree (1.4 M nodes) on the device."""
    from volrend_b200 import synth
    st = synth.make_tree("lego", depth=10, basis_dim=16, seed=0)
    return st, _load(st.npz_dict())


def _bench_views(n, kbd, seed):
    from volrend_b200 import synth
    f = synth.focal_for(800)
    cams = [_cam(800, 800, f, f, p) for p in synth.nerf_synthetic_test_poses(200)[::200 // n][:n]]
    assert fc.block_mode(n, 800, 800, kbd, _num_sms())[0], "not in block mode on this device"
    return cams, fc.windows(n, 800, 800, kbd, size=(9, 7), seed=seed, centre=True)


def test_finetune_step_grads(built, bench):
    """The finetune bench's step: 8 views of 800x800.  The gradient outside the slots the windows' rays can reach is
    exactly 0; the float output is vr_render_batch's over the whole frames."""
    import torch
    from volrend_b200 import RenderOptions
    st, tree = bench
    cams, wins = _bench_views(8, tree.info()["kernel_basis"], seed=1)
    dpix = fc.windowed(8, 800, 800, wins, 4, -1.0, 1.0, seed=2)
    g, _ = _grads(tree, cams, RenderOptions(), _dev(dpix))
    ot, slots = fc.cut_oracle_tree(st, cams, wins)
    slots = torch.from_numpy(slots).cuda()
    og, oA = fc.oracle_grads(ot, fc.oracle_cams(cams), {}, dpix, wins)
    rows = g.view(-1, st.data_dim)
    fc.assert_grads_close(rows[slots].cpu().numpy(), og, oA, "8 x 800x800")
    rows.index_fill_(0, slots, 0.0)
    assert int(torch.count_nonzero(rows)) == 0, "a gradient outside the windows' rays"


def test_refine_batch_error(built, bench):
    """The refine CLI's default batch: 16 views of 800x800."""
    import torch
    from volrend_b200 import RenderOptions
    st, tree = bench
    cams, wins = _bench_views(16, tree.info()["kernel_basis"], seed=3)
    err = fc.windowed(16, 800, 800, wins, 0, 0.25, 2.0, seed=4)
    s = _error(tree, cams, RenderOptions(), _dev(err))
    ot, slots = fc.cut_oracle_tree(st, cams, wins)
    slots = torch.from_numpy(slots).cuda()
    score, absum, hits = fc.oracle_error(ot, fc.oracle_cams(cams), {}, err, wins)
    fc.assert_error_close(s[slots].cpu().numpy(), score, absum, hits, float(err.max()), "16 x 800x800",
                          exact_set=False)
    s.index_fill_(0, slots, 0.0)
    assert int(torch.count_nonzero(s)) == 0, "an error term outside the windows' rays"
