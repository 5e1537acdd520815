"""`-m gpu`: every device path on trees in other node layouts (tests/layout_cases.py): depth-first, reverse
breadth-first (every non-root link backwards), shuffled, shuffled with free nodes, out-of-range links in a free node,
trailing zero nodes and noise in internal slots' rows, and wider data rows -- under both table parities.  A relaid tree
is the same tree, so everything is bit-identical to the canonical tree and to the reference's stored frames; there are
no tolerances.  Also the trees vr_tree_create must refuse (a defect in the part the root reaches), with their memory
given back, and quantised trees of one kernel basis function with no retained basis functions."""
import ctypes as C
import os

import numpy as np
import pytest

import edge_cases as ec
import golden_cases as gc
import layout_cases as lc
from conftest import ROOT
from oracle import query_oracle as qo
from wire_cases import golden_name, matches, wire_tree

pytestmark = pytest.mark.gpu
KERNELS = {"queue": 7, "inline": 3 + 16 * 193}     # the product kernels (vr_kernels.h)
FULL = ("shuffle", "dirty")                          # layouts that render every edge frame; the others render one
SEED = 7
RENDER = [(t, lay, p) for t in ec.TREES for lay in lc.LAYOUTS for p in (0, 1)
          if not (t == "quant_mixed" and lay != "shuffle")]
TREE_LAYOUTS = [(t, lay) for t in ec.TREES for lay in lc.LAYOUTS if not (t == "quant_mixed" and lay != "shuffle")]
WIRE = [(t, lay) for t in ("sh16_d6", "sh4_d5") for lay in lc.LAYOUTS]


def _ids(cases):
    return ["-".join(str(x) for x in c) for c in cases]


def _load(arrays, name=None, parity=None, slot_map=False, gpu_decode=True, ndc=True):
    from volrend_b200 import N3Tree
    t = N3Tree(gpu_decode=gpu_decode)
    t.load_npz(arrays)
    if ndc and name in ec.NDC:
        t.use_ndc = True
        t.ndc_width, t.ndc_height, t.ndc_focal = ec.NDC[name]
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


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view({1: np.uint8, 2: np.uint16, 4: np.uint32}[a.dtype.itemsize])


def _same(a, b, what):
    assert a.shape == b.shape, what
    assert np.array_equal(_bits(a), _bits(b)), what


def _single(tree, cam, opt, comp):
    """(float RGBA, RGBA8) of one launch_renderer."""
    import torch
    from volrend_b200 import launch_renderer
    img = torch.zeros((cam.height, cam.width, 4), dtype=torch.uint8, device="cuda")
    fo = torch.zeros((cam.height, cam.width, 4), dtype=torch.float32, device="cuda")
    if comp is None:
        launch_renderer(tree, cam, opt, img, None, None, True, float_out=fo)
    else:
        img.copy_(torch.from_numpy(comp[0]))
        launch_renderer(tree, cam, opt, img, torch.from_numpy(comp[1]).cuda(), None, False, float_out=fo)
    torch.cuda.synchronize()
    return fo.cpu().numpy(), img.cpu().numpy()


def _kernels(tree):
    from volrend_b200 import lib
    kbd = tree.info()["kernel_basis"]
    return {k: v for k, v in KERNELS.items() if lib().vr_variant_supported(kbd, v)}


class _Variant:
    def __init__(self, v):
        self.v = v

    def __enter__(self):
        from volrend_b200 import lib
        assert lib().vr_set_variant(self.v) == 0

    def __exit__(self, *a):
        from volrend_b200 import lib
        lib().vr_set_variant(0)


_RELAID = {}


def _relaid(name, layout):
    """(canonical SynthTree, its quantised npz or None, Relaid), cached for the module."""
    if (name, layout) not in _RELAID:
        st, npz = ec.edge_tree(name)
        _RELAID[(name, layout)] = (st, npz, lc.relayout(st, layout, npz, seed=SEED))
    return _RELAID[(name, layout)]


# ----------------------------------------------------------------------------------------------------------- render
@pytest.mark.parametrize("name,layout,parity", RENDER, ids=_ids(RENDER))
def test_render_equals_reference_frames(built, name, layout, parity):
    """Single views of both product kernels (where built for the basis) against the reference's stored frames; with
    every frame of the tree, also one batch of the 40x30 offscreen frames with options per view."""
    import torch
    from volrend_b200 import RenderOptions, render_batch
    _, _, r = _relaid(name, layout)
    tree = _load(r.arrays(), name, parity)
    frames = ec.frames_of(name) if layout in FULL else ec.frames_of(name)[:1]
    ks = _kernels(tree)
    assert ks
    for kname, v in ks.items():
        with _Variant(v):
            singles = {}
            for fr in frames:
                _, W, H, fx, fy, pose, kw, comp = ec.frame(fr, r.st)
                cam, opt = _cam(W, H, fx, fy, pose), RenderOptions(**kw)
                f, u = _single(tree, cam, opt, comp)
                ec.assert_identical(fr, f, u)
                singles[fr] = (f, u, cam, opt, comp)
            if layout not in FULL:
                continue
            off = [fr for fr, s in singles.items() if s[4] is None and (s[2].width, s[2].height) == (ec.W0, ec.H0)]
            imgs = torch.zeros((len(off), ec.H0, ec.W0, 4), dtype=torch.uint8, device="cuda")
            fos = torch.zeros((len(off), ec.H0, ec.W0, 4), dtype=torch.float32, device="cuda")
            render_batch(tree, [singles[fr][2] for fr in off], [singles[fr][3] for fr in off], imgs, float_out=fos)
            torch.cuda.synchronize()
            for i, fr in enumerate(off):
                _same(fos[i].cpu().numpy(), singles[fr][0], (fr, kname, "batch, options per view"))
                _same(imgs[i].cpu().numpy(), singles[fr][1], (fr, kname, "batch bytes, options per view"))


@pytest.mark.parametrize("name", [t for t in ec.TREES if t != "quant_mixed"])
def test_reference_renders_dirty_tree(built, tmp_path, name):
    """The reference loader and kernel on the written dirty tree (free nodes, one with links outside the array): the
    stored frames, so that the reference itself renders the relaid tree as the canonical one."""
    from oracle import ref_binding as rb
    from volrend_b200 import synth
    if not rb.available():
        pytest.skip("reference build (oracle/_ref) not present")
    _, _, r = _relaid(name, "dirty")
    path = str(tmp_path / f"{name}.npz")
    ec.write_tree_file(name, r.st, None, path)
    rt = rb.RefTree(path)
    try:
        for fr in ec.frames_of(name):
            _, W, H, fx, fy, pose, kw, comp = ec.frame(fr, r.st)
            rin, din = comp if comp is not None else (None, None)
            c12 = synth.c2w_to_colmajor12(pose)
            f = rt.render_f32(W, H, fx, fy, c12, rb.make_options(**kw), rgba_in=rin, depth_in=din)
            u = rt.render_u8(W, H, fx, fy, c12, rb.make_options(**kw), rgba_in=rin, depth_in=din)
            ec.assert_identical(fr, f, u)
    finally:
        rt.close()


# -------------------------------------------------------------------------------------------------- query / eval
def _query(tree, pts, rows=True):
    """vr_tree_query -> (data rows or None, cube_sz) of world points ``pts``."""
    import torch
    from volrend_b200 import _capi, lib
    x = torch.from_numpy(np.ascontiguousarray(pts, np.float32)).cuda()
    n = x.shape[0]
    data = torch.empty((n, tree.data_dim), dtype=torch.float16, device="cuda") if rows else None
    cube = torch.empty(n, dtype=torch.float32, device="cuda")
    _capi.check(lib().vr_tree_query(tree._handle, x.data_ptr(), n, data.data_ptr() if rows else None,
                                    cube.data_ptr(), None, None))
    torch.cuda.synchronize()
    return (data.cpu().numpy() if rows else None), cube.cpu().numpy()


def _probe(tree, p):
    import torch
    from volrend_b200 import _capi, lib
    kbd = tree.info()["kernel_basis"]
    out = torch.full((3 * max(kbd, 1),), float("nan"), dtype=torch.float32, device="cuda")
    _capi.check(lib().vr_probe_lumisphere(tree._handle, (C.c_float * 3)(*[float(v) for v in p]), out.data_ptr(), None))
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("name,layout", TREE_LAYOUTS, ids=_ids(TREE_LAYOUTS))
@pytest.mark.parametrize("parity", [0, 1])
def test_query_eval_probe_at_every_leaf(built, name, layout, parity):
    """vr_tree_query at the centre of every leaf returns the leaf's own row and cube size (every table entry and record
    the build wrote), as query_oracle does on the relaid arrays; vr_tree_eval there along random directions, and
    vr_probe_lumisphere at some of them, equal the canonical tree's."""
    st, npz, r = _relaid(name, layout)
    slots, depth, centres = lc.leaf_centres(st)
    pts = lc.centre_points(st, centres, depth)
    tree = _load(r.arrays(), name, parity, ndc=False)
    canon = _load(ec.tree_file_arrays(st, npz), name, parity, ndc=False)
    wide = layout == "wide"
    rows, cube = _query(tree, pts, rows=not wide)
    assert np.array_equal(_bits(cube), _bits((2.0 ** depth).astype(np.float32)))
    orows, ocube, _ = qo.query(r.st.child, r.st.data, r.st.offset, r.st.invradius3, pts)
    assert np.array_equal(_bits(cube), _bits(ocube))
    if not wide:
        assert np.array_equal(_bits(rows), _bits(st.data.reshape(-1, st.data_dim)[slots]))
        assert np.array_equal(_bits(rows), _bits(orows))
    dirs = np.random.default_rng(len(pts)).standard_normal((len(pts), 3)).astype(np.float32)
    from volrend_b200 import RenderOptions
    opt = RenderOptions()
    rgb, sigma = tree.eval(pts, dirs, opt)
    rgb0, sigma0 = canon.eval(pts, dirs, opt)
    _same(rgb, rgb0, "eval rgb")
    _same(sigma, sigma0, "eval sigma")
    for i in np.linspace(0, len(pts) - 1, 6).astype(int):
        _same(_probe(tree, pts[i]), _probe(canon, pts[i]), ("probe", i))


# --------------------------------------------------------------------------------------------------- leaf weights
@pytest.mark.parametrize("name,layout", TREE_LAYOUTS, ids=_ids(TREE_LAYOUTS))
def test_leaf_weights_follow_the_slot_map(built, name, layout):
    """Each relaid slot's weight is the canonical weight of its mapped slot, bit for bit; free nodes, internal slots
    and unshaded leaves stay -inf.  Tables are numbered by node index, so this checks the table entry -> slot map when
    table order is not node order."""
    from volrend_b200 import RenderOptions, leaf_weights
    st, npz, r = _relaid(name, layout)
    views = [v for v in ec.views_for(name) if v != "composite"][:3]
    cams = []
    for v in views:
        W, H, fx, fy, pose, _, _ = ec.view(v, name, st)
        if (W, H) == (ec.W0, ec.H0):
            cams.append(_cam(W, H, fx, fy, pose))
    assert cams
    for parity in (0, 1):
        canon = _load(ec.tree_file_arrays(st, npz), name, parity, slot_map=True)
        tree = _load(r.arrays(), name, parity, slot_map=True)
        w0 = leaf_weights(canon, cams, RenderOptions()).cpu().numpy().reshape(-1)
        w1 = leaf_weights(tree, cams, RenderOptions()).cpu().numpy().reshape(-1)
        m = r.slot_map
        assert np.isfinite(w0).any(), name
        _same(w1[m >= 0], w0[m[m >= 0]], (name, layout, parity))
        assert np.isneginf(w1[m < 0]).all()
        inner = r.st.child.reshape(-1) != 0
        assert np.isneginf(w1[inner]).all()


# ------------------------------------------------------------------------------------------------------ wireframe
@pytest.mark.parametrize("name,layout", WIRE, ids=_ids(WIRE))
def test_wireframe_equals_canonical_and_reference(built, name, layout):
    from volrend_b200 import N3Tree
    st = wire_tree(name)
    r = lc.relayout(st, layout, seed=SEED)
    canon = N3Tree.from_synth(st)
    for parity in (0, 1):
        tree = _load(r.arrays(), parity=parity)
        for d in (-1, 2, st.depth):
            v = tree.gen_wireframe(d)
            _same(v, canon.gen_wireframe(d), (name, layout, parity, d))
            assert matches(np.load(os.path.join(ROOT, "tests", "golden", "ref", golden_name(name, d) + ".npz")), v)


@pytest.mark.parametrize("name", [t for t in ec.TREES if t != "quant_mixed"])
def test_wireframe_of_edge_trees(built, name):
    st = ec.edge_tree(name)[0]
    canon = _load(st.npz_dict(), name)
    for layout in ("reverse", "dirty"):
        tree = _load(_relaid(name, layout)[2].arrays(), name)
        for d in (-1, 2, st.depth):
            _same(tree.gen_wireframe(d), canon.gen_wireframe(d), (name, layout, d))


# ---------------------------------------------------------------------------------------------------------- prune
@pytest.mark.parametrize("layout", lc.LAYOUTS)
@pytest.mark.parametrize("collapse", [False, True])
def test_pruned_relaid_tree_renders_as_pruned_canonical(built, layout, collapse):
    """prune_arrays of the relaid tree with its own weights (the canonical ones through the slot map) renders the
    bytes and floats of the pruned canonical tree."""
    from volrend_b200 import RenderOptions, leaf_weights, prune_arrays
    name = "mixed_sh16"
    st, _, r = _relaid(name, layout)
    frames = [f"{name}.{v}.default" for v in ("px", "nz", "inside", "face")]
    cams = [_cam(*ec.frame(fr, st)[1:6]) for fr in frames]
    outs = []
    for s in (st, r.st):
        t = _load(s.npz_dict(), slot_map=True)
        w = leaf_weights(t, cams, RenderOptions()).cpu().numpy()
        if s is r.st:
            _same(w.reshape(-1)[r.slot_map >= 0], outs[0][2][r.slot_map[r.slot_map >= 0]], "weights")
        child, data = prune_arrays(s.child, s.data, w, 1e-3, collapse=collapse)
        p = _load(dict(s.npz_dict(), child=child, data=data))
        outs.append(([_single(p, c, RenderOptions(), None) for c in cams], child.shape[0], w.reshape(-1)))
    (a, ca, _), (b, cb, _) = outs
    assert ca == cb
    for fr, (fa, ua), (fb, ub) in zip(frames, a, b):
        _same(fa, fb, (fr, "pruned floats"))
        _same(ua, ub, (fr, "pruned bytes"))


# ------------------------------------------------------------------------------------------------------ quantised
QUANT = [("SG", 7, 0), ("SG", 7, 1), ("SH", 1, 0)]


@pytest.mark.parametrize("fmt,basis,n_retain", QUANT, ids=[f"{f}{b}-r{n}" for f, b, n in QUANT])
@pytest.mark.parametrize("layout", ["canonical", "shuffle"])
def test_quantised_one_basis_kernel(built, fmt, basis, n_retain, layout):
    """Quantised trees whose kernel keeps one coefficient per channel (SG7: no 7-basis build; SH1), with no or one
    retained basis function: the GPU decode renders and probes exactly what the host decode does."""
    from volrend_b200 import RenderOptions, synth
    st = synth.make_tree("lego", depth=5, basis_dim=basis, seed=30 + basis + n_retain, fmt=fmt)
    npz = synth.quantise_tree(st, n_retain=n_retain, seed=4)
    if layout != "canonical":
        npz = lc.relayout(st, layout, npz, seed=SEED).npz
    g, h = _load(npz), _load(npz, gpu_decode=False)
    assert g._data is None and h._data is not None and g.info()["kernel_basis"] == 1
    cams = [_cam(64, 48, synth.focal_for(64), synth.focal_for(64), p) for p in synth.nerf_synthetic_test_poses(8)[2:5]]
    for v in _kernels(g).values():
        with _Variant(v):
            for c in cams:
                fg, ug = _single(g, c, RenderOptions(), None)
                fh, uh = _single(h, c, RenderOptions(), None)
                assert (fg[..., 3] > 0).any()
                _same(fg, fh, "GPU decode floats")
                _same(ug, uh, "GPU decode bytes")
    if fmt == "SH":
        for p in ([0.05, -0.1, 0.02], [0.3, 0.2, -0.1], [-0.2, 0.1, 0.25]):
            _same(_probe(g, p), _probe(h, p), ("probe", p))


# ---------------------------------------------------------------------------------------------------------- scale
def test_bench_tree_shuffled_equals_reference_frame(built):
    """The bench-size tree (1.4 M nodes: the chunked multi-threaded upload, the table scan at size) shuffled: pose 77
    at 800x800 equals the reference's stored frame of the canonical tree."""
    from volrend_b200 import RenderOptions, synth
    st = synth.make_tree("lego", depth=10, basis_dim=16, seed=0)
    r = lc.relayout(st, "shuffle", seed=SEED)
    del st
    tree = _load(r.arrays())
    W, H, fx, pose = gc.ref_frame_view("config2_v77")
    f, u = _single(tree, _cam(W, H, fx, fx, pose), RenderOptions(), None)
    gc.assert_matches_ref_frame("config2_v77", f, u, 0.0)


# ------------------------------------------------------------------------------------------------------- refusals
def _padded(st, extra_nodes=2_000_000):
    """``st`` with unreachable all-zero nodes appended, so that an upload that is not freed shows in the device's free
    memory (~0.2 GB per attempt for an RGBA tree)."""
    from dataclasses import replace
    dd = st.data_dim
    return replace(st, child=np.concatenate([st.child, np.zeros((extra_nodes, 2, 2, 2), np.int32)]),
                   data=np.concatenate([st.data, np.zeros((extra_nodes, 2, 2, 2, dd), np.float16)]), meta={})


def test_malformed_trees_are_refused_cleanly(built):
    """A defect the root reaches -- a link > capacity, == capacity, < 0 or to the root; a second parent at the same or
    another level; a cycle among non-root nodes -- is refused with VR_EINVAL and the build's message.  No march runs,
    every allocation of the attempt is freed, and the same tree without the defect loads."""
    import torch
    from volrend_b200 import N3Tree, VolrendError, _capi, lib
    st = _padded(ec.edge_tree("mixed_rgba")[0])
    cases = lc.malformed(st)
    assert len(cases) == 7

    def refuse(bad, msg):
        with pytest.raises(VolrendError) as e:
            N3Tree.from_synth(bad)
        assert e.value.code == _capi.VR_EINVAL and msg in str(e.value), str(e.value)

    first = next(iter(cases.values()))
    refuse(*first)                              # one-time allocations of the uploader
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    n0 = lib().vr_launch_count()
    for name, (bad, msg) in cases.items():
        refuse(bad, msg)
        refuse(bad, msg)
    torch.cuda.synchronize()
    assert lib().vr_launch_count() == n0
    assert torch.cuda.mem_get_info()[0] >= free0 - (128 << 20), "a refused upload kept device memory"
    assert N3Tree.from_synth(st).info()["capacity"] == st.capacity


def test_defects_in_free_nodes_are_accepted(built):
    """The malformed trees' defects placed in free nodes only (the dirty layout): accepted, capacity counts them."""
    st = ec.edge_tree("mixed_rgba")[0]
    r = lc.relayout(st, "dirty", seed=11)
    tree = _load(r.arrays())
    assert tree.info()["capacity"] == r.st.capacity > st.capacity
    fr = "mixed_rgba.px.default"
    _, W, H, fx, fy, pose, kw, _ = ec.frame(fr, st)
    from volrend_b200 import RenderOptions
    f, u = _single(tree, _cam(W, H, fx, fy, pose), RenderOptions(**kw), None)
    ec.assert_identical(fr, f, u)
