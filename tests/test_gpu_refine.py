"""`-m gpu`: the leaf-error pass (vr_tree_leaf_error), refined trees on the device and the coarse-to-fine fit
(volrend_b200.refine, finetune(refine_every=K)) on an H100.

The error sums are compared with the CPU restatement (oracle/error_oracle.c, orc_leaf_error, double): the set of slots
that receive terms exactly (the GPU buffer starts at -0, which a term of +0 turns into +0; errors are positive), the
values within 1e-4 * A + 1e-7, A being the sum of the absolute terms of the slot (the GPU adds its terms in float, in
the order its atomics land), and the work counters exactly."""
import ctypes as C
import os

import numpy as np
import pytest

import edge_cases as ec
import golden_cases as gc
import layout_cases as lc
from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)

pytestmark = pytest.mark.gpu
RTOL, ATOL = 1e-4, 1e-7
WEIGHT_TOL = 2e-6       # |GPU weight - oracle weight| (tests/test_gpu_leaf_weights.py)
NEG0 = 0x80000000
# |refined - original| of a float render, as tests/test_refine_cpu.py measured it with the march oracle (default step)
RENDER_DIFF = 0.01


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


def _err(n, H, W, seed):
    import torch
    g = torch.Generator().manual_seed(seed)
    return (torch.rand((n, H, W), generator=g) * 1.75 + 0.25).cuda()


def _gpu(tree, cams, opt, err, out=None, tile=None):
    """-> (score tensor, counters list); a new score buffer starts at -0."""
    import torch
    from volrend_b200 import leaf_error
    if out is None:
        out = torch.full((tree.capacity * 8,), -0.0, dtype=torch.float32, device="cuda")
    cnt = torch.zeros(5, dtype=torch.int64, device="cuda")
    leaf_error(tree, cams, opt, err, out=out, counters=cnt, tile=tile)
    torch.cuda.synchronize()
    return out, cnt.cpu().tolist()


def _close_to_oracle(g, score, absum, hits, err_max, what):
    g = g.cpu().numpy().reshape(-1)
    touched = g.view(np.uint32) != NEG0
    assert np.array_equal(touched, hits > 0), (what, "slots with terms differ", int((touched != (hits > 0)).sum()))
    d = np.abs(g.astype(np.float64) - score)
    # plus, per term, the weights pass's tolerance (WEIGHT_TOL) times the error: where att is within an ulp or two of
    # 1 (sigma_thresh 0 lets sigma ~ 0 through), 1 - att carries the difference of glibc's and libdevice's expf
    tol = RTOL * absum + ATOL + WEIGHT_TOL * err_max * hits
    assert (d <= tol).all(), (what, float((d - tol).max()))


def _check_view(tree, st, W, H, fx, fy, pose, kw, ndc, what, seed=0, tile=None):
    from oracle import binding as ob
    from oracle import error_binding as eb
    from volrend_b200 import RenderOptions, synth
    w, h = (tile[2], tile[3]) if tile else (W, H)
    err = _err(1, h, w, seed)
    g, cnt = _gpu(tree, [_cam(W, H, fx, fy, pose)], RenderOptions(**kw), err, tile=tile)
    ot = ob.OracleTree.from_synth(st, ndc=ndc)
    oc = ob.make_camera(W, H, fx, fy, synth.c2w_to_colmajor12(pose))
    score, absum, hits, oc_ = eb.leaf_error(ot, oc, ob.make_options(**kw), err[0].cpu().numpy(), tile=tile)
    _close_to_oracle(g, score, absum, hits, float(err.max()), what)
    assert cnt[:4] == [oc_["samples"], oc_["child_loads"], oc_["shaded"], oc_["rays_hit"]], (what, cnt, oc_)


GOLDEN = [(n, p) for n in gc.CASES for p in (0, 1)]


@pytest.mark.parametrize("name,parity", GOLDEN, ids=[f"{n}-{p}" for n, p in GOLDEN])
def test_golden_trees_match_oracle(built, name, parity):
    from volrend_b200 import synth
    st, W, H, pose, kw, ndc = gc.build_case(name)
    tree = _device_tree(st, ndc=ndc, parity=parity)
    f = synth.focal_for(W)
    for s in (1e-2, 0.0, -1.0):
        _check_view(tree, st, W, H, f, f, pose, dict(kw, sigma_thresh=s), ndc, f"{name} sigma_thresh {s}")


EDGE = [(n, p) for n in ec.TREES for p in (0, 1)]


@pytest.mark.parametrize("name,parity", EDGE, ids=[f"{n}-{p}" for n, p in EDGE])
def test_edge_trees_match_oracle(built, name, parity):
    st, npz = ec.edge_tree(name)              # quant_mixed: created quantised
    ndc = ec.NDC.get(name)
    tree = _device_tree(st, npz, ndc, parity)
    for i, v in enumerate(ec.views_for(name)):
        if v == "composite":
            continue
        W, H, fx, fy, pose, kw, _ = ec.view(v, name, st)
        for s in (1e-2, 0.0, -1.0):
            _check_view(tree, st, W, H, fx, fy, pose, dict(kw, sigma_thresh=s), ndc, f"{name}.{v} {s}", seed=i)


@pytest.fixture(scope="module")
def orbit():
    from volrend_b200 import RenderOptions, synth
    st, _, _, _, _, _ = gc.build_case("lego_sh16")
    tree = _device_tree(st)
    cams = [_cam(64, 48, synth.focal_for(64), synth.focal_for(64), p) for p in synth.nerf_synthetic_test_poses(24)]
    return st, tree, cams, RenderOptions()


def test_split_order_and_linearity(built, orbit):
    from oracle import binding as ob
    from oracle import error_binding as eb
    from volrend_b200 import synth
    st, tree, cams, opt = orbit
    err = _err(len(cams), 48, 64, 3)
    ot = ob.OracleTree.from_synth(st)
    score, absum, hits = np.zeros(st.capacity * 8), np.zeros(st.capacity * 8), np.zeros(st.capacity * 8)
    for v, c in enumerate(cams):
        oc = ob.make_camera(64, 48, c.fx, c.fy, synth.c2w_to_colmajor12(c.transform.T))
        s, a, h, _ = eb.leaf_error(ot, oc, ob.make_options(), err[v].cpu().numpy())
        score += s
        absum += a
        hits += h
    all_, _ = _gpu(tree, cams, opt, err)
    split, _ = _gpu(tree, cams[:10], opt, err[:10])
    split, _ = _gpu(tree, cams[10:], opt, err[10:], out=split)
    rev, _ = _gpu(tree, cams[::-1], opt, err.flip(0).contiguous())
    twice, _ = _gpu(tree, cams, opt, (err * 2).contiguous())
    tol = RTOL * absum + ATOL
    assert (np.abs(all_.cpu().numpy() - score) <= tol + WEIGHT_TOL * float(err.max()) * hits).all()
    a = all_.cpu().numpy().astype(np.float64)
    for other, k, what in ((split, 1, "split"), (rev, 1, "reversed"), (twice, 2, "2 err")):
        d = np.abs(other.cpu().numpy() - k * a)
        assert (d <= 2 * k * tol).all(), (what, float(d.max()))
    assert a.max() > 0


def test_tile_matches_oracle(built, orbit):
    st, tree, cams, opt = orbit
    c = cams[5]
    _check_view(tree, st, 64, 48, c.fx, c.fy, c.transform.T, {}, None, "tile", tile=(9, 7, 33, 26))


def test_counters_equal_the_weights_pass(built, orbit):
    import torch
    from volrend_b200 import leaf_weights
    st, tree, cams, opt = orbit
    err = _err(len(cams), 48, 64, 4)
    err[:, :, :20] = 0.0                                    # err 0: the same rays are marched
    g, ecnt = _gpu(tree, cams, opt, err)
    wcnt = torch.zeros(5, dtype=torch.int64, device="cuda")
    w = leaf_weights(tree, cams, opt, counters=wcnt)
    torch.cuda.synchronize()
    assert ecnt == wcnt.cpu().tolist()
    assert np.array_equal(g.cpu().numpy().view(np.uint32) != NEG0, ~np.isneginf(w.cpu().numpy().reshape(-1)))


def test_refusals(built):
    import torch
    from volrend_b200 import RenderOptions, _capi, leaf_error, lib, synth
    st = synth.make_tree("lego", depth=4, basis_dim=4, seed=33)
    cams = [_cam(16, 8, 20.0, 20.0, p) for p in synth.nerf_synthetic_test_poses(2)]
    err = _err(2, 8, 16, 0)
    plain = _device_tree(st, slot_map=False)
    with pytest.raises(RuntimeError, match="slot map"):
        leaf_error(plain, cams, RenderOptions(), err)
    L = lib()
    arr = (_capi.vr_camera * 2)(*[c._as_c() for c in cams])
    o = RenderOptions()._as_c()
    s = torch.zeros(st.capacity * 8, dtype=torch.float32, device="cuda")
    assert L.vr_tree_leaf_error(plain._handle, arr, 2, C.byref(o), None, err.data_ptr(), s.data_ptr(), None,
                                None) == _capi.VR_EUNSUPPORTED
    assert b"slot map" in L.vr_last_error()
    tree = _device_tree(st)
    assert L.vr_tree_leaf_error(tree._handle, arr, 2, C.byref(o), None, None, s.data_ptr(), None,
                                None) == _capi.VR_EINVAL
    assert L.vr_tree_leaf_error(tree._handle, arr, 2, C.byref(o), None, err.data_ptr(), None, None,
                                None) == _capi.VR_EINVAL
    host = np.zeros(err.numel(), np.float32)
    assert L.vr_tree_leaf_error(tree._handle, arr, 2, C.byref(o), None, host.ctypes.data, s.data_ptr(), None,
                                None) == _capi.VR_EINVAL
    assert L.vr_tree_leaf_error(tree._handle, arr, 2, C.byref(o), None, err.data_ptr(), host.ctypes.data, None,
                                None) == _capi.VR_EINVAL
    cnt = np.zeros(5, np.int64)
    assert L.vr_tree_leaf_error(tree._handle, arr, 2, C.byref(o), None, err.data_ptr(), s.data_ptr(), cnt.ctypes.data,
                                None) == _capi.VR_EINVAL
    assert b"counters_dev" in L.vr_last_error()
    assert not s.any()
    with pytest.raises(ValueError, match="err"):
        leaf_error(tree, cams, RenderOptions(), err[:1])
    with pytest.raises(ValueError, match="err"):
        leaf_error(tree, cams, RenderOptions(), err.cpu())
    with pytest.raises(ValueError, match="out"):
        leaf_error(tree, cams, RenderOptions(), err, out=s[:-1])


# ------------------------------------------------------------------------------------------- refined trees
def _refined(st, fraction, seed):
    from volrend_b200 import refine_npz, synth
    rng = np.random.default_rng(seed)
    z = refine_npz(st.npz_dict(), rng.random(st.capacity * 8).astype(np.float32), fraction)
    return z, synth.SynthTree(child=z["child"], data=z["data"], offset=st.offset, invradius3=st.invradius3,
                              data_dim=st.data_dim, data_format=st.data_format, depth=st.depth, extra=st.extra)


def _render_float(tree, cams, opt):
    import torch
    from volrend_b200 import render_batch
    fo = torch.empty((len(cams), cams[0].height, cams[0].width, 4), dtype=torch.float32, device="cuda")
    render_batch(tree, cams, opt, None, float_out=fo)
    torch.cuda.synchronize()
    return fo.cpu().numpy()


REFINED = [(n, p) for n in ("lego_sh16", "lego_rgba", "lego_asg4", "lego_sh16_ndc", "cfg1_sh1") for p in (0, 1)]


@pytest.mark.parametrize("name,parity", REFINED, ids=[f"{n}-{p}" for n, p in REFINED])
def test_refined_tree_renders_and_queries(built, name, parity, tmp_path):
    from oracle import binding as ob
    from oracle import ref_binding as rb
    from volrend_b200 import RenderOptions, synth
    from volrend_b200.compress import _write_npz
    st, W, H, pose, kw, ndc = gc.build_case(name)
    z, r = _refined(st, 0.3, parity)
    assert r.capacity > st.capacity
    tree = _device_tree(r, ndc=ndc, parity=parity)
    f = synth.focal_for(W)
    fo = _render_float(tree, [_cam(W, H, f, f, pose)], RenderOptions(**kw))[0]
    oc = ob.make_camera(W, H, f, f, synth.c2w_to_colmajor12(pose))
    of, _, _ = ob.render(ob.OracleTree.from_synth(r, ndc=ndc), oc, ob.make_options(**kw))
    assert np.abs(fo - of).max() <= 2e-6, float(np.abs(fo - of).max())
    orig = _render_float(_device_tree(st, ndc=ndc, parity=parity), [_cam(W, H, f, f, pose)], RenderOptions(**kw))[0]
    assert np.abs(fo - orig).max() <= RENDER_DIFF
    # every leaf of a new node holds its parent's row where vr_tree_query finds it
    slots, depth, centres = lc.leaf_centres(r)
    new = slots >= st.capacity * 8
    pts = lc.centre_points(r, centres[new], depth[new])
    rows = tree.query(pts)[0]
    parent = st.data.reshape(-1, st.data_dim)[_src(st, r)[slots[new]]]
    assert np.array_equal(np.asarray(rows).view(np.uint16), parent.view(np.uint16))
    if rb.available() and ndc is None:
        path = str(tmp_path / "refined.npz")
        _write_npz(path, z)
        ref = rb.RefTree(path)
        try:
            cam = _cam(W, H, f, f, pose)
            rf = ref.render_f32(W, H, f, f, cam.transform.reshape(12), rb.make_options(**kw))
            ours = _render_float(_device_tree(r, parity=parity), [cam], RenderOptions(**kw))[0]
            assert np.array_equal(ours.view(np.uint32), rf.view(np.uint32)), "our kernel vs the reference kernel"
        finally:
            ref.close()


def _src(st, r):
    """Source slot of every slot of the refined tree r of st: its parent slot for the new nodes' slots."""
    cap = st.capacity
    src = np.arange(r.capacity * 8)
    ch = np.asarray(r.child).reshape(-1)
    for s in range(cap * 8):
        if ch[s] != 0 and np.asarray(st.child).reshape(-1)[s] == 0:
            src[(s // 8 + ch[s]) * 8:(s // 8 + ch[s]) * 8 + 8] = s
    return src


def test_chain22_refined_to_the_cap_loads_and_renders(built):
    from oracle import binding as ob
    from volrend_b200 import RenderOptions, refine_npz, synth
    st, _ = ec.edge_tree("chain22")
    z = refine_npz(st.npz_dict(), np.ones(st.capacity * 8, np.float32), 1.0)
    r = synth.SynthTree(child=z["child"], data=z["data"], offset=st.offset, invradius3=st.invradius3,
                        data_dim=st.data_dim, data_format=st.data_format, depth=23)
    for parity in (0, 1):
        tree = _device_tree(r, parity=parity)
        assert tree.info()["max_depth"] == 23
        W, H, fx, fy, pose, kw, _ = ec.view("deep", "chain22", st)
        fo = _render_float(tree, [_cam(W, H, fx, fy, pose)], RenderOptions(**kw))[0]
        oc = ob.make_camera(W, H, fx, fy, synth.c2w_to_colmajor12(pose))
        of, _, _ = ob.render(ob.OracleTree.from_synth(r), oc, ob.make_options(**kw))
        assert np.abs(fo - of).max() <= 2e-6


# ------------------------------------------------------------------------------------------- coarse-to-fine fit
def _coarse_setup():
    """Targets: renders of a seeded depth-6 tree, 64x64, 24 poses.  Start: that tree with its deepest level averaged
    into its parents."""
    import torch
    from volrend_b200 import RenderOptions, prune, prune_arrays, synth
    fine = synth.make_tree("lego", depth=6, basis_dim=9, seed=7)
    W = H = 64
    f = synth.focal_for(W)
    cams = [_cam(W, H, f, f, p) for p in synth.nerf_synthetic_test_poses(24)]
    opt = RenderOptions()
    targets = torch.from_numpy(_render_float(_device_tree(fine), cams, opt)[..., :3].copy())
    levels, target = prune._structure(fine.child)
    cap, dd = fine.capacity, fine.data_dim
    child = fine.child.reshape(cap * 8).copy()
    data = fine.data.reshape(cap * 8, dd).astype(np.float32)
    parents = np.flatnonzero(np.isin(target, levels[-1]))
    rows = data.reshape(cap, 8, dd)[target[parents]].mean(1)
    child[parents] = 0
    data[parents] = rows
    c, d = prune_arrays(child.reshape(cap, 2, 2, 2), data.astype(np.float16).reshape(cap, 2, 2, 2, dd),
                        np.full(cap * 8, np.inf, np.float32), 0.0, collapse=False)
    coarse = synth.SynthTree(child=c, data=d, offset=fine.offset, invradius3=fine.invradius3, data_dim=dd,
                             data_format=fine.data_format, depth=5, extra=fine.extra)
    return coarse, cams, targets, opt


def _psnr(tree, cams, targets, opt):
    f = _render_float(tree, cams, opt)[..., :3]
    return -10 * np.log10(float(((f - targets.numpy()) ** 2).mean()))


def _loss(tree, cams, targets, opt):
    f = _render_float(tree, cams, opt)[..., :3]
    return float(((f - targets.numpy()) ** 2).mean())


def test_fit_through_a_refinement(built, monkeypatch):
    import importlib
    import torch
    ft = importlib.import_module("volrend_b200.finetune")   # the package exports the function of that name
    from volrend_b200 import finetune
    coarse, cams, targets, opt = _coarse_setup()
    train = cams[:20]
    tree = _device_tree(coarse)
    seen, losses = [], {}
    gather = ft._gather_fit

    def spy(master, adam, lr, src):
        new, adam2 = gather(master, adam, lr, src)
        seen.append((master.detach().clone(), {k: v.clone() for k, v in adam.state[master].items()},
                     src.clone(), new.detach().clone(), {k: v.clone() for k, v in adam2.state[new].items()}))
        return new, adam2

    monkeypatch.setattr(ft, "_gather_fit", spy)
    refines = []
    master, _ = finetune(tree, train, targets[:20], opt, steps=12, lr=1e-2, batch=4, seed=0, refine_every=5,
                         refine_fraction=0.2,
                         on_step=lambda s, l: losses.__setitem__(s, _loss(tree, train, targets[:20], opt)),
                         on_refine=lambda s, n, a, b: refines.append((s, n, a, b,
                                                                      _loss(tree, train, targets[:20], opt))))
    assert [r[0] for r in refines] == [5, 10] and len(seen) == 2
    for (s, n, a, b, after), (m0, st0, src, m1, st1) in zip(refines, seen):
        assert n > 0 and b == a + n
        dd = m0.shape[-1]
        src = src.cpu()
        for x0, x1 in ((m0, m1), (st0["exp_avg"], st1["exp_avg"]), (st0["exp_avg_sq"], st1["exp_avg_sq"])):
            x0, x1 = x0.reshape(-1, dd).cpu(), x1.reshape(-1, dd).cpu()
            assert torch.equal(x1[: a * 8], x0) and torch.equal(x1[a * 8:], x0[src[a * 8:]])
        assert float(st1["step"]) == float(st0["step"]) == s
        before = losses[s - 1]
        bound = 2 * np.sqrt(before) * RENDER_DIFF + RENDER_DIFF ** 2
        print(f"refine before step {s}: split {n}, nodes {a} -> {b}, loss {before:.6g} -> {after:.6g}")
        assert abs(after - before) <= bound, (before, after, bound)
    assert tuple(master.shape) == (tree.capacity, 2, 2, 2, coarse.data_dim)
    assert tree.child_.shape[0] == tree.capacity == refines[-1][3]


def test_end_to_end_coarse_to_fine(built):
    from volrend_b200 import finetune
    coarse, cams, targets, opt = _coarse_setup()
    train, held = cams[:20], cams[20:]
    out = {}
    for K in (0, 40):
        tree = _device_tree(coarse)
        p0 = _psnr(tree, held, targets[20:], opt)
        master, losses = finetune(tree, train, targets[:20], opt, steps=200, lr=1e-2, batch=4, seed=0,
                                  refine_every=K, refine_fraction=0.3)
        out[K] = (_loss(tree, train, targets[:20], opt), p0, _psnr(tree, held, targets[20:], opt), tree.capacity)
        print(f"refine_every {K}: nodes {coarse.capacity} -> {tree.capacity}, training loss "
              f"{losses[0]:.6g} -> {out[K][0]:.6g}, held-out PSNR {p0:.3f} -> {out[K][2]:.3f} dB")
    assert out[40][3] > coarse.capacity and out[0][3] == coarse.capacity
    # first H100 run (DESIGN.md 19): without refinement loss 4.69e-3 -> 2.68e-3, held-out PSNR 23.32 -> 24.15 dB;
    # refining every 40 steps (805 -> 27 907 nodes) loss -> 1.80e-3, PSNR -> 24.72 dB
    assert out[40][0] < 0.85 * out[0][0], out
    assert out[40][2] > out[0][2] + 0.25, out


def test_clis_on_png_targets(built, tmp_path, capsys):
    import importlib
    from volrend_b200 import write_png_file
    rf = importlib.import_module("volrend_b200.refine")
    ft = importlib.import_module("volrend_b200.finetune")
    coarse, cams, targets, opt = _coarse_setup()
    cams, targets = cams[:6], targets[:6]
    src = str(tmp_path / "t.npz")
    np.savez(src, **coarse.npz_dict())
    poses, pngs = [], []
    for i, c in enumerate(cams):
        p = str(tmp_path / f"p{i}.txt")
        np.savetxt(p, np.vstack([c.transform.T, [0, 0, 0, 1]]))
        poses.append(p)
        img = np.concatenate([np.clip(targets[i].numpy() * 255 + 0.5, 0, 255).astype(np.uint8),
                              np.full((64, 64, 1), 255, np.uint8)], -1)
        png = str(tmp_path / f"t{i}.png")
        assert write_png_file(png, img)
        pngs.append(png)
    view = ["--width", "64", "--height", "64", "--fx", str(cams[0].fx)]
    out = str(tmp_path / "r.npz")
    assert rf.main([src, out] + poses + ["--targets"] + pngs + view + ["--fraction", "0.25", "--batch", "4"]) == 0
    text = capsys.readouterr().out
    n_split = int(text.split("split ")[1].split(";")[0])
    assert n_split > 0 and f"nodes {coarse.capacity} -> {coarse.capacity + n_split}" in text
    with np.load(out) as z:
        assert z["child"].shape[0] == coarse.capacity + n_split and z["data"].dtype == np.float16
    out2 = str(tmp_path / "f.npz")
    assert ft.main([src, out2] + poses + ["--targets"] + pngs + view +
                   ["--steps", "12", "--batch", "2", "--refine-every", "5", "--refine-fraction", "0.2"]) == 0
    text = capsys.readouterr().out
    assert text.count("refine before step") == 2 and text.count("step ") - 2 == 12
    last = int(text.rsplit("nodes ", 1)[1].split("-> ")[1].split()[0])
    with np.load(out2) as z:
        assert z["child"].shape[0] == last > coarse.capacity
        assert z["data"].shape == (last, 2, 2, 2, coarse.data_dim)
