"""`-m gpu`: the leaf-gradient pass (vr_tree_leaf_grads), the in-place leaf update (vr_tree_update_data) and the
fitting loop (volrend_b200.finetune) on an H100.

The gradients are compared with the CPU restatement (oracle/grads_oracle.c, orc_leaf_grads, double) within
1e-4 * A + 1e-7, A being the sum of the absolute values of the terms the oracle added into the element: the GPU adds its
terms in float, in the order its atomics land.  The replayed render is compared with vr_render_batch bit for bit, and
so is everything the update touches: renders, queries, evals and the probe against a tree created from the same data."""
import ctypes as C
import os

import numpy as np
import pytest

import edge_cases as ec
import golden_cases as gc
from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)

pytestmark = pytest.mark.gpu
RTOL, ATOL = 1e-4, 1e-7


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


def _dpix(n, H, W, seed):
    import torch
    g = torch.Generator().manual_seed(seed)
    return (torch.rand((n, H, W, 4), generator=g) * 2 - 1).cuda()


def _render_float(tree, cams, opt):
    import torch
    from volrend_b200 import render_batch
    fo = torch.empty((len(cams), cams[0].height, cams[0].width, 4), dtype=torch.float32, device="cuda")
    img = torch.empty((len(cams), cams[0].height, cams[0].width, 4), dtype=torch.uint8, device="cuda")
    render_batch(tree, cams, opt, img, float_out=fo)
    torch.cuda.synchronize()
    return fo.cpu().numpy(), img.cpu().numpy()


def _grads(tree, cams, opt, dpix, out=None):
    import torch
    from volrend_b200 import leaf_grads
    fo = torch.full(tuple(dpix.shape), float("nan"), dtype=torch.float32, device="cuda")
    out = leaf_grads(tree, cams, opt, dpix, out=out, float_out=fo)
    torch.cuda.synchronize()
    return out, fo.cpu().numpy()


def _check_view(tree, st, W, H, fx, fy, pose, kw, ndc, what, seed=0):
    from oracle import binding as ob
    from oracle import grads_binding as gb
    from volrend_b200 import RenderOptions, synth
    cam = _cam(W, H, fx, fy, pose)
    opt = RenderOptions(**kw)
    dpix = _dpix(1, H, W, seed)
    g, fo = _grads(tree, [cam], opt, dpix)
    ref, _ = _render_float(tree, [cam], opt)
    assert np.array_equal(fo.view(np.uint32), ref.view(np.uint32)), (what, "replay != vr_render_batch")
    ot = ob.OracleTree.from_synth(st, ndc=ndc)
    oc = ob.make_camera(W, H, fx, fy, synth.c2w_to_colmajor12(pose))
    og, oA, _ = gb.leaf_grads(ot, oc, ob.make_options(**kw), dpix[0].cpu().numpy())
    g = g.cpu().numpy().reshape(og.shape).astype(np.float64)
    d = np.abs(g - og)
    bad = d > RTOL * oA + ATOL
    assert not bad.any(), (what, int(bad.sum()), float(d.max()), np.argwhere(bad)[:5].tolist())
    assert np.abs(og).max() > 0 or not (oA > 0).any(), what
    return g, og


GOLDEN = [(n, p) for n in gc.CASES if n not in ("lego_sh9_depth", "lego_sh9_composite") for p in (0, 1)]


@pytest.mark.parametrize("name,parity", GOLDEN, ids=[f"{n}-{p}" for n, p in GOLDEN])
def test_golden_trees_match_oracle(built, name, parity):
    from volrend_b200 import synth
    st, W, H, pose, kw, ndc = gc.build_case(name)
    tree = _device_tree(st, ndc=ndc, parity=parity)
    f = synth.focal_for(W)
    _check_view(tree, st, W, H, f, f, pose, kw, ndc, name)


EDGE = [(n, p) for n in ec.TREES for p in (0, 1)]


@pytest.mark.parametrize("name,parity", EDGE, ids=[f"{n}-{p}" for n, p in EDGE])
def test_edge_trees_match_oracle(built, name, parity):
    st, npz = ec.edge_tree(name)
    ndc = ec.NDC.get(name)
    tree = _device_tree(st, npz, ndc, parity)
    n = 0
    for fr in ec.frames_of(name):
        _, W, H, fx, fy, pose, kw, comp = ec.frame(fr, st)
        if comp is not None or W * H > ec.WHOLE_MAX_PIXELS:
            continue
        _check_view(tree, st, W, H, fx, fy, pose, dict(kw, render_depth=0), ndc, fr, seed=n)
        n += 1
    assert n > 0


def _views(st_name="lego", n=6, W=48, H=40):
    from volrend_b200 import synth
    poses = synth.nerf_synthetic_test_poses(n)
    f = synth.focal_for(W)
    return [_cam(W, H, f, f, p) for p in poses]


def test_accumulation_split_order_and_linearity(built):
    from volrend_b200 import RenderOptions, synth
    st = synth.make_tree("lego", depth=5, basis_dim=9, seed=31)
    tree = _device_tree(st)
    cams = _views(n=6)
    opt = RenderOptions()
    dpix = _dpix(6, cams[0].height, cams[0].width, 5)
    from oracle import binding as ob
    from oracle import grads_binding as gb
    ot = ob.OracleTree.from_synth(st)
    oA = np.zeros((st.capacity * 8, st.data_dim))
    for v, c in enumerate(cams):
        oc = ob.make_camera(c.width, c.height, c.fx, c.fy, synth.c2w_to_colmajor12(synth.nerf_synthetic_test_poses(6)[v]))
        gb.leaf_grads(ot, oc, ob.make_options(), dpix[v].cpu().numpy(), A=oA)
    all_, _ = _grads(tree, cams, opt, dpix)
    split, _ = _grads(tree, cams[:2], opt, dpix[:2])
    split, _ = _grads(tree, cams[2:], opt, dpix[2:], out=split)
    rev, _ = _grads(tree, cams[::-1], opt, dpix.flip(0).contiguous())
    twice, _ = _grads(tree, cams, opt, (dpix * 2).contiguous())
    a = all_.cpu().numpy().reshape(oA.shape).astype(np.float64)
    tol = RTOL * oA + ATOL
    for other, k, what in ((split, 1, "split"), (rev, 1, "reversed"), (twice, 2, "2 dpix")):
        d = np.abs(other.cpu().numpy().reshape(oA.shape) - k * a)
        assert (d <= k * tol).all(), (what, float(d.max()))
    assert np.abs(a).max() > 0


def _query_state(tree, st):
    """Everything that reads the leaf values besides the march: vr_tree_query's rows, vr_tree_eval, the probe."""
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
    try:
        rgb, sig = tree.eval(pts, dirs, RenderOptions())
        out["eval"] = np.concatenate([rgb, sig[:, None]], 1).view(np.uint32)
    except VolrendError:
        pass
    probe = torch.full((75,), float("nan"), dtype=torch.float32, device="cuda")
    xyz = (C.c_float * 3)(*[float(v) for v in pts[0]])
    if lib().vr_probe_lumisphere(tree._handle, xyz, probe.data_ptr(), None) == 0:
        torch.cuda.synchronize()
        out["probe"] = probe.cpu().numpy().view(np.uint32)
    return out


UPDATE = [(n, p) for n in ("mixed_sh16", "mixed_sh1", "mixed_rgba", "mixed_sg9", "aniso_ndc", "sigma_bits",
                           "quant_mixed", "root_mixed") for p in (0, 1)]


@pytest.mark.parametrize("name,parity", UPDATE, ids=[f"{n}-{p}" for n, p in UPDATE])
def test_update_data_matches_a_fresh_tree(built, name, parity):
    import torch
    from volrend_b200 import RenderOptions
    st, npz = ec.edge_tree(name)
    ndc = ec.NDC.get(name)
    tree = _device_tree(st, npz, ndc, parity)          # quant_mixed: created quantised
    info0 = tree.info()
    views = [v for v in ec.views_for(name) if v != "composite"][:3]
    cams = []
    for v in views:
        W, H, fx, fy, pose, kw, _ = ec.view(v, name, st)
        cams.append((_cam(W, H, fx, fy, pose), kw))
    before = [_render_float(tree, [c], RenderOptions(**kw)) for c, kw in cams]
    shape = (st.capacity, 2, 2, 2, st.data_dim)
    tree.update_data(torch.from_numpy(st.data.copy()).cuda())            # identity
    torch.cuda.synchronize()
    for (c, kw), (f0, u0) in zip(cams, before):
        f1, u1 = _render_float(tree, [c], RenderOptions(**kw))
        assert np.array_equal(f1.view(np.uint32), f0.view(np.uint32)) and np.array_equal(u1, u0), name
    rng = np.random.default_rng(parity)
    new = st.data.astype(np.float32) + rng.normal(0, 0.3, shape).astype(np.float32)
    with np.errstate(invalid="ignore"):                                   # sigma_bits: NaN and inf sigmas stay
        new[..., -1] = np.abs(new[..., -1]) * rng.choice([0.0, 1.0, 30.0], shape[:4])
    new_dev = torch.from_numpy(new).cuda()
    tree.update_data(new_dev)                                             # fp32: rounded with .half()
    torch.cuda.synchronize()
    assert tree.info() == info0
    assert tree.data_ is None and tree.quant_ is None
    fresh_st = ec.edge_tree(name)[0]
    fresh_st.data = new_dev.half().cpu().numpy()    # the device's rounding (NaN payloads differ from the CPU's)
    fresh = _device_tree(fresh_st, None, ndc, parity)
    for c, kw in cams:
        f1, u1 = _render_float(tree, [c], RenderOptions(**kw))
        f2, u2 = _render_float(fresh, [c], RenderOptions(**kw))
        assert np.array_equal(f1.view(np.uint32), f2.view(np.uint32)) and np.array_equal(u1, u2), name
    q1, q2 = _query_state(tree, fresh_st), _query_state(fresh, fresh_st)
    assert set(q1) == set(q2)
    for k in q1:
        assert np.array_equal(q1[k], q2[k]), (name, k)


def test_descent_direction(built):
    import torch
    from volrend_b200 import RenderOptions, synth
    st = synth.make_tree("lego", depth=5, basis_dim=9, seed=32)
    tree = _device_tree(st)
    cams = _views(n=4)
    opt = RenderOptions()
    target = torch.from_numpy(_render_float(tree, cams, opt)[0]).cuda()
    rng = np.random.default_rng(1)
    data = torch.from_numpy(st.data.astype(np.float32) + rng.normal(0, 0.5, st.data.shape).astype(np.float32)).cuda()
    tree.update_data(data)

    def mse():
        f = torch.from_numpy(_render_float(tree, cams, opt)[0]).cuda()
        return float((f[..., :3] - target[..., :3]).square().mean()), f

    l0, f = mse()
    diff = f[..., :3] - target[..., :3]
    dpix = torch.zeros_like(f)
    dpix[..., :3] = diff * (2.0 / diff.numel())
    g, _ = _grads(tree, cams, opt, dpix)
    step = 0.5 / float(g.abs().max())
    tree.update_data(data - step * g)
    l1, _ = mse()
    assert l1 < l0, (l0, l1)


def _fit_setup(seed=41):
    import torch
    from volrend_b200 import RenderOptions, synth
    st = synth.make_tree("lego", depth=5, basis_dim=9, seed=seed)
    W = H = 64
    f = synth.focal_for(W)
    poses = synth.nerf_synthetic_test_poses(24)
    cams = [_cam(W, H, f, f, p) for p in poses]
    opt = RenderOptions()
    clean = _device_tree(st)
    targets = torch.from_numpy(_render_float(clean, cams, opt)[0][..., :3].copy())
    rng = np.random.default_rng(seed)
    noisy = st.data.astype(np.float32)
    noisy[..., :-1] += rng.normal(0, 0.4, noisy[..., :-1].shape).astype(np.float32)
    noisy[..., -1] *= rng.uniform(0.5, 1.5, noisy.shape[:4]).astype(np.float32)
    st.data = noisy.astype(np.float16)
    return st, cams, targets, opt


def _psnr(tree, cams, targets, opt):
    f = _render_float(tree, cams, opt)[0][..., :3]
    return -10 * np.log10(float(((f - targets.numpy()) ** 2).mean()))


def test_end_to_end_fit(built):
    from volrend_b200 import finetune
    st, cams, targets, opt = _fit_setup()
    train, held = cams[:20], cams[20:]
    tree = _device_tree(st)
    p0 = _psnr(tree, held, targets[20:], opt)
    master, losses = finetune(tree, train, targets[:20], opt, steps=60, lr=2e-2, batch=4, seed=0)
    p1 = _psnr(tree, held, targets[20:], opt)
    print(f"fit: loss {losses[0]:.6g} -> {losses[-1]:.6g} (min {min(losses):.6g}), held-out PSNR {p0:.3f} -> {p1:.3f}")
    assert master.shape == st.data.shape and len(losses) == 60
    # first H100 run (DESIGN.md 18): loss 1.204e-3 -> 4.29e-5, held-out PSNR 29.51 -> 35.56 dB
    assert losses[-1] < 0.1 * losses[0], losses
    assert p1 > p0 + 4.0, (p0, p1)


def test_cli_on_png_targets(built, tmp_path, capsys):
    import importlib
    from volrend_b200 import write_png_file
    ft = importlib.import_module("volrend_b200.finetune")
    st, cams, targets, opt = _fit_setup(seed=42)
    cams, targets = cams[:6], targets[:6]
    src = str(tmp_path / "t.npz")
    np.savez(src, **st.npz_dict())
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
    out = str(tmp_path / "o.npz")
    rc = ft.main([src, out] + poses + ["--targets"] + pngs +
                 ["--width", "64", "--height", "64", "--fx", str(cams[0].fx), "--steps", "20", "--lr", "2e-2",
                  "--batch", "2", "--holdout", "1"])
    assert rc == 0
    text = capsys.readouterr().out
    before = float(text.split("held-out PSNR before: ")[1].split()[0])
    after = float(text.split("held-out PSNR after: ")[1].split()[0])
    assert after > before, text
    assert text.count("step ") == 20
    with np.load(out) as z, np.load(src) as s:
        assert z["data"].dtype == np.float16 and z["data"].shape == s["data"].shape
        assert np.array_equal(z["child"], s["child"]) and not np.array_equal(z["data"], s["data"])


def test_refusals(built):
    import torch
    from volrend_b200 import RenderOptions, VolrendError, _capi, leaf_grads, lib, synth
    st = synth.make_tree("lego", depth=4, basis_dim=4, seed=33)
    cams = _views(n=2, W=16, H=8)
    dpix = _dpix(2, 8, 16, 0)
    plain = _device_tree(st, slot_map=False)
    with pytest.raises(RuntimeError, match="slot map"):
        leaf_grads(plain, cams, RenderOptions(), dpix)
    with pytest.raises(RuntimeError, match="slot map"):
        plain.update_data(torch.zeros(st.data.shape, dtype=torch.float16, device="cuda"))
    L = lib()
    arr = (_capi.vr_camera * 2)(*[c._as_c() for c in cams])
    o = RenderOptions()._as_c()
    g = torch.zeros(st.capacity * 8 * st.data_dim, dtype=torch.float32, device="cuda")
    assert L.vr_tree_leaf_grads(plain._handle, arr, 2, C.byref(o), None, dpix.data_ptr(), g.data_ptr(), None,
                                None) == _capi.VR_EUNSUPPORTED
    assert L.vr_tree_update_data(plain._handle, g.data_ptr(), None) == _capi.VR_EUNSUPPORTED
    tree = _device_tree(st)
    with pytest.raises(VolrendError):
        leaf_grads(tree, cams, RenderOptions(render_depth=True), dpix)
    assert L.vr_tree_leaf_grads(tree._handle, arr, 2, C.byref(o), None, None, g.data_ptr(), None,
                                None) == _capi.VR_EINVAL
    assert L.vr_tree_leaf_grads(tree._handle, arr, 2, C.byref(o), None, dpix.data_ptr(), None, None,
                                None) == _capi.VR_EINVAL
    host = np.zeros(dpix.numel(), np.float32)
    assert L.vr_tree_leaf_grads(tree._handle, arr, 2, C.byref(o), None, host.ctypes.data, g.data_ptr(), None,
                                None) == _capi.VR_EINVAL
    assert L.vr_tree_update_data(tree._handle, None, None) == _capi.VR_EINVAL
    assert L.vr_tree_update_data(tree._handle, host.ctypes.data, None) == _capi.VR_EINVAL
    with pytest.raises(ValueError, match="dpix"):
        leaf_grads(tree, cams, RenderOptions(), dpix[:1])
    with pytest.raises(ValueError, match="dpix"):
        leaf_grads(tree, cams, RenderOptions(), dpix.cpu())
    with pytest.raises(ValueError, match="out"):
        leaf_grads(tree, cams, RenderOptions(), dpix, out=g[:-1])
    with pytest.raises(ValueError, match="out"):
        leaf_grads(tree, cams, RenderOptions(), dpix, out=g.double())
    with pytest.raises(ValueError, match="float_out"):
        leaf_grads(tree, cams, RenderOptions(), dpix, float_out=dpix[:1])
    with pytest.raises(ValueError, match="data"):
        tree.update_data(torch.zeros(st.data.shape, dtype=torch.float16))            # host tensor
    with pytest.raises(ValueError, match="data"):
        tree.update_data(torch.zeros((1,) + st.data.shape[1:], dtype=torch.float16, device="cuda"))
    if torch.cuda.device_count() > 1:
        other = torch.zeros(g.numel(), dtype=torch.float32, device="cuda:1")
        assert L.vr_tree_leaf_grads(tree._handle, arr, 2, C.byref(o), None, dpix.data_ptr(), other.data_ptr(), None,
                                    None) == _capi.VR_EINVAL
