"""`-m gpu`: per-view SSIM and its gradient (vr_image_ssim, volrend_b200.image_ssim), the evaluate tool and the D-SSIM
term of finetune on an H100.

Accuracy against the float64 oracle (oracle/ssim_oracle.py): ssim_v within 1e-6, and every dx element within
1e-4 * G + 1e-9, G being the view's largest |dx| of the oracle (DESIGN.md section 22)."""
import numpy as np
import pytest

import golden_cases as gc
from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)
from oracle import ssim_oracle as so

pytestmark = pytest.mark.gpu


def _gpu(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def _run(x, y, scale=1.0):
    import torch
    from volrend_b200 import image_ssim
    xt, yt = _gpu(x), _gpu(y)
    dx = torch.zeros_like(xt)
    s = image_ssim(xt, yt, dx=dx, dx_scale=scale)
    torch.cuda.synchronize()
    return s.cpu().numpy(), dx.cpu().numpy()


def _check(x, y, views=None, what="", rel=1e-4):
    """image_ssim of x against y (float32 as given) against the oracle on views ``views`` (all by default); dx within
    rel * G + 1e-9."""
    x = np.asarray(x, np.float32)
    y = np.asarray(y, np.float32)
    s, dx = _run(x, y)
    assert s.dtype == np.float64 and s.shape == (x.shape[0],)
    worst = 0.0
    for v in range(x.shape[0]) if views is None else views:
        s64, d64 = so.ssim_grad(x[v:v + 1], y[v:v + 1])
        assert abs(s[v] - s64[0]) <= 1e-6, (what, v, s[v], s64[0])
        G = float(np.abs(d64).max())
        err = np.abs(dx[v, ..., :3] - d64[0])
        assert np.all(err <= rel * G + 1e-9), (what, v, float(err.max()), G)
        worst = max(worst, float(err.max()) / max(G, 1e-30))
        if x.shape[-1] == 4:
            assert np.all(dx[v, ..., 3] == 0)
    print(f"{what}: worst |dx - dx64| / G = {worst:.2e}")
    return s, dx


def _images(seed, V, H, W, cx=4, cy=3, kind="random"):
    rng = np.random.default_rng(seed)
    x = rng.random((V, H, W, cx)).astype(np.float32)
    if kind == "random":
        y = rng.random((V, H, W, cy))
    elif kind == "near":
        y = x[..., :3] + rng.normal(0, 1e-3, (V, H, W, 3))
        if cy == 4:
            y = np.concatenate([y, rng.random((V, H, W, 1))], -1)
    elif kind == "flat":
        # flat 0 and near-1 regions (a white background), with a textured band between them
        x[:, : H // 3] = 0.0
        x[:, H // 3: 2 * H // 3, :, :3] = 0.999
        y = x[..., :3].astype(np.float64) + rng.normal(0, 0.02, (V, H, W, 3)) * (np.arange(W) > W // 2)[:, None]
        if cy == 4:
            y = np.concatenate([y, rng.random((V, H, W, 1))], -1)
    return x, np.asarray(y, np.float32)


# ------------------------------------------------------------------------------------------------- accuracy
@pytest.mark.parametrize("cx,cy", [(4, 3), (3, 3), (4, 4), (3, 4)])
@pytest.mark.parametrize("kind", ["random", "near", "flat"])
def test_matches_oracle(kind, cx, cy):
    x, y = _images(1, 2, 75, 69, cx, cy, kind)
    _check(x, y, what=f"{kind} {cx}/{cy}", rel=2e-4 if kind == "near" else 1e-4)


@pytest.mark.parametrize("H,W", [(11, 11), (11, 40), (37, 11), (33, 65), (97, 31)])
def test_odd_sizes(H, W):
    # near-identical images: the gradient is a small difference of large terms; 1.32e-4 * G at worst on the H100
    # runs (DESIGN.md section 22)
    x, y = _images(2, 3, H, W, kind="near")
    _check(x, y, what=f"{W}x{H}", rel=2e-4)


def test_identical_images():
    for kind in ("random", "flat"):
        x, _ = _images(3, 2, 70, 90, kind=kind)
        s, dx = _run(x, x)
        assert np.all(np.abs(s - 1.0) <= 1e-7), s
        assert np.abs(dx).max() <= 1e-9, float(np.abs(dx).max())
        x3 = np.ascontiguousarray(x[..., :3])
        s3, _ = _run(x, x3)
        assert np.array_equal(s, s3)


def test_800_one_view_and_1080p():
    x, y = _images(4, 1, 800, 800, kind="near")
    _check(x, y, what="800x800", rel=2e-4)
    x, y = _images(5, 1, 1080, 1920, kind="flat")
    _check(x, y, what="1920x1080")


def test_200_views_at_800():
    import torch
    from volrend_b200 import image_ssim
    rng = np.random.default_rng(6)
    base = rng.random((800, 800, 3)).astype(np.float32)
    xt = torch.empty((200, 800, 800, 4), dtype=torch.float32, device="cuda")
    yt = torch.empty((200, 800, 800, 3), dtype=torch.float32, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(6)
    b = _gpu(base)
    for v in range(200):
        xt[v, ..., :3] = b + 0.01 * (v % 7) * torch.randn((800, 800, 3), generator=g, device="cuda")
        xt[v, ..., 3] = 1.0
        yt[v] = b
    dx = torch.zeros_like(xt)
    s = image_ssim(xt, yt, dx=dx).cpu().numpy()
    dx = dx.cpu().numpy()
    for v in range(0, 200, 23):
        xv, yv = xt[v:v + 1].cpu().numpy(), yt[v:v + 1].cpu().numpy()
        s64, d64 = so.ssim_grad(xv, yv)
        assert abs(s[v] - s64[0]) <= 1e-6, (v, s[v], s64[0])
        G = float(np.abs(d64).max())
        assert np.all(np.abs(dx[v, ..., :3] - d64[0]) <= 1e-4 * G + 1e-9), v
    for v in range(200):       # the rest: the value only, which the kernel sums per view independently
        if v % 23:
            assert abs(s[v] - so.ssim(xt[v:v + 1].cpu().numpy(), yt[v:v + 1].cpu().numpy())[0]) <= 1e-6, v


def _render(tree, cams, opt):
    import torch
    from volrend_b200 import render_batch
    fo = torch.empty((len(cams), cams[0].height, cams[0].width, 4), dtype=torch.float32, device="cuda")
    render_batch(tree, cams, opt, None, float_out=fo)
    torch.cuda.synchronize()
    return fo


def _tree(st, ndc=None):
    from volrend_b200 import N3Tree
    t = N3Tree()
    t.load_npz(st.npz_dict())
    if ndc is not None:
        t.use_ndc = True
        t.ndc_width, t.ndc_height, t.ndc_focal = ndc
    t.load_cuda()
    return t


def _cams(W, H, poses):
    from volrend_b200 import synth
    from volrend_b200.views import cameras
    return cameras(poses, W, H, synth.focal_for(W), synth.focal_for(W))


@pytest.mark.parametrize("name", ["lego_sh16", "drums_sh9", "lego_rgba", "lego_sh16_ndc", "lego_sg9_rot"])
def test_renders_of_golden_trees(name):
    from volrend_b200 import RenderOptions, synth
    st, W, H, pose, kw, ndc = gc.build_case(name)
    opt = RenderOptions(**{k: v for k, v in kw.items() if k != "render_depth"})
    poses = [pose] if ndc is not None else synth.nerf_synthetic_test_poses(8)[:4]
    cams = _cams(W, H, poses)
    a = _render(_tree(st, ndc), cams, opt).cpu().numpy()
    rng = np.random.default_rng(7)
    st.data = (st.data.astype(np.float32) * rng.uniform(0.8, 1.2, st.data.shape)).astype(np.float16)
    b = _render(_tree(st, ndc), cams, opt).cpu().numpy()
    # Renders miss the 1e-4 * G gradient bound: worst 3.0e-2 * G (lego_sg9_rot) on the H100 runs, from windows on the
    # object in tiles whose shift is the background (DESIGN.md section 22); the values hold 1e-6.
    s, _ = _check(a, b, what=name, rel=6e-2)
    assert np.all(s < 1.0)


# ------------------------------------------------------------------------------------------------ behaviour
def test_bit_reproducible_and_accumulating():
    import torch
    from volrend_b200 import image_ssim
    x, y = _images(8, 3, 120, 130, kind="near")
    xt, yt = _gpu(x), _gpu(y)
    d0 = torch.randn(xt.shape, generator=torch.Generator().manual_seed(8)).cuda()
    dxa, dxb, dz = d0.clone(), d0.clone(), torch.zeros_like(xt)
    sa = image_ssim(xt, yt, dx=dxa, dx_scale=-0.75)
    sb = image_ssim(xt, yt, dx=dxb, dx_scale=-0.75)
    sz = image_ssim(xt, yt, dx=dz)
    sf = image_ssim(xt, yt)
    torch.cuda.synchronize()
    assert torch.equal(sa, sb) and torch.equal(sa, sz) and torch.equal(sa, sf)
    assert torch.equal(dxa, dxb)
    assert torch.equal(dxa[..., 3], d0[..., 3])                    # alpha keeps its bits
    assert torch.allclose(dxa[..., :3], d0[..., :3] - 0.75 * dz[..., :3], rtol=0, atol=1e-6)
    out = torch.full((3,), 7.0, dtype=torch.float64, device="cuda")
    assert image_ssim(xt, yt, out=out) is out and torch.equal(out, sa)


def test_refusals_leave_outputs_unchanged():
    import torch
    from volrend_b200 import VolrendError, _capi, image_ssim, lib
    x, y = _images(9, 2, 20, 24, kind="near")
    xt, yt = _gpu(x), _gpu(y)
    s = torch.full((2,), 5.0, dtype=torch.float64, device="cuda")
    dx = torch.full_like(xt, 3.0)
    L = lib()
    p = lambda t: t.data_ptr()
    host = torch.zeros(xt.shape)
    bad = [
        (p(xt), 4, p(yt), 3, -1, 20, 24, p(s), p(dx), 1.0),
        (p(xt), 4, p(yt), 3, 2, 10, 24, p(s), p(dx), 1.0),
        (p(xt), 4, p(yt), 3, 2, 20, 10, p(s), p(dx), 1.0),
        (p(xt), 5, p(yt), 3, 2, 20, 24, p(s), p(dx), 1.0),
        (p(xt), 4, p(yt), 2, 2, 20, 24, p(s), p(dx), 1.0),
        (p(xt), 4, p(yt), 3, 2, 20, 24, p(s), p(dx), float("nan")),
        (p(xt), 4, p(yt), 3, 2, 20, 24, p(s), p(dx), float("inf")),
        (None, 4, p(yt), 3, 2, 20, 24, p(s), p(dx), 1.0),
        (p(xt), 4, None, 3, 2, 20, 24, p(s), p(dx), 1.0),
        (p(xt), 4, p(yt), 3, 2, 20, 24, None, p(dx), 1.0),
        (p(host), 4, p(yt), 3, 2, 20, 24, p(s), p(dx), 1.0),
        (p(xt), 4, p(yt), 3, 2, 20, 24, p(s), p(host), 1.0),
    ]
    for args in bad:
        assert L.vr_image_ssim(*args, None) == _capi.VR_EINVAL, args
    n0 = L.vr_launch_count()
    assert L.vr_image_ssim(p(xt), 4, p(yt), 3, 0, 20, 24, p(s), p(dx), 1.0, None) == _capi.VR_OK
    assert L.vr_launch_count() == n0
    for kw in ({"dx_scale": float("nan")}, {"out": torch.zeros(2, dtype=torch.float32, device="cuda")},
               {"dx": torch.zeros((2, 20, 24, 3), device="cuda")}):
        with pytest.raises(ValueError):
            image_ssim(xt, yt, **kw)
    for a, b in ((xt[:, :10], yt[:, :10]), (xt, yt[:1]), (xt.cpu(), yt.cpu()), (xt.double(), yt.double()),
                 (xt[..., :2], yt)):
        with pytest.raises((ValueError, VolrendError)):
            image_ssim(a, b, out=s, dx=dx)
    torch.cuda.synchronize()
    assert torch.all(s == 5.0) and torch.all(dx == 3.0)


# -------------------------------------------------------------------------------------------------- fitting
def _fit_setup(seed=41, n=24):
    from volrend_b200 import RenderOptions, synth
    st = synth.make_tree("lego", depth=5, basis_dim=9, seed=seed)
    cams = _cams(64, 64, synth.nerf_synthetic_test_poses(n))
    opt = RenderOptions()
    targets = _render(_tree(st), cams, opt)[..., :3].cpu()
    rng = np.random.default_rng(seed)
    noisy = st.data.astype(np.float32)
    noisy[..., :-1] += rng.normal(0, 0.4, noisy[..., :-1].shape).astype(np.float32)
    noisy[..., -1] *= rng.uniform(0.5, 1.5, noisy.shape[:4]).astype(np.float32)
    st.data = noisy.astype(np.float16)
    return st, cams, targets, opt


def _slot_tree(st):
    from volrend_b200 import N3Tree
    t = N3Tree()
    t.load_npz(st.npz_dict())
    t.load_cuda(slot_map=True)
    return t


def test_zero_weight_never_calls_ssim(monkeypatch):
    from volrend_b200 import finetune, host
    st, cams, targets, opt = _fit_setup(n=8)

    def boom(*a, **k):
        raise AssertionError("image_ssim called with dssim_weight = 0")

    monkeypatch.setattr(host, "image_ssim", boom)
    _, losses = finetune(_slot_tree(st), cams, targets, opt, steps=3, lr=1e-2, batch=4, seed=0)
    assert len(losses) == 3
    with pytest.raises(AssertionError, match="image_ssim called"):
        finetune(_slot_tree(st), cams, targets, opt, steps=1, lr=1e-2, batch=4, seed=0, dssim_weight=0.5)


def test_descent_on_the_total_loss():
    import torch
    from volrend_b200 import image_ssim, leaf_grads
    st, cams, targets, opt = _fit_setup(n=4)
    tree = _slot_tree(st)
    lam = 0.8
    tgt = targets.cuda()
    data = torch.tensor(st.data.astype(np.float32), device="cuda")

    def total():
        f = _render(tree, cams, opt)
        return float((f[..., :3] - tgt).square().mean()) + lam * (1 - float(image_ssim(f, tgt).mean())), f

    l0, f = total()
    diff = f[..., :3] - tgt
    dpix = torch.zeros_like(f)
    dpix[..., :3] = diff * (2.0 / diff.numel())
    image_ssim(f, tgt, dx=dpix, dx_scale=-lam / len(cams))
    g = leaf_grads(tree, cams, opt, dpix)
    tree.update_data(data - (0.5 / float(g.abs().max())) * g)
    l1, _ = total()
    assert l1 < l0, (l0, l1)


def test_end_to_end_fit_raises_held_out_ssim():
    from volrend_b200 import evaluate, finetune
    st, cams, targets, opt = _fit_setup()
    train, held = cams[:20], cams[20:]
    res = {}
    for lam in (0.0, 0.5):
        tree = _slot_tree(st)
        m0, s0 = evaluate(tree, held, targets[20:], opt)
        finetune(tree, train, targets[:20], opt, steps=60, lr=2e-2, batch=4, seed=0, dssim_weight=lam)
        m1, s1 = evaluate(tree, held, targets[20:], opt)
        res[lam] = (s0.mean(), s1.mean(), -10 * np.log10(m0.mean()), -10 * np.log10(m1.mean()))
        print(f"dssim_weight {lam}: held-out SSIM {res[lam][0]:.4f} -> {res[lam][1]:.4f}, "
              f"PSNR {res[lam][2]:.3f} -> {res[lam][3]:.3f} dB")
    # first H100 run: held-out SSIM 0.9282 -> 0.9815 with dssim_weight 0.5 (0.9804 with MSE only), PSNR
    # 29.51 -> 35.46 dB (35.56 with MSE only)
    s0, s1 = res[0.5][:2]
    assert s1 > s0 + 0.03, res


# ------------------------------------------------------------------------------------------------- evaluate
def _write_cli_inputs(tmp_path, cams, images):
    from volrend_b200 import write_png_file
    poses, pngs = [], []
    for i, c in enumerate(cams):
        p = str(tmp_path / f"p{i}.txt")
        np.savetxt(p, np.vstack([c.transform.T, [0, 0, 0, 1]]))
        poses.append(p)
        png = str(tmp_path / f"t{i}.png")
        assert write_png_file(png, images[i])
        pngs.append(png)
    return poses, pngs


def test_cli_on_png_targets(tmp_path, capsys):
    import importlib
    import json
    from volrend_b200 import N3Tree, evaluate
    from volrend_b200.views import read_targets, target_batch
    ev = importlib.import_module("volrend_b200.evaluate")
    st, cams, targets, opt = _fit_setup(seed=42, n=5)
    src = str(tmp_path / "t.npz")
    np.savez(src, **st.npz_dict())
    rgba = [np.concatenate([np.clip(t.numpy() * 255 + 0.5, 0, 255).astype(np.uint8),
                            np.full((64, 64, 1), 200, np.uint8)], -1) for t in targets]
    poses, pngs = _write_cli_inputs(tmp_path, cams, rgba)
    js = str(tmp_path / "q.json")
    rc = ev.main([src] + poses + ["--targets"] + pngs + ["--width", "64", "--height", "64", "--fx", str(cams[0].fx),
                                                          "--batch", "2", "--background", "0.5", "--json", js])
    assert rc == 0
    text = capsys.readouterr().out
    assert text.count("view ") == 5 and "mean over 5 views" in text
    with open(js) as f:
        got = json.load(f)
    opt.background_brightness = 0.5
    tree = N3Tree(src)
    tg = read_targets(pngs, 5, 64, 64)
    mse, ssim = evaluate(tree, cams, tg, opt, batch=3)
    assert np.array_equal(np.array(got["mse"]), mse) and np.array_equal(np.array(got["ssim"]), ssim)
    assert got["mean_ssim"] == pytest.approx(ssim.mean(), rel=1e-15)
    f = _render(tree, cams, opt).cpu().numpy()
    t = target_batch(tg, range(5), 0.5, "cuda", 64, 64).cpu().numpy()
    # a flat render against targets of another brightness: 1.03e-6 at worst on the H100 runs (DESIGN.md section 22)
    assert np.all(np.abs(so.ssim(f, t) - ssim) <= 2e-6)
    assert np.allclose(mse, ((f[..., :3].astype(np.float64) - t) ** 2).mean(axis=(1, 2, 3)), rtol=1e-6)
    for v in range(5):
        assert f"view {v}: PSNR {-10 * np.log10(mse[v]):.3f} dB, SSIM {ssim[v]:.4f}" in text


def test_cli_on_compressed_and_ndc_trees(tmp_path, capsys):
    import importlib
    import json
    import torch
    from volrend_b200 import N3Tree, RenderOptions, compress_npz, image_ssim
    from volrend_b200.compress import _write_npz
    ev = importlib.import_module("volrend_b200.evaluate")
    cases = []
    st, cams, targets, opt = _fit_setup(seed=43, n=3)
    cases.append(("c", st, cams, None, compress_npz(st.npz_dict(), bits=8)))
    st, W, H, pose, _, ndc = gc.build_case("lego_sh16_ndc")
    from volrend_b200.views import cameras
    cases.append(("n", st, cameras([pose], W, H, 60.0, 60.0), ndc, st.npz_dict()))
    for tag, st, cams, ndc, z in cases:
        W, H = cams[0].width, cams[0].height
        src = str(tmp_path / f"{tag}.npz")
        _write_npz(src, z)
        if ndc is not None:
            pb = np.zeros(17, np.float32)
            pb[4], pb[9], pb[14] = ndc[1], ndc[0], ndc[2]
            np.save(src[:-4] + "_poses_bounds.npy", pb)
        rng = np.random.default_rng(10)
        imgs = [rng.integers(0, 256, (H, W, 3)).astype(np.uint8) for _ in cams]
        npy = str(tmp_path / f"{tag}.npy")
        np.save(npy, np.stack(imgs))
        poses = []
        for i, c in enumerate(cams):
            p = str(tmp_path / f"{tag}{i}.txt")
            np.savetxt(p, np.vstack([c.transform.T, [0, 0, 0, 1]]))
            poses.append(p)
        js = str(tmp_path / f"{tag}.json")
        assert ev.main([src] + poses + ["--targets", npy, "--width", str(W), "--height", str(H),
                                        "--fx", str(cams[0].fx), "--json", js]) == 0
        capsys.readouterr()
        with open(js) as f:
            got = json.load(f)
        # scored directly: the decoded tree's renders against the same images
        tree = N3Tree(src)
        assert tree.use_ndc == (ndc is not None)
        fo = _render(tree, cams, RenderOptions())
        tgt = torch.from_numpy(np.stack(imgs)).cuda().float() / 255.0
        want_s = image_ssim(fo, tgt).cpu().numpy()
        want_m = (fo[..., :3] - tgt).double().square().mean(dim=(1, 2, 3)).cpu().numpy()
        assert np.array_equal(np.array(got["ssim"]), want_s), tag
        assert np.array_equal(np.array(got["mse"]), want_m), tag
