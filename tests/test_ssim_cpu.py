"""`-m "not gpu"`: the float64 SSIM oracle (oracle/ssim_oracle.py, DESIGN.md section 22) on hand-worked cases, its
gradient against a torch float64 autograd restatement and central differences, the argument checks of the evaluate
and finetune command lines, and vr_image_ssim without a device."""
import ctypes as C

import numpy as np
import pytest

from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)
from oracle import ssim_oracle as so


def _pair(seed, V=2, H=14, W=13, cx=4, cy=3, noise=0.1):
    rng = np.random.default_rng(seed)
    x = rng.random((V, H, W, cx))
    y = np.clip(x[..., :cy] + noise * rng.standard_normal((V, H, W, cy)), 0, 1)
    return x, y


# ------------------------------------------------------------------------------------------- hand-worked values
def test_identical_images_give_one():
    x, _ = _pair(0)
    assert np.array_equal(so.ssim(x, x), np.ones(2))
    s, (a, b, c) = so.ssim_maps(x, x[..., :3], grad=True)
    assert np.all(s == 1.0)
    _, d = so.ssim_grad(x, x)
    assert np.abs(d).max() < 1e-12


@pytest.mark.parametrize("a,b", [(0.3, 0.6), (0.0, 1.0), (1.0, 1.0), (0.25, 0.0)])
def test_constant_planes(a, b):
    x = np.full((1, 15, 12, 3), a)
    y = np.full((1, 15, 12, 4), b)
    want = (2 * a * b + so.C1) / (a * a + b * b + so.C1)
    assert so.ssim(x, y)[0] == pytest.approx(want, rel=1e-12, abs=1e-15)


def test_eleven_by_eleven_is_one_output_pixel():
    x, y = _pair(1, H=11, W=11)
    s = so.ssim_maps(x, y)
    assert s.shape == (2, 3, 1, 1)
    # the single window is the whole image, weighted by the outer product of the filter
    f = so.gaussian()
    w = np.outer(f, f)
    xp, yp = x[0, :, :, 0], y[0, :, :, 0]
    mx, my = (w * xp).sum(), (w * yp).sum()
    sxx, syy = (w * xp * xp).sum() - mx * mx, (w * yp * yp).sum() - my * my
    sxy = (w * xp * yp).sum() - mx * my
    sxy = np.sign(sxy) * min(np.sqrt(sxx * syy), abs(sxy))
    want = (2 * mx * my + so.C1) * (2 * sxy + so.C2) / ((mx * mx + my * my + so.C1) * (sxx + syy + so.C2))
    assert s[0, 0, 0, 0] == pytest.approx(want, rel=1e-12)


def test_small_images_are_refused():
    with pytest.raises(ValueError, match="11x11"):
        so.ssim(np.zeros((1, 10, 20, 3)), np.zeros((1, 10, 20, 3)))


# ----------------------------------------------------------------------------------------------- flat windows
def _one_window(x, y):
    """Hand-worked SSIM and gradient of the single output pixel of 11x11 images x, y ([11, 11]) in exact terms: a flat
    image has mean equal to its value and variance and covariance exactly 0, and the clip rules take the tie."""
    f = so.gaussian()
    w = np.outer(f, f)
    flat_x, flat_y = np.all(x == x[0, 0]), np.all(y == y[0, 0])
    mx = x[0, 0] if flat_x else (w * x).sum()
    my = y[0, 0] if flat_y else (w * y).sum()
    sxx = 0.0 if flat_x else (w * x * x).sum() - mx * mx
    syy = 0.0 if flat_y else (w * y * y).sum() - my * my
    sxy = 0.0 if flat_x or flat_y else (w * x * y).sum() - mx * my
    A, B = 2 * mx * my + so.C1, 2 * sxy + so.C2
    C, D = mx * mx + my * my + so.C1, sxx + syy + so.C2
    s = A * B / (C * D)
    b, c = -s / D, 2 * A / (C * D)            # no clip is active: sxx * syy >= sxy^2 holds exactly
    direct = 2 * my * B / (C * D) - 2 * mx * s / C
    dx = w * (direct + 2 * (x - mx) * b + (y - my) * c) / 3
    return s, dx


@pytest.mark.parametrize("case", ["x_flat", "y_flat", "both_flat", "x_flat_zero", "both_flat_bright"])
def test_flat_windows_by_hand(case):
    rng = np.random.default_rng(11)
    x, y = rng.random((11, 11)), rng.random((11, 11))
    if case == "x_flat":
        x[:] = 0.999
    elif case == "y_flat":
        y[:] = 0.3
    elif case == "both_flat":
        x[:], y[:] = 0.25, 0.7
    elif case == "x_flat_zero":
        x[:] = 0.0
    else:
        x[:], y[:] = 0.999, 1.0
    s_h, dx_h = _one_window(x, y)
    X = np.repeat(x[None, :, :, None], 3, -1)
    Y = np.repeat(y[None, :, :, None], 3, -1)
    s, dx = so.ssim_grad(X, Y)
    assert s[0] == pytest.approx(s_h, rel=1e-13)
    for ch in range(3):
        assert np.allclose(dx[0, ..., ch], dx_h, rtol=1e-9, atol=1e-14 * np.abs(dx_h).max())
    if case != "both_flat" and case != "both_flat_bright":
        assert np.abs(dx_h).max() > 0        # the term through E[xy] (or E[x^2]) is on


# --------------------------------------------------------------------- the clip rules against torch autograd
def _torch_from_moments(mx, my, exx, eyy, exy):
    """The definition in torch, with the clip rules as torch.where (no sqrt at 0)."""
    import torch
    vx, vy = exx - mx * mx, eyy - my * my
    sxx = torch.where(vx >= 0, vx, torch.zeros_like(vx))
    syy = torch.where(vy >= 0, vy, torch.zeros_like(vy))
    sxy0 = exy - mx * my
    pr = sxx * syy
    rt = torch.where(pr > 0, torch.sqrt(torch.where(pr > 0, pr, torch.ones_like(pr))), torch.zeros_like(pr))
    sxy = torch.where(sxy0.abs() > rt, torch.sign(sxy0) * rt, sxy0)
    return ((2 * mx * my + so.C1) * (2 * sxy + so.C2) /
            ((mx * mx + my * my + so.C1) * (sxx + syy + so.C2)))


# (mx, my, exx, eyy, exy) with exact binary values, and what the clip rules must give
CLIP_CASES = {
    "inside": ((0.5, 0.25, 0.3125, 0.125, 0.15625), None),
    "variance_clipped": ((0.5, 0.25, 0.1875, 0.125, 0.125), "b0"),
    "covariance_clipped": ((0.5, 0.5, 0.3125, 0.5, 0.5), "c0"),
    "covariance_clipped_zero_variance": ((0.5, 0.5, 0.25, 0.5, 0.3125), "c0"),
    "covariance_tie": ((0.5, 0.5, 0.3125, 0.5, 0.375), "tie"),
    "negative_covariance_clipped": ((0.5, 0.5, 0.3125, 0.5, 0.0), "c0"),
}


@pytest.mark.parametrize("name", sorted(CLIP_CASES))
def test_clip_branches(name):
    import torch
    m, rule = CLIP_CASES[name]
    t = [torch.tensor(v, dtype=torch.float64, requires_grad=True) for v in m]
    s_t = _torch_from_moments(*t)
    s_t.backward()
    s, (a, b, c) = so.from_moments(*m, grad=True)
    assert float(s) == pytest.approx(float(s_t.detach()), rel=1e-14)
    assert float(a) == pytest.approx(float(t[0].grad), rel=1e-12, abs=1e-12)
    assert float(b) == pytest.approx(float(t[2].grad), rel=1e-12, abs=1e-12)
    assert float(c) == pytest.approx(float(t[4].grad), rel=1e-12, abs=1e-12)
    mx, my, exx, eyy, exy = m
    sxx, syy, sxy0 = exx - mx * mx, eyy - my * my, exy - mx * my
    if rule == "b0":
        assert sxx < 0 and float(b) == 0.0
    elif rule == "c0":
        assert abs(sxy0) > np.sqrt(max(sxx, 0) * max(syy, 0)) and float(c) == 0.0
        if sxx * syy == 0:      # the clip is active at a zero variance: no gradient through the root
            assert float(b) == pytest.approx(-float(s) / (sxx + syy + so.C2), rel=1e-14)
    elif rule == "tie":
        assert abs(sxy0) == np.sqrt(sxx * syy) and float(c) != 0.0


def _torch_ssim(x, y):
    import torch
    import torch.nn.functional as F
    f = torch.tensor(so.gaussian(), dtype=torch.float64)
    w = (f[:, None] * f[None, :])[None, None]
    V, H, W = x.shape[:3]
    xp = x[..., :3].permute(0, 3, 1, 2).reshape(V * 3, 1, H, W)
    yp = y[..., :3].permute(0, 3, 1, 2).reshape(V * 3, 1, H, W)
    flt = lambda a: F.conv2d(a, w)
    s = _torch_from_moments(flt(xp), flt(yp), flt(xp * xp), flt(yp * yp), flt(xp * yp))
    return s.reshape(V, -1).mean(1)


@pytest.mark.parametrize("seed,noise", [(0, 0.1), (1, 0.02), (2, 0.5)])
def test_gradient_matches_torch_autograd(seed, noise):
    import torch
    x, y = _pair(seed, V=3, H=17, W=15, noise=noise)
    x[0, 2:9, 3:12] = 0.999         # a flat bright patch
    xt = torch.tensor(x, requires_grad=True)
    st = _torch_ssim(xt, torch.tensor(y))
    st.sum().backward()
    s, d = so.ssim_grad(x, y)
    assert np.allclose(s, st.detach().numpy(), rtol=0, atol=1e-13)
    g = xt.grad.numpy()
    assert np.all(g[..., 3] == 0)
    assert np.allclose(d, g[..., :3], rtol=0, atol=1e-12 * np.abs(g).max())


def test_gradient_matches_central_differences():
    x, y = _pair(3, V=2, H=13, W=12)
    _, d = so.ssim_grad(x, y)
    h = 1e-6
    for idx in [(0, 3, 4, 1), (1, 0, 0, 2), (0, 12, 11, 0), (1, 7, 6, 1), (0, 5, 5, 2)]:
        xp, xm = x.copy(), x.copy()
        xp[idx] += h
        xm[idx] -= h
        num = (so.ssim(xp, y) - so.ssim(xm, y))[idx[0]] / (2 * h)
        assert num == pytest.approx(d[idx], rel=1e-6, abs=2e-10), idx


# ------------------------------------------------------------------------------------------- CLI and C-ABI
def _cli_inputs(tmp_path, w=16, h=12, n=2):
    import edge_cases as ec
    st = ec.mixed_tree(3, 4, "SH", 5)
    src = str(tmp_path / "t.npz")
    np.savez(src, **st.npz_dict())
    pose = str(tmp_path / "p.txt")
    np.savetxt(pose, np.vstack([np.eye(4)] * n))
    npy = str(tmp_path / "t.npy")
    np.save(npy, np.zeros((n, h, w, 3), np.uint8))
    return src, pose, npy


def test_evaluate_cli_argument_errors(tmp_path, capsys):
    import importlib
    ev = importlib.import_module("volrend_b200.evaluate")
    src, pose, npy = _cli_inputs(tmp_path)
    size = ["--width", "16", "--height", "12"]
    bad = [
        ([src, pose, "--targets", npy, "--batch", "0"] + size, "--batch"),
        ([src[:-4] + ".bin", pose, "--targets", npy] + size, "not an .npz"),
        ([str(tmp_path / "missing.npz"), pose, "--targets", npy] + size, "does not exist"),
        ([src, pose, "--targets", str(tmp_path / "missing.npy")] + size, "does not exist"),
        ([src, pose, "--targets", npy, "--width", "10", "--height", "12"], "11x11"),
        ([src, pose, "--targets", npy, "--width", "16", "--height", "10"], "11x11"),
        ([src, pose, "--targets", npy, "--width", "17", "--height", "12"], "the views"),
        ([src, pose, pose, "--targets", npy] + size, "targets for"),
        ([src, str(tmp_path / "nope.txt"), "--targets", npy] + size, "does not exist"),
    ]
    for argv, msg in bad:
        with pytest.raises(SystemExit) as e:
            ev.main(argv)
        assert e.value.code == 2, argv
        assert msg in capsys.readouterr().err, argv
    with pytest.raises(SystemExit):
        ev.main([src, pose] + size)        # --targets is required
    capsys.readouterr()


def test_finetune_cli_refuses_bad_dssim_weight(tmp_path, capsys):
    import importlib
    finetune = importlib.import_module("volrend_b200.finetune")
    src, pose, npy = _cli_inputs(tmp_path, w=6, h=8)
    base = [src, str(tmp_path / "o.npz"), pose, "--targets", npy, "--width", "6", "--height", "8"]
    for bad in ("-1", "nan", "inf", "-0.001"):
        with pytest.raises(SystemExit) as e:
            finetune.main(base + ["--dssim-weight", bad])
        assert e.value.code == 2
        assert "--dssim-weight" in capsys.readouterr().err
    assert not (tmp_path / "o.npz").exists()


def test_finetune_refuses_bad_dssim_weight():
    from types import SimpleNamespace
    from volrend_b200 import finetune
    for w in (-1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="dssim_weight"):
            finetune(None, [None], [None], None, steps=1, lr=1e-2, batch=1, seed=0, dssim_weight=w)
    # D-SSIM on images smaller than the SSIM window is refused before anything is rendered
    tree = SimpleNamespace(data_=np.zeros(1))
    cam = SimpleNamespace(width=10, height=32)
    with pytest.raises(ValueError, match="11x11"):
        finetune(tree, [cam], [None], None, steps=1, lr=1e-2, batch=1, seed=0, dssim_weight=0.5)


def test_finetune_cli_refuses_dssim_on_small_images(tmp_path, capsys):
    import importlib
    finetune = importlib.import_module("volrend_b200.finetune")
    src, pose, npy = _cli_inputs(tmp_path, w=6, h=8)
    with pytest.raises(SystemExit) as e:
        finetune.main([src, str(tmp_path / "o.npz"), pose, "--targets", npy, "--width", "6", "--height", "8",
                       "--dssim-weight", "0.5"])
    assert e.value.code == 2
    assert "11x11" in capsys.readouterr().err
    assert not (tmp_path / "o.npz").exists()


def test_image_ssim_without_a_device(built):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from volrend_b200 import _capi, lib
    L = lib()
    buf = C.c_void_p(0x1000)
    assert L.vr_image_ssim(buf, 4, buf, 3, 2, 16, 16, buf, buf, -0.5, None) == _capi.VR_ENODEVICE
    assert b"no CPU fallback" in L.vr_last_error()
    assert L.vr_image_ssim(buf, 3, buf, 3, 1, 11, 11, buf, None, 1.0, None) == _capi.VR_ENODEVICE
    # argument errors are found before the device is looked for
    assert L.vr_image_ssim(buf, 4, buf, 3, -1, 16, 16, buf, None, 1.0, None) == _capi.VR_EINVAL
    assert L.vr_image_ssim(buf, 4, buf, 3, 1, 10, 16, buf, None, 1.0, None) == _capi.VR_EINVAL
    assert L.vr_image_ssim(buf, 5, buf, 3, 1, 16, 16, buf, None, 1.0, None) == _capi.VR_EINVAL
    assert L.vr_image_ssim(buf, 4, buf, 3, 1, 16, 16, buf, None, float("nan"), None) == _capi.VR_EINVAL
    assert L.vr_image_ssim(None, 4, buf, 3, 1, 16, 16, buf, None, 1.0, None) == _capi.VR_EINVAL
