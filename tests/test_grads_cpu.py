"""`-m "not gpu"`: the CPU restatement of the leaf-gradient pass (oracle/grads_oracle.c, orc_leaf_grads) on one-ray
cases against the closed form, against central differences of orc_render's float output on edge-case and golden trees,
and the fine-tuning module's npz handling and CLI argument errors; VR_ENODEVICE from the two new entry points."""
import ctypes as C
import math

import numpy as np
import pytest

import edge_cases as ec
import golden_cases as gc
from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)

AXIS = (1, 1, 1, 1)   # pixel (1, 1) of a 2x2 frame: its ray runs along the camera's -back exactly


def _ray_along_x(y, z):
    from oracle import binding as ob
    c2w = [0, 0, -1, 0, 1, 0, -1, 0, 0, -1.0, y, z]   # right, up, back, centre (column-major)
    return ob.make_camera(2, 2, 1.0, 1.0, c2w)


def _root_tree(rows, fmt):
    """Root-only tree, unit box: leaf o has data row rows[o] (4 values: r, g, b, sigma), others 0."""
    from oracle import binding as ob
    child = np.zeros((1, 2, 2, 2), np.int32)
    data = np.zeros((1, 2, 2, 2, 4), np.float16)
    for o, r in rows.items():
        data.reshape(8, 4)[o] = r
    return ob.OracleTree(child, data, [0, 0, 0], [1, 1, 1], 4, fmt), data


def _closed_form(rows, fmt, g, bg, stop):
    """The pixel of a ray crossing leaves 0 then 4, each over Δδ = 1/2, as a function of their data rows: L = g . pix,
    differentiated by double central differences."""
    B0 = 0.28209479177387814

    def L(x):
        x = x.reshape(2, 4)
        T, S, stopped = 1.0, np.zeros(3), False
        for i in range(2):
            att = math.exp(-0.5 * x[i, 3])
            w = T * (1 - att)
            col = x[i, :3] if fmt == "RGBA" else 1 / (1 + np.exp(-B0 * x[i, :3]))
            S += w * col
            T *= att
            if T < stop:
                stopped = True
                break
        pix = np.append(S / (1 - T), 1.0) if stopped else np.append(S + T * bg, 1 - T)
        return float(np.dot(g, pix))

    x0 = np.array([rows[0], rows[4]], np.float64).reshape(-1)
    out = np.zeros_like(x0)
    for j in range(x0.size):
        h = 1e-6 * max(1.0, abs(x0[j]))
        xp, xm = x0.copy(), x0.copy()
        xp[j] += h
        xm[j] -= h
        out[j] = (L(xp) - L(xm)) / (2 * h)
    return out.reshape(2, 4)


@pytest.mark.parametrize("fmt", ["SH1", "RGBA"])
@pytest.mark.parametrize("case", ["runs_out", "stops_early"])
def test_one_ray_two_leaves_closed_form(fmt, case):
    from oracle import binding as ob
    from oracle import grads_binding as gb
    rows = {0: [0.75, -1.5, 2.0, 2.0], 4: [-0.5, 0.25, 1.25, 3.0 if case == "runs_out" else 10.0]}
    if fmt == "RGBA":
        rows = {o: [abs(v) / 2.5 for v in r[:3]] + [r[3]] for o, r in rows.items()}
    tree, data = _root_tree(rows, fmt)
    rows = {o: data.reshape(8, 4)[o].astype(np.float64) for o in rows}   # the fp16 values the march reads
    g = np.array([0.7, -1.3, 0.4, 2.1])
    bg, stop = 0.6, (0.0 if case == "runs_out" else 0.01)
    opt = ob.make_options(step_size=0.0, stop_thresh=stop, background_brightness=bg)
    dpix = np.tile(g.astype(np.float32), (1, 1, 1))
    grad, A, rgba = gb.leaf_grads(tree, _ray_along_x(0.25, 0.25), opt, dpix, tile=AXIS)
    f, _, _ = ob.render(tree, _ray_along_x(0.25, 0.25), opt, tile=AXIS)
    assert np.array_equal(rgba.view(np.uint32), f.view(np.uint32))
    assert (rgba[0, 0, 3] == 1.0) == (case == "stops_early")
    want = _closed_form(rows, fmt, g, bg, stop)
    # Δδ is 1/2 - 1e-6 (the box is shrunk by 1e-6 at both ends): relative 4e-6
    np.testing.assert_allclose(grad[[0, 4]], want, rtol=1e-4, atol=1e-7)
    assert not np.delete(grad, [0, 4], axis=0).any()
    assert (A >= np.abs(grad)).all()


def _loss(ot, cam, opt, dpix, tile):
    from oracle import binding as ob
    f, _, cnt = ob.render(ot, cam, opt, tile=tile, want_u8=False)
    return float(np.dot(f.astype(np.float64).reshape(-1), dpix.astype(np.float64).reshape(-1))), cnt


def _fd_check(ot, cam, opt, tile, seed, n_pick=8):
    """Central differences of sum(dpix * orc_render) with the fp16 neighbours of a data value as the step, for the
    entries of the largest oracle gradients: coefficients, sigma and (through dpix's alpha) the alpha channel."""
    from oracle import grads_binding as gb
    rng = np.random.default_rng(seed)
    h, w = tile[3], tile[2]
    dpix = rng.uniform(-1, 1, (h, w, 4)).astype(np.float32)
    grad, A, _ = gb.leaf_grads(ot, cam, opt, dpix, tile=tile)
    dd = ot.c.data_dim
    flat = ot.data.reshape(-1, dd)          # the array the oracle tree points at (fp16 bits)
    checked = {"coef": 0, "sigma": 0}
    for col_kind, cols in (("sigma", [dd - 1]), ("coef", list(range(dd - 1)))):
        mag = np.abs(grad[:, cols])
        order = np.argsort(-mag, axis=None)[:4 * n_pick]
        for flat_i in order:
            s, j = np.unravel_index(flat_i, mag.shape)
            col = cols[j]
            if mag[s, j] < 1e-4 or checked[col_kind] >= n_pick:
                continue
            bits = int(flat[s, col])
            v = float(np.array(bits, np.uint16).view(np.float16))
            if not math.isfinite(v) or abs(v) > 1e3:
                continue
            # a step of a few fp16 ulps, so that it is well above the float render's resolution; the step taken is the
            # actual difference of the two fp16 values
            h = 2e-3 * max(1.0, abs(v))
            up, dn = np.float16(v + h), np.float16(v - h)
            flat[s, col] = np.array(up, np.float16).view(np.uint16)
            lp, cp = _loss(ot, cam, opt, dpix, tile)
            flat[s, col] = np.array(dn, np.float16).view(np.uint16)
            lm, cm = _loss(ot, cam, opt, dpix, tile)
            flat[s, col] = bits
            _, c0 = _loss(ot, cam, opt, dpix, tile)
            if not (cp == cm == c0):
                continue                    # the step moved a sample across sigma_thresh or stop_thresh
            fd = (lp - lm) / (float(up) - float(dn))
            g = grad[s, col]
            assert abs(fd - g) <= 0.05 * abs(g) + 2e-3 * A[s, col] + 1e-5, (s, col, fd, g, A[s, col])
            checked[col_kind] += 1
    assert checked["coef"] > 0 and checked["sigma"] > 0, checked


@pytest.mark.parametrize("tree_name", ["mixed_sh16", "mixed_sh9", "mixed_sh1", "mixed_rgba", "mixed_sg9",
                                       "mixed_asg4", "aniso_ndc", "sigma_bits"])
def test_finite_differences_edge_trees(tree_name):
    from oracle import binding as ob
    from volrend_b200 import synth
    st, _ = ec.edge_tree(tree_name)
    fr = next(f for f in ec.frames_of(tree_name) if ec.frame(f, st)[7] is None)
    _, W, H, fx, fy, pose, kw, _ = ec.frame(fr, st)
    ot = ob.OracleTree.from_synth(st, ndc=ec.NDC.get(tree_name))
    cam = ob.make_camera(W, H, fx, fy, synth.c2w_to_colmajor12(pose))
    kw = dict(kw, render_depth=0, stop_thresh=0.0)    # no early stop: every step keeps the sample sequence
    tile = (max(W // 2 - 6, 0), max(H // 2 - 6, 0), min(12, W), min(12, H))
    _fd_check(ot, cam, ob.make_options(**kw), tile, seed=ec.TREES.index(tree_name))


@pytest.mark.parametrize("case", ["lego_sh16", "drums_sh9", "lego_sh25_bbox", "lego_rgba", "lego_sg9_rot",
                                  "lego_sh16_ndc"])
def test_finite_differences_golden_trees(case):
    from oracle import binding as ob
    from volrend_b200 import synth
    st, W, H, pose, kw, ndc = gc.build_case(case)
    ot = ob.OracleTree.from_synth(st, ndc=ndc)
    cam = ob.make_camera(W, H, synth.focal_for(W), synth.focal_for(W), synth.c2w_to_colmajor12(pose))
    tile = (W // 2 - 8, H // 2 - 8, 16, 16)
    _fd_check(ot, cam, ob.make_options(**kw), tile, seed=7)


def test_oracle_refuses_render_depth():
    from oracle import binding as ob
    from oracle import grads_binding as gb
    tree, _ = _root_tree({0: [0, 0, 0, 1.0]}, "SH1")
    with pytest.raises(RuntimeError):
        gb.leaf_grads(tree, _ray_along_x(0.25, 0.25), ob.make_options(render_depth=1), np.zeros((1, 1, 4)), tile=AXIS)


# ------------------------------------------------------------------------------------------- npz and CLI
def _files(tmp_path):
    from volrend_b200 import synth
    st = ec.mixed_tree(3, 4, "SH", 5)
    src = str(tmp_path / "t.npz")
    d = st.npz_dict()
    d["parent_depth"] = np.zeros(3, np.int32)
    np.savez(src, **d)
    qsrc = str(tmp_path / "q.npz")
    np.savez(qsrc, **synth.quantise_tree(st, n_retain=1, seed=3))
    pose = str(tmp_path / "p.txt")
    np.savetxt(pose, np.vstack([np.eye(4), np.eye(4)]))
    return st, src, qsrc, pose


def test_finetune_npz_keys_and_dtype(tmp_path):
    from volrend_b200 import finetune_npz, synth
    st, src, qsrc, _ = _files(tmp_path)
    with np.load(src) as z:
        new = np.asarray(z["data"], np.float32) * 0.5
        out = finetune_npz(z, new)
        assert set(out) == set(z.files) - {"parent_depth"}
        for k in out:
            if k != "data":
                assert np.array_equal(out[k], z[k]), k
        assert out["data"].dtype == z["data"].dtype == np.float16
        assert np.array_equal(out["data"], new.astype(np.float16))
        with pytest.raises(ValueError, match="shape"):
            finetune_npz(z, new[:1])
    d32 = dict(st.npz_dict(), data=st.data.astype(np.float32))
    assert finetune_npz(d32, st.data.astype(np.float64))["data"].dtype == np.float32
    with np.load(qsrc) as q, pytest.raises(ValueError, match="compressed"):
        finetune_npz(q, st.data)


def test_cli_argument_errors(tmp_path, capsys):
    import importlib
    from volrend_b200 import write_png_file
    finetune = importlib.import_module("volrend_b200.finetune")   # the package exports the function of that name
    st, src, qsrc, pose = _files(tmp_path)
    out = str(tmp_path / "o.npz")
    npy = str(tmp_path / "t.npy")
    np.save(npy, np.zeros((2, 8, 6, 3), np.uint8))
    bad_npy = str(tmp_path / "b.npy")
    np.save(bad_npy, np.zeros((2, 8, 6), np.uint8))
    three = str(tmp_path / "three.npy")
    np.save(three, np.zeros((3, 8, 6, 4), np.float32))
    png = str(tmp_path / "a.png")
    assert write_png_file(png, np.zeros((8, 6, 4), np.uint8))
    size = ["--width", "6", "--height", "8"]
    cases = [
        ([src, out, pose], "--targets"),
        ([src, out, pose, "--targets", npy, "--steps", "-1"] + size, "--steps"),
        ([src, out, pose, "--targets", npy, "--batch", "0"] + size, "--batch"),
        ([src, out, pose, "--targets", npy, "--lr", "0"] + size, "--lr"),
        ([src, out, pose, "--targets", npy, "--lr", "nan"] + size, "--lr"),
        ([src, src, pose, "--targets", npy] + size, "overwrite the input"),
        ([src, out, pose, "--targets", str(tmp_path / "missing.npy")] + size, "does not exist"),
        ([src, out, pose, "--targets", npy, "--width", "0"], "image size"),
        ([src, out, pose, "--targets", npy, "--holdout", "2"] + size, "--holdout"),
        ([src, out, pose, "--targets", npy, "--holdout", "-1"] + size, "--holdout"),
        ([src, out, pose, "--targets", three] + size, "3 targets for 2 poses"),
        ([src, out, pose, "--targets", bad_npy] + size, "not [views, height, width"),
        ([src, out, pose, "--targets", npy, "--width", "8", "--height", "6"], "the views 8x6"),
        ([src, out, pose, "--targets", png] + size, "1 targets for 2 poses"),
        ([src, out, pose, "--targets", png, png, "--width", "7", "--height", "8"], "the views 7x8"),
        ([src, out, pose, "--targets", png, npy] + size, "one .npy file or one .png per pose"),
        ([qsrc, out, pose, "--targets", npy] + size, "compressed"),
    ]
    for argv, msg in cases:
        with pytest.raises(SystemExit) as e:
            finetune.main(argv)
        assert e.value.code == 2, argv
        assert msg in capsys.readouterr().err, argv
    assert not (tmp_path / "o.npz").exists()


def test_view_png_targets_read_lazily_and_composited(tmp_path):
    import torch
    from volrend_b200 import write_png_file
    from volrend_b200.views import read_targets, target_rgb
    rgba = np.zeros((4, 5, 4), np.uint8)
    rgba[..., 0] = 255
    rgba[..., 3] = np.arange(5, dtype=np.uint8) * 60
    p = str(tmp_path / "a.png")
    assert write_png_file(p, rgba)
    t = read_targets([p, p], 2, 5, 4)
    assert len(t) == 2 and len(t[:1]) == 1
    img = t[1]
    assert img.shape == (4, 5, 4) and np.array_equal(img, rgba)
    rgb = target_rgb(img, 0.25, torch.device("cpu")).numpy()
    a = rgba[..., 3:4] / 255.0
    np.testing.assert_allclose(rgb, np.concatenate([a + 0.25 * (1 - a), 0.25 * (1 - a), 0.25 * (1 - a)], -1), atol=1e-6)


def test_new_entry_points_without_a_device(built):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from volrend_b200 import _capi, lib
    L = lib()
    fake = C.create_string_buffer(4096)
    cam = _capi.vr_camera(8, 8, 10.0, 10.0)
    o = _capi.vr_options()
    L.vr_default_options(C.byref(o))
    buf = C.c_void_p(0x1000)
    t = C.addressof(fake)
    assert L.vr_tree_leaf_grads(t, C.byref(cam), 1, C.byref(o), None, buf, buf, None, None) == _capi.VR_ENODEVICE
    assert b"no CPU fallback" in L.vr_last_error()
    assert L.vr_tree_leaf_grads(t, C.byref(cam), 1, C.byref(o), None, None, buf, None, None) == _capi.VR_EINVAL
    assert L.vr_tree_leaf_grads(t, C.byref(cam), 1, C.byref(o), None, buf, None, None, None) == _capi.VR_EINVAL
    assert L.vr_tree_leaf_grads(t, C.byref(cam), -1, C.byref(o), None, buf, buf, None, None) == _capi.VR_EINVAL
    assert L.vr_tree_leaf_grads(None, None, 0, None, None, None, None, None, None) == _capi.VR_OK
    assert L.vr_tree_update_data(t, buf, None) == _capi.VR_ENODEVICE
    assert L.vr_tree_update_data(None, buf, None) == _capi.VR_EINVAL
