"""`-m gpu`: the tree compressor (vr_tree_compress, volrend_b200.compress) against the numpy oracle, bit for bit, and
its output through the loaders."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _both(z, bits, retain, sigma_thresh=2.0):
    from oracle import quant_oracle as qo
    from volrend_b200.compress import compress_arrays
    data = np.ascontiguousarray(np.asarray(z["data"])).view(np.uint16)
    dd = int(z["data_dim"])
    flat = data.reshape(-1, dd)
    return compress_arrays(flat, dd, sigma_thresh, retain, bits), qo.compress_arrays(flat, dd, sigma_thresh, retain, bits)


def _assert_same(got, want):
    names = ["quant_colors", "quant_map", "sigma", "data_retained"]
    for n, g, w in zip(names, got[:4], want[:4]):
        if w is None:
            assert g is None, n
        else:
            assert g.shape == w.shape and np.array_equal(g, w), (n, int((g != w).sum()))
    assert got[4] == want[4]


@pytest.mark.parametrize("name,kind,depth,basis,fmt,retain,bits", [
    ("sh16_d6", "lego", 6, 16, "SH", 1, 16),
    ("sh16_d6_b5", "lego", 6, 16, "SH", 1, 5),
    ("sh9_r0", "lego", 6, 9, "SH", 0, 16),
    ("sh9_r4_b1", "lego", 6, 9, "SH", 4, 1),
    ("sh25_d5", "drums", 5, 25, "SH", 1, 16),
    ("sg7_extra", "lego", 5, 7, "SG", 1, 5),
])
def test_stand_in_trees_match_oracle(built, name, kind, depth, basis, fmt, retain, bits):
    import compress_cases as cc
    from volrend_b200 import synth
    st = synth.make_tree(kind, depth=depth, basis_dim=basis, fmt=fmt, seed=3)
    got, want = _both(cc.tree_dict(st), bits, retain)
    assert want[4] > 0
    _assert_same(got, want)


@pytest.mark.parametrize("bits", [1, 5, 16])
def test_adversarial_sets_match_oracle(built, bits):
    import compress_cases as cc
    sets = dict(cc.adversarial_sets())
    rng = np.random.default_rng(bits)
    for M in (2 ** bits - 1, 2 ** bits + 1):
        sets[f"M{M}"] = rng.standard_normal((M, 3)).astype(np.float16)
    for name, pts in sets.items():
        got, want = _both(cc.sh1_tree(pts), bits, 0)
        _assert_same(got, want)
    # no slot kept (every sigma at the threshold)
    got, want = _both(cc.sh1_tree(sets["three"], sigma=2.0), bits, 0)
    assert want[4] == 0
    _assert_same(got, want)


def test_exactly_65536_points_at_16_bits(built):
    import compress_cases as cc
    pts = np.random.default_rng(11).standard_normal((65536, 3)).astype(np.float16)
    got, want = _both(cc.sh1_tree(pts), 16, 0)
    assert want[4] == 65536
    _assert_same(got, want)
    assert np.unique(got[1][0]).size == 65536          # one point per bucket: the codebook is the point set


def test_bucket_sums_beyond_64_bits(built):
    """2^25 + 2^20 points in [64000, 65504] at bits 1: each bucket's exact sum exceeds 2^64 units of 2^-24, so the
    128-bit sum and its rounding to double run on the device (values vary, so the rounding matters)."""
    import compress_cases as cc
    M = (1 << 25) + (1 << 20)
    pts = np.random.default_rng(3).uniform(64000.0, 65504.0, (M, 3)).astype(np.float16)
    got, want = _both(cc.sh1_tree(pts), 1, 0)
    assert want[4] == M
    sizes = np.bincount(want[1][0].astype(np.int64))
    assert sizes.min() * 64000.0 * 2 ** 24 >= 2.0 ** 64
    _assert_same(got, want)


def test_sh16_depth8_all_sets(built):
    import compress_cases as cc
    from volrend_b200 import synth
    st = synth.make_tree("lego", depth=8, basis_dim=16, seed=0)
    got, want = _both(cc.tree_dict(st), 16, 1)
    assert got[0].shape[0] == 15 and want[4] > 200_000
    _assert_same(got, want)


def test_config2_tree_two_sets(built):
    """The bench tree (depth 10, SH16, seed 0): the last two basis functions (retain 14), 4.5 M points each."""
    import compress_cases as cc
    from volrend_b200 import synth
    st = synth.make_tree("lego", depth=10, basis_dim=16, seed=0)
    got, want = _both(cc.tree_dict(st), 16, 14)
    assert got[0].shape[0] == 2 and want[4] > 4_000_000
    _assert_same(got, want)


def test_repeatable_bytes(built):
    import compress_cases as cc
    from volrend_b200 import compress_npz, synth
    z = cc.tree_dict(synth.make_tree("lego", depth=7, basis_dim=16, seed=5))
    a, b = compress_npz(z), compress_npz(z)
    assert a.keys() == b.keys()
    for k in a:
        assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes(), k


def test_capi_rejects(built):
    import torch
    import compress_cases as cc
    from volrend_b200.compress import compress_device
    z = cc.sh1_tree(np.ones((16, 3), np.float16))
    d = torch.from_numpy(np.asarray(z["data"]).view(np.int16).reshape(-1, 4).copy()).cuda()
    for kw, msg in [(dict(bits=0), "bits"), (dict(bits=17), "bits"), (dict(retain=-1), "retain"),
                    (dict(retain=1), "no basis function")]:
        with pytest.raises(ValueError, match=msg):
            compress_device(d, 4, **{"retain": 0, **kw})
    with pytest.raises(ValueError, match="3 \\* basis_dim"):
        compress_device(d.reshape(-1)[:40].reshape(-1, 5), 5, retain=0)
    bad = d.clone()
    bad.view(torch.float16)[3, 1] = float("inf")
    with pytest.raises(ValueError, match="Inf or NaN"):
        compress_device(bad, 4, retain=0)
    bad.view(torch.float16)[3, 3] = 1.0                # not kept: its coefficients do not matter
    compress_device(bad, 4, retain=0)
    with pytest.raises(ValueError, match="contiguous"):
        compress_device(d.float(), 4, retain=0)
    with pytest.raises(ValueError, match="contiguous"):
        compress_device(d.t(), 4, retain=0)


def _render_pair(path):
    import torch
    from volrend_b200 import Camera, N3Tree, RenderOptions, launch_renderer, synth
    out = []
    for gpu_decode in (True, False):
        t = N3Tree(path, gpu_decode=gpu_decode)
        frames = []
        for i in (0, 37):
            cam = Camera(160, 120, synth.focal_for(160), synth.focal_for(160))
            cam.set_c2w(synth.nerf_synthetic_test_poses(200)[i])
            img = torch.zeros((120, 160, 4), dtype=torch.uint8, device="cuda")
            fo = torch.zeros((120, 160, 4), dtype=torch.float32, device="cuda")
            launch_renderer(t, cam, RenderOptions(), img, None, None, True, float_out=fo)
            torch.cuda.synchronize()
            frames.append((cam, fo.cpu().numpy(), img.cpu().numpy()))
        out.append(frames)
        t.free_cuda()
    return out


def test_written_file_renders_the_same_through_every_loader(built, tmp_path):
    import compress_cases as cc
    from oracle import ref_binding as rb
    from volrend_b200 import compress_npz, synth
    from volrend_b200.compress import _write_npz
    st = synth.make_tree("lego", depth=7, basis_dim=16, seed=2)
    path = str(tmp_path / "tree.npz")
    _write_npz(path, compress_npz(cc.tree_dict(st), retain=4))
    gpu, cpu = _render_pair(path)
    assert any(f.any() for _, f, _ in gpu)
    for (_, fg, ug), (_, fc, uc) in zip(gpu, cpu):
        assert np.array_equal(fg, fc) and np.array_equal(ug, uc)
    if rb.available():
        rt = rb.RefTree(path)                   # the reference loader reads the deflated npz through cnpy
        try:
            for cam, f, u in gpu:
                c12 = np.ascontiguousarray(cam.transform, np.float32).reshape(12)
                assert np.array_equal(f, rt.render_f32(cam.width, cam.height, cam.fx, cam.fy, c12, rb.make_options()))
                assert np.array_equal(u, rt.render_u8(cam.width, cam.height, cam.fx, cam.fy, c12, rb.make_options()))
        finally:
            rt.close()


def test_cli_end_to_end(built, tmp_path):
    import compress_cases as cc
    from oracle import quant_oracle as qo
    from volrend_b200 import synth
    st = synth.make_tree("lego", depth=6, basis_dim=9, seed=4)
    src = tmp_path / "scene.npz"
    np.savez(src, **cc.tree_dict(st))
    out_dir = tmp_path / "out"
    cmd = [sys.executable, "-m", "volrend_b200.compress", str(src), "--out_dir", str(out_dir), "--bits", "12",
           "--retain", "2", "--sigma_thresh", "0.5"]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert "MB ->" in r.stdout
    with np.load(out_dir / "scene.npz") as z:
        got = {k: z[k] for k in z.files}
    assert "data" not in got and "parent_depth" not in got and "depth_limit" not in got
    flat = np.ascontiguousarray(st.data).view(np.uint16).reshape(-1, st.data_dim)
    c, m, s, ret, _ = qo.compress_arrays(flat, st.data_dim, 0.5, 2, 12)
    assert np.array_equal(got["quant_colors"].view(np.uint16), c)
    assert np.array_equal(got["quant_map"].reshape(m.shape), m)
    assert np.array_equal(got["sigma"].view(np.uint16).reshape(-1), s)
    assert np.array_equal(got["data_retained"].view(np.uint16).reshape(ret.shape), ret)
