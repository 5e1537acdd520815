"""The tree compressor without a GPU: the numpy oracle on hand-checkable point sets, the dict assembly, a CPU round
trip through the loader, the CLI, and the C-ABI's answer when there is no device."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import compress_cases as cc
from oracle import quant_oracle as qo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
h = np.float16


def _cut(pts, bits):
    pts = np.asarray(pts, h).reshape(-1, 3).view(np.uint16)
    return qo.median_cut(pts[:, 0], pts[:, 1], pts[:, 2], bits)


def _f(colors):
    return colors.view(h)


# ---- the median cut and the means, on sets small enough to check by hand
def test_empty_set_gives_zero_codebook():
    colors, bucket = _cut(np.zeros((0, 3)), 16)
    assert colors.shape == (65536, 3) and not colors.any() and bucket.size == 0


def test_one_point_goes_to_the_odd_children():
    colors, bucket = _cut([[1.5, -2.0, 3.0]], 3)
    assert bucket.tolist() == [7]                     # 0 -> 1 -> 3 -> 7
    assert _f(colors)[7].tolist() == [1.5, -2.0, 3.0]
    assert not np.delete(colors, 7, 0).any()


def test_three_points():
    # x is the only axis with a range; level 0: sorted 1,2,3 -> {1} | {2,3}; level 1: {} | {1} and {2} | {3}
    colors, bucket = _cut([[3, 0, 0], [1, 0, 0], [2, 0, 0]], 2)
    assert bucket.tolist() == [3, 1, 2]
    assert _f(colors)[:4, 0].tolist() == [0, 1, 2, 3]


@pytest.mark.parametrize("bits", [1, 5, 8])
def test_sizes_follow_the_path(bits):
    rng = np.random.default_rng(bits)
    for M in (2 ** bits - 1, 2 ** bits + 1):
        _, bucket = _cut(rng.standard_normal((M, 3)), bits)
        sizes = qo.bucket_sizes(M, bits)
        assert np.array_equal(np.bincount(bucket, minlength=2 ** bits), sizes)
        assert sizes.max() - sizes.min() <= 1
        if M == 2 ** bits - 1:
            assert sizes[0] == 0 and (sizes[1:] == 1).all()   # the one empty bucket is the all-even path


def test_all_points_equal():
    colors, bucket = _cut(np.full((37, 3), 0.25), 4)
    sizes = qo.bucket_sizes(37, 4)
    assert np.array_equal(np.bincount(bucket, minlength=16), sizes)
    assert (_f(colors)[:16][sizes > 0] == h(0.25)).all() and not colors[:16][sizes == 0].any()
    # ties keep set order, so the buckets hold consecutive runs of points
    assert np.array_equal(bucket, np.repeat(np.arange(16), sizes))


def test_value_ties_keep_the_current_order():
    # level 0 cuts by y (the only range): y=0 points, in set order, then y=1 points; level 1 has no range left, so
    # each half splits in its current order
    pts = [[0, 0, 0], [0, 1, 0], [0, 0, 0], [0, 1, 0], [0, 0, 0], [0, 1, 0], [0, 0, 0], [0, 1, 0]]
    _, bucket = _cut(pts, 2)
    assert bucket.tolist() == [0, 2, 0, 2, 1, 3, 1, 3]


def test_child_order_is_the_sorted_order():
    # Q(1, 5) P(0, 5) T(.5, 0) U(.7, 10) and four at (20, 5).  Level 0 cuts by x (range 20): the even child is
    # P, T, U, Q in that order.  Level 1 cuts it by y (range 10 > 1): T, P, Q, U -- P before Q, because the child keeps
    # the sorted order.  A split that kept set order would put Q first and send it to bucket 0 instead of P.
    pts = [[1.0, 5, 0], [0.0, 5, 0], [0.5, 0, 0], [0.7, 10, 0]] + [[20, 5, 0]] * 4
    colors, bucket = _cut(pts, 2)
    assert bucket[:4].tolist() == [1, 0, 0, 1]
    assert _f(colors)[0].tolist() == [0.25, 2.5, 0]


def test_mixed_signed_zeros_are_one_value():
    pts = np.array([[0.0, -0.0, 0.0], [-0.0, 0.0, -0.0]] * 4, h)
    colors, bucket = _cut(pts, 3)
    assert bucket.tolist() == list(range(8))       # no axis has a range: the points split in set order
    assert (colors[:8] == 0).all()                 # the mean of a signed zero is +0


def test_axis_range_tie_takes_the_lowest_axis():
    pts = [[0, 0, 0], [2, 2, 0], [1, 0, 0], [0, 2, 0]]          # x range 2 == y range 2
    _, bucket = _cut(pts, 1)
    assert bucket.tolist() == [0, 1, 1, 0]                       # sorted by x: (0,0) (0,2) | (1,0) (2,2)
    _, bucket = _cut([[0, 0, 0], [0, 2, 0], [0, 1, 0], [0, 0, 3]], 1)   # z range 3 wins
    assert bucket.tolist() == [0, 0, 1, 1]                       # z: three zeros (set order), then 3


def test_exact_mean_where_a_double_running_sum_rounds():
    pts = cc.adversarial_sets()["big_sum"]
    colors, bucket = _cut(pts, 1)
    x = pts[:, 0].view(np.uint16)
    members = np.nonzero(bucket == 0)[0]
    S = sum(int(v) for v in qo.mult24(x[members]))                # exact, in units of 2^-24
    run = 0.0
    for v in qo.mult24(x[members]):                               # a double running sum drops every small term
        run += float(v)
    assert run != float(S)
    assert colors[0, 0] == np.float16(float(S) / members.size * 2.0 ** -24).view(np.uint16)


def test_exact_sum_beyond_64_bits():
    # more than 2^23 points of 65504 (2^39.99 units each): the exact sum needs more than 64 bits
    M = (1 << 23) + 5
    x = np.full(M, h(65504.0)).view(np.uint16)
    colors, _ = qo.median_cut(x, x, x, 1)
    assert (_f(colors)[:2] == h(65504.0)).all()


def test_zero_padding_rows():
    rng = np.random.default_rng(0)
    colors, bucket = _cut(rng.standard_normal((100, 3)), 5)
    assert not colors[32:].any() and bucket.max() < 32


def test_fp16_threshold():
    s = np.array([0.3, 0.2998, 0.3003, np.nan, -1.0, 2.0], h).view(np.uint16)
    # fp16(0.3) > fp16_rn(0.3) is false, an fp32 compare would keep it; NaN is never kept
    assert qo.kept_mask(s, 0.3).tolist() == [False, False, True, False, False, True]
    assert np.float32(np.float16(0.3)) > np.float32(0.3)


# ---- the dict and the loader
def test_dict_assembly_and_cpu_round_trip():
    from volrend_b200 import N3Tree, compress_npz, synth
    st = synth.make_tree("lego", depth=5, basis_dim=9, seed=1)
    z = cc.tree_dict(st)
    z["extra_key"] = np.arange(3)
    out = compress_npz(z, retain=2, bits=6, sigma_thresh=1.0, backend=qo.compress_arrays)
    assert "data" not in out and not any(k in out for k in ("parent_depth", "n_internal", "depth_limit"))
    assert out["extra_key"] is z["extra_key"] and out["child"] is z["child"]
    cap = st.capacity
    assert out["quant_colors"].shape == (7, 65536, 3) and out["quant_colors"].dtype == np.float16
    assert out["quant_map"].shape == (7, cap, 2, 2, 2) and out["quant_map"].dtype == np.uint16
    assert out["sigma"].shape == (cap, 2, 2, 2) and out["sigma"].dtype == np.float16
    assert out["data_retained"].shape == (2, cap, 2, 2, 2, 3) and out["data_retained"].dtype == np.float16
    t = N3Tree(gpu_decode=False)
    t.load_npz(out)
    dec = t.data_.view(np.uint16).reshape(-1, 28)
    src = st.data.view(np.uint16).reshape(-1, 28)
    keep = qo.kept_mask(src[:, -1], 1.0)
    assert keep.any() and not keep.all()
    assert np.array_equal(dec[keep, -1], src[keep, -1]) and not dec[~keep, -1].any()
    B = 9
    qc, qm = out["quant_colors"].view(np.uint16), out["quant_map"].reshape(7, -1)
    assert not qm[:, ~keep].any()                  # a dropped slot maps to row 0
    for j in range(B):
        for k in range(3):
            col = dec[:, k * B + j]
            if j < 2:
                assert np.array_equal(col[keep], src[keep, k * B + j]) and not col[~keep].any()
            else:
                assert np.array_equal(col, qc[j - 2][qm[j - 2], k])


def test_passes_legacy_keys_through_and_rejects_bad_input():
    from volrend_b200 import compress_npz
    z = cc.sh1_tree(np.ones((10, 3), h))
    del z["data_format"]
    out = compress_npz(z, retain=0, backend=qo.compress_arrays)
    assert "data_format" not in out and out["quant_colors"].shape == (1, 65536, 3) and "data_retained" not in out
    for kw, msg in [(dict(bits=0), "bits"), (dict(bits=17), "bits"), (dict(retain=-1), "retain"),
                    (dict(retain=1), "no basis function")]:
        with pytest.raises(ValueError, match=msg):
            compress_npz(z, **{"retain": 0, **kw}, backend=qo.compress_arrays)
    bad = dict(z, data_dim=np.int64(5), data=np.zeros((2, 2, 2, 2, 5), h))
    with pytest.raises(ValueError, match="3 \\* basis_dim"):
        compress_npz(bad, retain=0, backend=qo.compress_arrays)
    z["data"].reshape(-1, 4)[3, 2] = np.inf
    with pytest.raises(ValueError, match="Inf or NaN"):
        compress_npz(z, retain=0, backend=qo.compress_arrays)


# ---- the CLI
def _cli(*args):
    return subprocess.run([sys.executable, "-m", "volrend_b200.compress", *map(str, args)], cwd=ROOT,
                          capture_output=True, text=True)


def test_cli_noquant_skip_overwrite(tmp_path):
    z = cc.sh1_tree(np.ones((10, 3), h))
    z["n_free"] = np.int64(0)
    src = tmp_path / "a.npz"
    np.savez(src, **z)
    out_dir = tmp_path / "o"
    r = _cli(src, "--noquant", "--out_dir", out_dir)
    assert r.returncode == 0, r.stderr
    assert "deflate" in r.stdout and "MB ->" in r.stdout
    with np.load(out_dir / "a.npz") as got:
        assert sorted(got.files) == sorted(k for k in z if k != "n_free")
        assert np.array_equal(got["data"], z["data"])
    before = (out_dir / "a.npz").stat().st_mtime_ns
    r = _cli(src, "--noquant", "--out_dir", out_dir)
    assert "> skip" in r.stdout and (out_dir / "a.npz").stat().st_mtime_ns == before
    os.utime(out_dir / "a.npz", ns=(0, 0))
    r = _cli(src, "--noquant", "--overwrite", "--out_dir", out_dir)
    assert r.returncode == 0 and (out_dir / "a.npz").stat().st_mtime_ns != 0


def test_cli_skips_compressed_sources_and_rejects_weighted(tmp_path):
    from volrend_b200 import compress_npz
    z = compress_npz(cc.sh1_tree(np.ones((10, 3), h)), retain=0, backend=qo.compress_arrays)
    src = tmp_path / "c.npz"
    np.savez(src, **z)
    r = _cli(src, "--out_dir", tmp_path / "o")
    assert r.returncode == 0 and "already compressed" in r.stdout and not (tmp_path / "o" / "c.npz").exists()
    r = _cli(src, "--weighted", "--out_dir", tmp_path / "o")
    assert r.returncode != 0 and "--weighted is not supported" in r.stderr
    r = _cli(src, "--bits", "17", "--out_dir", tmp_path / "o")
    assert r.returncode != 0 and "bits" in r.stderr


def test_cli_error_leaves_no_output(tmp_path):
    z = cc.sh1_tree(np.ones((10, 3), h))
    src = tmp_path / "rgba.npz"
    np.savez(src, **z)
    r = _cli(src, "--retain", "1", "--out_dir", tmp_path / "o")   # SH1 with retain 1: nothing left to quantise
    assert r.returncode != 0 and "no basis function" in r.stderr
    assert os.listdir(tmp_path / "o") == []


# ---- the C-ABI without a device
def test_capi_without_device(built):
    import torch
    from volrend_b200 import _capi, lib
    L = lib()
    n = C.c_int64(-7)
    fake = C.create_string_buffer(64)          # never dereferenced: the argument and device checks come first
    p = C.addressof(fake)
    assert L.vr_tree_compress(p, 8, 4, 2.0, 0, 0, p, p, p, None, C.byref(n), None) == _capi.VR_EINVAL
    assert b"bits" in L.vr_last_error()
    assert L.vr_tree_compress(p, 8, 4, 2.0, 1, 16, p, p, p, p, C.byref(n), None) == _capi.VR_EINVAL
    assert L.vr_tree_compress(p, 8, 5, 2.0, 0, 16, p, p, p, None, C.byref(n), None) == _capi.VR_EINVAL
    assert L.vr_tree_compress(p, 8, 7, 2.0, 1, 16, p, p, p, None, C.byref(n), None) == _capi.VR_EINVAL   # retain, NULL
    assert L.vr_tree_compress(p, 8, 7, 2.0, -1, 16, p, p, p, None, C.byref(n), None) == _capi.VR_EINVAL
    if torch.cuda.is_available():
        return
    assert L.vr_tree_compress(p, 8, 7, 2.0, 1, 16, p, p, p, p, C.byref(n), None) == _capi.VR_ENODEVICE
    assert b"no CPU fallback" in L.vr_last_error()
    assert n.value == 0


def test_written_file_has_umask_permissions(tmp_path):
    from volrend_b200.compress import _write_npz
    path = tmp_path / "t.npz"
    old = os.umask(0o022)
    try:
        _write_npz(str(path), dict(a=np.arange(3)))
    finally:
        os.umask(old)
    assert (path.stat().st_mode & 0o777) == 0o644
    assert os.listdir(tmp_path) == ["t.npz"]
