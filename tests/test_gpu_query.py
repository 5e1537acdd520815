"""GPU: vr_tree_query / vr_tree_eval (N3Tree.query / eval) against the reference's query_single_from_root (goldens
and, where oracle/_ref is built, the live library), the numpy oracle, one-point calls, and the probe disc."""
import os
import tempfile

import numpy as np
import pytest

from oracle import query_oracle as qo
from oracle import ref_query
from probe_cases import W, H, focal, probe_case
from probe_cases import golden_path as probe_golden_path
from query_cases import QUERY_TREES, SIGMA_BITS, golden_path, query_tree, tree_space_points

pytestmark = pytest.mark.gpu


def _tree(z):
    from volrend_b200 import N3Tree
    t = N3Tree()
    t.load_npz(z)
    t.load_cuda()
    return t


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint16 if a.dtype == np.float16 else np.uint32)


@pytest.mark.parametrize("name", QUERY_TREES)
def test_query_matches_reference_golden(built, name):
    g = np.load(golden_path(name))
    t = _tree(query_tree(name))
    data, cube, local = t.query(g["points"])
    assert np.array_equal(_bits(data), g["data"]), int((_bits(data) != g["data"]).any(1).sum())
    assert np.array_equal(_bits(cube), _bits(g["cube"]))
    assert np.array_equal(_bits(local), _bits(g["local"]))


@pytest.mark.skipif(not ref_query.available(), reason="oracle/_ref/libref_query.so not built")
@pytest.mark.parametrize("name", ["lego_sh16", "lego_sh25_bbox", "lego_rgba", "quant_sh4", "chain"])
def test_query_matches_live_reference(built, name):
    z = query_tree(name)
    pts = np.concatenate([np.load(golden_path(name))["points"], tree_space_points(z, 20000, 5)])
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "t.npz")
        np.savez(path, **z)
        rt = ref_query.RefQueryTree(path)
        rd, rc, rl, _ = rt.query(pts)
        rt.close()
    data, cube, local = _tree(z).query(pts)
    assert np.array_equal(_bits(data), _bits(rd)) and np.array_equal(_bits(cube), _bits(rc))
    assert np.array_equal(_bits(local), _bits(rl))


@pytest.mark.parametrize("name", ["lego_sh16", "lego_sh4_stop0", "lego_sh25_bbox", "cfg1_sh1"])
def test_batched_equals_one_point_calls_and_oracle(built, name):
    z = query_tree(name)
    t = _tree(z)
    pts = tree_space_points(z, 5003, 11)          # not a multiple of 32: partial last group
    data, cube, local = t.query(pts)
    od, oc, ol = qo.query(t.child_, t.data_, t.offset, t.scale, pts)
    assert np.array_equal(_bits(data), _bits(od)) and np.array_equal(_bits(cube), _bits(oc))
    assert np.array_equal(_bits(local), _bits(ol))
    for i in range(0, 5003, 97):
        d1, c1, l1 = t.query(pts[i:i + 1])
        assert np.array_equal(_bits(d1[0]), _bits(data[i])) and c1[0] == cube[i] and np.array_equal(l1[0], local[i])
    rgb, sigma = t.eval(pts, np.tile(np.float32([[0.0, 0.6, 0.8]]), (len(pts), 1)))
    assert np.array_equal(_bits(sigma), _bits(data[:, -1].astype(np.float32)))


def _disc_dirs(cam, disp):
    """Pixel centres and directions of the probe disc, in the float operations of vr_probe.cu (numpy float32)."""
    f32 = np.float32
    m = np.ascontiguousarray(cam.transform, np.float32).reshape(12)
    out = []
    h = f32(disp) * f32(0.5)
    for y in range(0, min(disp + 5, cam.height)):
        for x in range(max(cam.width - disp - 5, 0), cam.width):
            xx, yy = x + 5 - cam.width + disp, y - 5
            a = f32(f32(xx) / h) + f32(-1)
            b = f32(f32(yy) / h) + f32(-1)
            c = qo.fma32(a, a, f32(b * b))
            if not c <= 1:
                continue
            s = np.sqrt(f32(f32(1) - c))
            d = [qo.fma32(-m[6 + k], s, qo.fma32(b, m[3 + k], -f32(a * m[k]))) for k in range(3)]
            out.append((y, x, d))
    return out


@pytest.mark.parametrize("name", ["sh16_centre", "sh16_minmax13", "sh9", "sh25_bbox", "rgba", "sg9_rot", "asg4"])
def test_eval_matches_probe_disc_float_output(built, name):
    import torch
    from volrend_b200 import Camera, N3Tree, RenderOptions, launch_renderer
    st, pose, optkw, probe, disp, _ = probe_case(name)
    tree = N3Tree.from_synth(st)
    cam = Camera(W, H, focal(), focal())
    cam.set_c2w(pose)
    o = RenderOptions(**optkw)
    o.enable_probe, o.probe, o.probe_disp_size = True, [float(v) for v in probe], int(disp)
    img = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    fo = torch.zeros((H, W, 4), dtype=torch.float32, device="cuda")
    launch_renderer(tree, cam, o, img, None, None, True, float_out=fo)
    fo = fo.cpu().numpy()
    px = _disc_dirs(cam, disp)
    assert len(px) > 100
    dirs = np.array([p[2] for p in px], np.float32).reshape(-1, 3)
    pts = np.tile(np.asarray(probe, np.float32)[None], (len(px), 1))
    rgb, _ = tree.eval(pts, dirs, o)
    disc = np.array([fo[y, x, :3] for y, x, _ in px], np.float32)
    assert np.array_equal(_bits(rgb + np.float32(0)), _bits(disc)), int((rgb != disc).any(1).sum())


@pytest.mark.parametrize("name", ["sh16_centre", "sh16_empty", "sh16_outside", "sh16_d37", "sh16_d500",
                                  "sh16_minmax13", "sh9", "sh25_bbox", "rgba", "sg9_rot", "asg4", "sh9_composite",
                                  "sh9_depth"])
def test_eval_matches_probe_golden_disc_bytes(built, name):
    """eval, quantised as render_kernel stores a disc pixel (volrend.cu:166-172: truncate o * 255, alpha 255), against
    the disc pixels of the reference's own frames (tests/golden/ref/probe_*.npz)."""
    from volrend_b200 import Camera, N3Tree, RenderOptions
    st, pose, optkw, probe, disp, _ = probe_case(name)
    ref = np.load(probe_golden_path(name))["ref_u8"]
    cam = Camera(W, H, focal(), focal())
    cam.set_c2w(pose)
    px = _disc_dirs(cam, disp)
    assert len(px) > 0
    dirs = np.array([p[2] for p in px], np.float32).reshape(-1, 3)
    pts = np.tile(np.asarray(probe, np.float32)[None], (len(px), 1))
    rgb, _ = N3Tree.from_synth(st).eval(pts, dirs, RenderOptions(**optkw))
    v = ((rgb + np.float32(0)) * np.float32(255)).astype(np.float64)
    with np.errstate(invalid="ignore"):                 # __float2uint_rz: NaN and negatives -> 0, saturating
        u = np.where(np.isnan(v) | (v < 0), 0, np.minimum(np.trunc(v), 2.0 ** 32 - 1))
    u8 = (u.astype(np.uint64) & 0xFF).astype(np.uint8)
    want = np.array([ref[y, x] for y, x, _ in px], np.uint8)
    assert (want[:, 3] == 255).all()
    bad = (u8 != want[:, :3]).any(1)
    assert not bad.any(), (int(bad.sum()), len(px))


def _sh_basis16(d):
    """Real SH basis up to degree 3 (lumisphere.hpp's constants), float64, of directions d [n, 3]."""
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    xx, yy, zz = x * x, y * y, z * z
    return np.stack([
        np.full_like(x, 0.28209479177387814), -0.4886025119029199 * y, 0.4886025119029199 * z,
        -0.4886025119029199 * x, 1.0925484305920792 * x * y, -1.0925484305920792 * y * z,
        0.31539156525252005 * (2 * zz - xx - yy), -1.0925484305920792 * x * z, 0.5462742152960396 * (xx - yy),
        -0.5900435899266435 * y * (3 * xx - yy), 2.890611442640554 * x * y * z,
        -0.4570457994644658 * y * (4 * zz - xx - yy), 0.3731763325901154 * z * (2 * zz - 3 * xx - 3 * yy),
        -0.4570457994644658 * x * (4 * zz - xx - yy), 1.445305721320277 * z * (xx - yy),
        -0.5900435899266435 * x * (xx - 3 * yy)], 1)


def test_eval_on_compressed_tree_agrees_with_decoded(built):
    """eval on a compress_npz tree against query + numpy: the SH sum of the decoded row's coefficients along the
    direction, through a sigmoid."""
    from volrend_b200 import RenderOptions
    from volrend_b200.compress import compress_npz
    z = query_tree("lego_sh16")
    tq = _tree(compress_npz(z, bits=8, sigma_thresh=0.0, retain=1))
    pts = tree_space_points(z, 4000, 3)
    rng = np.random.default_rng(4)
    dirs = rng.standard_normal((4000, 3)).astype(np.float32)
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    rgb, sigma = tq.eval(pts, dirs, RenderOptions(basis_minmax=[0, 15]))
    data, _, _ = tq.query(pts)
    od, _, _ = qo.query(tq.child_, tq.data_, tq.offset, tq.scale, pts)     # the reference's decode of the file
    assert np.array_equal(_bits(data), _bits(od))
    coef = od[:, :48].astype(np.float64).reshape(-1, 3, 16)
    want = 1.0 / (1.0 + np.exp(-np.einsum("ncj,nj->nc", coef, _sh_basis16(dirs.astype(np.float64)))))
    assert np.abs(rgb - want).max() <= 1e-5, float(np.abs(rgb - want).max())
    assert np.array_equal(_bits(sigma), _bits(od[:, -1].astype(np.float32)))


def test_torch_in_torch_out_without_host_copies(built):
    import torch
    from torch.profiler import ProfilerActivity, profile
    z = query_tree("lego_sh16")
    t = _tree(z)
    x = torch.from_numpy(tree_space_points(z, 10000, 8)).cuda()
    d = torch.nn.functional.normalize(torch.randn(10000, 3, device="cuda"), dim=1)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        data, cube, local = t.query(x)
        rgb, sigma = t.eval(x, d)
        torch.cuda.synchronize()
    for v in (data, cube, local, rgb, sigma):
        assert isinstance(v, torch.Tensor) and v.device == x.device
    assert data.dtype == torch.float16 and data.shape == (10000, t.data_dim)
    names = [e.name for e in prof.events()]
    assert not any("DtoH" in n or "Device -> Host" in n or "Memcpy DtoH" in n for n in names), \
        [n for n in names if "emcpy" in n]
    od, _, _ = qo.query(t.child_, t.data_, t.offset, t.scale, x.cpu().numpy())
    assert np.array_equal(_bits(data.cpu().numpy()), _bits(od))


def test_errors(built, small_trees):
    import torch
    from volrend_b200 import N3Tree, VolrendError, _capi, lib
    t = N3Tree.from_synth(small_trees["sg7_d5"])          # basis 7: only coefficient 0 is resident
    pts = np.zeros((5, 3), np.float32)
    with pytest.raises(VolrendError) as e:
        t.query(pts)
    assert e.value.code == _capi.VR_EUNSUPPORTED
    with pytest.raises(VolrendError):
        t.eval(pts, pts)
    # cube size, local coordinates and sigma need no colour record
    x = torch.zeros((5, 3), device="cuda")
    cube = torch.zeros(5, device="cuda")
    sig = torch.zeros(5, device="cuda")
    assert lib().vr_tree_query(t._handle, x.data_ptr(), 5, None, cube.data_ptr(), None, None) == 0
    assert lib().vr_tree_eval(t._handle, x.data_ptr(), None, 5, None, None, sig.data_ptr(), None) == 0
    assert lib().vr_tree_query(t._handle, x.data_ptr(), -1, None, None, None, None) == _capi.VR_EINVAL
    assert lib().vr_tree_query(t._handle, None, 5, None, cube.data_ptr(), None, None) == _capi.VR_EINVAL
    assert lib().vr_tree_query(None, x.data_ptr(), 5, None, cube.data_ptr(), None, None) == _capi.VR_EINVAL
    torch.cuda.synchronize()
    t2 = N3Tree.from_synth(small_trees["sh4_d5"])
    d, c, l = t2.query(np.zeros((0, 3), np.float32))
    assert d.shape == (0, t2.data_dim) and c.shape == (0,)
    d, c, l = t2.query(np.full((3, 3), np.nan, np.float32))
    od, oc, ol = qo.query(t2.child_, t2.data_, t2.offset, t2.scale, np.full((3, 3), np.nan, np.float32))
    assert np.array_equal(_bits(d), _bits(od)) and np.array_equal(l, ol)


def test_rows_beyond_2_pow_31_halves(built):
    import torch
    z = query_tree("lego_sh25_bbox")
    t = _tree(z)
    n = (1 << 31) // 76 + 4099                        # n * data_dim > 2^31
    assert n * t.data_dim > 2 ** 31
    x = torch.rand((n, 3), device="cuda") * 2 - 1
    data, cube, _ = t.query(x)
    torch.cuda.synchronize()
    idx = np.concatenate([np.arange(n - 3000, n), np.random.default_rng(1).integers(0, n, 2000)])
    it = torch.from_numpy(idx).cuda()
    xs = x[it].cpu().numpy()
    od, oc, _ = qo.query(t.child_, t.data_, t.offset, t.scale, xs)
    assert np.array_equal(_bits(data[it].cpu().numpy()), _bits(od))
    assert np.array_equal(cube[it].cpu().numpy(), oc)


def test_sigma_bit_patterns(built):
    """Negative, -0, +0 and NaN sigma come out of query as the source's fp16 bits and out of eval as their floats."""
    z = query_tree("sigma_bits")
    t = _tree(z)
    pts = tree_space_points(z, 6000, 9)
    data, _, _ = t.query(pts)
    sig = _bits(data)[:, -1]
    assert set(np.unique(sig).tolist()) == set(SIGMA_BITS.tolist())
    _, sigma = t.eval(pts, np.tile(np.float32([[0.0, 0.0, 1.0]]), (len(pts), 1)))
    want = data[:, -1].astype(np.float32)
    nan = np.isnan(want)
    assert nan.any() and np.array_equal(np.isnan(sigma), nan)
    assert np.array_equal(_bits(sigma[~nan]), _bits(want[~nan]))          # -0 stays -0


def test_side_stream_is_ordered_after_current_stream(built):
    """Inputs written and outputs allocated on the current stream are only read / written by a launch on another
    stream after that stream's earlier work; numpy results are complete when the call returns."""
    import torch
    z = query_tree("lego_sh16")
    t = _tree(z)
    pts = tree_space_points(z, 200000, 12)
    want, wc, wl = qo.query(t.child_, t.data_, t.offset, t.scale, pts)
    s = torch.cuda.Stream()
    for rep in range(2):
        torch.cuda._sleep(200_000_000)                 # delays the current stream's upload of pts
        data, cube, local = t.query(pts, stream=s)
        assert np.array_equal(_bits(data), _bits(want)) and np.array_equal(cube, wc), rep
        base = torch.from_numpy(pts).cuda()
        torch.cuda._sleep(200_000_000)
        x = base * 1.0                                 # written on the current stream behind the sleep
        d2, c2, _ = t.query(x, stream=s)
        s.synchronize()
        assert np.array_equal(_bits(d2.cpu().numpy()), _bits(want)), rep
        rgb, sig = t.eval(pts, np.tile(np.float32([[0.0, 0.6, 0.8]]), (len(pts), 1)), stream=s)
        assert np.array_equal(_bits(sig), _bits(want[:, -1].astype(np.float32))), rep
    torch.cuda.synchronize()


def test_buffers_on_the_wrong_device_or_host_are_refused(built):
    import torch
    from volrend_b200 import _capi, lib
    z = query_tree("cfg1_sh1")
    t = _tree(z)
    host = np.zeros((4, 3), np.float32)
    cube = torch.zeros(4, device="cuda")
    assert lib().vr_tree_query(t._handle, host.ctypes.data, 4, None, cube.data_ptr(), None, None) == _capi.VR_EINVAL
    x = torch.zeros((4, 3), device="cuda")
    hc = np.zeros(4, np.float32)
    assert lib().vr_tree_query(t._handle, x.data_ptr(), 4, None, hc.ctypes.data, None, None) == _capi.VR_EINVAL
    assert lib().vr_tree_eval(t._handle, x.data_ptr(), host.ctypes.data, 4, None, cube.data_ptr(), None, None) \
        == _capi.VR_EINVAL
    if torch.cuda.device_count() > 1:
        other = torch.zeros((4, 3), device="cuda:1")
        with pytest.raises(ValueError, match="cuda:1"):
            t.query(other)
    torch.cuda.synchronize()
