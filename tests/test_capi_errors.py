"""Error returns of the C-ABI: every failing call sets a message naming its own problem, each entry point checks its
arguments and the device in a fixed order, and batches too large for one launch are split without changing a byte."""
import ctypes as C

import numpy as np
import pytest

from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)

BUF = C.c_void_p(0x1000)   # never dereferenced: every call below that gets it fails its checks first


def _cam(w=8, h=8):
    from volrend_b200 import _capi
    c = _capi.vr_camera(w, h, 10.0, 10.0)
    c.c2w[:] = [1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0]   # column-major 3x4: identity rotation, origin
    return c


def _opt():
    from volrend_b200 import _capi, lib
    o = _capi.vr_options()
    lib().vr_default_options(C.byref(o))
    return o


def _set_unrelated_error():
    from volrend_b200 import lib
    assert lib().vr_set_variant(9) != 0
    assert b"variant 9" in lib().vr_last_error()


def test_png_failures_set_their_own_message(built, tmp_path):
    from volrend_b200 import _capi, lib
    L = lib()
    px = (C.c_uint8 * 64)()
    missing = str(tmp_path / "no_such_dir" / "f.png").encode()
    unwritten = str(tmp_path / "f.png").encode()
    cams = (_capi.vr_camera * 1)(_cam())
    paths = (C.c_char_p * 1)(unwritten)
    cases = [
        (lambda: L.vr_write_png(None, px, 4, 4), [b"null PNG path"]),
        (lambda: L.vr_write_png(missing, px, 4, 4), [missing, b"No such file or directory"]),
        (lambda: L.vr_write_png(unwritten, px, 0, 4), [unwritten, b"bad image size 0x4"]),
    ]
    for fn in (L.vr_render_frames_png, L.vr_render_frames_png_opts):
        cases += [
            (lambda fn=fn: fn(None, cams, -1, C.byref(_opt()), paths, 1), [b"n_views < 0"]),
            (lambda fn=fn: fn(None, None, 1, C.byref(_opt()), paths, 1), [b"null cameras"]),
            (lambda fn=fn: fn(None, cams, 1, C.byref(_opt()), None, 1), [b"null PNG paths"]),
        ]
    for call, words in cases:
        _set_unrelated_error()
        assert call() == _capi.VR_EINVAL
        msg = L.vr_last_error()
        assert b"variant" not in msg
        for w in words:
            assert w in msg, (w, msg)
    assert not (tmp_path / "f.png").exists()


def test_order_of_checks_without_a_device(built):
    """The return code of each entry point on a machine without a GPU: argument checks that come before the device
    check decide it, the device check decides every other case."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from volrend_b200 import _capi, lib
    L = lib()
    OK, EINVAL, ENODEV = _capi.VR_OK, _capi.VR_EINVAL, _capi.VR_ENODEVICE
    fake = C.create_string_buffer(4096)
    t = C.addressof(fake)
    cam, opt = C.byref(_cam()), C.byref(_opt())
    cams2 = (_capi.vr_camera * 2)(_cam(), _cam())
    mixed = (_capi.vr_camera * 2)(_cam(), _cam(16, 8))
    bad_tile = _capi.vr_rect(4, 0, 8, 8)
    xyz = (C.c_float * 3)(0.0, 0.0, 1.0)
    desc = _capi.vr_tree_desc()
    out = C.c_void_p()
    n = C.c_int64(0)
    off = (C.c_int32 * 3)(0, 0, 0)
    singular = (_capi.vr_camera * 1)(_capi.vr_camera(8, 8, 10.0, 10.0))
    table = [
        # (what, call, code)
        ("batch: null tree", lambda: L.vr_render_batch(None, cam, 1, opt, None, BUF, None, None, None), EINVAL),
        ("batch: no views", lambda: L.vr_render_batch(None, None, 0, None, None, None, None, None, None), OK),
        ("batch: n_views < 0", lambda: L.vr_render_batch(t, cam, -1, opt, None, BUF, None, None, None), EINVAL),
        ("batch", lambda: L.vr_render_batch(t, cam, 1, opt, None, BUF, None, None, None), ENODEV),
        ("batch: sizes differ", lambda: L.vr_render_batch(t, mixed, 2, opt, None, BUF, None, None, None), ENODEV),
        ("batch_opts", lambda: L.vr_render_batch_opts(t, cams2, 2, opt, None, BUF, None, None, None), ENODEV),
        ("render: tile outside", lambda: L.vr_render(t, cam, opt, C.byref(bad_tile), BUF, None, None, None), EINVAL),
        ("composite batch: no depth",
         lambda: L.vr_render_composite_batch(t, cam, 1, opt, None, BUF, None, None, None), EINVAL),
        ("composite batch: no views",
         lambda: L.vr_render_composite_batch(None, None, 0, None, None, None, None, None, None), OK),
        ("composite batch_opts", lambda: L.vr_render_composite_batch_opts(t, cams2, 2, opt, None, BUF, BUF, None, None),
         ENODEV),
        ("composite", lambda: L.vr_render_composite(t, cam, opt, None, BUF, BUF, None, None), ENODEV),
        ("bands: null tree", lambda: L.vr_render_bands(None, cam, opt, 4, 2, 0, BUF, None, None), EINVAL),
        ("bands batch: no views", lambda: L.vr_render_bands_batch(None, None, 0, None, 3, 0, 5, None, None, None), OK),
        ("bands batch: bad band_h", lambda: L.vr_render_bands_batch(t, cam, 1, opt, 3, 2, 0, BUF, None, None), ENODEV),
        ("trace: no counters", lambda: L.vr_debug_trace(t, cam, opt, BUF, None, None, None), ENODEV),
        ("surface: null surface", lambda: L.vr_render_surface(t, cam, opt, 0, 0, None), ENODEV),
        ("frames host: no views", lambda: L.vr_render_frames_host(t, cam, 0, opt, None), OK),
        ("frames host: null buffer", lambda: L.vr_render_frames_host(t, cam, 1, opt, None), EINVAL),
        ("frames host", lambda: L.vr_render_frames_host(t, cam, 1, opt, BUF), ENODEV),
        ("probe: no output", lambda: L.vr_draw_probe(t, cam, 1, opt, xyz, 3, None, None, None, 0, None), EINVAL),
        ("probe: no output, no views", lambda: L.vr_draw_probe(t, cam, 0, opt, xyz, 3, None, None, None, 0, None),
         EINVAL),
        ("probe: no views", lambda: L.vr_draw_probe(t, cam, 0, opt, xyz, 3, None, BUF, None, 0, None), OK),
        ("probe", lambda: L.vr_draw_probe(t, cam, 1, opt, xyz, 3, None, BUF, None, 0, None), ENODEV),
        ("probe: sizes differ", lambda: L.vr_draw_probe(t, mixed, 2, opt, xyz, 3, None, BUF, None, 0, None), ENODEV),
        ("lumisphere: null tree", lambda: L.vr_probe_lumisphere(None, xyz, BUF, None), EINVAL),
        ("lumisphere", lambda: L.vr_probe_lumisphere(t, xyz, BUF, None), ENODEV),
        ("query: n < 0", lambda: L.vr_tree_query(t, BUF, -1, BUF, None, None, None), EINVAL),
        ("query", lambda: L.vr_tree_query(t, BUF, 4, BUF, None, None, None), ENODEV),
        ("eval: null tree", lambda: L.vr_tree_eval(None, BUF, BUF, 4, opt, BUF, None, None), EINVAL),
        ("eval", lambda: L.vr_tree_eval(t, BUF, BUF, 4, opt, BUF, None, None), ENODEV),
        ("wireframe: null count", lambda: L.vr_tree_wireframe(t, 3, None, 0, None, None), EINVAL),
        ("wireframe", lambda: L.vr_tree_wireframe(t, 3, None, 0, C.byref(n), None), ENODEV),
        ("tree create: null", lambda: L.vr_tree_create(None, C.byref(out)), EINVAL),
        ("tree create quantized: null", lambda: L.vr_tree_create_quantized(None, C.byref(out)), EINVAL),
        ("tree create: N = 0", lambda: L.vr_tree_create(C.byref(desc), C.byref(out)), ENODEV),
        ("meshes: n_views < 0", lambda: L.vr_draw_meshes_batch(cams2, -1, None, off, BUF, BUF, None), EINVAL),
        ("meshes: singular camera", lambda: L.vr_draw_meshes_batch(singular, 1, None, off, BUF, BUF, None), EINVAL),
        ("meshes", lambda: L.vr_draw_meshes_batch(cams2, 2, None, off, BUF, BUF, None), ENODEV),
        ("normals: n_verts < 0", lambda: L.vr_mesh_estimate_normals(None, -1, None, 0, None), EINVAL),
        ("normals", lambda: L.vr_mesh_estimate_normals(None, 0, None, 0, None), ENODEV),
        ("compress: bits 0", lambda: L.vr_tree_compress(BUF, 8, 7, 2.0, 1, 0, BUF, BUF, BUF, BUF, C.byref(n), None),
         EINVAL),
        ("compress", lambda: L.vr_tree_compress(BUF, 8, 7, 2.0, 1, 16, BUF, BUF, BUF, BUF, C.byref(n), None), ENODEV),
    ]
    tree_less = ("tree create: N = 0", "meshes", "normals", "compress")
    for what, call, code in table:
        assert call() == code, what
        if code == ENODEV:
            assert b"no CUDA device" in L.vr_last_error(), what
        if what in tree_less:
            assert b"no CPU fallback" in L.vr_last_error(), what


# ------------------------------------------------------------------------------------ GPU: batches split in chunks
SPLIT = 8192 + 37   # the camera ring holds 8192 views: one full chunk and a short one


@pytest.fixture(scope="module")
def split_setup(small_trees):
    from volrend_b200 import Camera, N3Tree, synth
    cams = []
    for p in synth.nerf_synthetic_test_poses(SPLIT):
        c = Camera(8, 8, synth.focal_for(8), synth.focal_for(8))
        c.set_c2w(p)
        cams.append(c)
    return N3Tree.from_synth(small_trees["sh16_d6"]), cams


@pytest.mark.gpu
def test_bands_batch_split_equals_single_views(built, split_setup):
    import torch
    from volrend_b200 import RenderOptions, _capi, lib
    from volrend_b200.host import _cams_array
    tree, cams = split_setup
    L = lib()
    o = RenderOptions()._as_c()
    band, parts, part = 4, 2, 1
    rows = L.vr_band_rows(8, band, parts, part)
    s = torch.cuda.current_stream().cuda_stream
    shape = (SPLIT + 1, rows, 8, 4)   # + a guard view
    a, b = (torch.full(shape, 0xA5, dtype=torch.uint8, device="cuda") for _ in range(2))
    fa, fb = (torch.full(shape, float("nan"), dtype=torch.float32, device="cuda") for _ in range(2))
    _capi.check(L.vr_render_bands_batch(tree._handle, _cams_array(cams), SPLIT, C.byref(o), band, parts, part,
                                        a.data_ptr(), fa.data_ptr(), s))
    for i, c in enumerate(cams):
        _capi.check(L.vr_render_bands(tree._handle, C.byref(c._as_c()), C.byref(o), band, parts, part, b[i].data_ptr(),
                                      fb[i].data_ptr(), s))
    torch.cuda.synchronize()
    a, b, fa, fb = a.cpu().numpy(), b.cpu().numpy(), fa.cpu().numpy(), fb.cpu().numpy()
    assert (a[:SPLIT, ..., 3] == 255).all(), "a pixel kept the sentinel"
    assert (a[SPLIT] == 0xA5).all(), "the batch wrote past its views"
    assert np.array_equal(a, b)
    assert np.array_equal(fa.view(np.uint32), fb.view(np.uint32))
    assert len({a[i].tobytes() for i in range(0, SPLIT, 97)}) > 1, "every pose of the orbit looks the same"


@pytest.mark.gpu
def test_probe_split_equals_two_calls(built, split_setup):
    import torch
    from volrend_b200 import RenderOptions, _capi, lib
    from volrend_b200.host import _cams_array
    tree, cams = split_setup
    L = lib()
    o = RenderOptions()._as_c()
    xyz = (C.c_float * 3)(0.0, 0.0, 0.0)
    disp = 3   # an 8x8 frame is all candidate corner: x >= 8 - 3 - 5, y < 3 + 5
    s = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(11)
    img0 = torch.from_numpy(rng.integers(0, 256, (SPLIT, 8, 8, 4), dtype=np.uint8)).cuda()
    fo0 = torch.from_numpy(rng.random((SPLIT, 8, 8, 4), dtype=np.float32)).cuda()
    a, b, fa, fb = img0.clone(), img0.clone(), fo0.clone(), fo0.clone()
    _capi.check(L.vr_draw_probe(tree._handle, _cams_array(cams), SPLIT, C.byref(o), xyz, disp, None, a.data_ptr(),
                                fa.data_ptr(), 0, s))
    for v0, nv in ((0, 8192), (8192, SPLIT - 8192)):
        _capi.check(L.vr_draw_probe(tree._handle, _cams_array(cams[v0:v0 + nv]), nv, C.byref(o), xyz, disp, None,
                                    b[v0].data_ptr(), fb[v0].data_ptr(), 0, s))
    torch.cuda.synchronize()
    a, b, fa, fb = a.cpu().numpy(), b.cpu().numpy(), fa.cpu().numpy(), fb.cpu().numpy()
    drawn = (a != img0.cpu().numpy()).any(axis=(1, 2, 3))
    assert drawn[:8192].any() and drawn[8192:].any(), "the disc covers no pixel"
    assert np.array_equal(a, b)
    assert np.array_equal(fa.view(np.uint32), fb.view(np.uint32))
