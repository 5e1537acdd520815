"""The surface render path: vr_render_surface (and the surface form of vr_draw_probe) into a cudaArray, as the C++
drop-in launch_renderer, volrend_headless and VolumeRenderer::render() call it.  Its kernels are the kOutSurface
instantiations of both march kernels, which read the existing colour and the depth limit with surf2Dread and write the
pixel with surf2Dwrite: code of their own, apart from the linear-buffer path the other tests run.

The stored frames were written by the reference's own launch_renderer into a cudaArray through a surface, so the
surface bytes must equal them exactly, on the corpus the linear path is held to: the golden cases, the edge frames, the
probe cases and the bench-scale frames, under both kernels and both table parities.  Every surface frame must also
equal the bytes of launch_renderer into a linear buffer, which names the path when a stored-frame check fails.  Where
the kernel has no build for the tree's basis, the surface path must refuse with VR_EUNSUPPORTED and touch nothing.

Reached kOutSurface instantiations (variant: queue 7, inline 3 + 16 * 193), both parities unless noted:
  inline RGBA   golden lego_rgba, edge mixed_rgba, probe rgba, composite rgba_d5, reference frame live_rgba_d5
  inline 1      golden cfg1_sh1, edge mixed_sh1 / chain22 / chain23, composite sh1_full4
  inline 4 / queue 4     golden lego_sh4_stop0 / lego_asg4, edge root_only / sigma_bits / mixed_asg4 (composite:
                         root_only), composite sh4_d5 / asg4_d5
  inline 9 / queue 9     golden drums_sh9 / lego_sg9_rot / lego_sh9_depth / lego_sh9_composite, edge mixed_sh9 /
                         mixed_sg9 / root_mixed (composite), composite sh9_d6 / sg9_d5
  inline 16 / queue 16   golden lego_sh16 / lego_sh16_ndc, edge mixed_sh16 (composite) / aniso (composite) /
                         aniso_ndc / quant_mixed, composite sh16_d6, behaviour tests
  inline 25 / queue 25   golden lego_sh25_bbox, edge mixed_sh25, probe sh25_bbox, reference frames config4_v7 /
                         live_sh25_d5, composite sh25_d5
"""
import ctypes as C
import hashlib
import os
import subprocess

import numpy as np
import pytest

import edge_cases as ec
from conftest import ROOT
from golden_cases import CASES as GOLDEN, REF_FRAMES, build_case, composite_inputs, ref_frame_tree, ref_frame_view
from oracle import surface_binding as sb
from probe_cases import PROBE_CASES, H as PH, W as PW, focal as probe_focal, golden_path as probe_golden, probe_case
from test_gpu_edge_march import KERNELS, Case, _variant

PARITIES = (0, 1)
# the trees of conftest.small_trees with a kernel build: every kernel basis (RGBA, 1, 4, 9, 16, 25) and format
SMALL = ["sh1_full4", "sh4_d5", "sh9_d6", "sh16_d6", "sh25_d5", "rgba_d5", "sg9_d5", "asg4_d5"]


@pytest.fixture(scope="module")
def harness(built):
    if not sb.available():
        subprocess.check_call(["make", "oracle/libsurface_harness.so"], cwd=ROOT)
    sb.lib()
    return sb


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a, np.uint8).tobytes()).hexdigest()


def _load(st, parity=None, npz=None, ndc=None):
    """A device tree of st (or of the file arrays npz), under table parity ``parity`` when given."""
    from volrend_b200 import N3Tree
    if parity is not None:
        os.environ["VR_WIDE_PARITY"] = str(parity)
    try:
        t = N3Tree()
        t.load_npz(npz if npz is not None else st.npz_dict())
        if ndc is not None:
            t.use_ndc = True
            t.ndc_width, t.ndc_height, t.ndc_focal = ndc
        t.load_cuda()
    finally:
        os.environ.pop("VR_WIDE_PARITY", None)
    if parity is not None:
        assert t.info()["wide_parity"] == parity
    return t


def _cam(W, H, fx, pose, fy=None):
    from volrend_b200 import Camera
    c = Camera(W, H, fx, fx if fy is None else fy)
    c.set_c2w(pose)
    return c


def _supported(tree, kernel):
    from volrend_b200 import lib
    return bool(lib().vr_variant_supported(tree.info()["kernel_basis"], KERNELS[kernel]))


def _linear(tree, cam, opt, comp=None):
    """launch_renderer into a linear RGBA8 buffer (offscreen, or over comp = (rgba8, depth)), probe disc included."""
    import torch
    from volrend_b200 import launch_renderer
    img = torch.zeros((cam.height, cam.width, 4), dtype=torch.uint8, device="cuda")
    if comp is None:
        launch_renderer(tree, cam, opt, img, None, None, True)
    else:
        img.copy_(torch.from_numpy(np.ascontiguousarray(comp[0])))
        launch_renderer(tree, cam, opt, img, torch.from_numpy(np.ascontiguousarray(comp[1])).cuda(), None, False)
    torch.cuda.synchronize()
    return img.cpu().numpy()


def _surface(tree, cam, opt, comp=None, **kw):
    """The surface form of _linear: vr_render_surface into a cudaArray, then the surface disc when the probe is on."""
    rgba, depth = comp if comp is not None else (None, None)
    probe = (opt.probe, opt.probe_disp_size) if opt.enable_probe else None
    return sb.render_surface(tree, cam, opt, rgba_in=rgba, depth_in=depth, probe=probe, **kw)


def _same(got, want, what):
    bad = (got != want).any(-1)
    assert not bad.any(), (what, int(bad.sum()), np.argwhere(bad)[:4].tolist())


def _check(tree, cam, opt, comp, what, golden=None, sha=None):
    """Surface bytes == linear bytes (a difference names the surface path) == the reference's stored bytes."""
    s = _surface(tree, cam, opt, comp)
    _same(s, _linear(tree, cam, opt, comp), (what, "surface path differs from the linear path"))
    if golden is not None:
        _same(s, golden, (what, "differs from the reference's launch_renderer"))
    if sha is not None:
        assert _sha(s) == sha, (what, "differs from the reference's launch_renderer")
    return s


def _assert_refused(tree, cam, opt, what):
    """No kernel of the selected variant for the tree's basis: VR_EUNSUPPORTED, no launch, the array untouched."""
    from volrend_b200 import _capi, lib
    with sb.SurfaceFrame(cam.width, cam.height) as f:
        f.upload(np.full((cam.height, cam.width, 4), sb.SENTINEL, np.uint8))
        n0 = lib().vr_launch_count()
        assert f.render_rc(tree, cam, opt) == _capi.VR_EUNSUPPORTED, what
        assert b"not available for kernel basis" in lib().vr_last_error(), what
        assert lib().vr_launch_count() == n0, what
        assert (f.download() == sb.SENTINEL).all(), what


# ---------------------------------------------------------------------------------------------------- golden cases
@pytest.mark.gpu
@pytest.mark.parametrize("parity", PARITIES)
@pytest.mark.parametrize("kernel", sorted(KERNELS))
@pytest.mark.parametrize("name", GOLDEN)
def test_golden_cases(harness, name, kernel, parity):
    from volrend_b200 import RenderOptions, synth
    z = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
    st, W, H, pose, optkw, ndc = build_case(name)
    tree = _load(st, parity, ndc=ndc)
    cam, opt = _cam(W, H, synth.focal_for(W), pose), RenderOptions(**optkw)
    with _variant(KERNELS[kernel]):
        if not _supported(tree, kernel):
            _assert_refused(tree, cam, opt, name)
            return
        _check(tree, cam, opt, composite_inputs(name, W, H), name, golden=z["ref_u8"])


# ----------------------------------------------------------------------------------------------------- edge frames
@pytest.fixture(scope="module")
def edge_case_cache():
    return {}


@pytest.mark.gpu
@pytest.mark.parametrize("parity", PARITIES)
@pytest.mark.parametrize("kernel", sorted(KERNELS))
@pytest.mark.parametrize("name", ec.TREES)
def test_edge_frames(harness, edge_case_cache, name, kernel, parity):
    """Every frame of the tree (37x23, 1x1 and 1x64 frames, cameras inside the tree, depth limits 0, -1, +-inf and NaN
    in the composite frames) against its stored bytes and the Case's linear single view."""
    key = (name, kernel, parity)
    if key not in edge_case_cache:
        edge_case_cache[key] = Case(name, kernel, parity)
    c = edge_case_cache[key]
    with _variant(c.v):
        if not c.supported:
            _, W, H, fx, fy, pose, kw, _ = ec.frame(ec.frames_of(name)[0], c.st)
            from volrend_b200 import RenderOptions
            _assert_refused(c.tree, _cam(W, H, fx, pose, fy), RenderOptions(**kw), name)
            return
        assert c.singles
        for fr, (_, u, _, cam, opt, comp) in c.singles.items():
            s = _surface(c.tree, cam, opt, comp)
            _same(s, u, (fr, "surface path differs from the linear path"))
            assert _sha(s) == str(ec.load(fr)["sha_u8"]), (fr, "differs from the reference's launch_renderer")


# ---------------------------------------------------------------------------------------------------- probe cases
@pytest.fixture(scope="module")
def probe_trees():
    from volrend_b200 import N3Tree
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = N3Tree.from_synth(probe_case(name)[0])
        return cache[name]
    return get


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", sorted(KERNELS))
@pytest.mark.parametrize("name", list(PROBE_CASES))
def test_probe_cases(harness, probe_trees, name, kernel):
    """The surface march followed by the surface disc against the reference's frame with the probe on, and the march
    alone against its frame with the probe off."""
    from volrend_b200 import RenderOptions
    z = np.load(probe_golden(name), allow_pickle=False)
    tree = probe_trees(name)
    _, pose, optkw, probe, disp, comp = probe_case(name)
    cam = _cam(PW, PH, probe_focal(), pose)
    on = RenderOptions(**optkw)
    on.enable_probe, on.probe, on.probe_disp_size = True, [float(v) for v in probe], int(disp)
    off = RenderOptions(**optkw)
    with _variant(KERNELS[kernel]):
        if not _supported(tree, kernel):
            _assert_refused(tree, cam, off, name)
            return
        _check(tree, cam, off, comp, (name, "probe off"), golden=z["ref_u8_off"])
        _check(tree, cam, on, comp, (name, "probe on"), golden=z["ref_u8"])


# ---------------------------------------------------------------------------------------------- bench-scale frames
@pytest.fixture(scope="module")
def ref_trees():
    cache = {}

    def get(name):
        key = "config2" if name.startswith("config2") else name
        if key not in cache:
            cache.clear()           # one large tree on the device at a time
            st, npz = ref_frame_tree(name)
            cache[key] = _load(st, npz=npz)
        return cache[key]
    return get


@pytest.mark.gpu
@pytest.mark.parametrize("name", REF_FRAMES)
def test_reference_frames(harness, ref_trees, name):
    """The bench-scale frames (config 2: the CLI leg's 800x800 tree; config 4: 1920x1080 SH25) and the live and
    quantised frames, under each kernel built for the tree's basis."""
    from volrend_b200 import RenderOptions
    sha = str(np.load(os.path.join(ec.REF_DIR, name + ".npz"), allow_pickle=False)["sha_u8"])
    tree = ref_trees(name)
    W, H, fx, pose = ref_frame_view(name)
    cam = _cam(W, H, fx, pose)
    ran = 0
    for kernel in sorted(KERNELS):
        if _supported(tree, kernel):
            with _variant(KERNELS[kernel]):
                _check(tree, cam, RenderOptions(), None, (name, kernel), sha=sha)
            ran += 1
    assert ran >= 1


# ----------------------------------------------------------------------------------- composite on every kernel
def _composite_layers(W, H, seed):
    """Seeded colour, and ray-distance limits with stripes of 0, -1, +inf, NaN and -inf and finite ones elsewhere."""
    rng = np.random.default_rng(seed)
    rgba = rng.integers(0, 256, (H, W, 4)).astype(np.uint8)
    depth = rng.uniform(1.5, 5.0, (H, W)).astype(np.float32)
    for k, v in enumerate([0.0, -1.0, np.inf, np.nan, -np.inf]):
        depth[:, 3 * k:3 * k + 3] = v
    depth[: H // 4] = 1e9
    return rgba, depth


def _small_pose(name):
    from volrend_b200 import synth
    return synth.config1_pose() if name == "sh1_full4" else synth.nerf_synthetic_test_poses(8)[(len(name) * 3) % 8]


@pytest.mark.gpu
@pytest.mark.parametrize("parity", PARITIES)
@pytest.mark.parametrize("kernel", sorted(KERNELS))
@pytest.mark.parametrize("name", SMALL)
def test_composite_on_every_kernel(harness, small_trees, name, kernel, parity):
    """Offscreen and composite (colour and depth surfaces) frames of a 37x23 view: each kernel basis, each format."""
    from volrend_b200 import RenderOptions, synth
    st = small_trees[name]
    tree = _load(st, parity)
    cam, opt = _cam(37, 23, synth.focal_for(37), _small_pose(name)), RenderOptions()
    comp = _composite_layers(37, 23, seed=len(name))
    with _variant(KERNELS[kernel]):
        if not _supported(tree, kernel):
            _assert_refused(tree, cam, opt, name)
            return
        off = _check(tree, cam, opt, None, (name, "offscreen"))
        over = _check(tree, cam, opt, comp, (name, "composite"))
    assert (over != off).any(-1).mean() > 0.2, "the composite frame must show the colour under it"


# ------------------------------------------------------------------------------------------------ live reference
@pytest.mark.gpu
def test_live_reference_random_views(harness, small_trees, tmp_path):
    """Seeded random trees, poses, frame sizes (odd ones among them) and kernels, some composite: the surface bytes
    against the reference kernel's launch_renderer itself."""
    from oracle import ref_binding as rb
    from volrend_b200 import RenderOptions, synth
    if not rb.available():
        pytest.skip("oracle/_ref not built (it needs the reference sources at build time)")
    rng = np.random.default_rng(20261017)
    poses = synth.nerf_synthetic_test_poses(40)
    trees, refs = {}, {}
    try:
        for k in range(20):
            name = SMALL[k % len(SMALL)]
            if name not in trees:
                trees[name] = _load(small_trees[name])
                path = str(tmp_path / f"{name}.npz")
                small_trees[name].save_npz(path)
                refs[name] = rb.RefTree(path)
            tree = trees[name]
            W, H = int(rng.integers(1, 130)), int(rng.integers(1, 100))
            fx = float(synth.focal_for(W)) * float(rng.uniform(0.6, 1.6))
            cam = _cam(W, H, fx, poses[int(rng.integers(0, 40))])
            comp = _composite_layers(W, H, seed=k) if rng.random() < 0.35 else None
            kernels = [kk for kk in sorted(KERNELS) if _supported(tree, kk)]
            kernel = kernels[int(rng.integers(0, len(kernels)))]
            c12 = np.ascontiguousarray(cam.transform, np.float32).reshape(12)
            rin, din = comp if comp is not None else (None, None)
            want = refs[name].render_u8(W, H, cam.fx, cam.fy, c12, rb.make_options(), rgba_in=rin, depth_in=din)
            with _variant(KERNELS[kernel]):
                _check(tree, cam, RenderOptions(), comp, (k, name, kernel, W, H, comp is not None), golden=want)
    finally:
        for r in refs.values():
            r.close()


# ------------------------------------------------------------------------------------- behaviour of the surface form
@pytest.fixture(scope="module")
def sh16(small_trees):
    return _load(small_trees["sh16_d6"])


def _view(i, W=120, H=96):
    from volrend_b200 import synth
    return _cam(W, H, synth.focal_for(W), synth.nerf_synthetic_test_poses(12)[i])


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", sorted(KERNELS))
def test_array_larger_than_frame(harness, sh16, kernel):
    """An array 5 columns and 3 rows larger than the frame: the frame area is the exact-size render, offscreen and
    composite, and the margin keeps what was there."""
    from volrend_b200 import RenderOptions
    cam, opt = _view(5, 37, 23), RenderOptions()
    W, H = cam.width + 5, cam.height + 3
    rgba, depth = _composite_layers(W, H, seed=5)
    with _variant(KERNELS[kernel]):
        big = sb.render_surface(sh16, cam, opt, array_size=(W, H))
        _same(big[:cam.height, :cam.width], _surface(sh16, cam, opt), "frame area, offscreen")
        assert (big[cam.height:] == sb.SENTINEL).all() and (big[:, cam.width:] == sb.SENTINEL).all()
        big = sb.render_surface(sh16, cam, opt, rgba_in=rgba, depth_in=depth, array_size=(W, H))
        inner = (rgba[:cam.height, :cam.width], depth[:cam.height, :cam.width])
        _same(big[:cam.height, :cam.width], _linear(sh16, cam, opt, inner), "frame area, composite")
        assert np.array_equal(big[cam.height:], rgba[cam.height:]) and np.array_equal(big[:, cam.width:], rgba[:, cam.width:])


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", sorted(KERNELS))
def test_back_to_back_launches_leave_last_frame(harness, sh16, kernel):
    """8 surface launches into one array, each overlapping its predecessor's tail (programmatic dependent launch),
    then an offscreen launch followed at once by a composite launch over the same array."""
    from volrend_b200 import RenderOptions
    opt = RenderOptions()
    cams = [_view(i) for i in range(8)]
    with _variant(KERNELS[kernel]):
        with sb.SurfaceFrame(120, 96, depth=True) as f:
            for c in cams:
                f.render(sh16, c, opt)
            _same(f.download(), _linear(sh16, cams[-1], opt), "8 launches")
            depth = _composite_layers(120, 96, seed=8)[1]
            f.upload(None, depth)
            f.render(sh16, cams[0], opt)
            f.render(sh16, cams[1], opt, composite=True)
            got = f.download()
        _same(got, _linear(sh16, cams[1], opt, (_linear(sh16, cams[0], opt), depth)), "offscreen, then composite")


@pytest.mark.gpu
def test_launch_count_and_stream(harness, sh16):
    """One launch per surface render, two with the probe disc (none for an empty disc); a non-default stream gives
    the same bytes."""
    import torch
    from volrend_b200 import RenderOptions, lib
    cam = _view(3)
    opt = RenderOptions(enable_probe=True, probe=[0.0, 0.0, 0.0], probe_disp_size=40)
    for probe, n in ((None, 1), ((opt.probe, 40), 2), ((opt.probe, 0), 1)):
        n0 = lib().vr_launch_count()
        sb.render_surface(sh16, cam, opt, probe=probe)
        assert lib().vr_launch_count() - n0 == n, probe
    want = _surface(sh16, cam, opt)
    comp = _composite_layers(120, 96, seed=3)
    want_c = _surface(sh16, cam, opt, comp)
    s = torch.cuda.Stream()
    _same(_surface(sh16, cam, opt, stream=s), want, "stream")
    _same(_surface(sh16, cam, opt, comp, stream=s), want_c, "stream, composite")


@pytest.mark.gpu
def test_error_codes(harness, small_trees, sh16):
    """What a caller gets wrong: no launch, the array untouched, an error message naming the problem."""
    from volrend_b200 import Camera, N3Tree, RenderOptions, _capi, lib
    L = lib()
    opt = RenderOptions()
    o, cam = opt._as_c(), _view(0)
    with sb.SurfaceFrame(120, 96) as f:
        f.upload(np.full((96, 120, 4), sb.SENTINEL, np.uint8))
        n0 = L.vr_launch_count()
        assert L.vr_render_surface(sh16._handle, C.byref(cam._as_c()), C.byref(o), 0, 0, None) == _capi.VR_EINVAL
        assert b"null surface" in L.vr_last_error()
        for w, h in ((0, 96), (120, 0)):
            assert f.render_rc(sh16, Camera(w, h, 100.0, 100.0), opt) == _capi.VR_EINVAL
            assert b"bad camera size" in L.vr_last_error()
        cams2 = (_capi.vr_camera * 2)(cam._as_c(), cam._as_c())
        xyz = (C.c_float * 3)(0.0, 0.0, 0.0)
        tile = _capi.vr_rect(0, 0, 8, 8)
        assert L.vr_draw_probe(sh16._handle, cams2, 2, C.byref(o), xyz, 40, None, None, None, f.surface(), None) \
            == _capi.VR_EINVAL
        assert L.vr_draw_probe(sh16._handle, cams2, 1, C.byref(o), xyz, 40, C.byref(tile), None, None, f.surface(),
                               None) == _capi.VR_EINVAL
        assert b"surface form draws one full frame" in L.vr_last_error()
        assert L.vr_launch_count() == n0
        assert (f.download() == sb.SENTINEL).all()
    rgba = N3Tree.from_synth(small_trees["rgba_d5"])
    with _variant(KERNELS["queue"]):                    # the queue kernel has no RGBA build
        _assert_refused(rgba, cam, opt, "queue kernel, RGBA tree")


# ------------------------------------------------------------------------------------------------------ CPU check
def test_harness_builds_and_exports():
    """`make oracle` builds the harness, and it exports what the binding calls (loading needs no GPU)."""
    subprocess.check_call(["make", "-s", "oracle"], cwd=ROOT)
    assert sb.available()
    h = sb.lib()                                    # resolves every symbol of sb.SYMBOLS
    out = C.c_void_p(1)
    assert h.sh_alloc(0, 4, 0, C.byref(out)) != 0 and not out.value      # refused before any CUDA call
    assert h.sh_free(None) == 0
