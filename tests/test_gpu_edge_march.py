"""`-m gpu`: the edge-case march frames of tests/edge_cases.py through both product kernels (shading queue and inline
shading) under both table parities, on every render path: single views (float and bytes), tiles, batches with one set
of options and with options per view, a batch large enough for SM-local tile blocks, the composite batch, and bands.

Every single-view frame is bit-identical to the reference kernel's stored frame (and to the reference kernel itself
when oracle/_ref is built), within 2e-6 of the CPU oracle with exactly its work counters; every other path is
bit-identical to the single-view frames.  One test per path; the single views of each (tree, kernel, parity) are
rendered once and shared by them."""
import contextlib
import os

import numpy as np
import pytest

import edge_cases as ec
from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)

pytestmark = pytest.mark.gpu
QUEUE, INLINE = 7, 3 + 16 * 193         # the product kernels (vr_kernels.h)
KERNELS = {"queue": QUEUE, "inline": INLINE}
BLOCK_VIEWS = 2880                      # 40x30 views: enough blocks for the SM-local block path (set_work)
CASES = [(n, k, p) for n in ec.TREES for k in sorted(KERNELS) for p in (0, 1)]
IDS = [f"{n}-{k}-{p}" for n, k, p in CASES]


@contextlib.contextmanager
def _variant(v):
    from volrend_b200 import lib
    assert lib().vr_set_variant(v) == 0
    try:
        yield
    finally:
        lib().vr_set_variant(0)


def _device_tree(name, st, npz, parity, gpu_decode=True):
    from volrend_b200 import N3Tree
    os.environ["VR_WIDE_PARITY"] = str(parity)
    try:
        t = N3Tree(gpu_decode=gpu_decode)
        t.load_npz(ec.tree_file_arrays(st, npz))
        if name in ec.NDC:
            t.use_ndc = True
            t.ndc_width, t.ndc_height, t.ndc_focal = ec.NDC[name]
        t.load_cuda()
    finally:
        del os.environ["VR_WIDE_PARITY"]
    assert t.info()["wide_parity"] == parity
    return t


def _cam(W, H, fx, fy, pose):
    from volrend_b200 import Camera
    c = Camera(W, H, fx, fy)
    c.set_c2w(pose)
    return c


def _same(a, b, what):
    assert a.shape == b.shape, what
    if a.dtype == np.float32:
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), what
    else:
        assert np.array_equal(a, b), what


def _single(tree, cam, opt, comp):
    """(float RGBA, RGBA8, counters or None) of one launch_renderer."""
    import torch
    from volrend_b200 import launch_renderer
    img = torch.zeros((cam.height, cam.width, 4), dtype=torch.uint8, device="cuda")
    fo = torch.zeros((cam.height, cam.width, 4), dtype=torch.float32, device="cuda")
    cnt = None
    if comp is None:
        cnt = torch.zeros(5, dtype=torch.int64, device="cuda")
        launch_renderer(tree, cam, opt, img, None, None, True, float_out=fo, counters=cnt)
    else:
        img.copy_(torch.from_numpy(comp[0]))
        launch_renderer(tree, cam, opt, img, torch.from_numpy(comp[1]).cuda(), None, False, float_out=fo)
    torch.cuda.synchronize()
    return fo.cpu().numpy(), img.cpu().numpy(), (cnt.cpu().tolist() if cnt is not None else None)


class Case:
    """A tree on the device under one table parity, a kernel, and the single-view frames of all its views."""

    def __init__(self, name, kernel, parity):
        from volrend_b200 import RenderOptions, lib
        self.name, self.v = name, KERNELS[kernel]
        self.st, self.npz = ec.edge_tree(name)
        self.tree = _device_tree(name, self.st, self.npz, parity)
        self.kbd = self.tree.info()["kernel_basis"]
        self.supported = bool(lib().vr_variant_supported(self.kbd, self.v))
        self.singles = {}           # frame -> (f, u, counters, camera, options, composite)
        if not self.supported:
            return
        with _variant(self.v):
            for fr in ec.frames_of(name):
                _, W, H, fx, fy, pose, kw, comp = ec.frame(fr, self.st)
                cam, opt = _cam(W, H, fx, fy, pose), RenderOptions(**kw)
                self.singles[fr] = _single(self.tree, cam, opt, comp) + (cam, opt, comp)

    def offscreen(self, W=ec.W0, H=ec.H0):
        return [fr for fr, s in self.singles.items() if s[5] is None and (s[3].width, s[3].height) == (W, H)]

    def sizes(self):
        return sorted({(s[3].width, s[3].height) for s in self.singles.values() if s[5] is None})


@pytest.fixture(scope="module")
def cases():
    return {}


@pytest.fixture(scope="module")
def per_tree():
    """tree name -> {"oracle": {frame: oracle render}, "live": {frame: live reference render}}."""
    return {}


def _case(cases, name, kernel, parity):
    key = (name, kernel, parity)
    if key not in cases:
        cases[key] = Case(name, kernel, parity)
    c = cases[key]
    if not c.supported:
        assert kernel == "queue" and c.kbd < 4          # the queue kernel needs >= 4 basis functions
        pytest.skip(f"the {kernel} kernel has no {c.kbd}-basis build")
    return c


def _live_reference(per_tree, c, tmp_path):
    """The reference kernel's {frame: (float RGBA, RGBA8)} of the case's tree, or None without oracle/_ref."""
    from oracle import ref_binding as rb
    from volrend_b200 import synth
    if not rb.available():
        return None
    live = per_tree.setdefault(c.name, {}).setdefault("live", {})
    if not live:
        path = str(tmp_path / f"{c.name}.npz")
        ec.write_tree_file(c.name, c.st, c.npz, path)
        rt = rb.RefTree(path)
        for fr in ec.frames_of(c.name):
            _, W, H, fx, fy, pose, kw, comp = ec.frame(fr, c.st)
            rin, din = comp if comp is not None else (None, None)
            c12 = synth.c2w_to_colmajor12(pose)
            live[fr] = (rt.render_f32(W, H, fx, fy, c12, rb.make_options(**kw), rgba_in=rin, depth_in=din),
                        rt.render_u8(W, H, fx, fy, c12, rb.make_options(**kw), rgba_in=rin, depth_in=din))
        rt.close()
    return live


@pytest.mark.parametrize("name,kernel,parity", CASES, ids=IDS)
def test_single_views_match_reference_and_oracle(built, cases, per_tree, tmp_path, name, kernel, parity):
    c = _case(cases, name, kernel, parity)
    live = _live_reference(per_tree, c, tmp_path)
    oracle = per_tree.setdefault(name, {}).setdefault("oracle", {})
    for fr, (f, u, cnt, _, _, comp) in c.singles.items():
        ec.assert_identical(fr, f, u)                       # the stored frame of the reference kernel
        if live is not None:                                # and the kernel itself
            if ec.is_composite(fr):
                ec.assert_composite_tap(fr, f, live[fr][0])
            else:
                _same(f, live[fr][0], (fr, "live reference float RGBA"))
            _same(u, live[fr][1], (fr, "live reference bytes"))
        if fr not in oracle:
            oracle[fr] = ec.oracle_render(fr, c.st)
        fo, _, co = oracle[fr]                              # the CPU oracle: expf ulps, identical work counters
        assert np.array_equal(np.isnan(f), np.isnan(fo)), fr
        assert np.abs(np.nan_to_num(f) - np.nan_to_num(fo)).max() <= 2e-6, fr
        if cnt is not None:
            assert cnt[:4] == [co["samples"], co["child_loads"], co["shaded"], co["rays_hit"]], (fr, cnt, co)


@pytest.mark.parametrize("name,kernel,parity", CASES, ids=IDS)
def test_tiles_equal_single_views(built, cases, name, kernel, parity):
    """A tile away from the frame's edges (frames of at least 8x8 pixels)."""
    import torch
    from volrend_b200 import launch_renderer
    c = _case(cases, name, kernel, parity)
    with _variant(c.v):
        for fr, (f, u, _, cam, opt, comp) in c.singles.items():
            if comp is not None or cam.width < 8 or cam.height < 8:
                continue
            x0, y0, w, h = tile = (3, 5, cam.width - 7, cam.height - 9)
            img = torch.zeros((h, w, 4), dtype=torch.uint8, device="cuda")
            ft = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
            launch_renderer(c.tree, cam, opt, img, None, None, True, float_out=ft, tile=tile)
            torch.cuda.synchronize()
            _same(ft.cpu().numpy(), f[y0:y0 + h, x0:x0 + w], (fr, "tile"))
            _same(img.cpu().numpy(), u[y0:y0 + h, x0:x0 + w], (fr, "tile bytes"))


@pytest.mark.parametrize("name,kernel,parity", CASES, ids=IDS)
def test_batches_equal_single_views(built, cases, name, kernel, parity):
    """The offscreen frames of each size as one batch with options per view, and as one batch per distinct options."""
    import torch
    from volrend_b200 import render_batch
    c = _case(cases, name, kernel, parity)
    with _variant(c.v):
        for W, H in c.sizes():
            frs = c.offscreen(W, H)
            cams, opts = [c.singles[fr][3] for fr in frs], [c.singles[fr][4] for fr in frs]
            imgs = torch.zeros((len(frs), H, W, 4), dtype=torch.uint8, device="cuda")
            fos = torch.zeros((len(frs), H, W, 4), dtype=torch.float32, device="cuda")
            render_batch(c.tree, cams, opts, imgs, float_out=fos)
            torch.cuda.synchronize()
            for i, fr in enumerate(frs):
                _same(fos[i].cpu().numpy(), c.singles[fr][0], (fr, "batch, options per view"))
                _same(imgs[i].cpu().numpy(), c.singles[fr][1], (fr, "batch bytes, options per view"))
            for o in {repr(x): x for x in opts}.values():
                sub = [fr for fr, x in zip(frs, opts) if x == o]
                fos = torch.zeros((len(sub), H, W, 4), dtype=torch.float32, device="cuda")
                render_batch(c.tree, [c.singles[fr][3] for fr in sub], o, None, float_out=fos)
                torch.cuda.synchronize()
                for i, fr in enumerate(sub):
                    _same(fos[i].cpu().numpy(), c.singles[fr][0], (fr, "batch, one set of options"))


def _blocks(kbd, W, H, n):
    """Whether a batch launch of n views of W x H hands out SM-local blocks (the rule of set_work)."""
    import torch
    G, BW, BH = (1, 8, 8) if kbd == 25 else (4, 4, 4)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tx, ty = -(-W // 4), -(-H // 8)
    return n >= G and -(-tx // BW) * -(-ty // BH) * -(-n // G) >= 16 * sms


@pytest.mark.parametrize("name,kernel,parity", CASES, ids=IDS)
def test_block_batch_equals_single_views(built, cases, name, kernel, parity):
    """BLOCK_VIEWS views cycling through the 40x30 offscreen frames, options per view: the SM-local block path."""
    import torch
    from volrend_b200 import render_batch
    c = _case(cases, name, kernel, parity)
    frs = c.offscreen()
    assert frs
    n = BLOCK_VIEWS
    assert _blocks(c.kbd, ec.W0, ec.H0, n)
    with _variant(c.v):
        fos = torch.full((n, ec.H0, ec.W0, 4), float("nan"), dtype=torch.float32, device="cuda")
        render_batch(c.tree, [c.singles[frs[i % len(frs)]][3] for i in range(n)],
                     [c.singles[frs[i % len(frs)]][4] for i in range(n)], None, float_out=fos)
        torch.cuda.synchronize()
    want = torch.from_numpy(np.stack([c.singles[fr][0] for fr in frs])).cuda().view(torch.int32)
    got = fos.view(torch.int32)
    for i in range(len(frs)):
        assert torch.equal(got[i::len(frs)], want[i].expand_as(got[i::len(frs)])), frs[i]


@pytest.mark.parametrize("name,kernel,parity", CASES, ids=IDS)
def test_composite_batch_equals_single_views(built, cases, name, kernel, parity):
    """vr_render_composite_batch_opts over the 40x30 offscreen views (seeded colour, the depth limits 0, -1, +inf, NaN,
    -inf and finite ones of ec.composite_layers) and the composite views (their own colour and limits), against one
    vr_render_composite per view; the composite views also against their single-view frames."""
    import torch
    from volrend_b200 import _capi, lib
    from volrend_b200.host import _cams_array, _options_array
    c = _case(cases, name, kernel, parity)
    frs = c.offscreen() + [fr for fr, s in c.singles.items() if s[5] is not None]
    n = len(frs)
    rgba = np.random.default_rng(3).integers(0, 256, (n, ec.H0, ec.W0, 4)).astype(np.uint8)
    deps = np.stack([ec.composite_layers()[1]] * n)
    for i, fr in enumerate(frs):
        if c.singles[fr][5] is not None:
            rgba[i], deps[i] = c.singles[fr][5]
    cams, opts = [c.singles[fr][3] for fr in frs], [c.singles[fr][4] for fr in frs]
    a, d = torch.from_numpy(rgba).cuda(), torch.from_numpy(deps).cuda()
    fa = torch.zeros((n, ec.H0, ec.W0, 4), dtype=torch.float32, device="cuda")
    with _variant(c.v):
        _capi.check(lib().vr_render_composite_batch_opts(c.tree._handle, _cams_array(cams), n, _options_array(opts), None,
                                                         a.data_ptr(), d.data_ptr(), fa.data_ptr(),
                                                         torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        for i, fr in enumerate(frs):
            f1, u1, _ = _single(c.tree, cams[i], opts[i], (rgba[i], deps[i]))
            _same(fa[i].cpu().numpy(), f1, (fr, "composite batch"))
            _same(a[i].cpu().numpy(), u1, (fr, "composite batch bytes"))
            if c.singles[fr][5] is not None:
                _same(f1, c.singles[fr][0], (fr, "composite single view"))


@pytest.mark.parametrize("name,kernel,parity", CASES, ids=IDS)
def test_bands_equal_single_view(built, cases, name, kernel, parity):
    """vr_render_bands, two parts of 4-row bands of the first 40x30 offscreen frame."""
    import torch
    from volrend_b200 import dist as vd
    from volrend_b200 import lib, render_bands
    c = _case(cases, name, kernel, parity)
    fr = c.offscreen()[0]
    f, u, _, cam, opt, _ = c.singles[fr]
    with _variant(c.v):
        for part in range(2):
            rows = lib().vr_band_rows(ec.H0, 4, 2, part)
            img = torch.zeros((rows, ec.W0, 4), dtype=torch.uint8, device="cuda")
            fb = torch.zeros((rows, ec.W0, 4), dtype=torch.float32, device="cuda")
            assert render_bands(c.tree, cam, opt, 4, 2, part, img, float_out=fb) == rows
            torch.cuda.synchronize()
            r0 = 0
            for (_, y0, _, h) in vd.shard_bands(ec.W0, ec.H0, part, 2, 4):
                _same(fb[r0:r0 + h].cpu().numpy(), f[y0:y0 + h], (fr, "band", part))
                _same(img[r0:r0 + h].cpu().numpy(), u[y0:y0 + h], (fr, "band bytes", part))
                r0 += h


@pytest.mark.parametrize("kernel", sorted(KERNELS))
@pytest.mark.parametrize("parity", [0, 1])
def test_gpu_decode_equals_host_decode(built, cases, kernel, parity):
    """The quantised tree: the GPU decode renders exactly what the host decode does."""
    c = _case(cases, "quant_mixed", kernel, parity)
    host = _device_tree(c.name, c.st, c.npz, parity, gpu_decode=False)
    assert host._data is not None and c.tree._data is None
    with _variant(c.v):
        for fr, (f, u, _, cam, opt, comp) in c.singles.items():
            fh, uh, _ = _single(host, cam, opt, comp)
            _same(fh, f, (fr, "host decode"))
            _same(uh, u, (fr, "host decode bytes"))


def _padded_chain24(extra_nodes=2_000_000):
    """The 24-level chain plus unreachable leaf-only nodes, so that an upload that is not freed shows in the device's
    free memory (~0.26 GB per attempt)."""
    st = ec.varied_chain(24)
    st.child = np.concatenate([st.child, np.zeros((extra_nodes, 2, 2, 2), np.int32)])
    st.data = np.concatenate([st.data, np.zeros((extra_nodes, 2, 2, 2, 4), np.float16)])
    return st


def test_chain24_is_refused_cleanly(built):
    """A 24-level tree is deeper than kMaxTreeDepth: vr_tree_create refuses it with VR_EUNSUPPORTED and a message.
    The upload and the depth sweep run before the refusal; no render launch follows, every allocation of the attempt
    is freed, no device error is left behind, and the 23-level chain still loads and renders."""
    import torch
    from volrend_b200 import N3Tree, VolrendError, _capi, lib
    assert "chain24" in ec.REFUSED
    st = _padded_chain24()

    def refuse():
        with pytest.raises(VolrendError) as e:
            N3Tree.from_synth(st)
        assert e.value.code == _capi.VR_EUNSUPPORTED
        assert "deeper than 23 levels" in str(e.value)

    refuse()                                    # first attempt: one-time allocations of the uploader
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    n0 = lib().vr_launch_count()
    for _ in range(3):
        refuse()
    torch.cuda.synchronize()
    assert lib().vr_launch_count() == n0
    assert torch.cuda.mem_get_info()[0] >= free0 - (128 << 20), "a refused upload kept device memory"
    st23 = ec.varied_chain(23)
    t = N3Tree.from_synth(st23)
    assert t.info()["max_depth"] == 23
    _, W, H, fx, fy, pose, kw, _ = ec.frame("chain23.deep.default", st23)
    from volrend_b200 import RenderOptions
    f, u, _ = _single(t, _cam(W, H, fx, fy, pose), RenderOptions(**kw), None)
    ec.assert_identical("chain23.deep.default", f, u)
