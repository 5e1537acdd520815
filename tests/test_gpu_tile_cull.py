"""`-m gpu`: tile culling of batch launches (vr_cull.cu).  The uninstrumented batch march skips the tiles the coverage
pass leaves unmarked, and those rays take the miss path; the instrumented launch (``counters=``) and single-view
launches march every ray.  So every batch here must give the same RGBA8 bytes and float RGBA bits as the same call
with counters, or, for the entry points without counters (composite, bands), as one launch per view."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)

pytestmark = pytest.mark.gpu

import edge_cases as ec  # noqa: E402
import golden_cases as gc  # noqa: E402
import layout_cases as lc  # noqa: E402

PARITIES = ("0", "1")
GOLDEN = ["lego_sh16", "drums_sh9", "lego_sh25_bbox", "lego_rgba"]
EDGE = ["mixed_sh16", "mixed_rgba", "root_mixed", "chain22", "aniso", "quant_mixed", "sigma_bits"]
LAYOUT = ["shuffle", "dirty"]


def _device_tree(st, parity, slot_map=False, ndc=None):
    from volrend_b200 import N3Tree
    tree = N3Tree()
    tree.load_npz(st.npz_dict())
    if ndc is not None:
        tree.use_ndc = True
        tree.ndc_width, tree.ndc_height, tree.ndc_focal = ndc
    old = os.environ.get("VR_WIDE_PARITY")
    os.environ["VR_WIDE_PARITY"] = parity
    try:
        tree.load_cuda(slot_map=slot_map)
    finally:
        if old is None:
            del os.environ["VR_WIDE_PARITY"]
        else:
            os.environ["VR_WIDE_PARITY"] = old
    assert tree.info()["wide_parity"] == int(parity)
    return tree


def _cam(W, H, fx, fy, pose):
    from volrend_b200 import Camera
    c = Camera(W, H, fx, fy)
    c.set_c2w(np.asarray(pose, np.float32))
    return c


def _orbit(st, W, H, n, dist=(2.2, 3.0, 4.5)):
    """n views around the tree's box at a few distances, looking at its centre."""
    from volrend_b200 import synth
    centre = ec._to_world(st, [0.5, 0.5, 0.5])
    span = float(np.abs(ec._to_world(st, [1.0, 1.0, 1.0]) - ec._to_world(st, [0.0, 0.0, 0.0])).max())
    cams = []
    for i in range(n):
        a = 2.0 * np.pi * i / n
        d = dist[i % len(dist)] * span
        eye = centre + d * np.array([np.cos(a), np.sin(a), 0.4 + 0.3 * np.sin(3 * a)])
        cams.append(_cam(W, H, 0.9 * W, 0.9 * W, synth.look_at_c2w(eye, target=centre)))
    return cams


def _cases():
    """(id, SynthTree, cameras of one size, options dict)"""
    out = []
    for name in GOLDEN:
        st, W, H, pose, kw, _ = gc.build_case(name)
        out.append((name, st, [_cam(W, H, W * 1.1, W * 1.1, pose)] + _orbit(st, W, H, 7), kw))
    for name in EDGE:
        st = ec.edge_tree(name)[0]
        views = [v for v in ec.views_for(name) if ec.view(v, name, st)[:2] == (ec.W0, ec.H0)
                 and ec.view(v, name, st)[6] is None]
        cams, kw = [], {}
        for v in views:
            W, H, fx, fy, pose, vkw, _ = ec.view(v, name, st)
            if vkw:
                continue
            cams.append(_cam(W, H, fx, fy, pose))
        out.append((name, st, cams + _orbit(st, ec.W0, ec.H0, 5), kw))
    base = ec.edge_tree("mixed_sh16")[0]
    for layout in LAYOUT:
        st = lc.relayout(base, layout, seed=4).st
        out.append((f"mixed_sh16_{layout}", st, _orbit(st, ec.W0, ec.H0, 6), {}))
    return out


CASES = _cases()
OPTION_SETS = {
    "default": {},
    "depth": dict(render_depth=True),
    "thresh_neg": dict(sigma_thresh=-1.0),
    "thresh0": dict(sigma_thresh=0.0),
    "thresh_large": dict(sigma_thresh=1e4),
    "bbox_inner": dict(render_bbox=[0.2, 0.1, 0.3, 0.9, 0.8, 0.7]),
    "bbox_outer": dict(render_bbox=[-0.5, -0.5, -0.5, 1.5, 1.5, 1.5]),
}


def _opts(kw, extra):
    from volrend_b200 import RenderOptions
    d = dict(kw)
    d.update(extra)
    return RenderOptions(**d)


def _batch(tree, cams, opt, counters):
    import torch
    from volrend_b200 import render_batch
    n, H, W = len(cams), cams[0].height, cams[0].width
    img = torch.full((n, H, W, 4), 0xA5, dtype=torch.uint8, device="cuda")
    fo = torch.full((n, H, W, 4), float("nan"), dtype=torch.float32, device="cuda")
    cnt = torch.zeros(5, dtype=torch.int64, device="cuda") if counters else None
    render_batch(tree, cams, opt, img, float_out=fo, counters=cnt)
    torch.cuda.synchronize()
    return img.cpu().numpy(), fo.cpu().numpy().view(np.uint32)


def _same(got, want, what):
    assert np.array_equal(got[0], want[0]), f"{what}: {int((got[0] != want[0]).any(-1).sum())} RGBA8 pixels differ"
    assert np.array_equal(got[1], want[1]), f"{what}: {int((got[1] != want[1]).any(-1).sum())} float pixels differ"


@pytest.mark.parametrize("parity", PARITIES)
@pytest.mark.parametrize("case", range(len(CASES)), ids=[c[0] for c in CASES])
def test_batch_matches_instrumented(built, case, parity):
    name, st, cams, kw = CASES[case]
    tree = _device_tree(st, parity)
    for oname, extra in OPTION_SETS.items():
        opt = _opts(kw, extra)
        _same(_batch(tree, cams, opt, False), _batch(tree, cams, opt, True), f"{name} {oname}")
    # options per view: thresholds and modes that differ from view to view
    keys = list(OPTION_SETS)
    per = [_opts(kw, OPTION_SETS[keys[i % len(keys)]]) for i in range(len(cams))]
    _same(_batch(tree, cams, per, False), _batch(tree, cams, per, True), f"{name} per-view options")


@pytest.mark.parametrize("parity", PARITIES)
def test_ndc_tree(built, parity):
    st = ec.edge_tree("aniso_ndc")[0]
    tree = _device_tree(st, parity, ndc=ec.NDC["aniso_ndc"])
    W, H, fx, fy, pose, _, _ = ec.view("ndc", "aniso_ndc", st)
    cams = []
    for i in range(4):
        p = np.array(pose, np.float32)
        p[:3, 3] += np.float32(0.02) * np.array([i, -i, 0.5 * i], np.float32)
        cams.append(_cam(W, H, fx, fy, p))
    from volrend_b200 import RenderOptions
    for opt in (RenderOptions(), RenderOptions(render_depth=True)):
        _same(_batch(tree, cams, opt, False), _batch(tree, cams, opt, True), "ndc")


@pytest.mark.parametrize("parity", PARITIES)
def test_camera_inside_and_near_the_box(built, parity):
    from volrend_b200 import RenderOptions, synth
    st = synth.make_tree("lego", depth=7, basis_dim=16, seed=5)
    tree = _device_tree(st, parity)
    cams = []
    for k, p in enumerate([[0.5, 0.5, 0.5], [0.55, 0.38, 0.61], [0.02, 0.5, 0.5], [-0.01, 0.3, 0.7], [0.5, 1.004, 0.5]]):
        eye = ec._to_world(st, p)
        look = np.array([np.cos(k), np.sin(k), 0.3 - 0.2 * k])
        cams.append(_cam(96, 64, 40.0, 40.0, synth.look_at_c2w(eye, target=eye + look)))
    for opt in (RenderOptions(), RenderOptions(render_depth=True), RenderOptions(sigma_thresh=5.0)):
        _same(_batch(tree, cams, opt, False), _batch(tree, cams, opt, True), "camera inside")


def _singles_composite(tree, cams, opt, rgba, depth):
    import torch
    from volrend_b200 import lib
    from volrend_b200.host import _rect, _stream_ptr, check
    outs = []
    for i, c in enumerate(cams):
        img = rgba[i].clone()
        fo = torch.zeros(img.shape, dtype=torch.float32, device="cuda")
        check(lib().vr_render_composite(tree._handle, C.byref(c._as_c()), C.byref(opt._as_c()), _rect(None),
                                        img.data_ptr(), depth[i].data_ptr(), fo.data_ptr(), _stream_ptr(None)))
        outs.append((img, fo))
    torch.cuda.synchronize()
    return (np.stack([o[0].cpu().numpy() for o in outs]),
            np.stack([o[1].cpu().numpy() for o in outs]).view(np.uint32))


@pytest.mark.parametrize("parity", PARITIES)
def test_composite_with_depth_limit(built, parity):
    import torch
    from volrend_b200 import RenderOptions, lib
    from volrend_b200.host import _cams_array, _rect, _stream_ptr, check
    st, W, H, pose, kw, _ = gc.build_case("lego_sh16")
    tree = _device_tree(st, parity)
    cams = _orbit(st, W, H, 6)
    rng = np.random.default_rng(3)
    rgba0 = torch.from_numpy(rng.integers(0, 256, (6, H, W, 4)).astype(np.uint8)).cuda()
    dep = rng.uniform(1.0, 6.0, (6, H, W)).astype(np.float32)
    dep[:, :, ::7] = np.inf
    dep[:, ::5, :] = 0.0
    depth = torch.from_numpy(dep).cuda()
    for opt in (RenderOptions(**kw), RenderOptions(render_depth=True), RenderOptions(sigma_thresh=30.0)):
        img = rgba0.clone()
        fo = torch.zeros((6, H, W, 4), dtype=torch.float32, device="cuda")
        check(lib().vr_render_composite_batch(tree._handle, _cams_array(cams), len(cams), C.byref(opt._as_c()),
                                              _rect(None), img.data_ptr(), depth.data_ptr(), fo.data_ptr(),
                                              _stream_ptr(None)))
        torch.cuda.synchronize()
        got = (img.cpu().numpy(), fo.cpu().numpy().view(np.uint32))
        _same(got, _singles_composite(tree, cams, opt, rgba0, depth), "composite")


@pytest.mark.parametrize("parity", PARITIES)
def test_bands(built, parity):
    import torch
    from volrend_b200 import RenderOptions, lib, render_bands, render_bands_batch, synth
    st = synth.make_tree("lego", depth=7, basis_dim=9, seed=6)
    tree = _device_tree(st, parity)
    W, H = 72, 90
    cams = _orbit(st, W, H, 5)
    for band_h, parts, part in ((8, 3, 1), (4, 2, 0), (12, 4, 3)):   # 4 and 12: tiles straddle bands
        for opt in (RenderOptions(), RenderOptions(sigma_thresh=20.0)):
            rows = lib().vr_band_rows(H, band_h, parts, part)   # the compact output of one view
            img = torch.full((5, rows, W, 4), 0xA5, dtype=torch.uint8, device="cuda")
            fo = torch.zeros((5, rows, W, 4), dtype=torch.float32, device="cuda")
            n = render_bands_batch(tree, cams, opt, band_h, parts, part, img, float_out=fo)
            assert n == rows
            want_i, want_f = torch.full_like(img, 0xA5), torch.zeros_like(fo)
            for i, c in enumerate(cams):
                render_bands(tree, c, opt, band_h, parts, part, want_i[i], float_out=want_f[i])
            torch.cuda.synchronize()
            _same((img[:, :n].cpu().numpy(), fo[:, :n].cpu().numpy().view(np.uint32)),
                  (want_i[:, :n].cpu().numpy(), want_f[:, :n].cpu().numpy().view(np.uint32)), f"bands {band_h}")


@pytest.mark.parametrize("parity", PARITIES)
def test_after_update_data_fills_empty_space(built, parity):
    """Raising sigma in leaves that were empty must reach the coverage pass: rays that shaded nothing before do."""
    import torch
    from volrend_b200 import RenderOptions, synth
    st = synth.make_tree("lego", depth=6, basis_dim=16, seed=8)
    tree = _device_tree(st, parity, slot_map=True)
    cams = _orbit(st, 64, 48, 6)
    opt = RenderOptions()
    before = _batch(tree, cams, opt, False)
    data = st.data.reshape(st.capacity, 2, 2, 2, st.data_dim).copy()
    sig = data[..., -1].astype(np.float32)
    empty = sig <= opt.sigma_thresh
    assert empty.mean() > 0.3
    sig[empty] = 50.0
    data[..., -1] = sig.astype(np.float16)
    tree.update_data(torch.from_numpy(data).cuda())
    after = _batch(tree, cams, opt, False)
    _same(after, _batch(tree, cams, opt, True), "after update_data")
    assert not np.array_equal(after[0], before[0])


@pytest.mark.parametrize("parity", PARITIES)
@pytest.mark.parametrize("name", sorted(__import__("axis_ray_cases").CASES))
def test_axis_rays(built, name, parity):
    """Rays that run exactly along cell faces (tests/axis_ray_cases.py): pixel (1, 1) of each view, the case's axis
    ray, rendered as a 1x1 tile as the cases are meant to be (with step_size 0 only the axis ray moves on) -- the
    boundary case of the cell projection."""
    import torch
    import axis_ray_cases as ac
    from volrend_b200 import RenderOptions, render_batch
    case = ac.CASES[name]
    if len(case.views) < 2:
        pytest.skip("one view: not a batch")
    tree = _device_tree(case.st, parity)
    cams = [_cam(2, 2, 1.0, 1.0, v.pose) for v in case.views]
    opt = RenderOptions(**case.options())
    out = []
    for counters in (False, True):
        img = torch.full((len(cams), 1, 1, 4), 0xA5, dtype=torch.uint8, device="cuda")
        fo = torch.full((len(cams), 1, 1, 4), float("nan"), dtype=torch.float32, device="cuda")
        cnt = torch.zeros(5, dtype=torch.int64, device="cuda") if counters else None
        render_batch(tree, cams, opt, img, float_out=fo, counters=cnt, tile=ac.TILE)
        torch.cuda.synchronize()
        out.append((img.cpu().numpy(), fo.cpu().numpy().view(np.uint32)))
    _same(out[0], out[1], name)
