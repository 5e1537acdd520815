"""`-m gpu`: the batch work order (decode_item: tile rows outermost, views inside them).  Every batch entry point
must render each tile of each view exactly once: batches are compared bit for bit with per-view single launches on
buffers pre-filled with a sentinel (a skipped tile keeps it), and composite batches composite over their input (a
tile rendered twice would composite over its own output)."""
import ctypes as C

import numpy as np
import pytest

from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)

pytestmark = pytest.mark.gpu
QUEUE, INLINE = 7, 3 + 16 * 193
SENTINEL = 0xA5


def _cams(W, H, first, n):
    """n consecutive orbit poses of the bench sweep (neighbouring views see the same voxels)."""
    from volrend_b200 import Camera, synth
    out = []
    for p in synth.nerf_synthetic_test_poses(200)[first:first + n]:
        c = Camera(W, H, synth.focal_for(W), synth.focal_for(W))
        c.set_c2w(p)
        out.append(c)
    return out


@pytest.fixture(scope="module")
def trees(small_trees):
    from volrend_b200 import N3Tree
    return {k: N3Tree.from_synth(small_trees[k]) for k in ("sh16_d6", "sh25_d5")}


@pytest.fixture
def variant():
    from volrend_b200 import lib
    old = lib().vr_get_variant()
    yield lambda v: lib().vr_set_variant(v)
    lib().vr_set_variant(old)


def _filled(shape):
    import torch
    img = torch.full(shape + (4,), SENTINEL, dtype=torch.uint8, device="cuda")
    fo = torch.full(shape + (4,), float("nan"), dtype=torch.float32, device="cuda")
    return img, fo


def _singles(tree, cams, opt):
    import torch
    from volrend_b200 import launch_renderer
    H, W = cams[0].height, cams[0].width
    img, fo = _filled((len(cams), H, W))
    for i, c in enumerate(cams):
        launch_renderer(tree, c, opt, img[i], None, None, True, float_out=fo[i])
    torch.cuda.synchronize()
    return img.cpu().numpy(), fo.cpu().numpy()


def _batch(tree, cams, opt):
    import torch
    from volrend_b200 import render_batch
    img, fo = _filled((len(cams), cams[0].height, cams[0].width))
    render_batch(tree, cams, opt, img, float_out=fo)
    torch.cuda.synchronize()
    return img.cpu().numpy(), fo.cpu().numpy()


def _same(a, b):
    assert (a[0][..., 3] == 255).all(), "a pixel kept the sentinel"
    assert np.array_equal(a[0], b[0])
    assert np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))


@pytest.mark.parametrize("v", [INLINE, QUEUE])
def test_batch_uneven_grid_equals_single_views(built, trees, variant, v):
    """13 views of 37x29: neither the 4x8 tile grid nor the view count divides anything evenly."""
    from volrend_b200 import RenderOptions
    variant(v)
    cams = _cams(37, 29, 40, 13)
    opt = RenderOptions()
    _same(_batch(trees["sh16_d6"], cams, opt), _singles(trees["sh16_d6"], cams, opt))


@pytest.mark.parametrize("v", [INLINE, QUEUE])
def test_composite_batch_renders_each_tile_once(built, trees, variant, v):
    import torch
    from volrend_b200 import RenderOptions, _capi, lib
    from volrend_b200.host import _cams_array, _options_array
    variant(v)
    tree = trees["sh16_d6"]
    W, H, n = 37, 29, 13
    cams = _cams(W, H, 60, n)
    opt = RenderOptions()
    rng = np.random.default_rng(3)
    img0 = torch.from_numpy(rng.integers(0, 256, (n, H, W, 4), dtype=np.uint8)).cuda()
    dep = torch.full((n, H, W), 1e9, dtype=torch.float32, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    a, b = img0.clone(), img0.clone()
    fa, fb = _filled((n, H, W))[1], _filled((n, H, W))[1]
    _capi.check(lib().vr_render_composite_batch(tree._handle, _cams_array(cams), n, _options_array([opt]), None,
                                                a.data_ptr(), dep.data_ptr(), fa.data_ptr(), s))
    px = W * H
    for i, c in enumerate(cams):
        _capi.check(lib().vr_render_composite(tree._handle, C.byref(c._as_c()), C.byref(opt._as_c()), None,
                                              b.data_ptr() + 4 * px * i, dep.data_ptr() + 4 * px * i,
                                              fb.data_ptr() + 16 * px * i, s))
    torch.cuda.synchronize()
    _same((a.cpu().numpy(), fa.cpu().numpy()), (b.cpu().numpy(), fb.cpu().numpy()))


def test_two_part_band_batch_reassembles(built, trees):
    """vr_render_bands_batch, 2 parts: frame_row maps each part's compact rows back to the frame."""
    import torch
    from volrend_b200 import RenderOptions, lib, render_bands_batch
    tree = trees["sh16_d6"]
    W, H, n, band = 37, 29, 13, 4
    cams = _cams(W, H, 100, n)
    opt = RenderOptions()
    full = _batch(tree, cams, opt)
    got = np.full((n, H, W, 4), SENTINEL, np.uint8)
    for part in range(2):
        rows = lib().vr_band_rows(H, band, 2, part)
        img = torch.full((n + 1, rows, W, 4), SENTINEL, dtype=torch.uint8, device="cuda")   # + a guard view
        assert render_bands_batch(tree, cams, opt, band, 2, part, img) == rows
        torch.cuda.synchronize()
        img = img.cpu().numpy()
        assert (img[n] == SENTINEL).all(), "a band launch wrote past its views"
        for r in range(rows):
            got[:, (r // band * 2 + part) * band + r % band] = img[:n, r]
    assert np.array_equal(got, full[0])


def test_large_sh25_batch_equals_single_views(built, trees):
    """7 views of 1001x703 with 25 basis functions: enough tile blocks per SM for the batch's block queue."""
    from volrend_b200 import RenderOptions
    cams = _cams(1001, 703, 20, 7)
    opt = RenderOptions(basis_minmax=[0, 24])
    _same(_batch(trees["sh25_d5"], cams, opt), _singles(trees["sh25_d5"], cams, opt))
