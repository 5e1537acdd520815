"""`-m gpu`: SM-local tile blocks of batches (decode_item with blk_mode): 4x4 tiles of 4 consecutive views up to 16
basis functions, 8x8 tiles of one view with 25.  Batches are compared bit for bit with per-view single launches,
which keep the plain tile counter, on buffers pre-filled with a sentinel (a skipped tile keeps it); composite batches
composite over their input (a tile rendered twice would composite over its own output).  The sizes are chosen so that
the batch launches do use the blocks (`_blocks`, the rule of set_work), with view counts that are not a multiple of
the block's 4 views and tile grids that are not a multiple of its tiles."""
import ctypes as C

import numpy as np
import pytest

from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)

pytestmark = pytest.mark.gpu
SENTINEL = 0xA5
SHAPE = {"sh16_d6": (4, 4, 4), "sh25_d5": (1, 8, 8)}   # views, tiles wide, tiles high of a block (set_work)


def _blocks(W, H, n, kind="sh16_d6"):
    """Whether a batch launch of n views of W x H hands out SM-local blocks (set_work)."""
    import torch
    G, BW, BH = SHAPE[kind]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tx, ty = -(-W // 4), -(-H // 8)
    nb = -(-tx // BW) * -(-ty // BH) * -(-n // G)
    return n >= G and nb >= 16 * sms


def _cams(W, H, first, n):
    """n consecutive orbit poses of the bench sweep (neighbouring views see the same voxels)."""
    from volrend_b200 import Camera, synth
    poses = synth.nerf_synthetic_test_poses(200)
    out = []
    for i in range(n):
        c = Camera(W, H, synth.focal_for(W), synth.focal_for(W))
        c.set_c2w(poses[(first + i) % 200])
        out.append(c)
    return out


@pytest.fixture(scope="module")
def trees(small_trees):
    from volrend_b200 import N3Tree
    return {k: N3Tree.from_synth(small_trees[k]) for k in ("sh16_d6", "sh25_d5")}


def _opt(kind):
    from volrend_b200 import RenderOptions
    return RenderOptions(basis_minmax=[0, 24]) if kind == "sh25_d5" else RenderOptions()


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


# (views, W, H): 13 views of 113x89 tiles and 37 views of 61x59 tiles, neither a multiple of the blocks' views or
# tiles; neither width nor height a multiple of the 4x8-pixel tile
SHAPES = [(13, 451, 711), (37, 243, 469)]


@pytest.mark.parametrize("kind", ["sh16_d6", "sh25_d5"])
@pytest.mark.parametrize("n,W,H", SHAPES)
def test_view_blocks_equal_single_views(built, trees, kind, n, W, H):
    assert _blocks(W, H, n, kind)
    cams = _cams(W, H, 40, n)
    opt = _opt(kind)
    _same(_batch(trees[kind], cams, opt), _singles(trees[kind], cams, opt))


@pytest.mark.parametrize("kind", ["sh16_d6", "sh25_d5"])
def test_view_blocks_composite_renders_each_tile_once(built, trees, kind):
    import torch
    from volrend_b200 import _capi, lib
    from volrend_b200.host import _cams_array, _options_array
    tree = trees[kind]
    n, W, H = SHAPES[0]
    assert _blocks(W, H, n, kind)
    cams = _cams(W, H, 60, n)
    opt = _opt(kind)
    rng = np.random.default_rng(5)
    img0 = torch.from_numpy(rng.integers(0, 256, (n, H, W, 4), dtype=np.uint8)).cuda()
    dep = torch.from_numpy(rng.uniform(0.5, 3.0, (n, H, W)).astype(np.float32)).cuda()
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


def test_view_blocks_two_part_band_batch(built, trees):
    """vr_render_bands_batch, 2 parts, each part's rows a block batch of their own."""
    import torch
    from volrend_b200 import lib, render_bands_batch
    tree = trees["sh16_d6"]
    n, W, H, band = 37, 387, 675, 4
    cams = _cams(W, H, 100, n)
    opt = _opt("sh16_d6")
    ref = _singles(tree, cams, opt)[0]
    got = np.full((n, H, W, 4), SENTINEL, np.uint8)
    for part in range(2):
        rows = lib().vr_band_rows(H, band, 2, part)
        assert _blocks(W, rows, n)
        img = torch.full((n + 1, rows, W, 4), SENTINEL, dtype=torch.uint8, device="cuda")   # + a guard view
        assert render_bands_batch(tree, cams, opt, band, 2, part, img) == rows
        torch.cuda.synchronize()
        img = img.cpu().numpy()
        assert (img[n] == SENTINEL).all(), "a band launch wrote past its views"
        for r in range(rows):
            got[:, (r // band * 2 + part) * band + r % band] = img[:n, r]
    assert np.array_equal(got, ref)


def test_view_blocks_past_camera_ring_split(built, trees):
    """8192 + 37 views: one launch of 8192 views in blocks (5x5 tiles: one full block column and row, one partial),
    then one of 37 views with the plain tile counter."""
    n, W, H = 8192 + 37, 20, 40
    assert _blocks(W, H, 8192) and not _blocks(W, H, 37)
    cams = _cams(W, H, 0, n)
    opt = _opt("sh16_d6")
    _same(_batch(trees["sh16_d6"], cams, opt), _singles(trees["sh16_d6"], cams, opt))
