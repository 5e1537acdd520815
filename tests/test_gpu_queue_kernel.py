"""`-m gpu`: the shading-queue kernel (variant 7, vr_march_q.cuh) against the inline-shading kernel (variant
3 + 16*193, vr_march.cuh), bit for bit, at sizes where every CTA works through many tiles: batches with several option
sets and their counters, back-to-back single frames on one stream (they overlap through programmatic dependent
launch), a tile, a band and a composite launch."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
QUEUE, INLINE = 7, 3 + 16 * 193


def _cam(W, H, pose):
    from volrend_b200 import Camera, synth
    c = Camera(W, H, synth.focal_for(W), synth.focal_for(W))
    c.set_c2w(pose)
    return c


@pytest.mark.parametrize("basis,fmt", [(16, "SH"), (25, "SH"), (9, "SH"), (4, "SH"), (9, "SG")])
def test_queue_kernel_equals_inline_kernel(built, basis, fmt):
    import torch
    from volrend_b200 import N3Tree, RenderOptions, launch_renderer, lib, render_bands, render_batch, synth
    st = synth.make_tree("lego", depth=8, basis_dim=basis, seed=basis, fmt=fmt)
    tree = N3Tree.from_synth(st)
    W, H = 640, 480
    poses = synth.nerf_synthetic_test_poses(24)
    cams = [_cam(W, H, p) for p in poses]
    opts = [RenderOptions(), RenderOptions(stop_thresh=0.0, sigma_thresh=0.0), RenderOptions(render_depth=True),
            RenderOptions(step_size=1e-3, background_brightness=0.4)]
    res = {}
    for v in (QUEUE, INLINE):
        assert lib().vr_set_variant(v) == 0
        out = []
        for opt in opts:
            imgs = torch.zeros((len(cams), H, W, 4), dtype=torch.uint8, device="cuda")
            fo = torch.zeros((len(cams), H, W, 4), dtype=torch.float32, device="cuda")
            cnt = torch.zeros(5, dtype=torch.int64, device="cuda")
            render_batch(tree, cams, opt, imgs, float_out=fo)
            render_batch(tree, cams, opt, None, counters=cnt)
            torch.cuda.synchronize()
            out.append((fo.cpu().numpy(), imgs.cpu().numpy(), cnt.cpu().tolist()))
        # single-frame launches back to back on one stream (they overlap through PDL)
        single = torch.zeros((6, H, W, 4), dtype=torch.uint8, device="cuda")
        for rep in range(2):
            for i in range(6):
                launch_renderer(tree, cams[i], opts[0], single[i], None, None, True)
        # a tile and a band launch
        tile = torch.zeros((200, 300, 4), dtype=torch.float32, device="cuda")
        launch_renderer(tree, cams[3], opts[0], None, None, None, True, float_out=tile, tile=(100, 150, 300, 200))
        band = torch.zeros((max(1, H // 3 + 8), W, 4), dtype=torch.uint8, device="cuda")
        rows = render_bands(tree, cams[5], opts[0], 8, 3, 1, band)
        # composite mode
        comp = torch.full((H, W, 4), 77, dtype=torch.uint8, device="cuda")
        depth = torch.full((H, W), 3.5, dtype=torch.float32, device="cuda")
        launch_renderer(tree, cams[7], opts[0], comp, depth, None, False)
        torch.cuda.synchronize()
        res[v] = (out, single.cpu().numpy(), tile.cpu().numpy(), band[:rows].cpu().numpy(), comp.cpu().numpy())
    lib().vr_set_variant(0)
    a, b = res[QUEUE], res[INLINE]
    for (fa, ua, ca), (fb, ub, cb) in zip(a[0], b[0]):
        assert np.array_equal(fa, fb) and np.array_equal(ua, ub)
        assert ca == cb
    for x, y in zip(a[1:], b[1:]):
        assert np.array_equal(x, y)
    assert a[0][0][2][0] > 0 and (a[0][0][1][..., :3] != 255).any()      # something was rendered
