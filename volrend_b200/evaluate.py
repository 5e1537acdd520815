"""Score a tree's renders against test images: per-view PSNR and SSIM on the GPU.

    python -m volrend_b200.evaluate tree.npz pose.txt [pose.txt ...] --targets img.png [img.png ...]
                                    [-i intrinsics.txt] [-r] [--width 800] [--height 800] [--fx F] [--fy F]
                                    [--step_size S] [--sigma_thresh S] [--stop_thresh S] [--background B]
                                    [--batch 8] [--json out.json]

The renders are ``render_batch``'s float output, so nothing is lost to 8-bit rounding; RGBA targets are composited onto
the background brightness, as NeRF-synthetic test images are scored.  SSIM is :func:`volrend_b200.image_ssim`
(JaxNeRF's ``compute_ssim``, DESIGN.md section 22).  The tree may be any file ``N3Tree.open`` loads, compressed
(``quant_map``) and NDC trees included, so pruned and compressed trees can be scored.  The means printed last are the
means of the per-view values, as the NeRF-family papers report them.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

from .views import add_view_arguments, read_targets, target_batch, view_setup


def evaluate(tree, cams, targets, options, *, batch: int = 8, ssim: bool = True):
    """Per-view quality of the renders of ``tree`` (an ``N3Tree`` on the device) from ``cams`` (one image size)
    against ``targets`` (one image per camera, [H, W, 3 | 4], uint8 or float, indexed lazily), rendered with
    ``options`` (one ``RenderOptions``; its background brightness also composites RGBA targets) in batches of
    ``batch`` views.  Returns ``(mse, ssim)``: float64 numpy arrays [V] of the mean squared RGB error and the SSIM of
    every view (NaN for images smaller than the 11x11 SSIM window, and everywhere with ``ssim=False``, which skips it)."""
    import torch
    from .host import image_ssim, render_batch
    if batch < 1:
        raise ValueError(f"batch {batch} must be >= 1")
    if len(targets) != len(cams):
        raise ValueError(f"{len(targets)} targets for {len(cams)} views")
    if not tree.is_cuda_loaded():
        raise RuntimeError("N3Tree is not loaded on the device")
    dev = torch.device("cuda", tree._device)
    mse, sv = np.zeros(len(cams)), np.full(len(cams), np.nan)
    if not cams:
        return mse, sv
    H, W = cams[0].height, cams[0].width
    fo = torch.empty((min(batch, len(cams)), H, W, 4), dtype=torch.float32, device=dev)
    for v0 in range(0, len(cams), batch):
        idx = range(v0, min(v0 + batch, len(cams)))
        f = fo[:len(idx)]
        render_batch(tree, [cams[v] for v in idx], options, None, float_out=f)
        tgt = target_batch(targets, idx, options.background_brightness, dev, H, W)
        mse[v0:v0 + len(idx)] = (f[..., :3] - tgt).double().square().mean(dim=(1, 2, 3)).cpu().numpy()
        if ssim and min(H, W) >= 11:
            sv[v0:v0 + len(idx)] = image_ssim(f, tgt).cpu().numpy()
    return mse, sv


def psnr(mse) -> np.ndarray:
    """PSNR in dB of per-view MSE (max value 1)."""
    return -10.0 * np.log10(np.maximum(np.asarray(mse, np.float64), 1e-30))


# ---------------------------------------------------------------------------------------------------------- CLI
def _parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog="python -m volrend_b200.evaluate",
                                 description="Per-view PSNR and SSIM of a PlenOctree's renders against test images.")
    ap.add_argument("input", help="npz file storing octree data (any tree N3Tree.open loads, compressed included)")
    add_view_arguments(ap, targets=True)
    ap.add_argument("--batch", type=int, default=8, help="views rendered and scored per launch")
    ap.add_argument("--json", default="", help="also write the per-view values and their means to this file")
    return ap


def main(argv=None) -> int:
    ap = _parser()
    args = ap.parse_args(argv)
    if args.batch < 1:
        ap.error(f"--batch {args.batch} < 1")
    if not args.input.endswith(".npz"):
        ap.error(f"'{args.input}' is not an .npz tree")
    for p in [args.input] + args.targets:
        if not os.path.exists(p):
            ap.error(f"'{p}' does not exist")
    if args.width < 11 or args.height < 11:
        ap.error(f"image size {args.width}x{args.height}: SSIM needs at least 11x11")
    cams = view_setup(ap, args)
    try:
        targets = read_targets(args.targets, len(cams), args.width, args.height)
    except ValueError as e:
        ap.error(str(e))

    from .host import N3Tree, RenderOptions
    tree = N3Tree(args.input)
    options = RenderOptions(step_size=args.step_size, sigma_thresh=args.sigma_thresh, stop_thresh=args.stop_thresh,
                            background_brightness=args.background)
    mse, ssim = evaluate(tree, cams, targets, options, batch=args.batch)
    tree.free_cuda()
    p = psnr(mse)
    for v in range(len(cams)):
        print(f"view {v}: PSNR {p[v]:.3f} dB, SSIM {ssim[v]:.4f}")
    print(f"mean over {len(cams)} views: PSNR {p.mean():.3f} dB, SSIM {ssim.mean():.4f}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"mse": mse.tolist(), "psnr": p.tolist(), "ssim": ssim.tolist(),
                       "mean_psnr": float(p.mean()), "mean_ssim": float(ssim.mean())}, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
