#!/usr/bin/env python
"""Cost of per-frame render options: a 300-frame orbit of the bench tree (synthetic lego, SH16, depth 10) at 800x800
whose options change every frame, timed with CUDA events (kernel launches only, after warm-up; median of --reps):

  single   one single-view launch per frame (launch_renderer offscreen)
  opts     one batch with options per view (render_batch with a list: vr_render_batch_opts)
  opts_eq  the same batch with every view's options equal (the per-view kernels, no divergence in the options)
  uniform  the uniform batch of the same cameras with the first frame's options (vr_render_batch)
  anim     render_animation end to end to PNGs in a temporary directory (host clock, one run)

Prints one JSON line, with the card's name and power limit read in the same run.

    python tools/anim_bench.py [--frames 300] [--size 800] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl = [s.strip() for s in out.split(",")]
        return name, pl
    except Exception as e:   # the numbers still stand; say what could not be read
        return f"unknown ({e})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--size", type=int, default=800)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--depth", type=int, default=10)
    a = ap.parse_args()
    import torch
    from volrend_b200 import Camera, N3Tree, RenderOptions, launch_renderer, render_batch, synth
    from volrend_b200.anim import AnimKF, animation_frames, render_animation
    assert torch.cuda.is_available(), "needs a CUDA device"
    W = H = a.size
    tree = N3Tree.from_synth(synth.make_tree("lego", depth=a.depth, basis_dim=16, seed=0))
    # the orbit: two keyframes at the same place, one extra turn, options changing along the way
    k0 = AnimKF(fx=synth.focal_for(W), fy=synth.focal_for(W), t_max=1.0)
    k0.center = np.array([-3.0, 0.0, 2.0], np.float32)
    k0.v_back = (k0.center / np.linalg.norm(k0.center)).astype(np.float32)
    k0.opt = RenderOptions(step_size=1e-4, background_brightness=1.0, stop_thresh=1e-2, sigma_thresh=1e-2)
    k1 = AnimKF(fx=k0.fx * 1.2, fy=k0.fy * 1.2, t_max=a.frames / 30.0, loops=1)
    k1.center, k1.v_back = k0.center.copy(), k0.v_back.copy()
    k1.opt = RenderOptions(step_size=2e-4, background_brightness=0.0, stop_thresh=2e-2, sigma_thresh=2e-2,
                           render_bbox=[0.05, 0.05, 0.0, 0.95, 0.95, 1.0])
    frames = list(animation_frames([k0, k1], 30.0, (0, 0, 1), Camera(W, H)))
    cams = [c for _, c in frames]
    opts = [s.opt for s, _ in frames]
    n = len(cams)
    assert len({(o.step_size, o.background_brightness) for o in opts}) == n, "options must change every frame"
    img = torch.empty((n, H, W, 4), dtype=torch.uint8, device="cuda")

    def run_single():
        for i in range(n):
            launch_renderer(tree, cams[i], opts[i], img[i], None, None, True)

    legs = {"single": run_single,
            "opts": lambda: render_batch(tree, cams, opts, img),
            "opts_eq": lambda: render_batch(tree, cams, [opts[0]] * n, img),
            "uniform": lambda: render_batch(tree, cams, opts[0], img)}
    res = {}
    for name, fn in legs.items():
        fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        res[name + "_ms"] = float(np.median(ts))
        res[name + "_ms_per_frame"] = float(np.median(ts)) / n
        res[name + "_spread_ms"] = [float(min(ts)), float(max(ts))]
    # outputs of the per-view batch equal the single-view launches
    run_single()
    ref = img.clone()
    render_batch(tree, cams, opts, img)
    torch.cuda.synchronize()
    res["opts_equals_single"] = bool(torch.equal(ref, img))
    with tempfile.TemporaryDirectory() as d:
        t0 = time.perf_counter()
        paths = render_animation(tree, [k0, k1], 30.0, d, width=W, height=H)
        res["anim_s"] = time.perf_counter() - t0
        res["anim_frames"] = len(paths)
    name, pl = card()
    print(json.dumps({"bench": "anim", "frames": n, "size": [W, H], "tree": f"synthetic lego SH16 depth {a.depth}",
                      "gpu": name, "power_limit": pl, **res}))


if __name__ == "__main__":
    main()
