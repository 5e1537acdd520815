#!/usr/bin/env python
"""Times the octree grid (show_grid): generating it on the GPU, the reference's host walk, and
VolumeRenderer.render() with it; prints one JSON line.

  python tools/grid_bench.py [--steps 20] [--warmup 5] [--depth 10]

All on cuda:0 with the bench tree (synth lego SH16, depth --depth) at 800x800, NeRF-synthetic orbit pose 0:
  wire[m]           vr_tree_wireframe into a preallocated buffer, grid_max_depth m = 0..7: cells, MB written, median
                    ms (CUDA events around each call) and the write rate that implies; first_count_ms is the
                    one-time cell count of the first call (host clock, it synchronises)
  ref_host_ms[m]    the reference's N3Tree::gen_wireframe(m) on the host (oracle/_ref), when that build is present
  render_ms         VolumeRenderer.render() without the grid; render_grid_ms[m] with it, m = 3..7 (grid already
                    generated: the render does not regenerate it)
  draw_grid_ms[m]   vr_draw_meshes of the grid alone, orbit view and a close-up from 0.45x the orbit distance, where
                    the coarse grid's lines span much of the frame (the rasterizer's large-primitive path)
The GPU name, power limit and SM clock are read in the same process and printed beside the numbers."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from volrend_b200 import N3Tree, VolumeRenderer, draw_meshes, lib, synth  # noqa: E402
from volrend_b200._capi import check  # noqa: E402

W = H = 800


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms))


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                               "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--depth", type=int, default=int(os.environ.get("VR_BENCH_DEPTH", "10")))
    args = ap.parse_args()
    torch.cuda.set_device(0)
    res = {"impl": "ours", "what": "octree grid wireframe (vr_tree_wireframe) and VolumeRenderer.render with show_grid",
           "gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup, "tree": f"synth lego SH16 depth {args.depth}"}
    st = synth.make_tree("lego", depth=args.depth, basis_dim=16, seed=0)
    tree = N3Tree.from_synth(st)
    stream = torch.cuda.current_stream().cuda_stream

    t0 = time.perf_counter()
    n = C.c_int64()
    check(lib().vr_tree_wireframe(tree._handle, 0, None, 0, C.byref(n), stream))
    res["first_count_ms"] = round((time.perf_counter() - t0) * 1e3, 3)
    res["wire"] = {}
    for m in range(8):
        nv = tree.wireframe_vertex_count(m)
        buf = torch.empty(nv * 9, dtype=torch.float32, device="cuda")
        got = C.c_int64()

        def fill():
            check(lib().vr_tree_wireframe(tree._handle, m, buf.data_ptr(), nv, C.byref(got), stream))
        ms = timed(fill, args.steps, args.warmup)
        mb = nv * 36 / 1e6
        res["wire"][m] = {"cells": nv // 24, "MB": round(mb, 2), "ms": round(ms, 4), "GB_per_s": round(mb / ms, 1)}
        del buf

    from oracle import ref_binding as rb
    from oracle import ref_wire
    if ref_wire.available():
        from bench import StdoutToStderr      # the reference loader prints to stdout: keep the JSON line clean
        with tempfile.TemporaryDirectory() as tmp, StdoutToStderr():
            path = os.path.join(tmp, "bench.npz")
            st.save_npz(path)
            rt = rb.RefTree(path)
            reps = max(1, min(args.steps, 5))
            res["ref_host_ms"] = {m: round(float(np.median([ref_wire.wireframe_ms(rt, m) for _ in range(reps)])), 3) for m in range(8)}
            rt.close()
    else:
        res["ref_host_ms"] = "not measured (oracle/_ref not built)"

    pose = synth.nerf_synthetic_test_poses(200)[0]
    eye = pose[:3, 3].astype(np.float32)
    vr = VolumeRenderer()
    vr.resize(W, H)
    vr.camera.fx = vr.camera.fy = synth.focal_for(W)
    vr.camera.center = eye
    vr.camera.v_back = eye / np.linalg.norm(eye)
    vr.set(tree)
    res["render_ms"] = round(timed(vr.render, args.steps, args.warmup), 4)
    vr.options.show_grid = True
    res["render_grid_ms"], res["draw_grid_ms"], res["draw_grid_closeup_ms"] = {}, {}, {}
    img = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    dep = torch.full((H, W), 1e9, dtype=torch.float32, device="cuda")
    fill_ms = timed(lambda: dep.fill_(1e9), args.steps, args.warmup)
    for m in range(3, 8):
        vr.options.grid_max_depth = m
        vr.render()                           # generates the grid
        res["render_grid_ms"][m] = round(timed(vr.render, args.steps, args.warmup), 4)
        wire = vr._wire
        for key, scale in (("draw_grid_ms", 1.0), ("draw_grid_closeup_ms", 0.45)):
            vr.camera.center = eye * scale
            vr.camera._update()

            def draw():
                dep.fill_(1e9)
                draw_meshes(vr.camera, [wire], img, dep)
            res[key][m] = round(timed(draw, args.steps, args.warmup) - fill_ms, 4)
        vr.camera.center = eye
        vr.camera._update()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
