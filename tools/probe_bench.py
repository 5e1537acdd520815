#!/usr/bin/env python
"""Times the lumisphere probe (enable_probe); prints one JSON line.

  python tools/probe_bench.py [--steps 50] [--warmup 10] [--depth 10]

All on cuda:0 with the bench tree (synth lego SH16, depth --depth) at 800x800, NeRF-synthetic orbit pose 0, the probe
at the centre of the volume:
  overlay_ms[S]      vr_draw_probe alone over a finished frame, probe_disp_size S = 100, 400, 800
  launch_ms          launch_renderer (offscreen) without the probe; launch_probe_ms with it (S = 100)
  render_ms          VolumeRenderer.render() without the probe; render_probe_ms with it (the probe cube makes it take
                     the clear -> draw -> composite path, whose march then draws the disc)
Medians of --steps timed calls after --warmup untimed ones, CUDA events around each call.  The GPU name, power limit
and SM clock are read in the same process and printed beside the numbers."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from volrend_b200 import Camera, N3Tree, RenderOptions, VolumeRenderer, launch_renderer, lib, synth  # noqa: E402
from volrend_b200._capi import check  # noqa: E402


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                               "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unavailable ({e})"


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--depth", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("probe_bench needs a CUDA device")
    torch.cuda.set_device(0)
    W = H = 800
    st = synth.make_tree("lego", depth=a.depth, basis_dim=16, seed=0)
    tree = N3Tree.from_synth(st)
    pose = synth.nerf_synthetic_test_poses(200)[0]
    cam = Camera(W, H, synth.focal_for(W), synth.focal_for(W))
    cam.set_c2w(pose)
    centre = ((0.5 - np.asarray(st.offset, np.float64)) / np.asarray(st.invradius3, np.float64)).tolist()
    img = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    out = dict(gpu=gpu_info(), tree=f"synth lego SH16 depth {a.depth}", frame=f"{W}x{H}", steps=a.steps,
               warmup=a.warmup)

    base = RenderOptions(basis_minmax=[0, 15])
    launch_renderer(tree, cam, base, img, None, None, True)
    c, o = cam._as_c(), base._as_c()
    xyz = (C.c_float * 3)(*centre)
    out["overlay_ms"] = {}
    for S in (100, 400, 800):
        out["overlay_ms"][S] = timed(lambda: check(lib().vr_draw_probe(
            tree._handle, C.byref(c), 1, C.byref(o), xyz, S, None, img.data_ptr(), None, 0, stream)), a.steps, a.warmup)

    probe = RenderOptions(basis_minmax=[0, 15], enable_probe=True, probe=centre, probe_disp_size=100)
    out["launch_ms"] = timed(lambda: launch_renderer(tree, cam, base, img, None, None, True), a.steps, a.warmup)
    out["launch_probe_ms"] = timed(lambda: launch_renderer(tree, cam, probe, img, None, None, True), a.steps, a.warmup)

    vr = VolumeRenderer()
    vr.resize(W, H)
    vr.camera.fx = vr.camera.fy = synth.focal_for(W)
    vr.set(tree)
    out["render_ms"] = timed(vr.render, a.steps, a.warmup)
    vr.options.enable_probe, vr.options.probe, vr.options.probe_disp_size = True, centre, 100
    out["render_probe_ms"] = timed(vr.render, a.steps, a.warmup)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
