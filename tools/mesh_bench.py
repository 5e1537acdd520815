#!/usr/bin/env python
"""Times the CUDA mesh rasterizer and VolumeRenderer.render() with and without a mesh; prints one JSON line.

  python tools/mesh_bench.py [--steps 20] [--warmup 5] [--depth 10]

Legs, all at 800x800 on cuda:0 (median over --steps timed calls, each call bracketed by CUDA events after
--warmup untimed calls of the same shape):
  draw_cube_ms      vr_draw_meshes of Mesh.Cube() (12 triangles) seen from the NeRF-synthetic orbit
  draw_sphere_ms    Mesh.Sphere(225, 224) (~100k triangles) filling about half of the frame
  draw_quad_ms      a two-triangle quad covering the whole frame
  render_ms         VolumeRenderer.render() on the bench tree (synth lego SH16, depth --depth), no mesh
  render_cube_ms    the same with a visible Cube inside the volume (clear + draw + composite march)
  composite_march_ms / offscreen_march_ms  the two march launches of those renders on their own
The GPU name, power limit and SM clock are read in the same process and printed beside the numbers."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from volrend_b200 import Mesh, N3Tree, VolumeRenderer, draw_meshes, synth  # noqa: E402

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
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
        return out
    except Exception as e:  # noqa: BLE001
        return f"unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--depth", type=int, default=int(os.environ.get("VR_BENCH_DEPTH", "10")))
    args = ap.parse_args()
    torch.cuda.set_device(0)
    pose = synth.nerf_synthetic_test_poses(200)[0]
    vr = VolumeRenderer()
    vr.resize(W, H)
    vr.camera.fx = vr.camera.fy = synth.focal_for(W)
    eye = pose[:3, 3]
    vr.camera.center = eye.astype(np.float32)
    vr.camera.v_back = (eye / np.linalg.norm(eye)).astype(np.float32)
    vr.camera._update()
    cam = vr.camera

    img = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    dep = torch.full((H, W), 1e9, dtype=torch.float32, device="cuda")
    cube = Mesh.Cube()
    sphere = Mesh.Sphere(225, 224)
    sphere.scale = 1.4
    quad = Mesh(4, 2, 3)
    v = quad.vert.reshape(-1, 9)
    back = cam.v_back
    right, up = cam.v_right, cam.v_up
    ctr = eye - 1.0 * back                      # a plane one unit in front of the camera, 8 units wide
    for i, (a, b) in enumerate([(-1, -1), (1, -1), (1, 1), (-1, 1)]):
        v[i, :3] = ctr + 4 * a * right + 4 * b * up
        v[i, 3:9] = (0.5, 0.5, 0.5, *back)
    quad.faces[:] = (0, 1, 2, 0, 2, 3)
    for m in (cube, sphere, quad):
        m.update()

    def draw(m):
        def fn():
            dep.fill_(1e9)
            draw_meshes(cam, [m], img, dep)
        return fn

    fill_ms = timed(lambda: dep.fill_(1e9), args.steps, args.warmup)
    res = {"impl": "ours", "what": "mesh rasterizer (vr_draw_meshes) and VolumeRenderer.render at 800x800",
           "gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup,
           "n_tris": {"cube": 12, "sphere": int(sphere.faces.size // 3), "quad": 2}}
    for name, m in (("cube", cube), ("sphere", sphere), ("quad", quad)):
        res[f"draw_{name}_ms"] = round(timed(draw(m), args.steps, args.warmup) - fill_ms, 4)
        res[f"covered_{name}"] = int((dep != 1e9).sum().item())
    res["depth_fill_ms"] = round(fill_ms, 4)

    st = synth.make_tree("lego", depth=args.depth, basis_dim=16, seed=0)
    tree = N3Tree.from_synth(st)
    vr.set(tree)
    vr.meshes = []
    res["render_ms"] = round(timed(vr.render, args.steps, args.warmup), 4)
    inside = Mesh.Cube()
    inside.scale = 0.8
    vr.meshes = [inside]
    res["render_cube_ms"] = round(timed(vr.render, args.steps, args.warmup), 4)
    # its parts: the composite march alone (colour + ray-distance limits as the mesh pass left them), and the
    # offscreen march through launch_renderer for comparison
    from volrend_b200 import launch_renderer
    col, lim = vr._image.clone(), vr._depth.clone()
    res["composite_march_ms"] = round(timed(lambda: launch_renderer(tree, cam, vr.options, col, lim, None, False),
                                            args.steps, args.warmup), 4)
    res["offscreen_march_ms"] = round(timed(lambda: launch_renderer(tree, cam, vr.options, col, None, None, True),
                                            args.steps, args.warmup), 4)
    res["tree"] = f"synth lego SH16 depth {args.depth}"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
