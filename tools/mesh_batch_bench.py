#!/usr/bin/env python
"""Batched rendering of frames with meshes: the 300-frame orbit of tools/anim_bench.py on the bench tree (synthetic
lego, SH16, depth 10) at 800x800, timed with CUDA events (median of --reps after one warm-up pass).  Scenes:

  cube      Mesh.Cube() at scale 0.8 inside the volume
  sphere    Mesh.Sphere(225, 224) (~100k triangles)
  frustums  the 100-camera CameraFrustum drawlist of tests/golden/ref/mesh_dl_cams100.npz
  probe     no mesh, enable_probe on (probe cube + disc)

Legs per scene, in ms/frame:
  single    VolumeRenderer.render() per frame
  batch32 / batch64  VolumeRenderer.render_batch in chunks of 32 / 64 frames
  raster32  / march32  the two halves of batch32: draw_meshes_batch alone, vr_render_composite_batch_opts alone
Plus anim_s: render_animation with the frustum drawlist, end to end to PNGs (host clock, one run).
Prints one JSON line, with the card's name and power limit read in the same run.

    python tools/mesh_batch_bench.py [--frames 300] [--size 800] [--reps 3]
"""
import argparse
import contextlib
import copy
import io
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from anim_bench import card  # noqa: E402


def timed(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--size", type=int, default=800)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--depth", type=int, default=10)
    a = ap.parse_args()
    import torch
    from volrend_b200 import Camera, Mesh, N3Tree, RenderOptions, VolumeRenderer, draw_meshes_batch, host, lib, synth
    from volrend_b200.anim import AnimKF, MeshState, animation_frames, render_animation
    from volrend_b200.host import _cams_array, _options_array
    assert torch.cuda.is_available(), "needs a CUDA device"
    W = H = a.size
    tree = N3Tree.from_synth(synth.make_tree("lego", depth=a.depth, basis_dim=16, seed=0))
    k0 = AnimKF(fx=synth.focal_for(W), fy=synth.focal_for(W), t_max=1.0)
    k0.center = np.array([-3.0, 0.0, 2.0], np.float32)
    k0.v_back = (k0.center / np.linalg.norm(k0.center)).astype(np.float32)
    k1 = AnimKF(fx=k0.fx * 1.2, fy=k0.fy * 1.2, t_max=a.frames / 30.0, loops=1)
    k1.center, k1.v_back = k0.center.copy(), k0.v_back.copy()
    frames = list(animation_frames([k0, k1], 30.0, (0, 0, 1), Camera(W, H)))
    n = len(frames)
    rend = VolumeRenderer()
    rend.resize(W, H)
    rend.set(tree)
    cams = []
    for state, _ in frames:
        state.to_renderer(rend)
        cams.append(copy.deepcopy(rend.camera))
    opt = copy.deepcopy(rend.options)
    cube = Mesh.Cube()
    cube.scale = 0.8
    sphere = Mesh.Sphere(225, 224)
    z = np.load(os.path.join(ROOT, "tests", "golden", "ref", "mesh_dl_cams100.npz"))
    with contextlib.redirect_stdout(io.StringIO()):
        frustums = Mesh.open_drawlist_mem(bytes(z["input"]))
    probe = copy.deepcopy(opt)
    probe.enable_probe, probe.probe = True, [0.5, 0.5, 0.5]
    scenes = {"cube": ([cube], opt), "sphere": ([sphere], opt), "frustums": (frustums, opt), "probe": ([], probe)}
    for ms, _ in scenes.values():
        for m in ms:
            m.update()
    res = {}
    out = torch.empty((n, H, W, 4), dtype=torch.uint8, device="cuda")
    for name, (meshes, o) in scenes.items():
        rend.meshes, rend.options = meshes, o

        def single():
            for i, c in enumerate(cams):
                rend.camera = copy.deepcopy(c)
                out[i].copy_(rend.render())

        def batch(chunk):
            def fn():
                for v0 in range(0, n, chunk):
                    rend.render_batch(cams[v0:v0 + chunk], o, None, out=out[v0:v0 + chunk])
            return fn

        res[f"{name}_single_ms_per_frame"] = timed(single, a.reps) / n
        ref = out.clone()
        for chunk in (32, 64):
            host.RENDER_BATCH_CHUNK = chunk
            res[f"{name}_batch{chunk}_ms_per_frame"] = timed(batch(chunk), a.reps) / n
            res[f"{name}_batch{chunk}_equals_single"] = bool(torch.equal(ref, out))
        host.RENDER_BATCH_CHUNK = 32
        # the two halves of a 32-frame chunk, on their own
        draws = [[copy.copy(m) for m in meshes] + ([] if not o.enable_probe else [rend._probe])] * 32
        if o.enable_probe:
            rend._probe.visible = True
            rend._probe.translation = np.asarray(o.probe, np.float32)
        bc = [copy.deepcopy(c) for c in cams[:32]]
        for c in bc:
            c._update()
        img = out[:32]
        dep = torch.full((32, H, W), 1e9, dtype=torch.float32, device="cuda")
        res[f"{name}_raster32_ms_per_frame"] = timed(lambda: draw_meshes_batch(bc, draws, img, dep), a.reps) / 32
        arr, oarr = _cams_array(bc), _options_array([o] * 32)
        s = torch.cuda.current_stream().cuda_stream
        res[f"{name}_march32_ms_per_frame"] = timed(
            lambda: lib().vr_render_composite_batch_opts(tree._handle, arr, 32, oarr, None, img.data_ptr(),
                                                         dep.data_ptr(), None, s), a.reps) / 32
        rend._probe.visible = False
    kf = [k0.copy(), k1.copy()]
    for k in kf:
        k.mesh_state = {m.name: MeshState(np.asarray(m.rotation, np.float32), np.asarray(m.translation, np.float32),
                                          float(m.scale), bool(m.unlit)) for m in frustums}
    with tempfile.TemporaryDirectory() as d:
        t0 = time.perf_counter()
        paths = render_animation(tree, kf, 30.0, d, width=W, height=H, meshes=frustums)
        res["anim_frustums_s"] = time.perf_counter() - t0
        res["anim_frames"] = len(paths)
    gpu, pl = card()
    print(json.dumps({"bench": "mesh_batch", "frames": n, "size": [W, H], "tree": f"synthetic lego SH16 depth {a.depth}",
                      "gpu": gpu, "power_limit": pl, **{k: (round(v, 4) if isinstance(v, float) else v)
                                                        for k, v in res.items()}}))


if __name__ == "__main__":
    main()
