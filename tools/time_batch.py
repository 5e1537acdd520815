#!/usr/bin/env python
"""One timing line for one kernel variant:
200-view batch and back-to-back single-frame launches on the bench tree (cached as an .npz in /tmp).
usage: time_batch.py [label] [variant] [depth] [basis]"""
import ctypes as C
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from volrend_b200 import synth, N3Tree, Camera, RenderOptions, render_batch, lib  # noqa: E402

label = sys.argv[1] if len(sys.argv) > 1 else "default"
variant = int(sys.argv[2]) if len(sys.argv) > 2 else 0
depth = int(sys.argv[3]) if len(sys.argv) > 3 else 10
basis = int(sys.argv[4]) if len(sys.argv) > 4 else 16
path = f"/tmp/vr_tree_d{depth}_b{basis}.npz"
if not os.path.exists(path):
    synth.make_tree("lego", depth=depth, basis_dim=basis, seed=0).save_npz(path)
assert lib().vr_set_variant(variant) == 0
tree = N3Tree(path)
W = H = 800
cams = []
for p in synth.nerf_synthetic_test_poses(200):
    c = Camera(W, H, synth.focal_for(W), synth.focal_for(W))
    c.set_c2w(p)
    cams.append(c)
opt = RenderOptions()
imgs = torch.zeros((len(cams), H, W, 4), dtype=torch.uint8, device="cuda")
best = 1e9
for rep in range(5):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    render_batch(tree, cams, opt, imgs)
    e1.record()
    torch.cuda.synchronize()
    if rep:
        best = min(best, e0.elapsed_time(e1) / len(cams))
ccams = [c._as_c() for c in cams]
copt = opt._as_c()
stream = torch.cuda.current_stream().cuda_stream
single = 1e9
for rep in range(3):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for cc in ccams:
        lib().vr_render(tree._handle, C.byref(cc), C.byref(copt), None, imgs[0].data_ptr(), None, None, stream)
    e1.record()
    torch.cuda.synchronize()
    single = min(single, e0.elapsed_time(e1) / len(cams))
print(f"TIMING {label:28s} batch {best:.4f} ms/frame ({W * H / best / 1e3:7.0f} Mrays/s)   single-frame launches {single:.4f} ms/frame"
      f"   checksum {int(imgs[::50].long().sum())}", flush=True)
