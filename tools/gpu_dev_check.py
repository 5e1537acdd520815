#!/usr/bin/env python
"""Development probe for one gpurun call: parity of our kernel vs the CPU oracle and vs the
reference CUDA kernel (oracle/_ref), plus quick timings of every kernel variant.
Writes gpurun_out/dev_check.json.  Not a test and not the bench."""
import ctypes as C
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from volrend_b200 import synth, N3Tree, Camera, RenderOptions, launch_renderer, render_batch, lib  # noqa: E402
from oracle import binding as ob  # noqa: E402
from oracle import ref_binding as rb  # noqa: E402

VARIANTS = [int(v) for v in os.environ.get("VR_VARIANTS", "7,3091").split(",")]
out = {}
os.makedirs("gpurun_out", exist_ok=True)
dev = torch.device("cuda:0")
print(torch.cuda.get_device_name(0), flush=True)


def cmp(a, b):
    d = np.abs(a.astype(np.float64) - b.astype(np.float64))
    return dict(max=float(d.max()), mean=float(d.mean()), n_gt_1e4=int((d.max(-1) > 1e-4).sum()),
                n_gt_1e6=int((d.max(-1) > 1e-6).sum()), n_ne=int((d.max(-1) > 0).sum()), n=int(d.shape[0] * d.shape[1]))


def parity(name, st, W, H, pose, **optkw):
    path = f"/tmp/{name}.npz"
    st.save_npz(path)
    tree = N3Tree(path)
    cam = Camera(W, H, synth.focal_for(W), synth.focal_for(W))
    cam.set_c2w(pose)
    opt = RenderOptions(**optkw)
    res = {"info": tree.info()}
    ot = ob.OracleTree.from_synth(st)
    ocam = ob.make_camera(W, H, cam.fx, cam.fy, synth.c2w_to_colmajor12(pose))
    oopt = ob.make_options(**{k: v for k, v in optkw.items()})
    f_o, u_o, c_o = ob.render(ot, ocam, oopt)
    res["oracle_counters"] = c_o
    rt = rb.RefTree(path) if rb.available() else None
    if rt:
        ropt = rb.make_options(**optkw)
        f_r = rt.render_f32(W, H, cam.fx, cam.fy, synth.c2w_to_colmajor12(pose), ropt)
        u_r = rt.render_u8(W, H, cam.fx, cam.fy, synth.c2w_to_colmajor12(pose), ropt)
        res["oracle_vs_ref_f32"] = cmp(f_o, f_r)
        res["oracle_vs_ref_u8"] = cmp(u_o, u_r)
        q = np.zeros_like(u_r)
        q[..., :3] = np.floor(np.clip(f_r[..., :3] * np.float32(255.0), 0, None)).astype(np.uint32) & 0xff
        q[..., 3] = 255
        res["reftap_vs_refu8"] = cmp(q, u_r)
    for variant in VARIANTS:
        lib().vr_set_variant(variant)
        img = torch.zeros((H, W, 4), dtype=torch.uint8, device=dev)
        fo = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)
        cnt = torch.zeros(5, dtype=torch.int64, device=dev)
        launch_renderer(tree, cam, opt, img, None, None, True, float_out=fo)
        torch.cuda.synchronize()
        f_g, u_g = fo.cpu().numpy(), img.cpu().numpy()
        r = {"vs_oracle_f32": cmp(f_g, f_o), "vs_oracle_u8": cmp(u_g, u_o)}
        if rt:
            r["vs_ref_f32"] = cmp(f_g, f_r)
            r["vs_ref_u8"] = cmp(u_g, u_r)
        launch_renderer(tree, cam, opt, img, None, None, True, counters=cnt)
        torch.cuda.synchronize()
        r["counters"] = cnt.cpu().numpy().tolist()
        res[f"variant{variant}"] = r
    if rt:
        rt.close()
    out[name] = res
    print(name, json.dumps(res)[:3000], flush=True)
    return tree


t0 = time.time()
parity("cfg1", synth.make_config1_tree(), 64, 64, synth.config1_pose())
parity("lego7_sh16", synth.make_tree("lego", depth=7, basis_dim=16), 200, 200, synth.nerf_synthetic_test_poses(8)[3])
parity("lego7_sh9", synth.make_tree("lego", depth=7, basis_dim=9), 160, 120, synth.nerf_synthetic_test_poses(8)[5])
parity("lego6_sh25", synth.make_tree("lego", depth=6, basis_dim=25), 160, 120, synth.nerf_synthetic_test_poses(8)[1])
parity("lego6_sh4", synth.make_tree("lego", depth=6, basis_dim=4), 160, 120, synth.nerf_synthetic_test_poses(8)[2])
parity("lego6_rgba", synth.make_tree("lego", depth=6, fmt="RGBA"), 160, 120, synth.nerf_synthetic_test_poses(8)[6])
parity("lego6_sg9", synth.make_tree("lego", depth=6, basis_dim=9, fmt="SG"), 160, 120, synth.nerf_synthetic_test_poses(8)[7])
print("parity done", time.time() - t0, flush=True)

# ---- timing on the bench-size tree
depth = int(os.environ.get("VR_DEPTH", "10"))
st = synth.make_tree("lego", depth=depth, basis_dim=16)
print("tree", st.capacity, st.nbytes() / 1e6, "MB gen", time.time() - t0, flush=True)
path = "/tmp/lego_bench.npz"
st.save_npz(path)
tree = N3Tree.from_synth(st)
W = H = 800
poses = synth.nerf_synthetic_test_poses(200)
cams = []
for p in poses:
    c = Camera(W, H, synth.focal_for(W), synth.focal_for(W))
    c.set_c2w(p)
    cams.append(c)
opt = RenderOptions()
timing = {"tree_info": tree.info(), "nodes": st.capacity}
imgs = torch.zeros((len(cams), H, W, 4), dtype=torch.uint8, device=dev)
one = torch.zeros((H, W, 4), dtype=torch.uint8, device=dev)
cnt = torch.zeros(5, dtype=torch.int64, device=dev)
render_batch(tree, cams, opt, imgs, counters=cnt)
torch.cuda.synchronize()
cn = cnt.cpu().numpy().tolist()
timing["counters_200"] = cn
A = 4 * cn[1] + 2 * cn[0] + 6 * 16 * cn[2] + 4 * W * H * len(cams)
timing["A_bytes_per_frame"] = A / len(cams)
for variant in VARIANTS:
    lib().vr_set_variant(variant)
    for mode in ("batch",):
        for rep in range(3):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            if mode == "loop":
                for c in cams:
                    launch_renderer(tree, c, opt, one, None, None, True)
            else:
                render_batch(tree, cams, opt, imgs)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1)
        timing[f"v{variant}_{mode}_ms_per_frame"] = ms / len(cams)
        print(f"variant {variant} {mode}: {ms / len(cams):.4f} ms/frame  {W * H * len(cams) / ms / 1e3:.1f} Mrays/s  "
              f"{A / ms / 1e6:.1f} GB/s alg", flush=True)
if rb.available():
    rt = rb.RefTree(path)
    c12 = np.stack([synth.c2w_to_colmajor12(p) for p in poses])
    ropt = rb.make_options()
    for rep in range(3):
        ms = rt.time_frames(W, H, cams[0].fx, cams[0].fy, c12, ropt)
    timing["ref_ms_per_frame"] = ms / len(cams)
    print(f"reference kernel: {ms / len(cams):.4f} ms/frame {W * H * len(cams) / ms / 1e3:.1f} Mrays/s", flush=True)
    rt.close()
out["timing"] = timing
json.dump(out, open("gpurun_out/dev_check.json", "w"), indent=1, default=int)
print("done", time.time() - t0)

# ---- the unchanged reference CLI on both backends (main_headless.cpp)
import subprocess
pdir = "/tmp/lego_poses"
paths = synth.write_pose_files(poses, pdir, cams[0].fx)
root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for exe in ("oracle/_ref/volrend_headless", "oracle/_ref/volrend_headless_ref"):
    full = os.path.join(root, exe)
    if not os.path.exists(full):
        print("missing", exe)
        continue
    try:
        r = subprocess.run([full, path, "-i", os.path.join(pdir, "intrinsics.txt")] + paths, capture_output=True,
                           text=True, timeout=600)
        print(exe, "rc", r.returncode, r.stdout[-400:], r.stderr[-400:], flush=True)
        out.setdefault("cli", {})[exe] = dict(rc=r.returncode, stdout=r.stdout[-400:], stderr=r.stderr[-400:])
    except Exception as e:  # noqa: BLE001
        print(exe, "failed", e)
json.dump(out, open("gpurun_out/dev_check.json", "w"), indent=1, default=int)
