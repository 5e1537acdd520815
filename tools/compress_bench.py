#!/usr/bin/env python
"""Times the tree compressor (DESIGN.md section 12) on the bench tree (lego stand-in, depth 10, SH16, seed 0).

For the default flags (--bits 16 --sigma_thresh 2.0 --retain 1) and for --retain 4:
  * CUDA events, median of --reps runs after --warmup: upload (host -> device copy of `data`), the vr_tree_compress
    call, download (the four outputs);
  * kernel time per stage -- gather (kept slots, compaction, point sets), median cut (and the sort inside it), finish
    (means + map) -- from a torch.profiler trace of one more call;
  * host time to assemble the dict, deflate and write it (np.savez_compressed), median of --host-reps runs;
  * input file size (np.savez, as training writes it) and compressed size.
Also: the numpy restatement of the contract (oracle/quant_oracle.py, not svox) timed on one point set of the same
tree and checked equal to the device output for that set, and the PSNR of --views views rendered at 800x800 from the
compressed tree against the original (the stand-in's colours are random, so this says little about real scenes).

Prints the card name and power limit, then one JSON line.  Writes only to a temporary directory."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        return f"unknown ({e})"


def run_once(flat, dd, retain, bits, thresh):
    """CUDA events around the upload, the vr_tree_compress call and the download."""
    import torch
    from volrend_b200.compress import compress_device
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    ev[0].record()
    d = torch.from_numpy(flat.view(np.int16)).to("cuda")
    ev[1].record()
    outs, kept = compress_device(d, dd, thresh, retain, bits)
    ev[2].record()
    host = [None if t is None else t.cpu().numpy().view(np.uint16) for t in outs]
    ev[3].record()
    ev[3].synchronize()
    ms = dict(upload=ev[0].elapsed_time(ev[1]), compress_call=ev[1].elapsed_time(ev[2]),
              download=ev[2].elapsed_time(ev[3]))
    del d, outs
    return ms, host, kept


def stage_kernel_ms(flat, dd, retain, bits, thresh, tmp):
    """Kernel time per stage of one vr_tree_compress call, from a torch.profiler trace of a run of its own: kernels up
    to gather_kernel are the gather stage, finish_points_kernel / codebook_kernel the finish, everything between the
    median cut (of which the sort kernels and their digit scans are reported apart)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from volrend_b200.compress import compress_device
    d = torch.from_numpy(flat.view(np.int16)).to("cuda")
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        outs, _ = compress_device(d, dd, thresh, retain, bits)
        torch.cuda.synchronize()
    path = os.path.join(tmp, "trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        ev = json.load(f)
    ev = sorted((e for e in (ev["traceEvents"] if isinstance(ev, dict) else ev) if e.get("cat") == "kernel"),
                key=lambda e: float(e["ts"]))
    out, stage = dict(gather=0.0, median_cut=0.0, finish=0.0), "gather"
    sort_ms = 0.0
    for e in ev:
        name = e["name"]
        if "finish_points_kernel" in name or "codebook_kernel" in name:
            stage = "finish"
        out[stage] += float(e["dur"]) / 1e3
        if stage == "median_cut" and ("sort_kernel" in name or "digit_" in name or "DeviceScan" in name):
            sort_ms += float(e["dur"]) / 1e3
        if "gather_kernel" in name:
            stage = "median_cut"
    out["median_cut_sort"] = sort_ms
    del d, outs
    return {k: round(v, 3) for k, v in out.items()}


def psnr(a, b):
    mse = float(np.mean((np.clip(a, 0, 1).astype(np.float64) - np.clip(b, 0, 1)) ** 2))
    return float("inf") if mse == 0 else float(-10.0 * np.log10(mse))


def render_views(tree, views):
    import torch
    from volrend_b200 import Camera, RenderOptions, launch_renderer, synth
    poses = synth.nerf_synthetic_test_poses(200)
    out = []
    for i in views:
        cam = Camera(800, 800, synth.focal_for(800), synth.focal_for(800))
        cam.set_c2w(poses[i])
        img = torch.zeros((800, 800, 4), dtype=torch.uint8, device="cuda")
        fo = torch.zeros((800, 800, 4), dtype=torch.float32, device="cuda")
        launch_renderer(tree, cam, RenderOptions(), img, None, None, True, float_out=fo)
        torch.cuda.synchronize()
        out.append(fo.cpu().numpy()[..., :3])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--depth", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--host-reps", type=int, default=2)
    ap.add_argument("--views", type=int, nargs="*", default=[0, 50, 100])
    args = ap.parse_args()
    import torch
    import compress_cases as cc
    from oracle import quant_oracle as qo
    from volrend_b200 import N3Tree, compress_npz, synth
    from volrend_b200.compress import _write_npz
    c = card()
    print("card:", c, flush=True)
    torch.cuda.init()
    st = synth.make_tree("lego", depth=args.depth, basis_dim=16, seed=0)
    z = cc.tree_dict(st)
    dd = st.data_dim
    flat = np.ascontiguousarray(st.data).view(np.uint16).reshape(-1, dd)
    res = dict(card=c, tree=f"lego stand-in depth {args.depth} SH16 seed 0", n_child=int(flat.shape[0]), configs=[])
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, "tree.npz")
        np.savez(src, **z)
        in_mb = os.path.getsize(src) / 2 ** 20
        for retain in (1, 4):
            for _ in range(args.warmup):
                run_once(flat, dd, retain, 16, 2.0)
            runs = [run_once(flat, dd, retain, 16, 2.0) for _ in range(args.reps)]
            host, kept = runs[-1][1], runs[-1][2]
            med = {k: round(statistics.median(r[0][k] for r in runs), 3) for k in runs[0][0]}
            kernels = stage_kernel_ms(flat, dd, retain, 16, 2.0, tmp)
            out = os.path.join(tmp, f"tree_r{retain}.npz")
            hs = []
            for _ in range(args.host_reps):
                t0 = time.perf_counter()
                d = compress_npz(z, retain=retain, backend=lambda *a, _h=host, _k=kept: (*_h, _k))
                _write_npz(out, d)
                hs.append(time.perf_counter() - t0)
            row = dict(retain=retain, bits=16, sigma_thresh=2.0, n_kept=kept, device_ms=med, kernel_ms=kernels,
                       host_deflate_write_s=round(statistics.median(hs), 3), in_MB=round(in_mb, 2),
                       out_MB=round(os.path.getsize(out) / 2 ** 20, 2))
            print(f"retain {retain}: {json.dumps(row)}", flush=True)
            res["configs"].append(row)
            if retain == 1:
                # one point set through the numpy restatement, checked against the device output for that set
                B, j = (dd - 1) // 3, (dd - 1) // 3 - 1
                keep = qo.kept_mask(flat[:, -1], 2.0)
                kd = flat[keep]
                t0 = time.perf_counter()
                oc, ob = qo.median_cut(kd[:, j], kd[:, B + j], kd[:, 2 * B + j], 16)
                o_s = time.perf_counter() - t0
                q = j - retain
                eq = bool(np.array_equal(oc, host[0][q]) and np.array_equal(ob, host[1][q][keep]))
                res["oracle_one_set"] = dict(label="numpy restatement of the contract (oracle/quant_oracle.py), not svox",
                                             points=int(kd.shape[0]), seconds=round(o_s, 2), gpu_equal=eq)
                print("oracle:", json.dumps(res["oracle_one_set"]), flush=True)
                assert eq, "device output differs from the oracle on the checked set"
            orig = N3Tree.from_synth(st)
            ref = render_views(orig, args.views)
            orig.free_cuda()
            comp = N3Tree(out)
            got = render_views(comp, args.views)
            comp.free_cuda()
            row["psnr_db"] = [round(psnr(a, b), 2) for a, b in zip(got, ref)]
            print(f"retain {retain} PSNR vs original (views {args.views}): {row['psnr_db']}", flush=True)
            torch.cuda.empty_cache()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
