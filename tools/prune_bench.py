#!/usr/bin/env python
"""Measures pruning by ray weight (DESIGN.md section 17) on the bench tree (lego stand-in, depth 10, SH16, seed 0).

Weights from the 200 bench poses at 800x800 (config 2), then, at thresholds 0, 1e-3 and 1e-2, with and without
collapse:
  * leaves and nodes before and after, device_bytes of the loaded tree;
  * config-2 Mrays/s of the pruned tree against the original (vr_render_batch of the 200 views, CUDA events, median
    of --reps after --warmup, trees alternated);
  * PSNR of the pruned tree's renders against the original's on --psnr-views poses NOT used for the weights (the
    orbit shifted by half a step);
  * compressed file size (compress_npz defaults + deflate) with and without pruning.
Also the weights pass itself: ms per view next to the render ms per view of the same batch, alternated.

Prints the card name, power limit and max SM clock, then one JSON line; --out also writes the JSON there.  Writes
nothing else but temporary files."""
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

W = H = 800


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        return f"unknown ({e})"


def events_ms(fn, warmup, reps):
    import torch
    for _ in range(warmup):
        fn()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return statistics.median(out)


def psnr(a, b):
    mse = float(np.mean((np.clip(a, 0, 1).astype(np.float64) - np.clip(b, 0, 1)) ** 2))
    return float("inf") if mse == 0 else float(-10.0 * np.log10(mse))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--depth", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--psnr-views", type=int, default=8)
    ap.add_argument("--no-sizes", action="store_true", help="skip the compressed file sizes")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    from volrend_b200 import N3Tree, RenderOptions, compress_npz, leaf_weights, prune_npz, render_batch, synth
    from volrend_b200.compress import _write_npz
    from volrend_b200.views import cameras
    c = card()
    print("card:", c, flush=True)
    t0 = time.time()
    st = synth.make_tree("lego", depth=args.depth, basis_dim=16, seed=0)
    z = st.npz_dict()
    print(f"tree built in {time.time() - t0:.1f} s: capacity {st.capacity}", flush=True)
    f = synth.focal_for(W)
    cams = cameras(synth.nerf_synthetic_test_poses(200), W, H, f, f)
    held = cameras(synth.nerf_synthetic_test_poses(400)[1::2][:: max(1, 200 // args.psnr_views)][:args.psnr_views],
                   W, H, f, f)
    opt = RenderOptions()
    imgs = torch.empty((200, H, W, 4), dtype=torch.uint8, device="cuda")

    tree = N3Tree()
    tree.load_npz(z)
    tree.load_cuda(slot_map=True)
    info0 = tree.info()
    wbuf = torch.empty((st.capacity, 2, 2, 2), dtype=torch.float32, device="cuda")

    def weights_pass():
        wbuf.fill_(float("-inf"))
        leaf_weights(tree, cams, opt, out=wbuf)

    def fill_only():
        wbuf.fill_(float("-inf"))

    res = dict(card=c, tree=f"lego stand-in depth {args.depth} SH16 seed 0", views=200, size=f"{W}x{H}",
               capacity=st.capacity, device_bytes_with_slot_map=info0["device_bytes"])
    # the weights pass next to the render of the same batch, alternated
    timing = {"weights": [], "render": [], "fill": []}
    for _ in range(2):
        timing["weights"].append(events_ms(weights_pass, args.warmup, args.reps))
        timing["render"].append(events_ms(lambda: render_batch(tree, cams, opt, imgs), args.warmup, args.reps))
        timing["fill"].append(events_ms(fill_only, args.warmup, args.reps))
    weights_pass()
    weights = wbuf.cpu().numpy().reshape(-1).copy()
    res["weights_pass"] = {
        "ms_per_view_weights": [round(x / 200, 4) for x in timing["weights"]],
        "ms_per_view_render": [round(x / 200, 4) for x in timing["render"]],
        "ms_fill_minus_inf": [round(x, 3) for x in timing["fill"]],
        "note": "each weights time includes the -inf fill of the buffer (ms_fill_minus_inf, whole buffer)"}
    print("weights pass:", json.dumps(res["weights_pass"]), flush=True)
    leaf = z["child"].reshape(-1) == 0

    def render_ms(t):
        return events_ms(lambda: render_batch(t, cams, opt, imgs), args.warmup, args.reps)

    def held_frames(t):
        out = []
        for cam in held:
            fo = torch.zeros((1, H, W, 4), dtype=torch.float32, device="cuda")
            render_batch(t, [cam], opt, None, float_out=fo)
            torch.cuda.synchronize()
            out.append(fo.cpu().numpy()[0, ..., :3])
        return out

    ref_frames = held_frames(tree)
    tree.free_cuda()
    base = N3Tree()
    base.load_npz(z)
    base.load_cuda()
    info_base = base.info()
    sizes = {}
    with tempfile.TemporaryDirectory() as tmp:
        if not args.no_sizes:
            p = os.path.join(tmp, "orig.npz")
            _write_npz(p, compress_npz(z))
            sizes["original"] = os.path.getsize(p)
        res["original"] = dict(leaves=int(leaf.sum()), nodes=int(st.capacity), device_bytes=info_base["device_bytes"],
                               compressed_MB=round(sizes.get("original", 0) / 2 ** 20, 2))
        res["configs"] = []
        for thresh in (0.0, 1e-3, 1e-2):
            for collapse in (False, True):
                t1 = time.time()
                pz = prune_npz(z, weights, thresh, collapse)
                prune_s = time.time() - t1
                pt = N3Tree()
                pt.load_npz(pz)
                pt.load_cuda()
                ms_o, ms_p = [], []
                for _ in range(2):          # alternated
                    ms_o.append(render_ms(base))
                    ms_p.append(render_ms(pt))
                frames = held_frames(pt)
                row = dict(thresh=thresh, collapse=collapse, prune_host_s=round(prune_s, 2),
                           leaves_kept=int((leaf & (weights >= thresh)).sum()),
                           leaves_after=int((pz["child"].reshape(-1) == 0).sum()), nodes_after=int(pz["child"].shape[0]),
                           device_bytes=pt.info()["device_bytes"],
                           mrays_original=[round(W * H * 200 / m / 1e3, 1) for m in ms_o],
                           mrays_pruned=[round(W * H * 200 / m / 1e3, 1) for m in ms_p],
                           psnr_db_held_out=[round(psnr(a, b), 2) for a, b in zip(frames, ref_frames)])
                pt.free_cuda()
                if not args.no_sizes:
                    p = os.path.join(tmp, "pruned.npz")
                    _write_npz(p, compress_npz(pz))
                    row["compressed_MB"] = round(os.path.getsize(p) / 2 ** 20, 2)
                print(json.dumps(row), flush=True)
                res["configs"].append(row)
                del pz
                torch.cuda.empty_cache()
    base.free_cuda()
    res["card_after"] = card()
    line = json.dumps(res)
    print(line, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
