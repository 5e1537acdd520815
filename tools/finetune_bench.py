#!/usr/bin/env python
"""Measures fine-tuning (DESIGN.md section 18) on the bench tree (lego stand-in, depth 10, SH16, seed 0) with the 200
bench poses at 800x800 (config 2):
  * the gradient pass (vr_tree_leaf_grads) in ms per view next to the render (vr_render_batch, float output) of the
    same 200 views, CUDA events, median of --reps after --warmup, the two alternated twice; the gradient time includes
    the zero fill of the gradient buffer, which is also reported alone;
  * vr_tree_update_data (fp16 data already on the device);
  * one fitting step of --batch views (the loop of volrend_b200.finetune), split into render, loss, gradients, Adam
    and update, CUDA events around each part, median over --reps steps after --warmup;
  * device memory: the peak of torch's allocator (buffers, master copy, Adam state), the tree's device bytes and
    the device memory in use at the end (the driver's free memory before and after).

Prints the card name, power limit and max SM clock, then one JSON line; --out also writes the JSON there.  Writes
nothing else."""
import argparse
import json
import os
import statistics
import subprocess
import sys
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--depth", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=8, help="views per fitting step")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    from volrend_b200 import Camera, N3Tree, RenderOptions, leaf_grads, render_batch, synth
    if not torch.cuda.is_available():
        raise SystemExit("finetune_bench needs a CUDA device")
    c = card()
    print("card:", c, flush=True)
    t0 = time.time()
    st = synth.make_tree("lego", depth=args.depth, basis_dim=16, seed=0)
    print(f"tree built in {time.time() - t0:.1f} s: capacity {st.capacity}", flush=True)
    free0 = torch.cuda.mem_get_info()[0]
    f = synth.focal_for(W)
    cams = []
    for p in synth.nerf_synthetic_test_poses(200):
        cam = Camera(W, H, f, f)
        cam.set_c2w(p)
        cams.append(cam)
    opt = RenderOptions()
    tree = N3Tree()
    tree.load_npz(st.npz_dict())
    tree.load_cuda(slot_map=True)
    n = len(cams)
    fo = torch.empty((n, H, W, 4), dtype=torch.float32, device="cuda")
    dpix = torch.empty((n, H, W, 4), dtype=torch.float32, device="cuda").uniform_(-1e-6, 1e-6)
    grad = torch.zeros(st.data.shape, dtype=torch.float32, device="cuda")
    res = dict(card=c, tree=f"lego stand-in depth {args.depth} SH16 seed 0", views=n, size=f"{W}x{H}",
               capacity=st.capacity, data_dim=st.data_dim)

    def grads_pass():
        grad.zero_()
        leaf_grads(tree, cams, opt, dpix, out=grad)

    timing = {"grads": [], "render": [], "zero": []}
    for _ in range(2):
        timing["grads"].append(events_ms(grads_pass, args.warmup, args.reps))
        timing["render"].append(events_ms(lambda: render_batch(tree, cams, opt, None, float_out=fo), args.warmup,
                                          args.reps))
        timing["zero"].append(events_ms(grad.zero_, args.warmup, args.reps))
    res["grad_pass"] = {"ms_per_view_grads": [round(x / n, 4) for x in timing["grads"]],
                        "ms_per_view_render": [round(x / n, 4) for x in timing["render"]],
                        "ms_zero_fill": [round(x, 3) for x in timing["zero"]]}
    print("gradient pass:", json.dumps(res["grad_pass"]), flush=True)

    data16 = torch.from_numpy(st.data).cuda()
    res["update_data_ms"] = round(events_ms(lambda: tree.update_data(data16), args.warmup, args.reps), 3)
    print("update_data ms:", res["update_data_ms"], flush=True)
    del data16

    # one fitting step against renders of the tree itself (the values move, the cost does not depend on them)
    B = args.batch
    targets = fo[:, ..., :3]
    master = torch.tensor(np.asarray(st.data, np.float32), device="cuda").requires_grad_(True)
    adam = torch.optim.Adam([master], lr=1e-3)
    sfo = torch.empty((B, H, W, 4), dtype=torch.float32, device="cuda")
    sd = torch.zeros((B, H, W, 4), dtype=torch.float32, device="cuda")
    parts = {k: [] for k in ("render", "loss", "grads", "optimiser", "update", "step")}
    for it in range(args.warmup + args.reps):
        v0 = (it * B) % (n - B)
        vc, tg = cams[v0:v0 + B], targets[v0:v0 + B]
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
        ev[0].record()
        render_batch(tree, vc, opt, None, float_out=sfo)
        ev[1].record()
        diff = sfo[..., :3] - tg
        loss = diff.square().mean()
        sd[..., :3] = diff * (2.0 / diff.numel())
        ev[2].record()
        grad.zero_()
        leaf_grads(tree, vc, opt, sd, out=grad)
        ev[3].record()
        master.grad = grad
        adam.step()
        ev[4].record()
        tree.update_data(master.detach())
        ev[5].record()
        ev[5].synchronize()
        float(loss)
        if it >= args.warmup:
            for k, (a, b) in zip(("render", "loss", "grads", "optimiser", "update"), zip(ev[:-1], ev[1:])):
                parts[k].append(a.elapsed_time(b))
            parts["step"].append(ev[0].elapsed_time(ev[5]))
    res["fit_step"] = {"views": B, **{f"{k}_ms": round(statistics.median(v), 3) for k, v in parts.items()}}
    print("fitting step:", json.dumps(res["fit_step"]), flush=True)
    torch.cuda.synchronize()
    res["device_bytes_in_use_at_end"] = int(free0 - torch.cuda.mem_get_info()[0])
    res["peak_torch_allocated_bytes"] = int(torch.cuda.max_memory_allocated())
    res["tree_device_bytes"] = int(tree.info()["device_bytes"])
    print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
