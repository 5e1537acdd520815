#!/usr/bin/env python
"""Measures refinement (DESIGN.md section 19) on the bench tree (lego stand-in, depth 10, SH16, seed 0) with the 200
bench poses at 800x800 (config 2):
  * the error pass (vr_tree_leaf_error) in ms per view next to the render (vr_render_batch, float output) of the same
    200 views, CUDA events, median of --reps after --warmup, the two alternated twice; the error is a seeded uniform
    value in (0, 1] per pixel (the cost does not depend on it: every ray is marched);
  * per --fractions value, on the scores of that pass: the host time of refine_plan and of the gather of the data,
    the host time of the re-upload (vr_tree_create with the slot map, ending in a device synchronise), and nodes and
    device_bytes before and after;
  * config-2 Mrays/s of the tree refined with --render-fraction against the original, alternated twice;
  * one fitting step of --batch views on that refined tree (render, loss, gradients, Adam, update), median over
    --reps steps after --warmup.

Prints the card name, power limit and max SM clock, then one JSON line; --out also writes the JSON there.  Writes
nothing else."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from finetune_bench import H, W, card, events_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--depth", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=8, help="views per fitting step")
    ap.add_argument("--fractions", default="0.01,0.1,0.3")
    ap.add_argument("--render-fraction", type=float, default=0.1)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    from volrend_b200 import Camera, N3Tree, RenderOptions, leaf_error, leaf_grads, refine_plan, render_batch, synth
    if not torch.cuda.is_available():
        raise SystemExit("refine_bench needs a CUDA device")
    c = card()
    print("card:", c, flush=True)
    st = synth.make_tree("lego", depth=args.depth, basis_dim=16, seed=0)
    f = synth.focal_for(W)
    cams = []
    for p in synth.nerf_synthetic_test_poses(200):
        cam = Camera(W, H, f, f)
        cam.set_c2w(p)
        cams.append(cam)
    n = len(cams)
    opt = RenderOptions()

    def load(child, data):
        t = N3Tree()
        t.load_npz(dict(st.npz_dict(), child=child, data=data))
        t0 = time.perf_counter()
        t.load_cuda(slot_map=True)
        torch.cuda.synchronize()
        return t, (time.perf_counter() - t0) * 1e3

    tree, _ = load(st.child, st.data)
    fo = torch.empty((n, H, W, 4), dtype=torch.float32, device="cuda")
    err = torch.empty((n, H, W), dtype=torch.float32, device="cuda").uniform_(1e-3, 1.0)
    score = torch.zeros(st.capacity * 8, dtype=torch.float32, device="cuda")
    res = dict(card=c, tree=f"lego stand-in depth {args.depth} SH16 seed 0", views=n, size=f"{W}x{H}",
               capacity=st.capacity)

    def error_pass():
        score.zero_()
        leaf_error(tree, cams, opt, err, out=score)

    timing = {"error": [], "render": []}
    for _ in range(2):
        timing["error"].append(events_ms(error_pass, args.warmup, args.reps))
        timing["render"].append(events_ms(lambda: render_batch(tree, cams, opt, None, float_out=fo), args.warmup,
                                          args.reps))
    res["error_pass"] = {"ms_per_view_error": [round(x / n, 4) for x in timing["error"]],
                         "ms_per_view_render": [round(x / n, 4) for x in timing["render"]]}
    print("error pass:", json.dumps(res["error_pass"]), flush=True)

    error_pass()
    scores = score.cpu().numpy()
    res["leaves_with_positive_score"] = int((scores > 0).sum())
    dd = st.data_dim
    res["refine"] = []
    for frac in [float(x) for x in args.fractions.split(",")]:
        t0 = time.perf_counter()
        child, src = refine_plan(st.child, scores, frac)
        t1 = time.perf_counter()
        data = st.data.reshape(-1, dd)[src].reshape(-1, 2, 2, 2, dd)
        t2 = time.perf_counter()
        t, upload_ms = load(child, data)
        r = dict(fraction=frac, nodes_before=st.capacity, nodes_after=int(child.shape[0]),
                 device_bytes_before=int(tree.info()["device_bytes"]), device_bytes_after=int(t.info()["device_bytes"]),
                 refine_plan_ms=round((t1 - t0) * 1e3, 1), gather_ms=round((t2 - t1) * 1e3, 1),
                 upload_ms=round(upload_ms, 1))
        t.free_cuda()
        res["refine"].append(r)
        print("refine:", json.dumps(r), flush=True)
    child, src = refine_plan(st.child, scores, args.render_fraction)
    refined, _ = load(child, st.data.reshape(-1, dd)[src].reshape(-1, 2, 2, 2, dd))
    res["render_fraction"] = args.render_fraction

    rates = {"original": [], "refined": []}
    for _ in range(2):
        for k, t in (("original", tree), ("refined", refined)):
            ms = events_ms(lambda: render_batch(t, cams, opt, None, float_out=fo), args.warmup, args.reps)
            rates[k].append(round(n * W * H / ms / 1e3, 1))
    res["config2_mrays_per_s"] = rates
    print("config 2 Mrays/s:", json.dumps(rates), flush=True)
    tree.free_cuda()

    B = args.batch
    render_batch(refined, cams, opt, None, float_out=fo)
    targets = fo[..., :3].clone()
    cap = refined.capacity
    master = torch.tensor(np.asarray(refined.data_, np.float32), device="cuda").requires_grad_(True)
    grad = torch.zeros_like(master)
    adam = torch.optim.Adam([master], lr=1e-3)
    sfo = torch.empty((B, H, W, 4), dtype=torch.float32, device="cuda")
    sd = torch.zeros((B, H, W, 4), dtype=torch.float32, device="cuda")
    steps = []
    for it in range(args.warmup + args.reps):
        v0 = (it * B) % (n - B)
        vc, tg = cams[v0:v0 + B], targets[v0:v0 + B]
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        render_batch(refined, vc, opt, None, float_out=sfo)
        diff = sfo[..., :3] - tg
        sd[..., :3] = diff * (2.0 / diff.numel())
        grad.zero_()
        leaf_grads(refined, vc, opt, sd, out=grad)
        master.grad = grad
        adam.step()
        refined.update_data(master.detach())
        b.record()
        b.synchronize()
        if it >= args.warmup:
            steps.append(a.elapsed_time(b))
    res["fit_step_refined"] = {"views": B, "capacity": cap, "step_ms": round(statistics.median(steps), 3)}
    print("fitting step on the refined tree:", json.dumps(res["fit_step_refined"]), flush=True)
    print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
