#!/usr/bin/env python
"""Measures the total-variation prior (DESIGN.md section 20) on the bench tree (lego stand-in, depth 10, SH16, seed 0)
with the 200 bench poses at 800x800:
  * the neighbour build (vr_tree_leaf_neighbors): the first call of a tree (host time, it also counts the tree's cells
    and synchronises) and later calls (CUDA events), at creation and after splitting --fraction of the leaves that
    the error pass scores (refine_plan);
  * one leaf_tv call (both weights > 0, the fp32 master of the tree's data), its bytes computed from the shapes and
    the bandwidth that gives against the H100's 3.35 TB/s;
  * one fitting step of --batch views (render, loss, gradients, [TV,] Adam, update) without and with TV, the two
    alternated step by step in one run.
Times are medians of --reps after --warmup.  Prints the card name, power limit and max SM clock, then one JSON line;
--out also writes the JSON there.  Writes nothing else."""
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

HBM_TBS = 3.35


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--depth", type=int, default=10)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=8, help="views per fitting step")
    ap.add_argument("--fraction", type=float, default=0.1)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    from volrend_b200 import (Camera, N3Tree, RenderOptions, leaf_error, leaf_grads, leaf_neighbors, leaf_tv,
                              refine_plan, render_batch, synth)
    if not torch.cuda.is_available():
        raise SystemExit("tv_bench needs a CUDA device")
    c = card()
    print("card:", c, flush=True)
    st = synth.make_tree("lego", depth=args.depth, basis_dim=16, seed=0)
    f = synth.focal_for(W)
    cams = []
    for p in synth.nerf_synthetic_test_poses(200):
        cam = Camera(W, H, f, f)
        cam.set_c2w(p)
        cams.append(cam)
    opt = RenderOptions()
    dd = st.data_dim

    def load(child, data):
        t = N3Tree()
        t.load_npz(dict(st.npz_dict(), child=child, data=data))
        t.load_cuda(slot_map=True)
        return t

    def neighbours(t):
        nbr = torch.empty((t.capacity * 8, 3), dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        leaf_neighbors(t, out=nbr)
        torch.cuda.synchronize()
        first = (time.perf_counter() - t0) * 1e3
        later = events_ms(lambda: leaf_neighbors(t, out=nbr), args.warmup, args.reps)
        return nbr, dict(nodes=t.capacity, table_bytes=t.capacity * 8 * 3 * 4, first_call_ms=round(first, 2),
                         call_ms=round(later, 3), leaves=int((nbr >= 0).any(1).sum().item()) + 1)

    tree = load(st.child, st.data)
    res = dict(card=c, tree=f"lego stand-in depth {args.depth} SH16 seed 0", views=len(cams), size=f"{W}x{H}")
    nbr, res["neighbors_created"] = neighbours(tree)
    print("neighbours at creation:", json.dumps(res["neighbors_created"]), flush=True)

    score = torch.zeros(st.capacity * 8, dtype=torch.float32, device="cuda")
    err = torch.empty((len(cams), H, W), dtype=torch.float32, device="cuda").uniform_(1e-3, 1.0)
    leaf_error(tree, cams, opt, err, out=score)
    child, src = refine_plan(st.child, score.cpu().numpy(), args.fraction)
    del err, score
    refined = load(child, st.data.reshape(-1, dd)[src].reshape(-1, 2, 2, 2, dd))
    rnbr, r = neighbours(refined)
    res["neighbors_refined"] = dict(r, fraction=args.fraction)
    print("neighbours after refinement:", json.dumps(res["neighbors_refined"]), flush=True)
    del rnbr
    refined.free_cuda()
    del refined

    master = torch.tensor(np.asarray(tree.data_, np.float32), device="cuda").requires_grad_(True)
    grad = torch.zeros_like(master)
    energy = torch.zeros(1, dtype=torch.float64, device="cuda")
    ls, lc_ = 1e-2, 1e-3
    tv_ms = events_ms(lambda: leaf_tv(tree, nbr, master.detach(), ls, lc_, out=grad, energy=energy), args.warmup,
                      args.reps)
    n_slots, n_cols = tree.capacity * 8, 3 * 16 + 1
    # the table once, each listed value of the master read once, each gradient value read and written once
    nbytes = n_slots * 12 + n_slots * n_cols * (4 + 8)
    res["leaf_tv"] = dict(ms=round(tv_ms, 3), columns=n_cols, bytes=nbytes,
                          tb_per_s=round(nbytes / tv_ms / 1e9, 3), of_hbm=round(nbytes / tv_ms / 1e9 / HBM_TBS, 3))
    print("leaf_tv:", json.dumps(res["leaf_tv"]), flush=True)

    B = args.batch
    fo = torch.empty((len(cams), H, W, 4), dtype=torch.float32, device="cuda")
    render_batch(tree, cams, opt, None, float_out=fo)
    targets = fo[..., :3].clone()
    del fo
    adam = torch.optim.Adam([master], lr=1e-3)
    sfo = torch.empty((B, H, W, 4), dtype=torch.float32, device="cuda")
    sd = torch.zeros((B, H, W, 4), dtype=torch.float32, device="cuda")
    steps = {"plain": [], "tv": []}
    for it in range(args.warmup + args.reps):
        for key in ("plain", "tv"):
            v0 = (it * B) % (len(cams) - B)
            vc, tg = cams[v0:v0 + B], targets[v0:v0 + B]
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            render_batch(tree, vc, opt, None, float_out=sfo)
            diff = sfo[..., :3] - tg
            sd[..., :3] = diff * (2.0 / diff.numel())
            grad.zero_()
            leaf_grads(tree, vc, opt, sd, out=grad)
            if key == "tv":
                leaf_tv(tree, nbr, master.detach(), ls, lc_, out=grad, energy=energy)
            master.grad = grad
            adam.step()
            tree.update_data(master.detach())
            b.record()
            b.synchronize()
            if it >= args.warmup:
                steps[key].append(a.elapsed_time(b))
    res["fit_step"] = {"views": B, "plain_ms": round(statistics.median(steps["plain"]), 3),
                       "tv_ms": round(statistics.median(steps["tv"]), 3)}
    print("fitting step:", json.dumps(res["fit_step"]), flush=True)
    print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
