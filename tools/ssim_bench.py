#!/usr/bin/env python
"""Measures per-view SSIM (vr_image_ssim, DESIGN.md section 22):
  * forward (value only) and forward + backward (value and dx) on the fitting batch (8 views) and on the config-2 set
    (200 views), 800x800, x RGBA (render_batch's float_out) and y RGB (target_batch), CUDA events, median of --reps
    after --warmup, alternated --rounds times with a torch float32 conv2d restatement of the same definition (autograd
    for its backward);
  * the bytes and FLOPs the kernels need, from the shapes, the HBM and FP32 bounds they give on an H100 SXM data
    sheet (3.35 TB/s, 67 TFLOP/s FP32), and the share of the binding bound that the measured time reaches;
  * one 8-view fitting step (the loop of volrend_b200.finetune) on the bench tree (lego stand-in, depth 10, SH16,
    seed 0) with dssim_weight 0 and 0.2, alternated.

Prints the card name, power limit and SM clocks, then one JSON line; --out also writes the JSON there.  Writes
nothing else."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

W = H = 800
HBM_BPS, FP32_FLOPS = 3.35e12, 67e12
# FLOPs per output pixel and channel (an FMA counts 2): forward, 5 moments x 11 taps x 2 passes, plus the x*f, y*f
# products and the value; backward, the same moments on the tile's halo, the partials, the transposed filter of 3
# fields in 2 passes and the final combination.
FWD_FLOPS = 2 * (5 * 11 * 2) + 22 + 30
BWD_FLOPS = FWD_FLOPS + 40 + 2 * (3 * 11 * 2) + 5


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


def torch_ssim(x, y):
    """The definition in torch float32: per-view SSIM of [V, H, W, 4] x against [V, H, W, 3] y."""
    import torch
    import torch.nn.functional as F
    i = torch.arange(11, dtype=torch.float64, device=x.device)
    f = torch.exp(-0.5 * ((i - 5) / 1.5) ** 2)
    f = (f / f.sum()).float()
    V = x.shape[0]
    xp = x[..., :3].permute(0, 3, 1, 2).reshape(V * 3, 1, H, W)
    yp = y[..., :3].permute(0, 3, 1, 2).reshape(V * 3, 1, H, W)
    flt = lambda a: F.conv2d(F.conv2d(a, f.view(1, 1, 11, 1)), f.view(1, 1, 1, 11))
    mx, my = flt(xp), flt(yp)
    vx, vy = flt(xp * xp) - mx * mx, flt(yp * yp) - my * my
    sxx, syy = torch.where(vx >= 0, vx, 0 * vx), torch.where(vy >= 0, vy, 0 * vy)
    sxy0 = flt(xp * yp) - mx * my
    pr = sxx * syy
    rt = torch.where(pr > 0, torch.sqrt(torch.where(pr > 0, pr, torch.ones_like(pr))), torch.zeros_like(pr))
    sxy = torch.where(sxy0.abs() > rt, torch.sign(sxy0) * rt, sxy0)
    c1, c2 = 0.01 ** 2, 0.03 ** 2
    s = (2 * mx * my + c1) * (2 * sxy + c2) / ((mx * mx + my * my + c1) * (sxx + syy + c2))
    return s.reshape(V, -1).mean(1)


def oom_or(fn):
    """fn() or, when the torch restatement does not fit in device memory, "out of memory"."""
    import torch
    try:
        return fn()
    except torch.cuda.OutOfMemoryError:
        torch.cuda.empty_cache()
        return "out of memory"


def bounds(V, ms, backward):
    n_in, n_out = V * H * W, V * 3 * (H - 10) * (W - 10)
    nbytes = n_in * (16 + 12) * (2 if backward else 1) + (n_in * 16 * 2 if backward else 0)
    flops = n_out * (FWD_FLOPS + (BWD_FLOPS if backward else 0))
    t_hbm, t_fp32 = nbytes / HBM_BPS * 1e3, flops / FP32_FLOPS * 1e3
    bound = "HBM" if t_hbm >= t_fp32 else "FP32"
    return dict(bytes=nbytes, flops=flops, hbm_bound_ms=round(t_hbm, 4), fp32_bound_ms=round(t_fp32, 4),
                bound=bound, share_of_bound=round(max(t_hbm, t_fp32) / ms, 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--depth", type=int, default=10)
    ap.add_argument("--steps", type=int, default=10, help="timed fitting steps per setting and round")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    from volrend_b200 import N3Tree, RenderOptions, image_ssim, leaf_grads, render_batch, synth
    from volrend_b200.views import cameras
    if not torch.cuda.is_available():
        raise SystemExit("ssim_bench needs a CUDA device")
    c = card()
    print("card:", c, flush=True)
    res = dict(card=c, size=f"{W}x{H}", kernels={})
    g = torch.Generator(device="cuda").manual_seed(0)
    for V in (8, 200):
        x = torch.rand((V, H, W, 4), generator=g, device="cuda")
        y = (x[..., :3] + 0.05 * torch.randn((V, H, W, 3), generator=g, device="cuda")).contiguous()
        s = torch.empty(V, dtype=torch.float64, device="cuda")
        dx = torch.zeros_like(x)
        xr = x.clone().requires_grad_(True)

        def t_bwd():
            xr.grad = None
            torch_ssim(xr, y).sum().backward()

        t = {k: [] for k in ("fwd", "fwd_bwd", "torch_fwd", "torch_fwd_bwd")}
        for _ in range(args.rounds):
            t["fwd"].append(events_ms(lambda: image_ssim(x, y, out=s), args.warmup, args.reps))
            with torch.no_grad():
                t["torch_fwd"].append(oom_or(lambda: events_ms(lambda: torch_ssim(x, y), args.warmup, args.reps)))
            t["fwd_bwd"].append(events_ms(lambda: image_ssim(x, y, out=s, dx=dx), args.warmup, args.reps))
            t["torch_fwd_bwd"].append(oom_or(lambda: events_ms(t_bwd, args.warmup, args.reps)))
            xr.grad = None
            torch.cuda.empty_cache()
        # the two paths compute the same thing
        with torch.no_grad():
            st = torch_ssim(x, y).double()
        row = {k: [v if isinstance(v, str) else round(v, 3) for v in vs] for k, vs in t.items()}
        row["max_abs_ssim_vs_torch"] = float((s - st).abs().max())
        row["fwd_bounds"] = bounds(V, statistics.median(t["fwd"]), False)
        row["fwd_bwd_bounds"] = bounds(V, statistics.median(t["fwd_bwd"]), True)
        res["kernels"][f"{V}x{W}x{H}"] = row
        print(f"{V} views:", json.dumps(row), flush=True)
        del x, y, dx, xr
        torch.cuda.empty_cache()

    # one fitting step with and without the D-SSIM term
    st = synth.make_tree("lego", depth=args.depth, basis_dim=16, seed=0)
    f = synth.focal_for(W)
    cams = cameras(synth.nerf_synthetic_test_poses(200), W, H, f, f)
    opt = RenderOptions()
    tree = N3Tree()
    tree.load_npz(st.npz_dict())
    tree.load_cuda(slot_map=True)
    B = 8
    tfo = torch.empty((len(cams), H, W, 4), dtype=torch.float32, device="cuda")
    render_batch(tree, cams, opt, None, float_out=tfo)
    targets = tfo[..., :3].contiguous()
    del tfo
    master = torch.tensor(np.asarray(st.data, np.float32), device="cuda").requires_grad_(True)
    adam = torch.optim.Adam([master], lr=1e-3)
    grad = torch.zeros_like(master)
    fo = torch.empty((B, H, W, 4), dtype=torch.float32, device="cuda")
    dpix = torch.zeros((B, H, W, 4), dtype=torch.float32, device="cuda")

    def steps(lam, n, it0):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for it in range(it0, it0 + n):
            v0 = (it * B) % (len(cams) - B)
            vc, tg = cams[v0:v0 + B], targets[v0:v0 + B]
            render_batch(tree, vc, opt, None, float_out=fo)
            diff = fo[..., :3] - tg
            loss = diff.square().mean()
            dpix[..., :3] = diff * (2.0 / diff.numel())
            if lam > 0:
                image_ssim(fo, tg, dx=dpix, dx_scale=-lam / B)
            grad.zero_()
            leaf_grads(tree, vc, opt, dpix, out=grad)
            master.grad = grad
            adam.step()
            tree.update_data(master.detach())
            float(loss)
        b.record()
        b.synchronize()
        return a.elapsed_time(b) / n

    fit = {"dssim_0": [], "dssim_0.2": []}
    steps(0.0, args.warmup, 0)
    steps(0.2, args.warmup, 0)
    for r in range(args.rounds):
        fit["dssim_0"].append(round(steps(0.0, args.steps, 100 * r), 3))
        fit["dssim_0.2"].append(round(steps(0.2, args.steps, 100 * r), 3))
    res["fit_step_ms"] = {"views": B, "tree": f"lego stand-in depth {args.depth} SH16 seed 0", **fit}
    print("fitting step ms:", json.dumps(res["fit_step_ms"]), flush=True)
    print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
