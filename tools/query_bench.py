#!/usr/bin/env python
"""Throughput of the point queries (vr_tree_query, vr_tree_eval) against the reference's query_single_from_root
(oracle/_ref/libref_query.so, one thread per point), on the bench tree (depth-10 SH16) and config 4's depth-11 SH25
tree.  Prints one JSON line with the card name and power limit.  Needs a GPU; writes only to a temporary directory.

  python tools/query_bench.py [--reps 10] [--no-ref]

Rates are points per second of kernel time (CUDA events over --reps launches after a warm-up).  "compulsory" counts
the bytes every point must move through DRAM whatever the tree: its 12-byte input and its outputs (query: the data
row, cube_sz and local; eval: the direction, rgb and sigma).  Table words and colour records are left out: points of a
grid share leaves, so those reads mostly hit in L2, and counting one record per point would exceed the bandwidth the
card has.  Divided by kernel time, the compulsory bytes are compared with the 3.35 TB/s of the H100 SXM data sheet."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

PEAK_BPS = 3.35e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        return f"unknown ({e})"


def points(tree, kind, n_side, seed=0):
    """World points on the GPU: a raster-order grid of cell centres (z fastest) or uniform random ones."""
    import torch
    if kind == "grid":
        g = (torch.arange(n_side, device="cuda", dtype=torch.float64) + 0.5) / n_side
        t = torch.stack(torch.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    else:
        gen = torch.Generator(device="cuda").manual_seed(seed)
        t = torch.rand((n_side, 3), device="cuda", dtype=torch.float64, generator=gen)
    off = torch.tensor(tree.offset, dtype=torch.float64, device="cuda")
    sc = torch.tensor(tree.scale, dtype=torch.float64, device="cuda")
    return ((t - off) / sc).float().contiguous()


def time_call(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def measure(tree, x, reps, ref_tree=None):
    import torch
    from volrend_b200 import RenderOptions, lib
    from volrend_b200._capi import check
    n = x.shape[0]
    dd = tree.data_dim
    data = torch.empty((n, dd), dtype=torch.float16, device="cuda")
    cube = torch.empty(n, device="cuda")
    local = torch.empty((n, 3), device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    q_ms = time_call(lambda: check(lib().vr_tree_query(tree._handle, x.data_ptr(), n, data.data_ptr(), cube.data_ptr(),
                                                        local.data_ptr(), s)), reps)
    d = torch.nn.functional.normalize(torch.randn((n, 3), device="cuda"), dim=1)
    rgb = torch.empty((n, 3), device="cuda")
    sig = torch.empty(n, device="cuda")
    o = RenderOptions()._as_c()
    e_ms = time_call(lambda: check(lib().vr_tree_eval(tree._handle, x.data_ptr(), d.data_ptr(), n, C.byref(o),
                                                       rgb.data_ptr(), sig.data_ptr(), s)), reps)
    q_bytes = n * (12 + 2 * dd + 4 + 12)
    e_bytes = n * (24 + 12 + 4)
    out = dict(points=n, query_ms=round(q_ms, 3), query_pts_per_s=n / q_ms * 1e3,
               query_compulsory_GBps=q_bytes / q_ms / 1e6, query_share_of_3_35TBps=q_bytes / q_ms * 1e3 / PEAK_BPS,
               eval_ms=round(e_ms, 3), eval_pts_per_s=n / e_ms * 1e3, eval_compulsory_GBps=e_bytes / e_ms / 1e6,
               eval_share_of_3_35TBps=e_bytes / e_ms * 1e3 / PEAK_BPS)
    if ref_tree is not None:
        # outputs past 2 GB are timed without the host copy of the reference's results (and not compared)
        compare = n * (2 * dd + 16) <= (2 << 30)
        rd, rc, rl, r_ms = ref_tree.query(x.cpu().numpy(), reps=reps, outputs=compare)
        out.update(ref_ms=round(r_ms, 3), ref_pts_per_s=n / r_ms * 1e3, speedup_vs_ref=r_ms / q_ms)
        if compare:
            out["identical_to_ref"] = bool(np.array_equal(rd.view(np.uint16), data.cpu().numpy().view(np.uint16))
                                           and np.array_equal(rc, cube.cpu().numpy())
                                           and np.array_equal(rl.view(np.uint32), local.cpu().numpy().view(np.uint32)))
    del data, cube, local, rgb, sig, d
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--no-ref", action="store_true", help="skip the reference kernel")
    args = ap.parse_args()
    import torch
    from oracle import ref_query
    from volrend_b200 import N3Tree, synth
    assert torch.cuda.is_available(), "query_bench needs a CUDA device"
    use_ref = ref_query.available() and not args.no_ref
    res = dict(card=card(), reps=args.reps, workloads={})
    trees = [("bench_sh16_d10", lambda: synth.make_tree("lego", depth=10, basis_dim=16, seed=0),
              [("grid256", "grid", 256, True), ("grid512", "grid", 512, True), ("uniform16.7M", "uniform", 1 << 24, True)]),
             ("config4_sh25_d11", lambda: synth.make_tree("gyroid_small", depth=11, basis_dim=25, seed=0, band_cells=1.0),
              [("grid256", "grid", 256, True)])]
    with tempfile.TemporaryDirectory() as tmp:
        for tname, make, loads in trees:
            st = make()
            tree = N3Tree.from_synth(st)
            rt = None
            if use_ref:
                path = os.path.join(tmp, tname + ".npz")
                st.save_npz(path)
                rt = ref_query.RefQueryTree(path)
            del st
            for wname, kind, size, with_ref in loads:
                x = points(tree, kind, size)
                res["workloads"][f"{tname}/{wname}"] = measure(tree, x, args.reps, rt if with_ref else None)
                del x
                torch.cuda.empty_cache()
                print(tname, wname, res["workloads"][f"{tname}/{wname}"], file=sys.stderr, flush=True)
            if rt is not None:
                rt.close()
            tree.free_cuda()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
