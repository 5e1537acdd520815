"""Time tree construction from voxel cells: the GPU build (``build_arrays``: the count call and the fill call, as a
user runs it) against the host oracle (``oracle/build_oracle.py``), on three inputs:

  bench     the leaves of the bench tree (lego stand-in, depth 10, SH16): a multi-resolution cell list
  dense256  a dense 256^3 SH9 grid (every cell listed, random rows)
  shell512  a sigma-sparse 512^3 SH9 grid: the cells of the ``shell`` SDF band (|sdf| < 2 cells) at level 9

GPU times are CUDA-event medians after warm-ups; peak device memory is the high-water mark of the stream-ordered pool
the build's scratch comes from, plus the output tensors.  The oracle runs once per input (it takes seconds to minutes);
inputs above --oracle-max-cells are not run on it.  Prints one JSON line per input and writes them to --out.

    python tools/build_bench.py [--reps 5] [--warmup 2] [--oracle-max-cells 20000000] [--out build.json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def _pool():
    import torch
    cu = C.CDLL("libcuda.so.1")
    dev, pool = C.c_int(), C.c_void_p()
    assert cu.cuDeviceGet(C.byref(dev), torch.cuda.current_device()) == 0
    assert cu.cuDeviceGetDefaultMemPool(C.byref(pool), dev) == 0
    return cu, pool


def _pool_high(reset=False) -> int:
    cu, pool = _pool()
    v = C.c_uint64(0)
    if reset:
        assert cu.cuMemPoolSetAttribute(pool, 8, C.byref(v)) == 0         # CU_MEMPOOL_ATTR_USED_MEM_HIGH
        return 0
    assert cu.cuMemPoolGetAttribute(pool, 8, C.byref(v)) == 0
    return v.value


def inputs():
    import torch
    from volrend_b200 import grid_cells, leaf_cells, synth
    st = synth.make_tree("lego", depth=10, basis_dim=16, seed=0)
    c, r = leaf_cells(st.child, st.data)
    yield "bench", torch.from_numpy(c).cuda(), torch.from_numpy(r).cuda()
    g = torch.randn((256, 256, 256, 28), dtype=torch.float16, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    c, r = grid_cells(g)
    del g
    yield "dense256", c, r
    R = 512
    i = torch.arange(R, device="cuda", dtype=torch.float32)
    ctr = (i + 0.5) / R
    keep = []
    for x in range(R):                                   # one x slab at a time: the band of the sphere r = 0.325
        d = torch.sqrt((ctr[x] - 0.5) ** 2 + (ctr[:, None] - 0.5) ** 2 + (ctr[None, :] - 0.5) ** 2) - 0.325
        yz = torch.nonzero(d.abs() < 2.0 / R)
        keep.append(torch.cat([torch.full((yz.shape[0], 1), x, device="cuda", dtype=torch.int64), yz], 1))
    xyz = torch.cat(keep).to(torch.int32)
    c = torch.cat([torch.full((xyz.shape[0], 1), 9, device="cuda", dtype=torch.int32), xyz], 1).contiguous()
    r = torch.randn((c.shape[0], 28), dtype=torch.float16, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    yield "shell512", c, r


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--oracle-max-cells", type=int, default=20_000_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from oracle import build_oracle as bo
    from volrend_b200 import build_arrays
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    results = []
    for name, cells, rows in inputs():
        n = int(cells.shape[0])
        rec = dict(input=name, cells=n, data_dim=int(rows.shape[1]), gpu=gpu)
        for merge in (False, True):
            for _ in range(args.warmup):
                child, data = build_arrays(cells, rows, merge=merge)
            torch.cuda.synchronize()
            del child, data
            times = []
            for _ in range(args.reps):
                _pool_high(reset=True)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                child, data = build_arrays(cells, rows, merge=merge)
                b.record()
                b.synchronize()
                times.append(a.elapsed_time(b))
                peak = _pool_high() + child.numel() * 4 + data.numel() * 2
                nodes = int(child.shape[0])
                del child, data
            ms = float(np.median(times))
            key = "merge" if merge else "plain"
            rec[key] = dict(gpu_ms_median=round(ms, 3), gpu_ms_all=[round(t, 3) for t in times], nodes=nodes,
                            cells_per_s=round(n / (ms * 1e-3)), peak_device_bytes=int(peak))
        if n <= args.oracle_max_cells:
            c, r = cells.cpu().numpy(), rows.cpu().numpy()
            t0 = time.perf_counter()
            oc, od = bo.build(c, r)
            rec["oracle_s"] = round(time.perf_counter() - t0, 2)
            child, data = build_arrays(cells, rows)
            rec["oracle_equal"] = bool(np.array_equal(oc, child.cpu().numpy()) and
                                       np.array_equal(od.view(np.uint16), data.cpu().numpy().view(np.uint16)))
            del oc, od, child, data
        else:
            rec["oracle_s"] = None
        print(json.dumps(rec), flush=True)
        results.append(rec)
        del cells, rows
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
