"""Time vr_tree_isosurface on the bench stand-in tree (DESIGN.md section 23).

    python tools/iso_bench.py [--levels 8 9 10] [--calls 5] [--out iso_bench.json]

For each lattice level L: the count-only call and the fill call (count + fill + normals + colours; and without
colours), CUDA events around each call, medians of --calls calls after warm-ups, in two alternated rounds; the lattice
samples per second against vr_tree_query on the same R^3 points (cube sizes only, in chunks), triangles per second,
the default pool's high-water mark and the mesh sizes.  The -Xptxas -v lines of the new kernels are read from
build/obj/ptxas_iso.log.  Needs a CUDA device; there is no fallback.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import re
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _pool():
    import torch
    cu = C.CDLL("libcuda.so.1")
    dev, pool = C.c_int(), C.c_void_p()
    assert cu.cuDeviceGet(C.byref(dev), torch.cuda.current_device()) == 0
    assert cu.cuDeviceGetDefaultMemPool(C.byref(pool), dev) == 0
    return cu, pool


def _pool_high(reset: bool) -> int:
    cu, pool = _pool()
    v = C.c_uint64(0)
    if reset:
        assert cu.cuMemPoolSetAttribute(pool, 8, C.byref(v)) == 0       # CU_MEMPOOL_ATTR_USED_MEM_HIGH
        return 0
    assert cu.cuMemPoolGetAttribute(pool, 8, C.byref(v)) == 0
    return int(v.value)


def _time(fn) -> float:
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def _ptxas():
    path = os.path.join(ROOT, "build", "obj", "ptxas_iso.log")
    out, cur = {}, None
    for line in open(path):
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = re.sub(r"^_ZN3vrb\w*?_vr_iso_cu_\w{8}", "", m.group(1))
            out[cur] = {}
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            out[cur]["spill_st"], out[cur]["spill_ld"] = int(m.group(1)), int(m.group(2))
        m = re.search(r"Used (\d+) registers.*?(?:(\d+) bytes smem)?$", line.strip())
        if m and cur:
            out[cur]["regs"], out[cur]["smem"] = int(m.group(1)), int(m.group(2) or 0)
    return out


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--levels", type=int, nargs="+", default=[8, 9, 10])
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        print("iso_bench needs a CUDA device", file=sys.stderr)
        return 1
    from volrend_b200 import N3Tree, lib, synth, _capi
    from volrend_b200._capi import check
    st = synth.make_tree("lego", depth=10, basis_dim=16, seed=0)
    s = np.asarray(st.data, np.float16)[..., -1].astype(np.float32).reshape(-1)
    s = s[np.isfinite(s) & (s > 0)]
    level = float(np.float32(np.quantile(s, 0.5)))
    tree = N3Tree.from_synth(st)
    L_ = lib()
    sp = torch.cuda.current_stream().cuda_stream
    name = torch.cuda.get_device_name()
    props = os.popen("nvidia-smi --query-gpu=power.limit,clocks.max.sm --format=csv,noheader").read().strip()
    res = dict(device=name, power_limit_and_max_sm_clock=props, tree="synth lego depth 10 SH16 seed 0",
               level=level, kernels=_ptxas(), levels={})
    for L in args.levels:
        nv, nf = C.c_int64(), C.c_int64()

        def count():
            check(L_.vr_tree_isosurface(tree._handle, L, C.c_float(level), None, 0, None, 0, None, 0, C.byref(nv),
                                        C.byref(nf), sp))
        count()
        n_v, n_f = nv.value, nf.value
        vert = torch.empty((n_v, 9), dtype=torch.float32, device="cuda")
        faces = torch.empty((n_f, 3), dtype=torch.int32, device="cuda")

        def fill(flags):
            def f():
                check(L_.vr_tree_isosurface(tree._handle, L, C.c_float(level), None, flags, vert.data_ptr(), n_v,
                                            faces.data_ptr(), n_f, C.byref(nv), C.byref(nf), sp))
            return f
        for _ in range(2):
            count(); fill(0)(); fill(_capi.VR_ISO_COLOR)()
        torch.cuda.synchronize()
        _pool_high(True)
        fill(_capi.VR_ISO_COLOR)()
        torch.cuda.synchronize()
        high = _pool_high(False)
        rounds = []
        for r in range(2):
            rounds.append(dict(count_ms=statistics.median(_time(count) for _ in range(args.calls)),
                               fill_ms=statistics.median(_time(fill(_capi.VR_ISO_COLOR)) for _ in range(args.calls)),
                               fill_nocolor_ms=statistics.median(_time(fill(0)) for _ in range(args.calls))))
        # vr_tree_query over the same R^3 lattice points (world coordinates), cube sizes only, in chunks
        R = 1 << L
        c = ((torch.arange(R, device="cuda", dtype=torch.float32) + 0.5) / R - float(st.offset[0])) / float(st.invradius3[0])
        chunk_planes = max(1, (1 << 26) // (R * R))
        cube = torch.empty(chunk_planes * R * R, dtype=torch.float32, device="cuda")
        q_ms = []
        for rr in range(2):
            tot = 0.0
            for i0 in range(0, R, chunk_planes):
                i1 = min(R, i0 + chunk_planes)
                cx = ((torch.arange(i0, i1, device="cuda", dtype=torch.float32) + 0.5) / R - float(st.offset[0])) / float(st.invradius3[0])
                cy = ((torch.arange(R, device="cuda", dtype=torch.float32) + 0.5) / R - float(st.offset[1])) / float(st.invradius3[1])
                cz = ((torch.arange(R, device="cuda", dtype=torch.float32) + 0.5) / R - float(st.offset[2])) / float(st.invradius3[2])
                xyz = torch.stack(torch.meshgrid(cx, cy, cz, indexing="ij"), -1).reshape(-1, 3).contiguous()
                n = xyz.shape[0]
                tot += _time(lambda: check(L_.vr_tree_query(tree._handle, xyz.data_ptr(), n, None, cube.data_ptr(),
                                                            None, sp)))
            q_ms.append(tot)
        del c
        cnt = min(r["count_ms"] for r in rounds)
        fl = min(r["fill_ms"] for r in rounds)
        res["levels"][L] = dict(
            n_verts=n_v, n_faces=n_f, rounds=rounds, query_ms_rounds=q_ms,
            iso_count_samples_per_s=R ** 3 / (cnt * 1e-3), query_samples_per_s=R ** 3 / (min(q_ms) * 1e-3),
            triangles_per_s_fill=n_f / (fl * 1e-3), pool_high_bytes=high,
            output_bytes=n_v * 36 + n_f * 12)
        del vert, faces
        torch.cuda.empty_cache()
        print(json.dumps({L: res["levels"][L]}))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res["kernels"]))
    return 0


if __name__ == "__main__":
    sys.exit(main())
