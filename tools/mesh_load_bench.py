#!/usr/bin/env python
"""Times mesh loading with GPU normal estimation (DESIGN.md section 11).

  * vr_mesh_estimate_normals alone, CUDA events, median of 20 after 5 warm-ups, on: legoman (the reference's
    sample OBJ, from its golden), a UV sphere just under the reference's float-index bound (Sphere(1000, 1800),
    1.8 M vertices, 3.6 M faces) and a 20 M-triangle soup;
  * Mesh.open_drawlist end to end on a `mesh` drawlist of that sphere (host clock, synchronised);
  * the reference's Mesh::open_drawlist_mem on the same bytes through oracle/_ref/libref_mesh.so (host clock),
    when that harness is built.

Prints the card name and power limit first.  Writes nothing into the tree (the drawlist goes to a temporary file).
"""
import contextlib
import io
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
    except Exception as e:             # the timings below still say what they measured
        return f"unknown ({e})"


def time_kernel(mesh, reps=20, warm=5):
    import torch
    from volrend_b200 import _capi, lib
    from volrend_b200.host import _stream_ptr
    mesh.update()
    vd, fd = mesh._vert_dev, mesh._faces_dev
    nv, nf = vd.numel() // 9, (fd.numel() // 3 if fd is not None else 0)
    s = _stream_ptr(None)
    ms = []
    for i in range(warm + reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        _capi.check(lib().vr_mesh_estimate_normals(vd.data_ptr(), nv, fd.data_ptr() if fd is not None else None, nf, s))
        b.record()
        b.synchronize()
        if i >= warm:
            ms.append(a.elapsed_time(b))
    return statistics.median(ms), nv, nf


def main():
    import torch
    from volrend_b200 import Mesh
    import mesh_io_cases as mc
    from oracle import ref_mesh
    print("card:", card(), flush=True)
    torch.cuda.init()
    _, data, _, _, _ = mc.load_golden("mesh_obj_legoman.npz")
    with contextlib.redirect_stdout(io.StringIO()):
        lego = Mesh.load_mem_basic_obj(data)
    sphere = Mesh.Sphere(1000, 1800)
    n_soup = 20_000_000
    soup = Mesh(3 * n_soup, 0, 3)
    rng = np.random.default_rng(0)
    soup.vert.reshape(-1, 9)[:, :3] = rng.standard_normal((3 * n_soup, 3), dtype=np.float32)
    rows = []
    for name, m in [("legoman", lego), ("sphere 1000x1800", sphere), ("soup 20M tris", soup)]:
        ms, nv, nf = time_kernel(m)
        rows.append((name, nv, nf if nf else nv // 3, ms))
        print(f"vr_mesh_estimate_normals {name}: {nv} vertices, {nf if nf else nv // 3} faces: {ms:.3f} ms "
              "(median of 20)", flush=True)
        m._vert_dev = m._faces_dev = None
        torch.cuda.empty_cache()
    del soup
    pts = np.asarray(sphere.vert, np.float32).reshape(-1, 9)[:, :3].reshape(-1)
    b = io.BytesIO()
    np.savez(b, s="mesh", s__points=pts, s__faces=np.asarray(sphere.faces, np.int32))
    blob = b.getvalue()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "sphere.draw.npz")
        with open(path, "wb") as f:
            f.write(blob)
        times = []
        for i in range(4):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            with contextlib.redirect_stdout(io.StringIO()):
                (m,) = Mesh.open_drawlist(path)
            torch.cuda.synchronize()
            times.append((time.perf_counter() - t0) * 1e3)
        print(f"Mesh.open_drawlist sphere drawlist ({len(blob) / 1e6:.1f} MB): {statistics.median(times[1:]):.1f} ms "
              f"(median of 3 after 1 warm-up; first {times[0]:.1f} ms)", flush=True)
    if ref_mesh.available():
        with contextlib.redirect_stdout(io.StringIO()):
            rt = [ref_mesh.open_drawlist_mem_ms(blob) for _ in range(3)]
        print(f"reference Mesh::open_drawlist_mem same bytes: {statistics.median(rt):.1f} ms (median of 3)", flush=True)
    else:
        print("reference harness not built: no reference time", flush=True)


if __name__ == "__main__":
    main()
