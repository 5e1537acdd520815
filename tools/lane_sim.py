#!/usr/bin/env python
"""Design tool: dump the bench tree's topology + sigma and a few poses, build tools/lane_sim.c and run
it.  Ranks lane-scheduling policies of the march kernel on the CPU (no GPU needed).
MEM=1 replays the memory traffic of the batch work orders instead -- per-SM L1 (L1KB, default 156) and L2 (L2MB,
default 50) hit rates, DRAM bytes and the per-SM balance of the plain and the SM-affine block orders (give it
consecutive orbit poses: MEM=1 VIEWS=40-55)."""
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from volrend_b200 import synth  # noqa: E402


def main():
    depth = int(os.environ.get("DEPTH", 10))
    size = int(os.environ.get("SIZE", 800))
    views = []
    for v in os.environ.get("VIEWS", "0,37,90").split(","):
        a, _, b = v.partition("-")
        views += list(range(int(a), int(b or a) + 1))
    kind = os.environ.get("KIND", "lego")
    dump = f"/tmp/lane_sim_{kind}_{depth}_{size}.bin"
    st = synth.make_tree(kind, depth=depth, basis_dim=1, seed=0)
    poses = synth.nerf_synthetic_test_poses(200)
    cams = np.stack([synth.c2w_to_colmajor12(poses[v]) for v in views]).astype(np.float32)
    with open(dump, "wb") as f:
        np.array([st.capacity, size, size, len(views)], np.int64).tofile(f)
        fx = synth.focal_for(size)
        np.concatenate([st.offset, st.invradius3, [fx, fx]]).astype(np.float32).tofile(f)
        st.child.reshape(-1).astype(np.int32).tofile(f)
        np.ascontiguousarray(st.data[..., st.data_dim - 1]).view(np.uint16).reshape(-1).tofile(f)
        cams.tofile(f)
    exe = "/tmp/lane_sim"
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-o", exe, os.path.join(ROOT, "tools", "lane_sim.c"),
                           "-lm", "-pthread"])
    subprocess.check_call([exe, dump])


if __name__ == "__main__":
    main()
