"""`-m "not gpu"`: the edge-case march frames of tests/edge_cases.py on the CPU.  Every tree passes the host loader, the
oracle renders every frame in bounded time and within MAX_SAMPLES_PER_RAY samples per ray (so no case that reaches a
GPU can hang a kernel), and the oracle matches the stored frames of the reference's CUDA kernel."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import edge_cases as ec
from conftest import ROOT


@pytest.mark.parametrize("name", ec.TREES)
def test_host_loader_accepts_tree(name):
    """N3Tree.load_npz (the host half of open_arrays / open) reads the tree as it is, and its links form a tree whose
    leaves sit at every level the case claims."""
    from volrend_b200 import N3Tree
    st, npz = ec.edge_tree(name)
    t = N3Tree(gpu_decode=False)
    t.load_npz(ec.tree_file_arrays(st, npz))
    assert t.capacity == st.capacity and t.N == 2 and t.data_dim == st.data_dim
    assert np.array_equal(t.child_, st.child)
    assert np.array_equal(t.data_.view(np.uint16), st.data.view(np.uint16))
    assert np.array_equal(t.scale, st.invradius3) and np.array_equal(t.offset, st.offset)
    # BFS links: every non-root node has exactly one parent, after it; leaf levels 1..depth all present
    child = st.child.reshape(-1, 8).astype(np.int64)
    n, s = np.nonzero(child)
    tgt = n + child[n, s]
    assert (child[n, s] > 0).all() and (tgt < st.capacity).all()
    assert np.array_equal(np.sort(tgt), np.arange(1, st.capacity))
    depth = np.zeros(st.capacity, np.int64)
    depth[tgt] = -1
    for a, b in sorted(zip(n, tgt)):
        depth[b] = depth[a] + 1
    leaf_levels = set((depth[:, None] + 1).repeat(8, 1)[child == 0].tolist())
    assert leaf_levels == set(range(1, st.depth + 1)), sorted(leaf_levels)
    if name.startswith(("mixed", "root", "chain")):      # every leaf is shaded, coarse ones included
        sig = st.data.reshape(-1, 8, st.data_dim)[..., -1].astype(np.float32)
        assert (sig[child == 0] > 0).all()


def test_refused_trees_are_listed():
    assert set(ec.REFUSED) == {"chain24"}
    assert not set(ec.REFUSED) & set(ec.TREES)


def _max_samples_per_ray(tree_name):
    """{frame: (max samples of one ray, total)} by the oracle, one 1x1 tile per pixel."""
    from oracle import binding as ob
    from volrend_b200 import synth
    st, _ = ec.edge_tree(tree_name)
    ot = ob.OracleTree.from_synth(st, ndc=ec.NDC.get(tree_name))
    out = {}
    for fr in ec.frames_of(tree_name):
        _, W, H, fx, fy, pose, kw, comp = ec.frame(fr, st)
        cam, opt = ob.make_camera(W, H, fx, fy, synth.c2w_to_colmajor12(pose)), ob.make_options(**kw)
        worst = total = 0
        for y in range(H):
            for x in range(W):
                rin, din = (None, None) if comp is None else (comp[0][y:y + 1, x:x + 1], comp[1][y:y + 1, x:x + 1])
                _, _, cnt = ob.render(ot, cam, opt, tile=(x, y, 1, 1), rgba_in=rin, depth_in=din, want_float=False,
                                      want_u8=False, nthreads=1)
                worst = max(worst, cnt["samples"])
                total += cnt["samples"]
        out[fr] = (worst, total)
    return out


@pytest.mark.parametrize("name", ec.TREES)
def test_oracle_terminates_within_sample_bound(built, name):
    """Each ray of each frame ends within MAX_SAMPLES_PER_RAY samples, and the whole tree's frames within a timeout
    (in a process of their own, so that a march that never ends fails the test instead of hanging it)."""
    r = subprocess.run([sys.executable, os.path.abspath(__file__), name], cwd=ROOT, capture_output=True, text=True,
                       timeout=600, env=dict(os.environ, PYTHONPATH=ROOT))
    assert r.returncode == 0, r.stderr
    got = json.loads(r.stdout.strip().splitlines()[-1])
    assert set(got) == set(ec.frames_of(name))
    for fr, (worst, total) in got.items():
        assert worst <= ec.MAX_SAMPLES_PER_RAY, (fr, worst)
        if not fr.endswith("bbox_degen.default") and not fr.endswith("bbox_inv.default"):
            assert total > 0, fr                  # every other frame marches some ray


@pytest.mark.parametrize("name", ec.FRAMES)
def test_oracle_matches_reference_frame(built, name):
    """The oracle against the reference kernel's stored frame: floats within 2.4e-7 (glibc against libdevice expf), and
    bytes identical except where the reference's float sits within that bound of a byte boundary."""
    st, _ = ec.edge_tree(name.split(".")[0])
    f, u, _ = ec.oracle_render(name, st)
    z = ec.load(name)
    assert f.shape == tuple(z["shape"])
    if "f32" in z:
        f, u, rf, ru = f.reshape(-1, 4), u.reshape(-1, 4), z["f32"].reshape(-1, 4), z["u8"].reshape(-1, 4)
    else:
        idx = z["index"]
        f, u, rf, ru = f.reshape(-1, 4)[idx], u.reshape(-1, 4)[idx], z["f32_sample"], z["u8_sample"]
    assert np.array_equal(np.isnan(f), np.isnan(rf)), name
    d = np.abs(np.nan_to_num(f) - np.nan_to_num(rf))
    assert d.max() <= 2.4e-7, (name, float(d.max()))
    s = rf.astype(np.float64) * 255
    near = np.abs(s - np.round(s)) <= 255 * 2.4e-7
    diff = u != ru
    assert (np.abs(u.astype(int) - ru.astype(int)) <= 1).all(), name
    assert near[diff].all(), (name, "a byte differs away from a byte boundary")


def _box_rays(name):
    """Tree-space (origins, directions) of the rays of frame ``name`` (float64) and its render box (lo, hi)."""
    st, _ = ec.edge_tree(name.split(".")[0])
    _, W, H, fx, fy, pose, kw, _ = ec.frame(name, st)
    px, py = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    vx, vy = (px - W * 0.5) / fx, -(py - H * 0.5) / fy
    R = pose[:3, :3].astype(np.float64)
    d = vx[..., None] * R[:, 0] + vy[..., None] * R[:, 1] - R[:, 2]
    sc = st.invradius3.astype(np.float64)
    o = pose[:3, 3].astype(np.float64) * sc + st.offset
    return o, (d * sc).reshape(-1, 3), np.array(kw["render_bbox"][:3]), np.array(kw["render_bbox"][3:])


def test_graze_view_grazes_the_render_box():
    """The graze frame's rays meet the box's front face (x = 0.75) on its edges, and many leave through a side face
    (y or z), so the slab test's t_min ~ t_max at a box edge, with its 1e-6 inset, is rendered."""
    o, d, lo, hi = _box_rays("mixed_sh16.graze.default")
    with np.errstate(divide="ignore"):
        t1, t2 = (lo - o) / d, (hi - o) / d
    tn, tf = np.minimum(t1, t2), np.maximum(t1, t2)
    hit = tn.max(-1) < tf.min(-1)
    assert (tn.argmax(-1)[hit] == 0).all()                           # every hit enters through the front face
    assert (hit & (tf.argmin(-1) != 0)).sum() >= 100                 # and many leave through a side face
    front = o + ((hi[0] - o[0]) / d[:, :1]) * d                      # where each ray crosses the plane x = 0.75
    on_edge = np.isclose(front[:, 1:], lo[1:], atol=1e-9, rtol=0).any(-1)
    assert on_edge.sum() >= 30                                       # column 0 and row 0: on the edges y, z = 0.25


@pytest.mark.parametrize("name", [f"{t}.{v}.default" for t in ("chain22", "chain23") for v in ec.DEEP])
def test_deep_chain_views_march_through_the_chain(built, name):
    """Every ray of the deep views starts with a lookup at its leaf's level and goes on for several samples through
    the chain's other levels."""
    st, _ = ec.edge_tree(name.split(".")[0])
    _, W, H, _, _, _, _, _ = ec.frame(name, st)
    _, _, c = ec.oracle_render(name, st)
    level = st.depth - ec.DEEP[name.split(".")[1]][0]
    assert c["rays_hit"] == W * H and c["samples"] >= 4 * W * H
    assert c["child_loads"] >= (level + 3) * W * H


def test_every_frame_has_a_golden():
    missing = [f for f in ec.FRAMES if not os.path.exists(ec.golden_path(f))]
    assert not missing, f"run tools/make_golden.py --edge on a GPU: {missing[:5]}"


if __name__ == "__main__":
    print(json.dumps(_max_samples_per_ray(sys.argv[1])))
