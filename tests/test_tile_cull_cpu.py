"""CPU: the tile culling of batch launches (volrend_b200/csrc/vr_cull.cu) never culls a tile that holds a shading ray.
tools/lane_sim.c restates the policy -- the same 32^3 max-sigma grid, the same dilation, one bit per 4x8 tile -- and
replays every ray of the frame with the CPU oracle's arithmetic; CULL=1 counts, per view, the tiles with a shaded
sample that the mask leaves unmarked (must be none) and the tiles it marks that never shade.  The trees are the golden,
edge and relaid trees the GPU tests use and the bench tree at a reduced size."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from conftest import ROOT

import edge_cases as ec  # noqa: E402
import golden_cases as gc  # noqa: E402
import layout_cases as lc  # noqa: E402


@pytest.fixture(scope="module")
def lane_sim(tmp_path_factory):
    cc = shutil.which("gcc") or shutil.which("cc")
    if not cc:
        pytest.skip("no C compiler")
    exe = str(tmp_path_factory.mktemp("cull") / "lane_sim")
    subprocess.check_call([cc, "-O2", "-ffp-contract=off", "-o", exe, os.path.join(ROOT, "tools", "lane_sim.c"),
                           "-lm", "-pthread"])
    return exe


def _orbit(st, n, dist=(2.2, 3.0, 4.5)):
    """n column-major c2w (12 floats) around the tree's box at a few distances, looking at its centre."""
    from volrend_b200 import synth
    centre = ec._to_world(st, [0.5, 0.5, 0.5])
    span = float(np.abs(ec._to_world(st, [1.0, 1.0, 1.0]) - ec._to_world(st, [0.0, 0.0, 0.0])).max())
    out = []
    for i in range(n):
        a = 2.0 * np.pi * i / n + 0.3
        eye = centre + dist[i % len(dist)] * span * np.array([np.cos(a), np.sin(a), 0.4 + 0.3 * np.sin(3 * a)])
        out.append(synth.c2w_to_colmajor12(synth.look_at_c2w(eye, target=centre)))
    return out


def _run(exe, path, st, W, H, fx, cams, thresh=None):
    with open(path, "wb") as f:       # the dump format of tools/lane_sim.py
        np.array([st.capacity, W, H, len(cams)], np.int64).tofile(f)
        np.concatenate([st.offset, st.invradius3, [fx, fx]]).astype(np.float32).tofile(f)
        st.child.reshape(-1).astype(np.int32).tofile(f)
        np.ascontiguousarray(np.asarray(st.data)[..., st.data_dim - 1]).astype(np.float16).view(np.uint16) \
            .reshape(-1).tofile(f)
        np.stack(cams).astype(np.float32).tofile(f)
    env = dict(os.environ, CULL="1")
    if thresh is not None:
        env["THRESH"] = repr(float(thresh))
    r = subprocess.run([exe, path], capture_output=True, text=True, env=env)
    views = [tuple(int(v) for v in m) for m in
             re.findall(r"cull view \d+: tiles (\d+) marked (\d+) shading (\d+) unmarked_shading (\d+) "
                        r"marked_never_shading (\d+)", r.stdout)]
    total = [ln for ln in r.stdout.splitlines() if ln.startswith("cull total")]
    assert len(views) == len(cams) and total, r.stdout + r.stderr
    return r.returncode, views, total[0]


def _check(rc, views, total, what):
    print(f"{what}: {total}")
    for v, (tiles, marked, shading, bad, never) in enumerate(views):
        assert bad == 0, f"{what} view {v}: {bad} tiles with a shading ray are culled"
        assert shading <= marked <= tiles
    assert rc == 0


def _trees():
    out = []
    for name in ["lego_sh16", "drums_sh9", "lego_sh25_bbox", "lego_rgba", "cfg1_sh1"]:
        out.append((name, gc.build_case(name)[0]))
    for name in ["mixed_sh16", "mixed_rgba", "root_mixed", "chain22", "aniso", "sigma_bits"]:
        out.append((name, ec.edge_tree(name)[0]))
    base = ec.edge_tree("mixed_sh16")[0]
    for layout in ["shuffle", "dirty"]:
        out.append((f"mixed_sh16_{layout}", lc.relayout(base, layout, seed=4).st))
    return out


TREES = _trees()


@pytest.mark.parametrize("thresh", [None, 0.0, 3.0])
@pytest.mark.parametrize("case", range(len(TREES)), ids=[t[0] for t in TREES])
def test_no_shading_tile_is_culled(lane_sim, tmp_path, case, thresh):
    name, st = TREES[case]
    rc, views, total = _run(lane_sim, str(tmp_path / "d.bin"), st, 96, 72, 80.0, _orbit(st, 6), thresh)
    _check(rc, views, total, f"{name} thresh={thresh}")


def test_below_every_sigma_marks_everything(lane_sim, tmp_path):
    st = TREES[0][1]
    rc, views, total = _run(lane_sim, str(tmp_path / "d.bin"), st, 64, 48, 60.0, _orbit(st, 3), thresh=-1e30)
    _check(rc, views, total, "thresh=-1e30")
    assert all(marked == tiles for tiles, marked, _, _, _ in views)


def test_bench_tree_reduced(lane_sim, tmp_path):
    """The bench tree (lego, depth 10) at 200x200 on three of the bench poses: nothing that shades is culled, and the
    mask keeps most of what culling exactly the non-shading tiles would save."""
    from volrend_b200 import synth
    st = synth.make_tree("lego", depth=10, basis_dim=1, seed=0)
    poses = synth.nerf_synthetic_test_poses(200)
    cams = [synth.c2w_to_colmajor12(poses[v]) for v in (0, 37, 90)]
    rc, views, total = _run(lane_sim, str(tmp_path / "d.bin"), st, 200, 200, synth.focal_for(200), cams)
    _check(rc, views, total, "bench tree 200x200")
    m = re.search(r"tiles_culled ([\d.]+) \(bound ([\d.]+)\)", total)
    assert float(m.group(1)) >= 0.5 * float(m.group(2)), total
