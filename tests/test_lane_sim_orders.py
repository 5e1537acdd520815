"""CPU: every work order of tools/lane_sim.c's memory replay -- the plain orders and the SM-affine blocks of one or
several views -- visits every (view, tile) exactly once, also when neither the view count nor the tile grid is a
multiple of a block."""
import os
import shutil
import subprocess

import pytest

from conftest import ROOT


@pytest.fixture(scope="module")
def lane_sim(tmp_path_factory):
    cc = shutil.which("gcc") or shutil.which("cc")
    if not cc:
        pytest.skip("no C compiler")
    exe = str(tmp_path_factory.mktemp("lane_sim") / "lane_sim")
    subprocess.check_call([cc, "-O2", "-ffp-contract=off", "-o", exe, os.path.join(ROOT, "tools", "lane_sim.c"),
                           "-lm", "-pthread"])
    return exe


@pytest.mark.parametrize("views,W,H", [(13, 148, 232), (37, 148, 232), (1, 37, 29), (8, 800, 800)])
def test_orders_visit_every_tile_once(lane_sim, views, W, H):
    r = subprocess.run([lane_sim, "--check-orders", str(views), str(W), str(H)], capture_output=True, text=True)
    lines = r.stdout.strip().splitlines()
    assert r.returncode == 0, r.stdout
    assert len(lines) >= 14 and all(ln.endswith(" ok") for ln in lines), r.stdout
    assert any("views, view inner" in ln for ln in lines)
