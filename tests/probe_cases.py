"""Deterministic inputs of the lumisphere probe goldens (tests/golden/ref/probe_*.npz): shared by
tools/make_golden.py --probe, which runs the reference's launch_renderer with enable_probe on an H100, and by the
CPU and GPU probe tests."""
import os

import numpy as np

from golden_cases import build_case, composite_inputs
from volrend_b200 import synth

W, H = 160, 120
REF_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref")

# name -> (golden_cases tree/pose/options case, where the probe sits, probe_disp_size, option overrides)
PROBE_CASES = {
    "sh16_centre": ("lego_sh16", "centre", 100, {}),
    "sh16_empty": ("lego_sh16", "empty", 100, {}),
    "sh16_outside": ("lego_sh16", "outside", 100, {}),
    "sh16_d37": ("lego_sh16", "centre", 37, {}),
    "sh16_d1": ("lego_sh16", "centre", 1, {}),
    "sh16_d0": ("lego_sh16", "centre", 0, {}),
    "sh16_d500": ("lego_sh16", "centre", 500, {}),
    "sh16_dmax": ("lego_sh16", "centre", 2 ** 31 - 1, {}),
    "sh16_dneg": ("lego_sh16", "centre", -3, {}),
    "sh16_minmax13": ("lego_sh16", "centre", 100, dict(basis_minmax=[1, 3])),
    "sh9": ("drums_sh9", "centre", 100, {}),
    "sh25_bbox": ("lego_sh25_bbox", "centre", 100, {}),
    "rgba": ("lego_rgba", "centre", 100, {}),
    "sg9_rot": ("lego_sg9_rot", "centre", 100, {}),
    "asg4": ("lego_asg4", "centre", 100, {}),
    "sh9_composite": ("lego_sh9_composite", "centre", 100, {}),
    "sh9_depth": ("lego_sh9_depth", "centre", 100, {}),
}

# tree coordinates of the three probe positions (the world point is offset + scale * probe, volrend.cu:180-182)
_TREE_POINT = {"centre": (0.5, 0.5, 0.5), "empty": (0.02, 0.03, 0.97), "outside": (1.7, -0.4, 0.5)}


def probe_case(name: str):
    """-> (SynthTree, pose 4x4, options dict, probe world xyz, disp_size, composite inputs or None)."""
    base, where, disp, over = PROBE_CASES[name]
    st, _, _, pose, optkw, ndc = build_case(base)
    assert ndc is None
    optkw = dict(optkw)
    bd = int(str(st.data_format)[len(str(st.data_format).rstrip("0123456789")):] or -1)
    if bd > 0 and "basis_minmax" not in optkw:
        # the reference sums basis_minmax[0]..[1] of the probed leaf's coefficients; keep the range inside the
        # tree's basis (what VolumeRenderer.set() does), where its output is defined
        optkw["basis_minmax"] = [0, bd - 1]
    optkw.update(over)
    t = np.asarray(_TREE_POINT[where], np.float64)
    probe = ((t - np.asarray(st.offset, np.float64)) / np.asarray(st.invradius3, np.float64)).astype(np.float32)
    return st, pose, optkw, probe, disp, composite_inputs(base, W, H)


def focal() -> float:
    return synth.focal_for(W)


def golden_path(name: str) -> str:
    return os.path.join(REF_DIR, "probe_" + name + ".npz")
