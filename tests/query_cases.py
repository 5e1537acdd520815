"""Trees and point sets of the point-query goldens (tests/golden/ref/query_*.npz, written by
``tools/make_golden.py --query`` from the reference's own query_single_from_root, oracle/ref_query.cu)."""
from __future__ import annotations

import zlib

import numpy as np

from golden_cases import build_case
from wire_cases import chain_tree
from volrend_b200 import synth

# golden-case trees (tests/golden_cases.py), a quantised tree, the 23-level chain tree and a tree whose leaves hold
# negative, signed-zero and NaN sigma
QUERY_TREES = ["cfg1_sh1", "lego_sh4_stop0", "drums_sh9", "lego_sh16", "lego_sh25_bbox", "lego_rgba", "lego_sg9_rot",
               "lego_asg4", "lego_sh16_ndc", "quant_sh4", "chain", "sigma_bits"]
# fp16 sigma bit patterns of the sigma_bits tree, slot i taking SIGMA_BITS[i % 6]: -2.5, -0, +0, NaN, a negative NaN
# with another payload, 3.0
SIGMA_BITS = np.array([0xC100, 0x8000, 0x0000, 0x7E00, 0xFE01, 0x4200], np.uint16)
# point sets, in this order, concatenated in every golden
SETS = ["grid", "uniform", "outside", "nonfinite", "dyadic"]


def quantised(st: synth.SynthTree, seed: int = 21) -> dict:
    """npz dict of ``st`` in the quant_colors / quant_map format (one retained basis function), random codebooks."""
    rng = np.random.default_rng(seed)
    cap = st.child.shape[0]
    bd = (st.data_dim - 1) // 3
    nq = bd - 1
    data = st.data.reshape(cap * 8, st.data_dim)
    z = dict(child=st.child, offset=st.offset, invradius3=st.invradius3, data_dim=np.int64(st.data_dim),
             data_format=np.array(st.data_format))
    z["quant_colors"] = rng.normal(0, 0.5, (nq, 65536, 3)).astype(np.float16)
    z["quant_map"] = rng.integers(0, 65536, (nq, cap, 2, 2, 2)).astype(np.uint16)
    z["sigma"] = data[:, -1].reshape(cap, 2, 2, 2).copy()
    z["data_retained"] = np.stack([data[:, k * bd] for k in range(3)], -1).reshape(1, cap, 2, 2, 2, 3).copy()
    return z


def query_tree(name: str):
    """-> npz dict of the tree (what N3Tree.load_npz and the reference loader read)."""
    if name == "chain":
        st = chain_tree()
    elif name == "quant_sh4":
        return quantised(synth.make_tree("lego", depth=5, basis_dim=4, seed=14))
    elif name == "sigma_bits":
        st = synth.make_tree("lego", depth=5, basis_dim=4, seed=22)
        d = st.data.reshape(-1, st.data_dim).view(np.uint16).copy()
        d[:, -1] = SIGMA_BITS[np.arange(d.shape[0]) % len(SIGMA_BITS)]
        st.data = d.view(np.float16).reshape(st.data.shape)
    else:
        st = build_case(name)[0]
    z = dict(child=st.child, data=st.data, offset=st.offset, invradius3=st.invradius3, data_dim=np.int64(st.data_dim),
             data_format=np.array(st.data_format))
    if st.extra is not None:
        z["extra_data"] = st.extra
    return z


def _to_world(z: dict, t: np.ndarray) -> np.ndarray:
    off = np.asarray(z["offset"], np.float64)
    sc = np.asarray(z["invradius3"], np.float64)
    with np.errstate(invalid="ignore"):
        return ((np.asarray(t, np.float64) - off) / sc).astype(np.float32)


def point_sets(name: str, z: dict) -> dict:
    """set name -> float32 [n, 3] world points."""
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    g = (np.arange(10, dtype=np.float64) + 0.5) / 10
    grid = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)       # raster order, z fastest
    vals = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, 1.0, 1 - 1e-6, 0.5, 2.0], np.float32)
    nonfinite = np.stack(np.meshgrid(vals, vals, vals, indexing="ij"), -1).reshape(-1, 3)
    # cell faces k / 2^d at every depth down to the tree's, their float neighbours, and the clamp bound
    d = rng.integers(1, 24, (600, 3))
    k = np.floor(rng.random((600, 3)) * (2.0 ** d))
    faces = (k / 2.0 ** d).astype(np.float32)
    wiggle = rng.integers(-1, 2, (600, 3))
    faces = np.where(wiggle == 0, faces, np.nextafter(faces, np.where(wiggle > 0, 2, -1).astype(np.float32)))
    ends = np.array([[1 - 1e-6] * 3, [np.float32(1) - np.float32(1e-6)] * 3, [1.0] * 3, [0.0] * 3, [0.5, 0.25, 0.75]],
                    np.float32)
    if name == "chain":     # the corner and centre of each cell along the chain, down to its 23rd level
        c = np.zeros(3)
        for lv in range(23):
            o = (5 * lv + 3) % 8
            ends = np.concatenate([ends, [c, c + 2.0 ** -(lv + 1)]]).astype(np.float32)
            c = c + np.array([(o >> 2) & 1, (o >> 1) & 1, o & 1]) * 2.0 ** -(lv + 1)
    return {
        "grid": _to_world(z, grid),
        "uniform": _to_world(z, rng.random((1000, 3))),
        "outside": _to_world(z, rng.uniform(-1.0, 2.0, (500, 3))),
        # non-finite and boundary values straight in world coordinates
        "nonfinite": nonfinite.astype(np.float32),
        "dyadic": _to_world(z, np.concatenate([faces, ends]).astype(np.float64)),
    }


def all_points(name: str, z: dict):
    """-> (float32 [n, 3] points of every set, int8 [n] set index)."""
    s = point_sets(name, z)
    pts = np.concatenate([s[k] for k in SETS]).astype(np.float32)
    lab = np.concatenate([np.full(len(s[k]), i, np.int8) for i, k in enumerate(SETS)])
    return pts, lab


def tree_space_points(z: dict, n: int, seed: int) -> np.ndarray:
    """n uniform world points inside the tree's box."""
    rng = np.random.default_rng(seed)
    return _to_world(z, rng.random((n, 3)))


def golden_path(name: str) -> str:
    import os
    return os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref", "query_" + name + ".npz")
