"""Trees and cuts of the grid-wireframe goldens (tests/golden/ref/wire_*.npz, written by
``tools/make_golden.py --wire`` from the reference's own N3Tree::gen_wireframe)."""
from __future__ import annotations

import hashlib

import numpy as np

from volrend_b200 import synth

# outputs up to this many floats are stored whole; larger ones as a SHA-256 plus a sample of vertices
WHOLE_MAX_FLOATS = 1 << 18
SAMPLE_VERTS = 2048
CHAIN_LEVELS = 23       # leaf level of the chain tree: deeper than a 64-bit key holds (21 levels)


def chain_tree(levels: int = CHAIN_LEVELS) -> synth.SynthTree:
    """One internal child per level (octants vary from level to level), the rest leaves: leaves down to ``levels``."""
    cap = levels
    child = np.zeros((cap, 8), np.int32)
    for i in range(cap - 1):
        child[i, (5 * i + 3) % 8] = 1                   # node i+1, relative to node i
    data = np.zeros((cap, 8, 4), np.float16)
    data[..., 3] = np.float16(0.5)
    data[..., :3] = np.float16(0.25)
    return synth.SynthTree(child=child.reshape(cap, 2, 2, 2), data=data.reshape(cap, 2, 2, 2, 4),
                           offset=np.array([0.5, 0.5, 0.5], np.float32),
                           invradius3=np.array([0.5, 0.5, 0.5], np.float32), data_dim=4, data_format="SH1",
                           depth=levels)


def _xf_tree() -> synth.SynthTree:
    st = synth.make_tree("drums", depth=5, basis_dim=1, seed=9)
    st.offset = np.array([0.4132, 0.5378, 0.4719], np.float32)
    st.invradius3 = np.array([0.2917, 0.3311, 0.3779], np.float32)
    return st


def wire_tree(name: str) -> synth.SynthTree:
    if name == "sh4_d5":
        return synth.make_tree("lego", depth=5, basis_dim=4, seed=3)        # tests/conftest.py small_trees
    if name == "sh16_d6":
        return synth.make_tree("lego", depth=6, basis_dim=16, seed=1)
    if name == "xf_d5":
        return _xf_tree()
    if name == "chain":
        return chain_tree()
    raise KeyError(name)


WIRE_DEPTHS = {
    "sh4_d5": [-1, 0, 2, 3, 5, 8],
    "sh16_d6": [-1, 0, 2, 3, 6, 9],
    "xf_d5": [1, 3, 5],
    "chain": [0, 20, 21, 22, 23, 40],
}
WIRE_CASES = [(name, d) for name, depths in WIRE_DEPTHS.items() for d in depths]


def golden_name(name: str, max_depth: int) -> str:
    return f"wire_{name}_m{max_depth}".replace("-", "n")


def sample_index(n_verts: int) -> np.ndarray:
    rng = np.random.default_rng(n_verts)
    idx = rng.integers(0, n_verts, SAMPLE_VERTS)
    return np.unique(np.concatenate([idx, [0, n_verts - 1]])).astype(np.int64)


def sha256(v: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(v, np.float32).tobytes()).hexdigest()


def record(name: str, max_depth: int, v: np.ndarray) -> dict:
    """What the golden file keeps of gen_wireframe's output ``v`` (float32, flat)."""
    v = np.ascontiguousarray(v, np.float32)
    rec = dict(case=np.array(name), max_depth=np.int64(max_depth), n_floats=np.int64(v.size), sha256=np.array(sha256(v)))
    if v.size <= WHOLE_MAX_FLOATS:
        rec["verts"] = v
    else:
        idx = sample_index(v.size // 9)
        rec["sample_idx"] = idx
        rec["sample"] = v.reshape(-1, 9)[idx]
    return rec


def matches(rec, v: np.ndarray) -> bool:
    """Byte-identical to the stored output (whole, or SHA-256 over every byte)."""
    v = np.ascontiguousarray(v, np.float32)
    if int(rec["n_floats"]) != v.size:
        return False
    if "verts" in rec:
        return np.array_equal(np.asarray(rec["verts"]).view(np.uint32), v.view(np.uint32))
    return str(rec["sha256"]) == sha256(v)
