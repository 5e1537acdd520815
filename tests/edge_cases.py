"""Trees, views and options of the edge-case march goldens (tests/golden/ref/edge_*.npz, written by
``tools/make_golden.py --edge`` from the reference's own CUDA kernel).

The trees step outside what ``synth.make_tree`` makes: leaves that carry colour and density at every level (root
octants included, so leaves that the wide tables replicate into several entries are shaded), chains down to the
deepest accepted level, an anisotropic off-centre tree transform, fp16 edge values of sigma and colour, and a quantised
tree.  The views put rays where the march goes wrong: exactly zero direction components, rays inside cell faces,
cameras inside the tree (down to the deepest chain cell), grazing, degenerate and inverted render boxes, unequal and
very short focal lengths, sizes that are not multiples of the 4x8 warp tile, and composite depth limits of 0, < 0,
+inf and NaN.

Every frame is ``(tree, view, options)``; ``FRAMES`` lists them, ``frame(name)`` builds one.  The step size stays at
its default (1e-4 in tree units, far above ulp(t) for the t of these views), so that a sample on a cell face always
moves on.
"""
from __future__ import annotations

import hashlib
import os

import numpy as np

from wire_cases import chain_tree
from volrend_b200 import synth

REF_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref")
# frames of at most this many pixels are stored whole; larger ones as SHA-256 plus a pixel sample (ref_frame_record)
WHOLE_MAX_PIXELS = 2048
# bound on the samples of any one ray of any frame (the CPU test checks it with the oracle before a GPU sees the case)
MAX_SAMPLES_PER_RAY = 4096

# fp16 sigma bit patterns of the sigma_bits tree, slot i taking SIGMA_BITS[i % len]: -2.5, -0, +0, NaN, a negative NaN
# with another payload, fp16 max, +inf, the smallest and the largest subnormal, 3.0, 1.0
SIGMA_BITS = np.array([0xC100, 0x8000, 0x0000, 0x7E00, 0xFE01, 0x7BFF, 0x7C00, 0x0001, 0x03FF, 0x4200, 0x3C00],
                      np.uint16)
# colour coefficient bit patterns mixed into the sigma_bits tree: +-fp16 max, +-smallest subnormal, largest subnormal
COLOUR_BITS = np.array([0x7BFF, 0xFBFF, 0x0001, 0x8001, 0x03FF], np.uint16)

# Trees the library refuses, with the reason; the reference renders them, no frame of them is stored.
REFUSED = {"chain24": "24 leaf levels: deeper than kMaxTreeDepth (23), vr_tree_create returns VR_EUNSUPPORTED"}


# ----------------------------------------------------------------------------------------------------------- trees
def _extra(fmt: str, basis: int, rng):
    if fmt == "SG":
        mu = rng.standard_normal((basis, 3)).astype(np.float32)
        mu /= np.linalg.norm(mu, axis=1, keepdims=True)
        lam = rng.uniform(0.5, 8.0, (basis, 1)).astype(np.float32)
        return np.concatenate([lam, mu], 1)
    if fmt == "ASG":
        ex = np.zeros((basis, 11), np.float32)
        for i in range(basis):
            q, _ = np.linalg.qr(rng.standard_normal((3, 3)))
            ex[i, 0:2] = rng.uniform(0.5, 6.0, 2)
            ex[i, 2:5], ex[i, 5:8], ex[i, 8:11] = q[:, 0], q[:, 1], q[:, 2]
        return ex
    return None


def _fill_leaves(child, levels, fmt, basis, rng):
    """fp16 data of every slot: leaves get sigma for an optical depth of 0.05..2 across their cell (8 % of them a
    sub-threshold haze) and random colour; ``levels[n]`` is node n's depth (cube [-1, 1]^3 in world units)."""
    cap = child.shape[0]
    data_dim = 4 if fmt == "RGBA" else 3 * basis + 1
    cell = 2.0 ** (1 - (np.asarray(levels, np.float64) + 1))                 # world edge of a child cell
    tau = rng.uniform(0.05, 2.0, (cap, 8))
    sigma = tau / cell[:, None]
    haze = rng.random((cap, 8)) < 0.08
    sigma = np.where(haze, 0.005, sigma)
    data = np.zeros((cap, 8, data_dim), np.float32)
    data[..., -1] = sigma
    if fmt == "RGBA":
        data[..., :3] = rng.random((cap, 8, 3))
    else:
        co = rng.standard_normal((cap, 8, 3 * basis)) * 0.6
        co[..., 0::basis] *= 2.0
        data[..., :3 * basis] = co
    data[child.reshape(cap, 8) != 0] = 0.0                                     # internal slots carry nothing
    return data.astype(np.float16).reshape(cap, 2, 2, 2, data_dim), data_dim


def mixed_tree(depth: int, basis: int = 16, fmt: str = "SH", seed: int = 0, p_refine: float = 0.3,
               root_leaves=(1, 6)) -> synth.SynthTree:
    """Random refinement with leaves at every level 1..depth: the first node of each depth refines one octant and
    keeps at least one leaf, the root keeps ``root_leaves`` as leaves.  Every leaf is shaded."""
    rng = np.random.default_rng(seed)
    masks, levels = [], [0]
    seen_depth = set()
    i = 0
    while i < len(levels):
        d = levels[i]
        m = np.zeros(8, bool)
        if d + 1 < depth:
            m = rng.random(8) < p_refine
            if d == 0:
                m[:] = True
                m[list(root_leaves)] = False
            if d not in seen_depth:
                m[rng.integers(8)] = True
                if m.all():
                    m[rng.integers(8)] = False
        seen_depth.add(d)
        masks.append(m)
        levels.extend([d + 1] * int(m.sum()))
        i += 1
    cap = len(levels)
    child = np.zeros((cap, 8), np.int32)
    nxt = 1
    for n, m in enumerate(masks):
        for s in np.flatnonzero(m):
            child[n, s] = nxt - n
            nxt += 1
    fmt_name = "RGBA" if fmt == "RGBA" else f"{fmt}{basis}"
    data, data_dim = _fill_leaves(child, levels, fmt, basis, rng)
    return synth.SynthTree(child=child.reshape(cap, 2, 2, 2), data=data, offset=np.full(3, 0.5, np.float32),
                           invradius3=np.full(3, 0.5, np.float32), data_dim=data_dim, data_format=fmt_name,
                           depth=depth, extra=_extra(fmt, basis, rng))


def root_only_tree() -> synth.SynthTree:
    """capacity 1: the root's 8 octants are all shaded leaves."""
    rng = np.random.default_rng(31)
    child = np.zeros((1, 8), np.int32)
    data, data_dim = _fill_leaves(child, [0], "SH", 4, rng)
    return synth.SynthTree(child=child.reshape(1, 2, 2, 2), data=data, offset=np.full(3, 0.5, np.float32),
                           invradius3=np.full(3, 0.5, np.float32), data_dim=data_dim, data_format="SH4", depth=1)


def varied_chain(levels: int) -> synth.SynthTree:
    """``wire_cases.chain_tree`` with sigma and colour that vary per level: optical depth 0.1..1.5 across a cell of the
    coarse levels; sigma capped at 40 + 20 * level, so that a ray that starts in a deep cell loses at most ~0.1 of
    optical depth per sample there and goes on through the chain's other levels."""
    st = chain_tree(levels)
    lv = np.arange(levels, dtype=np.float64)
    cell = 2.0 ** (1 - (lv + 1))
    tau = 0.1 + 1.4 * ((lv * 7) % 11) / 10
    d = np.zeros((levels, 8, 4), np.float32)
    d[..., 3] = np.minimum(tau / cell, 40.0 + 20.0 * lv)[:, None]
    d[..., 0] = (np.sin(lv * 1.3) * 2)[:, None]
    d[..., 1] = (np.cos(lv * 0.7) * 2)[:, None]
    d[..., 2] = ((lv % 5) - 2.0)[:, None]
    d[..., 2] += np.linspace(-0.5, 0.5, 8)[None, :]
    d[st.child.reshape(levels, 8) != 0] = 0.0
    st.data = d.astype(np.float16).reshape(levels, 2, 2, 2, 4)
    return st


def chain_leaf_centre(level: int):
    """Tree-space centre (float64) of a leaf at ``level`` (>= 1) of a chain with at least that many levels: the
    octant opposite the chain's internal child of the node at depth ``level - 1``."""
    c = np.zeros(3)
    for lv in range(level - 1):
        o = (5 * lv + 3) % 8
        c = c + np.array([(o >> 2) & 1, (o >> 1) & 1, o & 1]) * 2.0 ** -(lv + 1)
    o = ((5 * (level - 1) + 3) % 8) ^ 7
    return c + np.array([(o >> 2) & 1, (o >> 1) & 1, o & 1]) * 2.0 ** -level + 2.0 ** -(level + 1)


def sigma_bits_tree() -> synth.SynthTree:
    st = mixed_tree(6, basis=4, seed=41)
    cap = st.capacity
    d = st.data.reshape(cap * 8, st.data_dim).view(np.uint16).copy()
    d[:, -1] = SIGMA_BITS[np.arange(cap * 8) % len(SIGMA_BITS)]
    rows = np.arange(0, cap * 8, 3)
    d[rows, (rows // 3) % (st.data_dim - 1)] = COLOUR_BITS[rows % len(COLOUR_BITS)]
    d[st.child.reshape(-1) != 0] = 0
    st.data = d.view(np.float16).reshape(st.data.shape)
    return st


TREES = ["mixed_sh16", "mixed_sh9", "mixed_sh25", "mixed_sh1", "mixed_rgba", "mixed_sg9", "mixed_asg4",
         "root_only", "root_mixed", "chain22", "chain23", "aniso", "aniso_ndc", "sigma_bits", "quant_mixed"]
NDC = {"aniso_ndc": (40.0, 30.0, 36.0)}


def edge_tree(name: str):
    """-> (SynthTree with decoded data, npz dict of the file when it is not the tree itself (quantised) or None)."""
    mixed = {"mixed_sh16": (16, "SH", 101), "mixed_sh9": (9, "SH", 102), "mixed_sh25": (25, "SH", 103),
             "mixed_sh1": (1, "SH", 104), "mixed_rgba": (-1, "RGBA", 105), "mixed_sg9": (9, "SG", 106),
             "mixed_asg4": (4, "ASG", 107)}
    if name in mixed:
        basis, fmt, seed = mixed[name]
        return mixed_tree(8, basis, fmt, seed), None
    if name == "root_only":
        return root_only_tree(), None
    if name == "root_mixed":            # 4 root leaves, 4 subtrees down to level 4
        return mixed_tree(4, 9, "SH", 108, p_refine=0.4, root_leaves=(0, 3, 5, 6)), None
    if name.startswith("chain"):
        return varied_chain(int(name[len("chain"):])), None
    if name in ("aniso", "aniso_ndc"):
        st = mixed_tree(6, 16, "SH", 109)
        if name == "aniso":
            st.offset = np.array([0.4132, 0.5378, 0.4719], np.float32)
            st.invradius3 = np.array([0.2917, 0.4311, 0.3779], np.float32)
        else:                       # the NDC frustum maps to [-1, 1]^2 x [-1, 1]: a box around it, off centre
            st.offset = np.array([0.48, 0.53, 0.55], np.float32)
            st.invradius3 = np.array([0.45, 0.41, 0.47], np.float32)
        return st, None
    if name == "sigma_bits":
        return sigma_bits_tree(), None
    if name == "quant_mixed":
        from volrend_b200 import N3Tree
        st = mixed_tree(6, 16, "SH", 110)
        npz = synth.quantise_tree(st, n_retain=1, seed=3)
        host = N3Tree(gpu_decode=False)
        host.load_npz(npz)                              # the reference's CPU decode (n3tree.cpp:279-340)
        st.data = host.data_.copy()
        return st, npz
    raise KeyError(name)


def tree_file_arrays(st: synth.SynthTree, npz) -> dict:
    """The arrays of the case's tree.npz: the quantised ones when there are, else the tree's."""
    return npz if npz is not None else st.npz_dict()


def write_tree_file(name: str, st: synth.SynthTree, npz, path: str) -> None:
    """tree.npz of case ``name`` at ``path``, with the ``*_poses_bounds.npy`` that makes the loaders use NDC
    (n3tree.cpp:22-52) for the NDC cases."""
    np.savez(path, **tree_file_arrays(st, npz))
    pb = path[:-4] + "_poses_bounds.npy"
    if name in NDC:
        p = np.zeros((1, 17), np.float32)
        p[0, 0] = p[0, 6] = p[0, 12] = 1.0          # identity rotation
        p[0, 9], p[0, 4], p[0, 14] = NDC[name]      # width, height, focal (n3tree.cpp:27-29)
        p[0, 15], p[0, 16] = 1.0, 10.0
        np.save(pb, p)
    elif os.path.exists(pb):
        os.remove(pb)


# ----------------------------------------------------------------------------------------------------------- views
W0, H0 = 40, 30         # even: pixel column 20 and row 15 have exactly zero camera-space x and y
AXES = {"px": (1, 0, 0), "nx": (-1, 0, 0), "py": (0, 1, 0), "ny": (0, -1, 0), "pz": (0, 0, 1), "nz": (0, 0, -1)}
VIEWS_ALL = list(AXES) + ["inside", "face", "graze", "bbox_degen", "bbox_inv", "aspect", "wide", "odd", "one",
                          "column", "composite"]
VIEWS_SHORT = ["px", "nz", "inside", "face", "odd"]
# chain views from inside a leaf k levels above the deepest one, looking along the given direction
DEEP = {"deep": (0, (-0.4, 1.0, 0.3)), "deep1": (1, (0.7, -0.2, 0.5)), "deep2": (2, (-0.3, -0.6, -0.9))}


def _to_world(st, t) -> np.ndarray:
    return (np.asarray(t, np.float64) - st.offset.astype(np.float64)) / st.invradius3.astype(np.float64)


def _axis_pose(st, axis, dist=2.5):
    a = np.asarray(axis, np.float64)
    half = 0.5 / st.invradius3.astype(np.float64)
    eye = _to_world(st, [0.5, 0.5, 0.5]) + a * dist * half.max()
    up = (0, 1, 0) if a[2] != 0 else (0, 0, 1)
    return synth.look_at_c2w(eye, target=eye - a, up=up)


def composite_layers():
    """(existing RGBA8, ray-distance limit) of the composite views: limits 0, -1, +inf, NaN, -inf and NaN in stripes of
    5 columns, finite limits in the rest of the frame."""
    rng = np.random.default_rng(7)
    rgba = rng.integers(0, 256, (H0, W0, 4)).astype(np.uint8)
    depth = rng.uniform(1.5, 4.0, (H0, W0)).astype(np.float32)
    for k, v in enumerate([0.0, -1.0, np.inf, np.nan, -np.inf, np.nan]):
        depth[:, k * 5:(k + 1) * 5] = v
    return rgba, depth


def view(name: str, tree_name: str, st):
    """-> (W, H, fx, fy, row-major c2w 4x4, options dict, composite (rgba8, depth) or None)."""
    if tree_name in NDC:        # forward-facing camera in front of the NDC frustum (volrend.cu:34-54)
        pose = np.eye(4, dtype=np.float32)
        pose[:3, 3] = [0.05, -0.03, 0.2]
        W, H = (W0, H0) if name != "odd" else (37, 23)
        return W, H, 36.0, 36.0, pose, {}, None
    f = 36.0
    if name in AXES:
        return W0, H0, f, f, _axis_pose(st, AXES[name]), {}, None
    if name == "inside":        # camera inside the box: every ray starts at t = 0 in some leaf
        eye = _to_world(st, [0.55, 0.38, 0.61])
        return W0, H0, 14.0, 14.0, synth.look_at_c2w(eye, target=eye + np.array([0.3, 1.0, -0.2])), {}, None
    if name in DEEP:            # camera at the centre of a chain leaf k levels above the deepest: the first lookup of
        k, look = DEEP[name]    # every ray is there, and the rays go on through the chain's other levels
        eye = _to_world(st, chain_leaf_centre(st.depth - k))
        return W0, H0, 14.0, 14.0, synth.look_at_c2w(eye, target=eye + np.asarray(look)), {}, None
    if name == "face":          # on the dyadic planes y = 1/2 and z = 5/8 looking along +x: the centre column runs
        eye = _to_world(st, [-0.5, 0.5, 0.625])         # inside the plane y = 1/2, the centre row inside z = 5/8
        return W0, H0, f, f, synth.look_at_c2w(eye, target=eye + np.array([1.0, 0.0, 0.0])), {}, None
    if name == "graze":         # along -x from tree x = 4.5: the rays of column 0 and row 0 meet the box's front face
        # (x = 0.75) on its edges y = 0.25 and z = 0.25, and the outer rays leave through the side faces
        return (W0, H0, 300.0, 225.0, _axis_pose(st, AXES["px"], dist=8.0),
                dict(render_bbox=[0.25, 0.25, 0.25, 0.75, 0.75, 0.75]), None)
    if name == "bbox_degen":
        return W0, H0, f, f, _axis_pose(st, (0.6, -0.64, 0.48)), dict(render_bbox=[0.5, 0.25, 0.5, 0.5, 0.75, 0.5]), None
    if name == "bbox_inv":
        return W0, H0, f, f, _axis_pose(st, (0.6, -0.64, 0.48)), dict(render_bbox=[0.8, 0.7, 0.9, 0.2, 0.3, 0.1]), None
    if name == "aspect":
        return W0, H0, 50.0, 22.0, _axis_pose(st, (-0.36, 0.48, 0.8)), {}, None
    if name == "wide":          # ~160 degree horizontal field of view
        return W0, H0, 3.5, 3.5, _axis_pose(st, (0.0, -0.6, 0.8), dist=1.2), {}, None
    if name == "odd":
        return 37, 23, 33.0, 33.0, _axis_pose(st, (0.48, 0.6, -0.64)), {}, None
    if name == "one":
        return 1, 1, 1000.0, 1000.0, _axis_pose(st, (0.36, -0.8, 0.48)), {}, None
    if name == "column":
        return 1, 64, 60.0, 60.0, _axis_pose(st, (-0.8, -0.36, 0.48)), {}, None
    if name == "composite":
        return W0, H0, f, f, _axis_pose(st, (0.48, -0.6, 0.64)), {}, composite_layers()
    raise KeyError(name)


def views_for(tree_name: str):
    if tree_name == "mixed_sh16":
        return VIEWS_ALL
    if tree_name in NDC:
        return ["ndc", "odd"]
    if tree_name.startswith("chain"):
        return VIEWS_SHORT + list(DEEP)
    if tree_name.startswith("root") or tree_name == "aniso":
        return VIEWS_SHORT + ["py", "pz", "composite"]
    return VIEWS_SHORT


OPTIONS = {"default": {}, "thresh0": dict(sigma_thresh=0.0), "thresh_neg": dict(sigma_thresh=-1.0)}


def options_for(tree_name: str):
    return list(OPTIONS) if tree_name == "sigma_bits" else ["default"]


FRAMES = [f"{t}.{v}.{o}" for t in TREES for v in views_for(t) for o in options_for(t)]


def frame(name: str, st=None):
    """-> (tree name, W, H, fx, fy, pose, options dict, composite or None) of frame ``tree.view.options``."""
    t, v, o = name.split(".")
    if st is None:
        st = edge_tree(t)[0]
    W, H, fx, fy, pose, kw, comp = view(v, t, st)
    kw = dict(kw)
    kw.update(OPTIONS[o])
    return t, W, H, fx, fy, pose, kw, comp


def frames_of(tree_name: str):
    return [f for f in FRAMES if f.split(".")[0] == tree_name]


def oracle_render(name: str, st, tile=None, nthreads=None):
    """The CPU oracle's (float RGBA, RGBA8, counters) of frame ``name`` of tree ``st``."""
    from oracle import binding as ob
    t, W, H, fx, fy, pose, kw, comp = frame(name, st)
    ot = ob.OracleTree.from_synth(st, ndc=NDC.get(t))
    cam = ob.make_camera(W, H, fx, fy, synth.c2w_to_colmajor12(pose))
    rin, din = comp if comp is not None else (None, None)
    return ob.render(ot, cam, ob.make_options(**kw), tile=tile, rgba_in=rin, depth_in=din, nthreads=nthreads)


# ------------------------------------------------------------------------------------------------ stored frames
def golden_path(name: str) -> str:
    return os.path.join(REF_DIR, "edge_" + name.replace(".", "__") + ".npz")


def record(name: str, f: np.ndarray, u: np.ndarray) -> dict:
    """What is stored of the reference's float RGBA f and RGBA8 u of frame ``name``."""
    from golden_cases import ref_frame_record
    rec = ref_frame_record(name, f, u)
    if f.shape[0] * f.shape[1] <= WHOLE_MAX_PIXELS:
        rec["f32"], rec["u8"] = f, u
    return rec


def _sha(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def load(name: str):
    return np.load(golden_path(name), allow_pickle=False)


def is_composite(name: str) -> bool:
    return name.split(".")[1] == "composite"


def assert_composite_tap(name: str, f: np.ndarray, ref: np.ndarray) -> None:
    """Float RGBA of a composite frame against the reference's float tap: alpha exact, colour within 1 ulp."""
    ulps = np.abs(np.ascontiguousarray(f, np.float32).view(np.int32).astype(np.int64)
                  - np.ascontiguousarray(ref, np.float32).view(np.int32).astype(np.int64)).reshape(-1, 4)
    assert ulps[:, :3].max() <= 1 and ulps[:, 3].max() == 0, (name, int(ulps.max()))


def assert_identical(name: str, f: np.ndarray, u: np.ndarray | None) -> None:
    """Float RGBA (and bytes, when given) bit-identical to the stored reference frame.  Composite frames: the
    reference's float tap (oracle/ref_harness.cu) restates the final ``out += rgba_in / 255 * (1 - alpha)`` of
    volrend.cu:159-163 in a kernel of its own, which nvcc contracts differently from the byte kernel, so there colour
    channels may differ by 1 ulp; alpha and the bytes of the reference's own kernel stay exact."""
    z = load(name)
    assert f.shape == tuple(z["shape"]), (name, f.shape)
    idx = z["index"]
    fs = np.ascontiguousarray(f, np.float32).reshape(-1, 4)[idx]
    if is_composite(name):
        if "f32" in z:
            assert_composite_tap(name, f, z["f32"])
        else:
            assert_composite_tap(name, fs, z["f32_sample"])
        assert u is not None and _sha(np.ascontiguousarray(u, np.uint8)) == str(z["sha_u8"]), name
        return
    bad = (fs.view(np.uint32) != z["f32_sample"].view(np.uint32)).any(-1)
    assert not bad.any(), (name, "float RGBA differs from the reference kernel", int(bad.sum()),
                           float(np.nanmax(np.abs(fs - z["f32_sample"]))))
    assert _sha(np.ascontiguousarray(f, np.float32)) == str(z["sha_f32"]), (name, "float RGBA differs outside the sample")
    if u is not None:
        assert np.array_equal(u.reshape(-1, 4)[idx], z["u8_sample"]), name
        assert _sha(np.ascontiguousarray(u, np.uint8)) == str(z["sha_u8"]), name
