"""Synthetic N3Tree (PlenOctree) + camera-pose generators.

No real scene (lego/drums ``tree.npz``) exists on the build or GPU boxes and there is
no network, so every BASELINE.json config is driven by seeded procedural stand-ins
written in exactly the on-disk schema the unchanged volrend loader accepts
(reference ``src/n3tree.cpp:228-362``; schema in SURVEY.md App. C):

* ``child``  int32 ``[capacity, 2, 2, 2]``  relative node offset, 0 = leaf
  (``include/volrend/internal/n3tree_query.hpp:36-46``)
* ``data``   fp16  ``[capacity, 2, 2, 2, data_dim]`` leaf record
  ``[R coeffs | G coeffs | B coeffs | sigma]`` (``include/volrend/cuda/rt_core.cuh:118-165``)
* ``offset`` f32[3], ``invradius3`` f32[3]  world -> tree: ``tree = offset + scale * world``
* ``data_dim`` int64, ``data_format`` unicode string ("SH16", "SH1", "RGBA", ...)

Pose files follow ``scripts/extract_test_poses.py:14-30`` / ``main_headless.cpp:40-74``
(whitespace 4x4 row-major camera-to-world, NeRF/OpenGL convention).
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass, field

import numpy as np

# ----------------------------------------------------------------------------------------
# signed distance fields (tree coordinates, unit cube [0,1]^3)
# ----------------------------------------------------------------------------------------


def _sd_box(p, c, h):
    q = np.abs(p - np.asarray(c, np.float32)) - np.asarray(h, np.float32)
    return np.linalg.norm(np.maximum(q, 0.0), axis=-1) + np.minimum(q.max(axis=-1), 0.0)


def _sd_sphere(p, c, r):
    return np.linalg.norm(p - np.asarray(c, np.float32), axis=-1) - r


def _sd_cyl_z(p, c, r, hz):
    d = p - np.asarray(c, np.float32)
    dxy = np.sqrt(d[..., 0] ** 2 + d[..., 1] ** 2) - r
    dz = np.abs(d[..., 2]) - hz
    return np.minimum(np.maximum(dxy, dz), 0.0) + np.sqrt(
        np.maximum(dxy, 0.0) ** 2 + np.maximum(dz, 0.0) ** 2)


def _sd_torus_z(p, c, R, r):
    d = p - np.asarray(c, np.float32)
    q = np.sqrt(d[..., 0] ** 2 + d[..., 1] ** 2) - R
    return np.sqrt(q * q + d[..., 2] ** 2) - r


def sdf_shell(p):
    """Config 1: a sphere of radius 0.325 about the cube centre (shell r in [0.25, 0.4])."""
    return _sd_sphere(p, (0.5, 0.5, 0.5), 0.325)


def sdf_lego(p):
    """Config 2/3/5 stand-in: a bulldozer-ish union of boxes, studs, wheels and a boom so
    the surface has lego-like area, concavities and thin parts."""
    d = _sd_box(p, (0.5, 0.5, 0.36), (0.30, 0.17, 0.06))            # chassis
    d = np.minimum(d, _sd_box(p, (0.42, 0.5, 0.50), (0.12, 0.13, 0.085)))  # cabin
    d = np.minimum(d, _sd_box(p, (0.66, 0.5, 0.46), (0.10, 0.10, 0.04)))   # hood
    d = np.minimum(d, _sd_box(p, (0.86, 0.5, 0.33), (0.025, 0.24, 0.09)))  # blade
    for sy in (-1.0, 1.0):                                           # tracks + wheels
        d = np.minimum(d, _sd_box(p, (0.5, 0.5 + sy * 0.215, 0.27), (0.33, 0.035, 0.055)))
        for wx in (0.24, 0.41, 0.59, 0.76):
            c = np.array((wx, 0.5 + sy * 0.215, 0.27), np.float32)
            dd = p - c
            rxz = np.sqrt(dd[..., 0] ** 2 + dd[..., 2] ** 2) - 0.07
            dy = np.abs(dd[..., 1]) - 0.045
            d = np.minimum(d, np.minimum(np.maximum(rxz, dy), 0.0) + np.sqrt(
                np.maximum(rxz, 0.0) ** 2 + np.maximum(dy, 0.0) ** 2))
    for sx in range(6):                                              # studs
        for sy in range(3):
            d = np.minimum(d, _sd_cyl_z(p, (0.27 + 0.09 * sx, 0.41 + 0.09 * sy, 0.43), 0.024, 0.016))
    d = np.minimum(d, _sd_torus_z(p, (0.36, 0.5, 0.66), 0.075, 0.018))   # beacon ring
    d = np.minimum(d, _sd_cyl_z(p, (0.36, 0.5, 0.60), 0.012, 0.05))
    d = np.minimum(d, _sd_box(p, (0.74, 0.5, 0.60), (0.16, 0.02, 0.02)))  # boom
    return d


def sdf_drums(p):
    """Config 3 stand-in: several thin drum shells / cymbal discs (lots of thin surface)."""
    d = np.full(p.shape[:-1], 1e9, np.float32)
    for (cx, cy, cz, r, h) in ((0.35, 0.40, 0.40, 0.13, 0.08), (0.65, 0.40, 0.40, 0.13, 0.08),
                               (0.50, 0.66, 0.34, 0.18, 0.12), (0.28, 0.66, 0.46, 0.09, 0.05),
                               (0.72, 0.66, 0.46, 0.09, 0.05)):
        d = np.minimum(d, _sd_cyl_z(p, (cx, cy, cz), r, h))
    for (cx, cy, cz, r) in ((0.22, 0.30, 0.70, 0.12), (0.78, 0.30, 0.72, 0.12), (0.5, 0.25, 0.76, 0.10)):
        d = np.minimum(d, _sd_cyl_z(p, (cx, cy, cz), r, 0.006))
        d = np.minimum(d, _sd_cyl_z(p, (cx, cy, cz - 0.2), 0.008, 0.2))
    return d


def sdf_gyroid(p):
    """Config 4: gyroid sheet clipped to a ball -- huge, thin, view-independent surface."""
    w = 2.0 * math.pi * 3.0
    q = p * np.float32(w)
    g = (np.sin(q[..., 0]) * np.cos(q[..., 1]) + np.sin(q[..., 1]) * np.cos(q[..., 2])
         + np.sin(q[..., 2]) * np.cos(q[..., 0]))
    d = np.abs(g) / np.float32(w * 1.5)          # ~distance to the sheet (|grad| <= 1.5 w)
    ball = _sd_sphere(p, (0.5, 0.5, 0.5), 0.46)
    return np.maximum(d, ball)


def sdf_gyroid_small(p):
    """Config 4 (depth 11): the same gyroid sheet clipped to a small ball, so that a 2048^3
    refinement stays around a million nodes."""
    w = 2.0 * math.pi * 4.0
    q = p * np.float32(w)
    g = (np.sin(q[..., 0]) * np.cos(q[..., 1]) + np.sin(q[..., 1]) * np.cos(q[..., 2])
         + np.sin(q[..., 2]) * np.cos(q[..., 0]))
    d = np.abs(g) / np.float32(w * 1.5)
    ball = _sd_sphere(p, (0.5, 0.5, 0.5), 0.17)
    return np.maximum(d, ball)


def _scaled(fn, s):
    """Shrink a shape about the cube centre by 1/s (keeps distances metric)."""
    def g(p):
        return fn((p - np.float32(0.5)) * np.float32(s) + np.float32(0.5)) / np.float32(s)
    return g


SDFS = {"shell": sdf_shell, "lego": _scaled(sdf_lego, 1.25), "drums": _scaled(sdf_drums, 1.35),
        "gyroid": sdf_gyroid, "gyroid_small": sdf_gyroid_small}


# ----------------------------------------------------------------------------------------
# tree container
# ----------------------------------------------------------------------------------------


@dataclass
class SynthTree:
    child: np.ndarray            # int32 [cap,2,2,2]
    data: np.ndarray             # fp16  [cap,2,2,2,data_dim]
    offset: np.ndarray           # f32[3]
    invradius3: np.ndarray       # f32[3]
    data_dim: int
    data_format: str
    depth: int                   # max leaf depth (root's children are depth 1)
    extra: np.ndarray | None = None
    meta: dict = field(default_factory=dict)

    @property
    def capacity(self) -> int:
        return int(self.child.shape[0])

    def nbytes(self) -> int:
        return self.child.nbytes + self.data.nbytes

    def npz_dict(self) -> dict:
        """The arrays of the App. C schema, as ``np.load`` of the saved file returns them."""
        kw = dict(data_dim=np.int64(self.data_dim), data_format=np.array(self.data_format),
                  invradius3=self.invradius3.astype(np.float32), offset=self.offset.astype(np.float32),
                  child=self.child, data=self.data)
        if self.extra is not None:
            kw["extra_data"] = self.extra.astype(np.float32)
        return kw

    def save_npz(self, path: str) -> None:
        """Write the App. C schema; readable by the unchanged loader (n3tree.cpp:228-362)."""
        np.savez(path, **self.npz_dict())


def _hash_u01(ix, iy, iz, salt):
    """Cheap deterministic per-cell uniform in [0,1) (so trees don't depend on traversal order)."""
    h = (ix.astype(np.uint64) * np.uint64(73856093)) ^ (iy.astype(np.uint64) * np.uint64(19349663)) \
        ^ (iz.astype(np.uint64) * np.uint64(83492791)) ^ np.uint64(salt * 2654435761 & 0xFFFFFFFF)
    h ^= h >> np.uint64(13)
    h *= np.uint64(0x5BD1E995)
    h ^= h >> np.uint64(15)
    return ((h & np.uint64(0xFFFFFF)).astype(np.float32)) / np.float32(1 << 24)


def make_tree(kind: str = "lego", depth: int = 9, basis_dim: int = 16, seed: int = 0,
              fmt: str = "SH", full: bool = False, band_cells: float = 2.0,
              sigma_scale: float | None = None, opaque_cells: float = 5.0, world_radius: float = 1.5,
              coeff_std: float = 0.6, max_nodes: int = 6_000_000) -> SynthTree:
    """Build a sparse (or ``full``) octree whose finest cells hug ``SDFS[kind]``.

    A cell at level L (grid 2^L) is refined while it intersects the band
    ``|sdf| < band_cells * finest_cell``; finest-level cells inside the band get
    sigma > 0 and random SH/SG/RGB coefficients, every other leaf is empty (sigma = 0).
    ``fmt``: "SH" | "SG" | "ASG" | "RGBA".
    """
    rng = np.random.default_rng(seed)
    sdf = SDFS[kind]
    if fmt == "RGBA":
        data_dim, basis = 4, -1
        data_format = "RGBA"
    else:
        data_dim, basis = 3 * basis_dim + 1, basis_dim
        data_format = f"{fmt}{basis_dim}"
    finest = 1.0 / (1 << depth)
    band = band_cells * finest
    offs = np.stack(np.meshgrid(np.arange(2), np.arange(2), np.arange(2), indexing="ij"), -1).astype(np.int64)

    level_coords = [np.zeros((1, 3), np.int64)]
    level_refine = []            # per node-level: bool [n,2,2,2] which children are internal
    for lvl in range(depth):
        coords = level_coords[-1]
        cc = coords[:, None, None, None, :] * 2 + offs[None]           # [n,2,2,2,3] child-cell coords
        cell = 1.0 / (1 << (lvl + 1))
        if lvl + 1 < depth:
            if full:
                refine = np.ones(cc.shape[:-1], bool)
            else:
                ctr = ((cc.astype(np.float32) + 0.5) * np.float32(cell))
                d = np.empty(cc.shape[:-1], np.float32)
                step = max(1, 2_000_000 // 8)
                for s in range(0, len(coords), step):
                    d[s:s + step] = sdf(ctr[s:s + step])
                refine = np.abs(d) < (0.8660254 * cell + band)
                if lvl == 0:
                    refine[:] = True                                    # keep the top well-formed
        else:
            refine = np.zeros(cc.shape[:-1], bool)
        level_refine.append(refine)
        nxt = cc[refine]
        if lvl + 1 < depth:
            level_coords.append(nxt.reshape(-1, 3))
        if sum(len(c) for c in level_coords) > max_nodes:
            raise RuntimeError("synthetic tree exceeds max_nodes; lower depth or band_cells")

    counts = [len(c) for c in level_coords]
    starts = np.concatenate([[0], np.cumsum(counts)])
    cap = int(starts[-1])
    child = np.zeros((cap, 2, 2, 2), np.int32)
    for lvl in range(depth - 1):
        refine = level_refine[lvl]
        n = counts[lvl]
        node_ids = (starts[lvl] + np.arange(n, dtype=np.int64))[:, None, None, None]
        child_ids = np.zeros(refine.shape, np.int64)
        child_ids[refine] = starts[lvl + 1] + np.arange(int(refine.sum()), dtype=np.int64)
        rel = np.where(refine, child_ids - node_ids, 0)
        child[starts[lvl]:starts[lvl] + n] = rel.astype(np.int32)

    data = np.zeros((cap, 2, 2, 2, data_dim), np.float16)
    # finest-level leaves: children of the last node level
    coords = level_coords[depth - 1]
    cc = coords[:, None, None, None, :] * 2 + offs[None]
    ctr = ((cc.astype(np.float32) + 0.5) * np.float32(finest))
    d = np.empty(cc.shape[:-1], np.float32)
    step = max(1, 2_000_000 // 8)
    for s in range(0, len(coords), step):
        d[s:s + step] = sdf(ctr[s:s + step])
    inside = np.abs(d) < band
    if sigma_scale is None:
        # T < 0.01 after ~opaque_cells finest cells: sigma * (cell * 2*world_radius) * n ~= 4.6
        sigma_scale = 4.6 / (opaque_cells * finest * 2.0 * world_radius)
    u = _hash_u01(cc[..., 0], cc[..., 1], cc[..., 2], seed + 1)
    v = _hash_u01(cc[..., 0], cc[..., 1], cc[..., 2], seed + 2)
    sigma = sigma_scale * np.exp((u - 0.5) * 2.0)                       # log-uniform x[1/e, e]
    fuzz = v < 0.08                                                    # a little sub-threshold haze
    sigma = np.where(fuzz, v * 0.25, sigma)
    sigma = np.where(inside, sigma, 0.0).astype(np.float32)
    sigma = np.minimum(sigma, 60000.0)
    base = int(starts[depth - 1])
    leaf_block = data[base:base + len(coords)]
    leaf_block[..., data_dim - 1] = sigma.astype(np.float16)
    nz = inside
    n_nz = int(nz.sum())
    if fmt == "RGBA":
        rgb = rng.random((n_nz, 3), dtype=np.float32)
        leaf_block[nz, :3] = rgb.astype(np.float16)
    else:
        co = rng.standard_normal((n_nz, 3 * basis), dtype=np.float32) * np.float32(coeff_std)
        # DC term carries most of the colour, like trained PlenOctrees
        co[:, 0::basis] *= 2.0
        if basis > 1:
            falloff = (1.0 / (1.0 + np.sqrt(np.arange(basis, dtype=np.float32))))
            co *= np.tile(falloff, 3)[None, :] * 1.6
        leaf_block[nz, :3 * basis] = co.astype(np.float16)
    if full and depth <= 6:
        pass
    extra = None
    if fmt == "SG":
        # [lambda, mu_x, mu_y, mu_z] per lobe (lumisphere.hpp:30-36)
        mu = rng.standard_normal((basis, 3)).astype(np.float32)
        mu /= np.linalg.norm(mu, axis=1, keepdims=True)
        lam = rng.uniform(0.5, 8.0, (basis, 1)).astype(np.float32)
        extra = np.concatenate([lam, mu], 1)
    elif fmt == "ASG":
        # [lambda_x, lambda_y, mu_x(3), mu_y(3), mu_z(3)] per lobe (lumisphere.hpp:14-28)
        ex = np.zeros((basis, 11), np.float32)
        for i in range(basis):
            q, _ = np.linalg.qr(rng.standard_normal((3, 3)))
            ex[i, 0:2] = rng.uniform(0.5, 6.0, 2)
            ex[i, 2:5], ex[i, 5:8], ex[i, 8:11] = q[:, 0], q[:, 1], q[:, 2]
        extra = ex
    inv = np.full(3, 1.0 / (2.0 * world_radius), np.float32)
    return SynthTree(child=child, data=data, offset=np.full(3, 0.5, np.float32), invradius3=inv,
                     data_dim=data_dim, data_format=data_format, depth=depth, extra=extra,
                     meta=dict(kind=kind, seed=seed, nodes_per_level=counts, shaded_leaves=n_nz,
                               sigma_scale=float(sigma_scale), world_radius=world_radius))


def make_config1_tree(seed: int = 0) -> SynthTree:
    """BASELINE config 1 (SURVEY.md 8d): full depth-4 SH1 tree, 585 nodes, shell-shaped sigma
    r in [0.25, 0.4] with sigma ~ U(5, 60), DC ~ N(0,1); world cube [-1,1]^3."""
    rng = np.random.default_rng(seed)
    t = make_tree("shell", depth=4, basis_dim=1, seed=seed, full=True, world_radius=1.0)
    offs = np.stack(np.meshgrid(np.arange(2), np.arange(2), np.arange(2), indexing="ij"), -1)
    # recompute finest-level leaves with the exact config-1 recipe
    cap = t.capacity
    n_last = 512
    base = cap - n_last
    # coordinates of last-level nodes in BFS order (full tree => lexicographic refinement order)
    coords = np.zeros((1, 3), np.int64)
    for _ in range(3):
        coords = (coords[:, None, None, None, :] * 2 + offs[None]).reshape(-1, 3)
    cc = coords[:, None, None, None, :] * 2 + offs[None]
    ctr = (cc.astype(np.float32) + 0.5) / 16.0
    r = np.linalg.norm(ctr - 0.5, axis=-1)
    inside = (r >= 0.25) & (r <= 0.4)
    sigma = rng.uniform(5.0, 60.0, inside.shape).astype(np.float32)
    dc = rng.standard_normal(inside.shape + (3,)).astype(np.float32)
    blk = np.zeros((n_last, 2, 2, 2, 4), np.float16)
    blk[..., 3] = np.where(inside, sigma, 0.0).astype(np.float16)
    blk[..., :3] = dc.astype(np.float16)
    t.data[base:] = blk
    t.meta["shaded_leaves"] = int(inside.sum())
    return t


# ----------------------------------------------------------------------------------------
# cameras
# ----------------------------------------------------------------------------------------


def look_at_c2w(eye, target=(0.0, 0.0, 0.0), up=(0.0, 0.0, 1.0)) -> np.ndarray:
    """4x4 camera-to-world, NeRF/OpenGL convention: camera looks down -z, +y up
    (reference ``src/cuda/volrend.cu:27-28``, ``src/camera.cpp:47-55``)."""
    eye = np.asarray(eye, np.float64)
    back = eye - np.asarray(target, np.float64)
    back /= np.linalg.norm(back)
    right = np.cross(np.asarray(up, np.float64), back)
    right /= np.linalg.norm(right)
    upv = np.cross(back, right)
    m = np.eye(4)
    m[:3, 0], m[:3, 1], m[:3, 2], m[:3, 3] = right, upv, back, eye
    return m.astype(np.float32)


def nerf_synthetic_test_poses(n: int = 200, radius: float = 4.031128874, elev_deg: float = 30.0) -> np.ndarray:
    """The NeRF-synthetic ``transforms_test.json`` spiral: n views on a circle of the
    camera sphere (radius 4.0311), elevation 30 deg, azimuth sweeping 360 deg."""
    out = np.zeros((n, 4, 4), np.float32)
    el = math.radians(elev_deg)
    for i in range(n):
        az = 2.0 * math.pi * i / n
        eye = (radius * math.cos(el) * math.cos(az), radius * math.cos(el) * math.sin(az), radius * math.sin(el))
        out[i] = look_at_c2w(eye)
    return out


def random_sphere_poses(n: int, radius: float, seed: int = 0) -> np.ndarray:
    rng = np.random.default_rng(seed)
    out = np.zeros((n, 4, 4), np.float32)
    for i in range(n):
        v = rng.standard_normal(3)
        v /= np.linalg.norm(v)
        if abs(v[2]) > 0.95:
            v = np.array([0.6, 0.0, 0.8])
        out[i] = look_at_c2w(v * radius)
    return out


def config1_pose() -> np.ndarray:
    """Config 1 camera: world (0,-3.2,1.6) looking at the origin, +z up."""
    return look_at_c2w((0.0, -3.2, 1.6))


def focal_for(width: int, full_focal: float = 1111.11, full_width: int = 800) -> float:
    return full_focal * width / full_width


def write_pose_files(poses: np.ndarray, out_dir: str, fx: float, fy: float | None = None) -> list[str]:
    """Emit ``pose/NNNN.txt`` + ``intrinsics.txt`` as scripts/extract_test_poses.py:14-30 does."""
    os.makedirs(os.path.join(out_dir, "pose"), exist_ok=True)
    paths = []
    for i, p in enumerate(poses):
        path = os.path.join(out_dir, "pose", f"{i:04d}.txt")
        np.savetxt(path, p.reshape(4, 4), fmt="%.9g")
        paths.append(path)
    K = np.eye(4, dtype=np.float64)
    K[0, 0] = fx
    K[1, 1] = fx if fy is None else fy
    np.savetxt(os.path.join(out_dir, "intrinsics.txt"), K, fmt="%.9g")
    return paths


def c2w_to_colmajor12(c2w: np.ndarray) -> np.ndarray:
    """4x4 (or 3x4) row-major c2w -> the 12 floats of glm::mat4x3 (column-major: right, up,
    back, centre), i.e. what ``Camera::transform`` holds (camera.cpp:52-55)."""
    m = np.asarray(c2w, np.float32)[:3, :4]
    return np.ascontiguousarray(m.T).reshape(12).copy()


def quantise_tree(st: SynthTree, n_retain: int = 1, seed: int = 0) -> dict:
    """A compressed (scripts/compress_octree.py:93-118 schema) version of ``st``: geometry and sigma
    are kept, the colour coefficients come from random 65536-entry codebooks (one per quantised basis
    function) plus ``n_retain`` un-quantised leading basis functions.  Returns the npz dict; its
    decode (src/n3tree.cpp:279-340) defines the tree's colours."""
    fmt = st.data_format.rstrip("0123456789")
    if fmt == "RGBA":
        raise ValueError("RGBA trees are not quantised")
    n_total = (st.data_dim - 1) // 3
    n_quant = n_total - n_retain
    assert n_quant >= 1
    rng = np.random.default_rng(seed)
    cap = st.capacity
    colors = (rng.standard_normal((n_quant, 65536, 3), dtype=np.float32) * 0.8).astype(np.float16)
    qmap = rng.integers(0, 65536, (n_quant, cap, 2, 2, 2), dtype=np.int64).astype(np.uint16)
    npz = dict(data_dim=np.int64(st.data_dim), data_format=np.array(st.data_format),
               invradius3=st.invradius3.astype(np.float32), offset=st.offset.astype(np.float32), child=st.child,
               quant_colors=colors, quant_map=qmap, sigma=np.ascontiguousarray(st.data[..., st.data_dim - 1]))
    if n_retain > 0:
        npz["data_retained"] = (rng.standard_normal((n_retain, cap, 2, 2, 2, 3), dtype=np.float32) * 1.2).astype(np.float16)
    if st.extra is not None:
        npz["extra_data"] = st.extra.astype(np.float32)
    return npz
