"""numpy restatement of vr_tree_isosurface (DESIGN.md section 23): the level-L lattice of leaf sigma, the vertices on
its crossing edges in their fixed order and the faces of the generator's triangle table.  TEST INFRASTRUCTURE ONLY: the
CPU tests check its topology and geometry, the GPU tests check the kernel against it bit for bit.  It shares no code
with volrend_b200.isosurface or the kernel; the lattice values come from query_oracle's descent."""
from __future__ import annotations

import numpy as np

from oracle import query_oracle as qo
from tools import gen_iso_table as gen

_TABLE = gen.build_table()
MAX_TRIS = max(len(t) for t in _TABLE)
TRI_COUNT = np.array([len(t) for t in _TABLE], np.int64)
TRIS = np.zeros((256, MAX_TRIS, 3), np.int64)
for _c, _t in enumerate(_TABLE):
    if _t:
        TRIS[_c, :len(_t)] = np.array(_t, np.int64)
EDGE_CORNER = np.array([gen.edge_corner(e) for e in range(12)], np.int64)
EDGE_AXIS = np.arange(12) // 4
CORNER = np.array([gen.corner_xyz(c) for c in range(8)], np.int64)


def lattice(child, data, depth: int) -> np.ndarray:
    """float32 [R+2, R+2, R+2] (R = 2^depth): sigma of the leaf holding each lattice point (i + 0.5) / R of the unit
    cube, index i + 1 along x, y, z; padding (index 0 and R + 1) is 0.  NaN reads as 0, +-inf as +-65504."""
    R = 1 << depth
    c = (np.arange(R, dtype=np.float32) + np.float32(0.5)) / np.float32(R)
    pts = np.stack(np.meshgrid(c, c, c, indexing="ij"), -1).reshape(-1, 3)
    rows, _, _ = qo.query(child, data, np.zeros(3, np.float32), np.ones(3, np.float32), pts)
    s = rows[:, -1].astype(np.float32)
    s = np.where(np.isnan(s), np.float32(0), s)
    s = np.clip(s, np.float32(-65504), np.float32(65504)).astype(np.float32)
    out = np.zeros((R + 2,) * 3, np.float32)
    out[1:-1, 1:-1, 1:-1] = s.reshape(R, R, R)
    return out


def mesh(s: np.ndarray, level: float, offset=(0.0, 0.0, 0.0), scale=(1.0, 1.0, 1.0)) -> dict:
    """The isosurface of a padded lattice ``s`` [R+2]^3 (index = lattice index + 1) at ``level``:
    ``pos`` float32 [n, 3] world positions, ``faces`` uint32 [m, 3], ``inside`` int64 [n, 3] lattice indices of each
    vertex's inside endpoint, ``edge`` int64 [n, 4] its owner point (lattice index) and axis."""
    s = np.asarray(s, np.float32)
    n1 = s.shape[0]
    R = n1 - 2
    lv = np.float32(level)
    ins = s > lv
    cross = np.zeros(s.shape + (3,), bool)
    cross[:-1, :, :, 0] = ins[:-1] != ins[1:]
    cross[:, :-1, :, 1] = ins[:, :-1] != ins[:, 1:]
    cross[:, :, :-1, 2] = ins[:, :, :-1] != ins[:, :, 1:]
    flat = cross.reshape(-1)
    vid = (np.cumsum(flat) - 1).astype(np.int64).reshape(cross.shape)
    p, d = np.nonzero(cross.reshape(-1, 3))
    g = np.stack(np.unravel_index(p, s.shape), -1)                     # padded owner point
    e = np.eye(3, dtype=np.int64)[d]
    sa, sb = s[tuple(g.T)], s[tuple((g + e).T)]
    t = ((lv - sa) / (sb - sa)).astype(np.float32)
    c = (g - 1).astype(np.float32) + np.float32(0.5)
    c[np.arange(len(d)), d] = (c[np.arange(len(d)), d] + t).astype(np.float32)
    u = (c / np.float32(R)).astype(np.float32)
    off = np.asarray(offset, np.float32)[None, :]
    sc = np.asarray(scale, np.float32)[None, :]
    pos = ((u - off) / sc).astype(np.float32)
    a_in = ins[tuple(g.T)]
    inside = np.where(a_in[:, None], g, g + e) - 1
    # faces: cubes by lower corner in C order, triangles in table order
    case = np.zeros((R + 1,) * 3, np.int64)
    for k in range(8):
        x, y, z = CORNER[k]
        case |= ins[x:x + R + 1, y:y + R + 1, z:z + R + 1].astype(np.int64) << k
    cubes = np.nonzero(TRI_COUNT[case.reshape(-1)])[0]
    cc = case.reshape(-1)[cubes]
    lo = np.stack(np.unravel_index(cubes, case.shape), -1)
    cnt = TRI_COUNT[cc]
    rep = np.repeat(np.arange(len(cubes)), cnt)
    tri = np.arange(len(rep)) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    edges = TRIS[cc[rep], tri]                                          # [m, 3]
    pt = lo[rep][:, None, :] + CORNER[EDGE_CORNER[edges]]
    faces = vid[pt[..., 0], pt[..., 1], pt[..., 2], EDGE_AXIS[edges]]
    assert (faces >= 0).all()
    return dict(pos=pos, faces=faces.astype(np.uint32), inside=inside.astype(np.int64),
                edge=np.concatenate([g - 1, d[:, None]], 1).astype(np.int64))


def isosurface(child, data, offset, scale, depth: int, level: float) -> dict:
    """:func:`mesh` of the tree's level-``depth`` lattice, in world coordinates of ``offset`` / ``scale``."""
    return mesh(lattice(child, data, depth), level, offset, scale)
