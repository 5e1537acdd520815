"""numpy restatement of N3Tree::gen_wireframe (reference src/n3tree.cpp:365-434): the octree grid as line segments.
TEST INFRASTRUCTURE ONLY (the product generates it on the GPU, volrend_b200/csrc/vr_wire.cu).

Works from the host ``child`` array (int32 [capacity, 2, 2, 2], relative offsets, 0 = leaf) and restates:
* which cells: from the root (depth 0), a cell of a node of depth d is emitted when it is a leaf or d >= max_depth,
  otherwise the walk descends into it;
* their order: the reference's depth-first pre-order, octants x-major then y then z, which is ascending Morton order
  of the cell corners left-aligned to the deepest emitted level;
* their vertices: 24 per cell (12 edges), 9 float32 each, bounds ((float)i / 2^level - offset) / scale in float32.
"""
from __future__ import annotations

import numpy as np

VERTS_PER_CELL = 24
FLOATS_PER_CELL = VERTS_PER_CELL * 9


def _vertex_selectors() -> np.ndarray:
    """[24, 3] 0/1: whether vertex v lies on the low or the high bound of its cell along each axis.  For each (a, b)
    in (0,0), (0,1), (1,0), (1,1): the x-, y- and z-parallel edges whose two other axes (in axis order) take (a, b),
    each from its low end to its high end."""
    sel = []
    for a in (0, 1):
        for b in (0, 1):
            for edge in range(3):
                others = [ax for ax in range(3) if ax != edge]
                for end in (0, 1):
                    s = [0, 0, 0]
                    s[edge] = end
                    s[others[0]], s[others[1]] = a, b
                    sel.append(s)
    return np.asarray(sel, np.int64)


SEL = _vertex_selectors()


def cells(child, max_depth: int):
    """Emitted cells in the reference's order: (corner int64 [n, 3] on the grid of each cell's level, level [n])."""
    child = np.asarray(child, np.int32).reshape(-1, 8)
    octs = np.array([(i, j, k) for i in range(2) for j in range(2) for k in range(2)], np.int64)   # child order
    node = np.zeros(1, np.int64)
    corner = np.zeros((1, 3), np.int64)
    out_c, out_l = [], []
    depth = 0
    while node.size:
        c = child[node]                                          # [n, 8]
        cc = (corner[:, None, :] * 2 + octs[None]).reshape(-1, 3)
        link = c.reshape(-1).astype(np.int64)
        stop = (link == 0) | (depth >= max_depth)
        out_c.append(cc[stop])
        out_l.append(np.full(int(stop.sum()), depth + 1, np.int64))
        node = np.repeat(node, 8)[~stop] + link[~stop]
        corner = cc[~stop]
        depth += 1
    corner = np.concatenate(out_c)
    level = np.concatenate(out_l)
    lc = int(level.max())
    aligned = corner << (lc - level)[:, None]
    # Morton digits, most significant level first; np.lexsort takes its primary key last
    digits = [((aligned[:, 0] >> s) & 1) * 4 + ((aligned[:, 1] >> s) & 1) * 2 + ((aligned[:, 2] >> s) & 1)
              for s in range(lc)]
    order = np.lexsort(digits)
    return corner[order], level[order]


def wireframe(child, offset, scale, max_depth: int) -> np.ndarray:
    """The float32 vertex array gen_wireframe(max_depth) returns (flat, 9 floats per vertex)."""
    corner, level = cells(child, max_depth)
    off = np.asarray(offset, np.float32).reshape(3)
    sc = np.asarray(scale, np.float32).reshape(3)
    gs = (np.int64(1) << level).astype(np.float32)[:, None]
    lo = ((corner.astype(np.float32) / gs) - off) / sc
    hi = (((corner + 1).astype(np.float32)) / gs - off) / sc
    bounds = np.stack([lo, hi], 1)                                    # [n, 2, 3]
    v = np.zeros((corner.shape[0], VERTS_PER_CELL, 9), np.float32)
    for ax in range(3):
        v[:, :, ax] = bounds[:, SEL[:, ax], ax]
    v[:, :, 8] = 1.0
    return v.reshape(-1)
