"""Host oracle of ``vr_tree_build`` (DESIGN.md section 21): every cell is inserted into a dict of nodes, creating its
ancestors on the way down from the root, then the nodes are numbered by a breadth-first walk, octants in order.  It
shares no code with ``volrend_b200.build``.

A node is keyed by its cell ``(level, x, y, z)`` (the root is ``(0, 0, 0, 0)``); each of its 8 slots is ``None`` (an
unlisted leaf, +0), ``("row", bytes)`` (a listed cell or, after a merge, a collapsed node) or ``("node", key)``.
"""
from __future__ import annotations

import numpy as np

MAX_LEVEL = 23
ROOT = (0, 0, 0, 0)


def _octant(x: int, y: int, z: int) -> int:
    return (x & 1) << 2 | (y & 1) << 1 | (z & 1)


def _node(nodes: dict, key) -> list:
    """The slots of node ``key``, created (with its ancestors) when missing.  A listed cell in the way is an overlap."""
    slots = nodes.get(key)
    if slots is not None:
        return slots
    level, x, y, z = key
    parent = _node(nodes, (level - 1, x >> 1, y >> 1, z >> 1))
    o = _octant(x, y, z)
    if parent[o] is not None:
        raise ValueError(f"cell {key} is inside a listed cell")
    parent[o] = ("node", key)
    slots = nodes[key] = [None] * 8
    return slots


def _merge(nodes: dict, zero: bytes) -> None:
    """Bottom-up, a node whose 8 slots are rows with equal bits (None reads +0) becomes that row in its parent."""
    for key in sorted(nodes, key=lambda k: -k[0]):
        if key == ROOT:
            continue
        slots = nodes[key]
        if any(s is not None and s[0] == "node" for s in slots):
            continue
        vals = {zero if s is None else s[1] for s in slots}
        if len(vals) != 1:
            continue
        level, x, y, z = key
        nodes[(level - 1, x >> 1, y >> 1, z >> 1)][_octant(x, y, z)] = ("row", vals.pop())
        del nodes[key]


def build(cells, rows, merge: bool = False):
    """``(child int32 [n_nodes, 2, 2, 2], data fp16 [n_nodes, 2, 2, 2, data_dim])`` of the cells ``[n, 4]`` (level, i,
    j, k) with fp16 ``rows`` ``[n, data_dim]``.  Raises ValueError for a level outside [1, 23], a coordinate outside
    [0, 2^level) and duplicate or overlapping cells."""
    cells = np.asarray(cells).reshape(-1, 4).astype(np.int64)
    rows = np.ascontiguousarray(np.asarray(rows, np.float16))
    if rows.ndim != 2 or rows.shape[0] != cells.shape[0]:
        raise ValueError(f"rows must have shape [{cells.shape[0]}, data_dim]")
    dd = rows.shape[1]
    bits = rows.view(np.uint16)
    nodes = {ROOT: [None] * 8}
    for n, (level, x, y, z) in enumerate(cells.tolist()):
        if not 1 <= level <= MAX_LEVEL:
            raise ValueError(f"cell {n}: level {level} outside [1, {MAX_LEVEL}]")
        if not all(0 <= v < 1 << level for v in (x, y, z)):
            raise ValueError(f"cell {n}: coordinate outside [0, 2^{level})")
        parent = _node(nodes, (level - 1, x >> 1, y >> 1, z >> 1))
        o = _octant(x, y, z)
        if parent[o] is not None:
            raise ValueError(f"cell {n} {(level, x, y, z)} is listed twice or contains a listed cell")
        parent[o] = ("row", bits[n].tobytes())
    zero = bytes(2 * dd)
    if merge:
        _merge(nodes, zero)
    order, index = [ROOT], {ROOT: 0}            # breadth first, octants in order
    for key in order:
        for s in nodes[key]:
            if s is not None and s[0] == "node":
                index[s[1]] = len(order)
                order.append(s[1])
    child = np.zeros((len(order), 8), np.int32)
    data = np.zeros((len(order), 8, dd), np.uint16)
    for i, key in enumerate(order):
        for o, s in enumerate(nodes[key]):
            if s is None:
                continue
            if s[0] == "node":
                child[i, o] = index[s[1]] - i
            else:
                data[i, o] = np.frombuffer(s[1], np.uint16)
    return child.reshape(-1, 2, 2, 2), data.view(np.float16).reshape(-1, 2, 2, 2, dd)
