"""Restatement of the total-variation prior between neighbouring leaves (DESIGN.md 20) -- TEST INFRASTRUCTURE.

Shares nothing with the device path (no wide tables, no slot map, no walk of the wireframe):
  * leaves: a plain recursive walk of ``child`` from the root gives every reachable leaf slot, its depth d (root's
    slots: 1) and its integer cell i in [0, 2^d)^3;
  * neighbours: n_a(s) is the leaf found by an integer descent from the root at the point (i + e_a) 2^-d (at depth k
    the octant bit of axis b is bit (24 - k) of that point on the 2^24 grid), none when i_a + 1 = 2^d;
  * energy and gradient in float64, straight from the formulas:
      E = sum_G (lam_G / N_leaf) sum_s sum_{c in G} sqrt(1e-8 + sum_a (v[n_a, c] - v[s, c])^2)
      term (s, c): -sum_a D_a / r to s, +D_a / r to n_a, times lam_G / N_leaf.
``neighbors_levels`` is a level-by-level (numpy) form of the same rules, for trees of millions of nodes; the tests
check it against the recursive form.
"""
import sys

import numpy as np

EPS = 1e-8
GRID = 24


def _links(child):
    child = np.asarray(child)
    return child.reshape(child.shape[0], 8).astype(np.int64)


def leaves(child):
    """-> list of (slot, depth, (ix, iy, iz)) of every reachable leaf, depth first."""
    ch = _links(child)
    out = []

    def walk(node, depth, x, y, z):
        for o in range(8):
            cx, cy, cz = 2 * x + ((o >> 2) & 1), 2 * y + ((o >> 1) & 1), 2 * z + (o & 1)
            c = int(ch[node, o])
            if c != 0:
                walk(node + c, depth + 1, cx, cy, cz)
            else:
                out.append((node * 8 + o, depth, (cx, cy, cz)))

    limit = sys.getrecursionlimit()
    sys.setrecursionlimit(max(limit, 1000))
    try:
        walk(0, 1, 0, 0, 0)
    finally:
        sys.setrecursionlimit(limit)
    return out


def leaf_at(child, p):
    """Slot of the leaf holding the point p (three ints on the 2^24 grid of the unit cube)."""
    ch = _links(child)
    node, depth = 0, 1
    while True:
        o = (((p[0] >> (GRID - depth)) & 1) << 2) | (((p[1] >> (GRID - depth)) & 1) << 1) | ((p[2] >> (GRID - depth)) & 1)
        c = int(ch[node, o])
        if c == 0:
            return node * 8 + o
        node, depth = node + c, depth + 1


def neighbors(child):
    """int32 [capacity * 8, 3]: n_a(slot), -1 where there is none and for every slot that is not a reachable leaf."""
    cap = np.asarray(child).shape[0]
    nbr = np.full((cap * 8, 3), -1, np.int32)
    for slot, d, i in leaves(child):
        for a in range(3):
            if i[a] + 1 < (1 << d):
                j = list(i)
                j[a] += 1
                nbr[slot, a] = leaf_at(child, [v << (GRID - d) for v in j])
    return nbr


def neighbors_levels(child):
    """``neighbors`` level by level: the leaves of each depth, then all their descents at once."""
    ch = _links(child)
    cap = ch.shape[0]
    nbr = np.full((cap * 8, 3), -1, np.int32)
    oct_ = np.array([[(o >> 2) & 1, (o >> 1) & 1, o & 1] for o in range(8)], np.int64)
    nodes, corner, d = np.zeros(1, np.int64), np.zeros((1, 3), np.int64), 1
    while nodes.size:
        sl = (nodes[:, None] * 8 + np.arange(8)).reshape(-1)
        cell = (2 * corner[:, None, :] + oct_[None]).reshape(-1, 3)
        link = ch.reshape(-1)[sl]
        leaf = link == 0
        for a in range(3):
            has = leaf & (cell[:, a] + 1 < (1 << d))
            p = cell[has].copy()
            p[:, a] += 1
            p <<= GRID - d
            node = np.zeros(p.shape[0], np.int64)
            found = np.full(p.shape[0], -1, np.int64)
            k = 1
            while (found < 0).any():
                live = found < 0
                o = (((p[:, 0] >> (GRID - k)) & 1) << 2) | (((p[:, 1] >> (GRID - k)) & 1) << 1) | ((p[:, 2] >> (GRID - k)) & 1)
                s = node * 8 + o
                c = ch.reshape(-1)[s]
                found = np.where(live & (c == 0), s, found)
                node = np.where(live, node + c, node)
                k += 1
            nbr[sl[has], a] = found
        nodes, corner, d = (sl[~leaf] // 8 + link[~leaf]), cell[~leaf], d + 1
    return nbr


def columns(data_dim, fmt, basis_dim):
    """(colour columns, sigma column) of a data row: the columns the leaf-gradient pass writes.  fmt: 'RGBA', 'SH',
    'SG' or 'ASG'; a basis size other than 1, 4, 9, 16 or 25 keeps coefficient 0 of each channel only."""
    if fmt == "RGBA" or basis_dim < 0:
        return [0, 1, 2], data_dim - 1
    k = basis_dim if basis_dim in (1, 4, 9, 16, 25) else 1
    return [c * basis_dim + j for c in range(3) for j in range(k)], data_dim - 1


def tv(child, data, lam_sigma, lam_color, colour_cols, sigma_col, nbr=None):
    """-> (E, grad float64 [capacity * 8, data_dim], A float64 [capacity * 8, data_dim]): the energy, its gradient and
    the per-element sum of the absolute values of the terms.  Each group's terms are formed for all leaves at once."""
    v = np.asarray(data, np.float64).reshape(-1, np.asarray(data).shape[-1])
    nb = neighbors(child) if nbr is None else np.asarray(nbr)
    slots = np.array([s for s, _, _ in leaves(child)], np.int64)
    grad = np.zeros_like(v)
    absum = np.zeros_like(v)
    E = 0.0
    for lam, cols in ((lam_sigma, [sigma_col]), (lam_color, list(colour_cols))):
        if lam == 0:
            continue
        w = lam / slots.size
        cols = np.asarray(cols, np.int64)
        n = nb[slots].astype(np.int64)                                  # [leaves, 3]
        has = n >= 0
        own = v[slots][:, cols]                                          # [leaves, cols]
        D = np.where(has[:, :, None], v[np.maximum(n, 0)][:, :, cols] - own[:, None, :], 0.0)   # [leaves, 3, cols]
        r = np.sqrt(EPS + (D * D).sum(1))                                # [leaves, cols]
        E += w * r.sum()
        t = w * D / r[:, None, :]                                        # term of (leaf, axis, column)
        np.add.at(grad, (slots[:, None], cols[None, :]), -t.sum(1))
        np.add.at(absum, (slots[:, None], cols[None, :]), np.abs(t).sum(1))
        for a in range(3):
            k = has[:, a]
            np.add.at(grad, (n[k, a][:, None], cols[None, :]), t[k, a])
            np.add.at(absum, (n[k, a][:, None], cols[None, :]), np.abs(t[k, a]))
    return E, grad, absum
