"""The same trees in other node layouts, and the malformed trees ``vr_tree_create`` refuses.

``synth.make_tree`` and ``edge_cases.mixed_tree`` number nodes breadth first: every link is positive, table order
equals depth order equals node order, every node is reachable and internal slots hold zero data.  The reference
accepts much more (``ptr += skip * N3`` with any signed skip, n3tree_query.hpp:36-46; it never reads an unreachable
node or an internal slot's data), and trained trees carry free nodes.  Each transform here returns the same tree --
the same leaves at the same positions with the same rows -- in another layout:

  dfs        depth-first pre-order, octants in order: links positive, not level-sorted
  reverse    the root at 0, every other node in reverse breadth-first order: every non-root link is negative
  shuffle    a seeded random order of the non-root nodes: links of both signs
  dirty      shuffle, plus free nodes interleaved with the real ones (random data, links among themselves with a
             cycle, links into the tree, and one free node whose links leave [1, capacity): > capacity, == capacity,
             0 and < 0), trailing all-zero nodes, and random fp16 (NaN, +-Inf, -0 among them) in internal slots' rows
  wide       breadth-first as given, with extra data columns between the colour coefficients and sigma

Quantised trees (``npz`` with ``quant_map``) are relaid along the capacity axis of every per-slot array.
"""
from __future__ import annotations

from dataclasses import dataclass, replace

import numpy as np

from volrend_b200 import synth

LAYOUTS = ["dfs", "reverse", "shuffle", "dirty", "wide"]
WIDE_EXTRA = 3                          # columns the wide layout inserts before sigma
N_TRAIL = 3                             # all-zero nodes the dirty layout appends
# fp16 bit patterns mixed into the internal slots' rows of the dirty layout: NaN, -NaN, +Inf, -Inf, -0
SPECIAL_BITS = np.array([0x7E00, 0xFE01, 0x7C00, 0xFC00, 0x8000], np.uint16)
PER_SLOT = {"quant_map": 1, "data_retained": 1, "sigma": 0}     # quantised arrays: index of their capacity axis


@dataclass
class Relaid:
    st: synth.SynthTree        # the tree in the new layout (decoded data)
    npz: dict | None           # the quantised arrays in the new layout, when the tree is quantised
    slot_map: np.ndarray       # int64 [capacity * 8]: new slot -> slot of the canonical tree, -1 for free nodes
    n_free: int                # free nodes (unreachable, not all-zero) among the new nodes

    def arrays(self) -> dict:
        """What N3Tree.load_npz and the reference loader read."""
        return self.npz if self.npz is not None else self.st.npz_dict()


def targets(child) -> np.ndarray:
    """int64 [capacity, 8]: the node each internal slot links to, -1 for leaves."""
    ch = np.asarray(child, np.int64).reshape(-1, 8)
    return np.where(ch != 0, np.arange(ch.shape[0])[:, None] + ch, -1)


def bfs_levels(child) -> list:
    """Nodes of each depth in breadth-first order (parents in order, octants in order), from a valid tree."""
    tgt = targets(child)
    levels = [np.zeros(1, np.int64)]
    while True:
        t = tgt[levels[-1]].reshape(-1)
        t = t[t >= 0]
        if t.size == 0:
            return levels
        levels.append(t)


def dfs_order(child) -> np.ndarray:
    tgt = targets(child)
    out, stack = [], [0]
    while stack:
        n = stack.pop()
        out.append(n)
        kids = tgt[n][tgt[n] >= 0]
        stack.extend(kids[::-1].tolist())
    return np.array(out, np.int64)


def _relabel(st: synth.SynthTree, npz, new_of: np.ndarray, cap_new: int) -> Relaid:
    """Node n of ``st`` becomes node new_of[n] of a tree of cap_new nodes; the other nodes are all zero."""
    cap, dd = st.capacity, st.data_dim
    tgt = targets(st.child)
    rel = np.where(tgt >= 0, new_of[np.maximum(tgt, 0)] - new_of[:, None], 0)
    child = np.zeros((cap_new, 8), np.int32)
    child[new_of] = rel
    data = np.zeros((cap_new, 8, dd), np.float16)
    data[new_of] = st.data.reshape(cap, 8, dd)
    slot_map = np.full((cap_new, 8), -1, np.int64)
    slot_map[new_of] = np.arange(cap * 8).reshape(cap, 8)
    out = replace(st, child=child.reshape(cap_new, 2, 2, 2), data=data.reshape(cap_new, 2, 2, 2, dd), meta={})
    q = None
    if npz is not None:
        q = dict(npz)
        q["child"] = out.child
        for k, ax in PER_SLOT.items():
            if k in npz:
                a = np.asarray(npz[k])
                shape = list(a.shape)
                shape[ax] = cap_new
                b = np.zeros(shape, a.dtype)
                idx = [slice(None)] * a.ndim
                idx[ax] = new_of
                b[tuple(idx)] = a
                q[k] = b
    return Relaid(out, q, slot_map.reshape(-1), 0)


def _from_order(st, npz, order) -> Relaid:
    new_of = np.empty(st.capacity, np.int64)
    new_of[order] = np.arange(st.capacity)
    return _relabel(st, npz, new_of, st.capacity)


def _shuffled(st, rng) -> np.ndarray:
    rest = np.arange(1, st.capacity)
    return np.concatenate([[0], rng.permutation(rest)]).astype(np.int64)


def _dirty(st: synth.SynthTree, npz, seed: int) -> Relaid:
    rng = np.random.default_rng(seed)
    cap, dd = st.capacity, st.data_dim
    n_free = max(4, cap // 6)
    cap_new = cap + n_free + N_TRAIL
    pos = 1 + rng.permutation(cap + n_free - 1)          # positions 1 .. cap + n_free - 1, shuffled
    new_of = np.empty(cap, np.int64)
    new_of[0] = 0
    new_of[1:] = pos[:cap - 1]
    free = np.sort(pos[cap - 1:])
    r = _relabel(st, npz, new_of, cap_new)
    child = r.st.child.reshape(cap_new, 8)
    data = r.st.data.reshape(cap_new, 8, dd).view(np.uint16)
    # internal slots of the real nodes: random rows with NaN, +-Inf and -0 mixed in
    inner = child != 0
    noise = rng.integers(0, 1 << 16, (int(inner.sum()), dd), dtype=np.uint16)
    noise = np.where(rng.random(noise.shape) < 0.3, SPECIAL_BITS[rng.integers(0, len(SPECIAL_BITS), noise.shape)], noise)
    data[inner] = noise
    # free nodes: random rows, and links: a cycle through all of them (slot 0), random in-range links (slot 1), links
    # into the tree (slot 2); the last one links outside [1, capacity) in slots 3..6
    data[free] = rng.integers(0, 1 << 16, (n_free, 8, dd), dtype=np.uint16)
    nxt = np.roll(free, -1)
    child[free, 0] = nxt - free
    child[free, 1] = rng.choice(free, n_free) - free
    child[free, 2] = rng.choice(new_of[1:] if cap > 1 else free, n_free) - free
    bad = free[-1]
    for s, t in zip((3, 4, 5, 6), (cap_new + 3, cap_new, 0, -2)):
        child[bad, s] = t - bad
    r.st.child = child.reshape(cap_new, 2, 2, 2)
    r.st.data = data.view(np.float16).reshape(cap_new, 2, 2, 2, dd)
    if r.npz is not None:
        r.npz["child"] = r.st.child
    r.n_free = n_free
    return r


def _wide(st: synth.SynthTree, npz, seed: int) -> Relaid:
    if npz is not None:
        raise ValueError("quantised trees have data_dim 3 * basis_dim + 1")
    rng = np.random.default_rng(seed)
    cap, dd = st.capacity, st.data_dim
    r = _from_order(st, None, np.arange(cap))
    d = np.zeros((cap, 8, dd + WIDE_EXTRA), np.uint16)
    src = st.data.reshape(cap, 8, dd).view(np.uint16)
    d[..., :dd - 1] = src[..., :dd - 1]
    d[..., dd - 1:dd - 1 + WIDE_EXTRA] = rng.integers(0, 1 << 16, (cap, 8, WIDE_EXTRA), dtype=np.uint16)
    d[..., -1] = src[..., -1]
    r.st.data = d.view(np.float16).reshape(cap, 2, 2, 2, dd + WIDE_EXTRA)
    r.st.data_dim = dd + WIDE_EXTRA
    return r


def relayout(st: synth.SynthTree, layout: str, npz: dict | None = None, seed: int = 0) -> Relaid:
    """``st`` (canonical: every node reachable) in ``layout``; ``npz``: its quantised arrays, if it is quantised."""
    if layout == "dfs":
        return _from_order(st, npz, dfs_order(st.child))
    if layout == "reverse":
        bfs = np.concatenate(bfs_levels(st.child))
        return _from_order(st, npz, np.concatenate([[0], bfs[1:][::-1]]))
    if layout == "shuffle":
        return _from_order(st, npz, _shuffled(st, np.random.default_rng(seed)))
    if layout == "dirty":
        return _dirty(st, npz, seed)
    if layout == "wide":
        return _wide(st, npz, seed)
    raise KeyError(layout)


def leaf_centres(st: synth.SynthTree):
    """-> (slot int64 [n], depth int [n], tree-space centre float64 [n, 3]) of every leaf reachable from the root."""
    tgt = targets(st.child)
    nodes, lo, dep = np.zeros(1, np.int64), np.zeros((1, 3)), 1
    slots, depths, centres = [], [], []
    oct_ = np.array([[(o >> 2) & 1, (o >> 1) & 1, o & 1] for o in range(8)], np.float64)
    while nodes.size:
        h = 2.0 ** -dep
        sl = (nodes[:, None] * 8 + np.arange(8)).reshape(-1)
        corner = (lo[:, None, :] + oct_[None] * h).reshape(-1, 3)
        t = tgt.reshape(-1)[sl]
        leaf = t < 0
        slots.append(sl[leaf])
        depths.append(np.full(int(leaf.sum()), dep))
        centres.append(corner[leaf] + h / 2)
        nodes, lo, dep = t[~leaf], corner[~leaf], dep + 1
    return np.concatenate(slots), np.concatenate(depths), np.concatenate(centres)


def centre_points(st: synth.SynthTree, centres: np.ndarray, depth: np.ndarray) -> np.ndarray:
    """World points (float32) whose fused ``offset + scale * xyz`` lands on the leaf centres ``centres`` (tree space)
    where a float32 point does, else within a few ulps of it, strictly inside the leaf's cell at ``depth``."""
    from oracle import query_oracle as qo
    off, sc = st.offset.astype(np.float32), st.invradius3.astype(np.float32)
    want = centres.astype(np.float32)
    x = ((centres - off.astype(np.float64)) / sc.astype(np.float64)).astype(np.float32)
    for _ in range(8):
        got = qo.fma32(sc[None, :], x, off[None, :])
        miss = got != want
        if not miss.any():
            break
        x = np.where(miss, np.nextafter(x, np.where(got < want, np.inf, -np.inf).astype(np.float32)), x)
    got = qo.fma32(sc[None, :], x, off[None, :]).astype(np.float64)
    assert (np.abs(got - centres) < 2.0 ** -(np.asarray(depth)[:, None] + 1)).all(), "a point left its leaf's cell"
    return x


# ------------------------------------------------------------------------------------------- malformed trees
LINKS_OUTSIDE = "links outside"
TWO_PATHS = "two paths"


def malformed(st: synth.SynthTree) -> dict:
    """name -> (SynthTree, the refusal's message) of ``st`` (depth >= 4, every node reachable) with one defect in the
    part the root reaches.  A leaf slot of a reached node becomes a link: outside [1, capacity) (> capacity,
    == capacity, < 0, == 0 the root), to a node another node of its level already links to, to a deeper node that
    already has a parent, or to an ancestor of its own node (a cycle among non-root nodes)."""
    lv = bfs_levels(st.child)
    assert len(lv) >= 4
    ch = st.child.reshape(-1, 8)
    out = {}

    def leaf_slot(nodes, avoid=()):
        for n in nodes:
            if n in avoid:
                continue
            for s in range(8):
                if ch[n, s] == 0:
                    return int(n), s
        raise AssertionError("no leaf slot")

    def with_link(n, s, tgt):
        c = ch.copy()
        c[n, s] = tgt - n
        return replace(st, child=c.reshape(st.child.shape), meta={})

    n, s = leaf_slot(lv[2])
    cap = st.capacity
    out["outside_above"] = (with_link(n, s, cap + 5), LINKS_OUTSIDE)
    out["outside_at_capacity"] = (with_link(n, s, cap), LINKS_OUTSIDE)
    out["outside_negative"] = (with_link(n, s, -3), LINKS_OUTSIDE)
    out["outside_root"] = (with_link(n, s, 0), LINKS_OUTSIDE)
    tgt = targets(st.child)
    # a second parent at the same level: another node of lv[2] links to a child of the first one
    p = next(int(m) for m in lv[2] if (tgt[m] >= 0).any())
    kid = int(tgt[p][tgt[p] >= 0][0])
    n2, s2 = leaf_slot(lv[2], avoid=(p,))
    out["two_parents_same_level"] = (with_link(n2, s2, kid), TWO_PATHS)
    # a second parent two levels up
    n1, s1 = leaf_slot(lv[1])
    out["two_parents_other_level"] = (with_link(n1, s1, int(lv[3][0])), TWO_PATHS)
    # a cycle among non-root nodes: a node of lv[3] links back to its grandparent (in lv[1])
    d3 = next(int(m) for m in lv[3] if (ch[m] == 0).any())
    par = {int(c): int(m) for m in np.concatenate(lv) for c in tgt[m][tgt[m] >= 0]}
    s3 = int(np.flatnonzero(ch[d3] == 0)[0])
    out["cycle"] = (with_link(d3, s3, par[par[d3]]), TWO_PATHS)
    return out
