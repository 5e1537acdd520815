"""Shapes, windows and reference sums of the fitting passes' tests (tests/test_fit_shapes_cpu.py,
tests/test_gpu_fit_shapes.py).

The gradient pass (vr_tree_leaf_grads) and the error pass (vr_tree_leaf_error) run on batches the size the fitting
loop uses: thousands of warp tiles, so that set_work (vr_kernels_inst.cu) hands them out in SM-local blocks.  Their
CPU references (oracle/grads_oracle.c, oracle/error_oracle.c) cost a ray per pixel, so the tests give each view a
``dpix`` / ``err`` that is random inside a small window and exactly 0 elsewhere, and run the references on the windows
alone.  That is sound: a pixel with g = 0 adds only +-0 terms on the GPU (G.gs, G.kt and G.gat are all 0; the error
pass adds weight * 0), so every slot that no window ray shades stays exactly 0, and the reference summed over the
windows is the reference of the whole batch.  test_fit_shapes_cpu.py checks this on the references themselves."""
from __future__ import annotations

from dataclasses import replace

import numpy as np

import layout_cases as lc

KTW, KTH = 4, 8             # pixels of a warp tile (vr_march.cuh kTW, kTH)
BLK_TILES = 64              # warp tiles of a block (vr_types.h kBlkTiles)
RTOL, ATOL = 1e-4, 1e-7     # |GPU - oracle| <= RTOL * A + ATOL (tests/test_gpu_finetune.py)
WEIGHT_TOL = 2e-6           # the weights pass's per-term tolerance (tests/test_gpu_refine.py)
NEG0 = 0x80000000


# ------------------------------------------------------------------------------------------------ block mode
def block_shape(kbd: int):
    """-> (views, tiles wide, tiles high) of a block: up to 16 basis functions 4 views x 4x4 tiles, 25 one view x 8x8
    tiles."""
    return (1, 8, 8) if kbd == 25 else (4, 4, 4)


def block_mode(n_views: int, w: int, h: int, kbd: int, num_sms: int):
    """set_work's decision for a launch of ``n_views`` views of w x h pixels of a tree of kernel basis ``kbd``:
    -> (blocks on, number of blocks)."""
    g, bw, bh = block_shape(kbd)
    tiles_x, tiles_y = -(-w // KTW), -(-h // KTH)
    nb = -(-tiles_x // bw) * -(-tiles_y // bh) * -(-n_views // g)
    on = n_views >= g and n_views >= 2 and nb >= 16 * num_sms and nb * BLK_TILES <= 0x7FFFFFFF
    return on, nb


def block_pixels(kbd: int):
    """(width, height) in pixels of a block's tiles."""
    _, bw, bh = block_shape(kbd)
    return bw * KTW, bh * KTH


def block_batch(kbd: int, num_sms: int, w: int, h: int):
    """-> (n_big, n_small): the fewest views, not a multiple of 4, whose w x h batch is in block mode, and a view count
    of at least 4 whose batch is not.  ``w`` x ``h`` must not be a multiple of the block."""
    bpw, bph = block_pixels(kbd)
    assert w % bpw and h % bph, "the image must end inside a block"
    n = 5
    while n % 4 == 0 or not block_mode(n, w, h, kbd, num_sms)[0]:
        n += 1
    small = n // 4 if kbd != 25 else n // 8
    small = max(small - small % 4 + 1, 5)           # an odd count, so the last view group is padded too
    assert not block_mode(small, w, h, kbd, num_sms)[0]
    return n, small


# ------------------------------------------------------------------------------------------------ windows
def windows(n_views: int, w: int, h: int, kbd: int, size=(9, 7), seed: int = 0, centre=False):
    """Per view a window (x0, y0, ww, wh) of ``size`` that straddles a block edge (so also a tile edge) in x and in y,
    at an offset that varies with the view; every fifth view's window sits in the image's bottom-right corner, where the
    last tiles and blocks are cut by the image edge.  ``centre``: edges from the middle half of the image only."""
    rng = np.random.default_rng(seed)
    bpw, bph = block_pixels(kbd)
    ww, wh = size
    out = []
    for v in range(n_views):
        if v % 5 == 4:
            out.append((w - ww, h - wh, ww, wh))
            continue
        xs = [e for e in range(bpw, w, bpw) if not centre or w // 4 <= e <= 3 * w // 4]
        ys = [e for e in range(bph, h, bph) if not centre or h // 4 <= e <= 3 * h // 4]
        ex, ey = int(rng.choice(xs)), int(rng.choice(ys))
        x0 = min(max(ex - 1 - v % (ww - 1), 0), w - ww)
        y0 = min(max(ey - 1 - (v // 2) % (wh - 1), 0), h - wh)
        out.append((x0, y0, ww, wh))
    return out


def windowed(n_views: int, w: int, h: int, wins, channels: int, lo: float, hi: float, seed: int):
    """float32 [n, h, w, channels] (channels 0: [n, h, w]), uniform in [lo, hi) inside each view's window, 0 elsewhere."""
    rng = np.random.default_rng(seed)
    shape = (n_views, h, w) + ((channels,) if channels else ())
    a = np.zeros(shape, np.float32)
    for v, (x0, y0, ww, wh) in enumerate(wins):
        a[v, y0:y0 + wh, x0:x0 + ww] = rng.uniform(lo, hi, (wh, ww) + shape[3:]).astype(np.float32)
    return a


# ------------------------------------------------------------------------------------------------ references
def oracle_cams(cams):
    """oracle/binding.py cameras of volrend_b200 Cameras."""
    from oracle import binding as ob
    return [ob.make_camera(c.width, c.height, c.fx, c.fy, np.asarray(c.transform, np.float32).reshape(12)) for c in cams]


def oracle_grads(ot, ocams, kw: dict, dpix: np.ndarray, wins=None, nthreads=None):
    """orc_leaf_grads summed over the views: -> (grad, A) float64 [capacity * 8, data_dim].  ``wins``: per view the
    window the reference runs on (``dpix`` is frame-sized and must be 0 outside it); None: the whole frame.  Windows
    run on one thread: the reference's threads each sum into a whole copy of the buffers."""
    from oracle import binding as ob
    from oracle import grads_binding as gb
    opt = ob.make_options(**kw)
    nthreads = nthreads or (1 if wins is not None else None)
    shape = (ot.c.capacity * 8, ot.c.data_dim)
    grad, A = np.zeros(shape), np.zeros(shape)
    for v, oc in enumerate(ocams):
        x0, y0, w, h = wins[v] if wins is not None else (0, 0, oc.width, oc.height)
        gb.leaf_grads(ot, oc, opt, dpix[v, y0:y0 + h, x0:x0 + w], tile=(x0, y0, w, h), grad=grad, A=A,
                      nthreads=nthreads)
    return grad, A


def oracle_error(ot, ocams, kw: dict, err: np.ndarray, wins=None, nthreads=None):
    """orc_leaf_error summed over the views: -> (score, absum, hits) [capacity * 8]; ``wins`` as in oracle_grads."""
    from oracle import binding as ob
    from oracle import error_binding as eb
    opt = ob.make_options(**kw)
    nthreads = nthreads or (1 if wins is not None else None)
    n = ot.c.capacity * 8
    score, absum, hits = np.zeros(n), np.zeros(n), np.zeros(n)
    for v, oc in enumerate(ocams):
        x0, y0, w, h = wins[v] if wins is not None else (0, 0, oc.width, oc.height)
        s, a, k, _ = eb.leaf_error(ot, oc, opt, err[v, y0:y0 + h, x0:x0 + w], tile=(x0, y0, w, h), nthreads=nthreads)
        score += s
        absum += a
        hits += k
    return score, absum, hits


def assert_grads_close(g, og, oA, what, terms=True):
    """GPU gradients (any shape of og's size) within RTOL * A + ATOL of the reference's; ``terms``: and not all
    zero."""
    g = np.asarray(g, np.float64).reshape(og.shape)
    d = np.abs(g - og)
    bad = d > RTOL * oA + ATOL
    assert not bad.any(), (what, int(bad.sum()), float(d.max()), np.argwhere(bad)[:5].tolist())
    assert not terms or ((oA > 0).any() and np.abs(og).max() > 0), (what, "no term at all")


def assert_error_close(g, score, absum, hits, err_max, what, exact_set=True):
    """The error sums within RTOL * absum + ATOL + WEIGHT_TOL * err_max * hits of the reference's.  ``exact_set``: also
    the set of slots that received terms (the GPU buffer started at -0), which holds when every pixel's err is
    positive; a windowed err of 0 turns the slots of the other pixels' samples to +0."""
    g = np.asarray(g, np.float32).reshape(-1)
    if exact_set:
        touched = g.view(np.uint32) != NEG0
        assert np.array_equal(touched, hits > 0), (what, "slots with terms differ", int((touched != (hits > 0)).sum()))
    d = np.abs(g.astype(np.float64) - score)
    tol = RTOL * absum + ATOL + WEIGHT_TOL * err_max * hits
    assert (d <= tol).all(), (what, float((d - tol).max()), int((d > tol).sum()))
    assert score.max() > 0, (what, "no term at all")


# ------------------------------------------------------------------------------------------------ big trees
def frustum_nodes(st, views, margin: float = 1.0) -> np.ndarray:
    """bool [capacity]: the nodes whose cell meets the pyramid of some view's window, widened by ``margin`` pixels.
    ``views``: (Camera, (x0, y0, w, h)).  Every sample of a window ray lies in such a cell, so cutting the tree below
    the other nodes changes nothing any window ray meets (the rays start at the camera: the pyramid's apex)."""
    tgt = lc.targets(st.child)
    off = np.asarray(st.offset, np.float64)
    sc = np.asarray(st.invradius3, np.float64)
    planes = []                             # (world normals [4, 3], apex [3]): inside where n . (p - apex) >= 0
    for c, (x0, y0, w, h) in views:
        m = np.asarray(c.transform, np.float64)     # rows: right, up, back, centre
        vx0, vx1 = (x0 - margin - c.width * 0.5) / c.fx, (x0 + w - 1 + margin - c.width * 0.5) / c.fx
        vy1, vy0 = -(y0 - margin - c.height * 0.5) / c.fy, -(y0 + h - 1 + margin - c.height * 0.5) / c.fy
        # camera space (right, up, back), depth -z:  x + vx0 z >= 0, -x - vx1 z >= 0, likewise y
        ncam = np.array([[1, 0, vx0], [-1, 0, -vx1], [0, 1, vy0], [0, -1, -vy1]], np.float64)
        planes.append((ncam @ m[:3], m[3]))
    octs = np.array([[(o >> 2) & 1, (o >> 1) & 1, o & 1] for o in range(8)], np.float64)
    keep = np.zeros(st.capacity, bool)
    keep[0] = True
    nodes, lo, size = np.zeros(1, np.int64), np.zeros((1, 3)), 1.0
    while nodes.size:
        size /= 2
        corner = (lo[:, None, :] + octs[None] * size).reshape(-1, 3)
        t = tgt[nodes].reshape(-1)
        inner = t >= 0
        corner, t = corner[inner], t[inner]
        half = size / sc / 2
        centre = (corner - off) / sc + half
        hit = np.zeros(t.size, bool)
        for n, apex in planes:
            reach = (centre - apex) @ n.T + np.abs(n) @ half          # max of n . (p - apex) over the cell
            hit |= (reach >= -1e-9).all(1)
        keep[t[hit]] = True
        nodes, lo = t[hit], corner[hit]
    return keep


def cut_oracle_tree(st, cams, wins):
    """The reference's tree of ``st`` cut to the nodes the windows' rays can meet (its sums then cost only those
    nodes), and int64 [its capacity * 8], the slot of ``st`` of each of its slots."""
    from oracle import binding as ob
    small, slots = compact(st, frustum_nodes(st, list(zip(cams, wins))))
    return ob.OracleTree.from_synth(small), slots


def compact(st, keep: np.ndarray):
    """The tree of the nodes ``keep`` (which must be closed under parents): links to other nodes become leaves of
    zero data.  -> (SynthTree, int64 [new capacity * 8] slot of ``st`` of every new slot)."""
    old = np.flatnonzero(keep)
    cap, dd, k = st.capacity, st.data_dim, old.size
    new_of = np.full(cap, -1, np.int64)
    new_of[old] = np.arange(k)
    tgt = lc.targets(st.child)[old]
    linked = (tgt >= 0) & keep[np.maximum(tgt, 0)]
    child = np.where(linked, new_of[np.maximum(tgt, 0)] - np.arange(k)[:, None], 0).astype(np.int32)
    data = st.data.reshape(cap, 8, dd)[old].copy()
    data[(tgt >= 0) & ~linked] = 0
    out = replace(st, child=child.reshape(k, 2, 2, 2), data=data.reshape(k, 2, 2, 2, dd), meta={})
    return out, (old[:, None] * 8 + np.arange(8)).reshape(-1)
