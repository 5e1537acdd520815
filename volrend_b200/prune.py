"""Prune a PlenOctree ``.npz`` by ray weight: drop the leaves no view gives a compositing weight of at least ``thresh``.

    python -m volrend_b200.prune tree.npz out.npz pose.txt [pose.txt ...] [-i intrinsics.txt] [-r]
                                 [--width 800] [--height 800] [--fx F] [--fy F]
                                 [--step_size S] [--sigma_thresh S] [--stop_thresh S] [--thresh 1e-3] [--no-collapse]

The weights are the maximum over the views of every shaded sample's weight T * (1 - att) in each leaf, computed on the
GPU by the march itself (``vr_tree_leaf_weights``, see :func:`volrend_b200.leaf_weights`); the pruning is host numpy.
DESIGN.md section 17 states the rules:

* a leaf slot is dropped iff its weight is below ``thresh`` or NaN (a slot no view shades keeps -inf and is dropped);
  a dropped leaf's whole data row becomes +0;
* with ``collapse``, bottom-up, an internal slot whose 8 children are all dropped leaves becomes a dropped leaf itself;
  the root node always stays;
* nodes no longer reachable from the root are removed; the others keep their relative order, and the child links are
  rewritten as offsets relative to the new node indices.

Prune first, then compress (``python -m volrend_b200.compress``): compressed input is refused.
"""
from __future__ import annotations

import argparse
import math
import sys

import numpy as np

from .compress import _write_npz, carried_keys, check_uncompressed
from .views import add_view_arguments, open_inputs

N = 2
_ADVICE = "prune the uncompressed tree first, then compress"


def _structure(child: np.ndarray):
    """(levels, target) of a [cap, 2, 2, 2] child array: the node indices of each depth reachable from the root (root
    first) and, per slot, the node an internal slot links to (-1 for leaves and slots of unreachable nodes).  Raises
    ValueError for links outside [1, capacity) and for nodes reached twice."""
    cap = child.shape[0]
    ch = child.reshape(cap, 8).astype(np.int64)
    target = np.full(cap * 8, -1, np.int64)
    seen = np.zeros(cap, bool)
    seen[0] = True
    levels = [np.zeros(1, np.int64)]
    while True:
        nodes = levels[-1]
        slots = (nodes[:, None] * 8 + np.arange(8)).reshape(-1)
        rel = ch.reshape(-1)[slots]
        slots, rel = slots[rel != 0], rel[rel != 0]
        if slots.size == 0:
            return levels, target
        tgt = slots // 8 + rel
        if ((tgt < 1) | (tgt >= cap)).any():
            raise ValueError("child array has links outside [1, capacity)")
        if seen[tgt].any() or np.unique(tgt).size != tgt.size:
            raise ValueError("child array is not a tree: a node is reachable along two paths")
        seen[tgt] = True
        target[slots] = tgt
        levels.append(np.sort(tgt))


def _check_arrays(child, data, weights):
    child = np.asarray(child)
    data = np.asarray(data)
    if child.ndim != 4 or child.shape[1:] != (N, N, N) or child.shape[0] < 1:
        raise ValueError(f"child must have shape [capacity, 2, 2, 2], not {child.shape}")
    cap = child.shape[0]
    if data.ndim != 5 or data.shape[:4] != child.shape or data.dtype.itemsize != 2:
        raise ValueError(f"data must be a half-precision [capacity, 2, 2, 2, data_dim] array, not {data.dtype} {data.shape}")
    w = np.asarray(weights, np.float32)
    if w.size != cap * 8:
        raise ValueError(f"weights have {w.size} elements, the tree {cap * 8} slots")
    return child, data, w.reshape(cap * 8)


def prune_arrays(child, data, weights, thresh: float, collapse: bool = True):
    """(child', data') of the tree ``child`` int32 [cap, 2, 2, 2] / ``data`` fp16 [cap, 2, 2, 2, data_dim] pruned by the
    per-slot ``weights`` (``capacity * 8`` floats, slot = node * 8 + octant, as :func:`leaf_weights` returns them):
    leaves whose weight is below ``thresh`` or NaN are dropped (data row +0), with ``collapse`` internal slots whose
    children are all dropped leaves become dropped leaves, and unreachable nodes are removed (module docstring)."""
    thresh = float(thresh)
    if math.isnan(thresh):
        raise ValueError("thresh is NaN")
    child, data, w = _check_arrays(child, data, weights)
    cap = child.shape[0]
    levels, target = _structure(child)
    leaf = target < 0                                   # slots of unreachable nodes never matter
    dropped = leaf & ~(w >= thresh)                     # NaN compares false: dropped
    parent = np.full(cap, -1, np.int64)                 # node -> the slot that links to it
    parent[target[target >= 0]] = np.nonzero(target >= 0)[0]
    if collapse:
        for nodes in reversed(levels[1:]):
            gone = dropped.reshape(cap, 8)[nodes].all(axis=1)
            ps = parent[nodes[gone]]
            dropped[ps] = True
            leaf[ps] = True
    keep = np.zeros(cap, bool)                          # reachable from the root through the remaining links
    keep[0] = True
    frontier = np.zeros(1, np.int64)
    while frontier.size:
        slots = (frontier[:, None] * 8 + np.arange(8)).reshape(-1)
        slots = slots[~leaf[slots]]
        frontier = target[slots]
        keep[frontier] = True
    nodes = np.nonzero(keep)[0]
    new_index = np.cumsum(keep) - 1
    slots = (nodes[:, None] * 8 + np.arange(8)).reshape(-1)
    internal = ~leaf[slots]
    out_child = np.zeros(slots.size, np.int32)
    out_child[internal] = (new_index[target[slots[internal]]] - new_index[slots[internal] // 8]).astype(np.int32)
    dd = data.shape[-1]
    flat = np.ascontiguousarray(data).reshape(cap * 8, dd)
    out_data = flat[slots].copy()
    out_data.view(np.uint16)[dropped[slots]] = 0
    return out_child.reshape(-1, N, N, N), out_data.reshape(-1, N, N, N, dd)


def prune_npz(z, weights, thresh: float, collapse: bool = True) -> dict:
    """The pruned form of the tree dict ``z`` (``N3Tree`` npz keys): ``child`` and ``data`` pruned by
    :func:`prune_arrays`, the training-time keys ``compress_npz`` drops dropped too, every other key passed through.
    Compressed input (``quant_map``) is refused: prune first, then compress."""
    check_uncompressed(z, _ADVICE)
    child, data = prune_arrays(z["child"], z["data"], weights, thresh, collapse)
    out = {k: z[k] for k in carried_keys(z, ("child", "data"))}
    out["child"] = child
    out["data"] = data
    return out


# ---------------------------------------------------------------------------------------------------------- CLI
def _parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog="python -m volrend_b200.prune",
                                 description="Prune a PlenOctree npz by ray weight: leaves whose maximum compositing "
                                             "weight over the given views is below --thresh are dropped.")
    ap.add_argument("input", help="npz file storing octree data (uncompressed)")
    ap.add_argument("output", help="where to write the pruned npz")
    add_view_arguments(ap)
    ap.add_argument("--thresh", type=float, default=1e-3, help="leaves with a maximum weight below this are dropped")
    ap.add_argument("--no-collapse", dest="collapse", action="store_false",
                    help="keep internal nodes whose children are all dropped")
    ap.add_argument("--batch", type=int, default=64, help="views per weights launch")
    return ap


def main(argv=None) -> int:
    ap = _parser()
    args = ap.parse_args(argv)
    if math.isnan(args.thresh):
        ap.error("--thresh is NaN")
    if args.batch < 1:
        ap.error(f"--batch {args.batch} < 1")
    tree, cams, _, d, opt = open_inputs(ap, args, _ADVICE)

    from .host import leaf_weights
    w = None
    for v0 in range(0, len(cams), args.batch):
        w = leaf_weights(tree, cams[v0:v0 + args.batch], opt, out=w)
    weights = w.cpu().numpy().reshape(-1)
    tree.free_cuda()

    out = prune_npz(d, weights, args.thresh, args.collapse)
    leaf = np.asarray(d["child"]).reshape(-1) == 0
    kept = int((leaf & (weights >= args.thresh)).sum())
    print(f"views {len(cams)}: leaves kept {kept}, dropped {int(leaf.sum()) - kept}; "
          f"nodes {np.asarray(d['child']).shape[0]} -> {out['child'].shape[0]}")
    _write_npz(args.output, out)
    return 0


if __name__ == "__main__":
    sys.exit(main())
