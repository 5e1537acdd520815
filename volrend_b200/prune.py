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
import os
import sys

import numpy as np

from .compress import DROPPED_KEYS, _write_npz

N = 2


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
    keys = list(z.files if hasattr(z, "files") else z)
    if "quant_map" in keys or "quant_colors" in keys:
        raise ValueError("the tree is already compressed (quant_map): prune the uncompressed tree first, then compress")
    for k in ("child", "data"):
        if k not in keys:
            raise ValueError(f"the tree has no '{k}' array")
    child, data = prune_arrays(z["child"], z["data"], weights, thresh, collapse)
    out = {k: z[k] for k in keys if k not in ("child", "data") and k not in DROPPED_KEYS}
    out["child"] = child
    out["data"] = data
    return out


# ---------------------------------------------------------------------------------------------------------- CLI
def read_poses(path: str) -> list:
    """Row-major 4x4 camera-to-world matrices of a pose file, one or more per file (volrend_headless)."""
    with open(path) as f:
        vals = np.array(f.read().split(), np.float32)
    n = vals.size // 16 + (1 if vals.size % 16 >= 12 else 0)
    vals = np.concatenate([vals, np.zeros(n * 16 - vals.size, np.float32)]) if n * 16 > vals.size else vals
    return [vals[16 * i:16 * i + 16].reshape(4, 4) for i in range(n)]


def read_intrinsics(path: str):
    """(fx, fy) of a 4x4 intrinsics file: the first and the sixth number (volrend_headless)."""
    with open(path) as f:
        vals = f.read().split()
    if len(vals) < 6:
        raise ValueError(f"intrinsics file {path} has {len(vals)} numbers, not a 4x4 matrix")
    return float(vals[0]), float(vals[5])


def add_view_arguments(ap: argparse.ArgumentParser) -> None:
    """The camera, pose and march options of the tools that run views over a tree (prune, finetune):
    volrend_headless's pose files, -i, -r and image size, and the step and thresholds."""
    ap.add_argument("poses", nargs="+", help="camera-to-world pose .txt files (row-major 4x4, one or more per file)")
    ap.add_argument("-i", "--intrin", default="", help="intrinsics matrix 4x4; if set, overrides the fx/fy")
    ap.add_argument("-r", "--reverse_yz", action="store_true", help="use OpenCV camera space convention instead of NeRF")
    ap.add_argument("--width", type=int, default=800, help="image width")
    ap.add_argument("--height", type=int, default=800, help="image height")
    ap.add_argument("--fx", type=float, default=-1.0, help="focal length in x (default 1111.11)")
    ap.add_argument("--fy", type=float, default=-1.0, help="focal length in y (default fx)")
    ap.add_argument("--step_size", type=float, default=1e-4, help="ray march step size")
    ap.add_argument("--sigma_thresh", type=float, default=1e-2, help="sigma threshold of a shaded sample")
    ap.add_argument("--stop_thresh", type=float, default=1e-2, help="transmittance below which a ray stops")


def view_setup(ap: argparse.ArgumentParser, args):
    """Checks add_view_arguments' values (ap.error on a bad one) -> (row-major 4x4 poses, fx, fy)."""
    if args.width < 1 or args.height < 1:
        ap.error(f"image size {args.width}x{args.height} must be positive")
    for p in args.poses + ([args.intrin] if args.intrin else []):
        if not os.path.exists(p):
            ap.error(f"'{p}' does not exist")
    fx = 1111.11 if args.fx < 0 else args.fx
    fy = fx if args.fy < 0 else args.fy
    if args.intrin:
        fx, fy = read_intrinsics(args.intrin)
    poses = [m for p in args.poses for m in read_poses(p)]
    if not poses:
        ap.error("no camera poses in the pose files")
    if args.reverse_yz:
        poses = [m @ np.diag([1, -1, -1, 1]).astype(np.float32) for m in poses]
    return poses, fx, fy


def load_tree_arrays(d: dict, path: str):
    """An N3Tree of the npz dict ``d`` read from ``path``, on the device with the slot map; NDC trees (a
    ``<tree>_poses_bounds.npy`` beside the file) as ``N3Tree.open`` loads them."""
    from .host import N3Tree
    tree = N3Tree()
    tree.load_npz(d)
    pb = path[:-4] + "_poses_bounds.npy"
    if path.endswith(".npz") and os.path.exists(pb):
        tree.use_ndc = True
        tree._unpack_llff_poses_bounds(np.load(pb))
    tree.load_cuda(slot_map=True)
    return tree


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
    if args.width < 1 or args.height < 1:
        ap.error(f"image size {args.width}x{args.height} must be positive")
    if math.isnan(args.thresh):
        ap.error("--thresh is NaN")
    if args.batch < 1:
        ap.error(f"--batch {args.batch} < 1")
    if os.path.abspath(args.input) == os.path.abspath(args.output):
        ap.error("the output would overwrite the input")
    if not os.path.exists(args.input):
        ap.error(f"'{args.input}' does not exist")
    poses, fx, fy = view_setup(ap, args)
    with np.load(args.input) as z:
        d = {k: z[k] for k in z.files}
    if "quant_map" in d or "quant_colors" in d:
        ap.error(f"{args.input} is already compressed: prune the uncompressed tree first, then compress")

    from .host import Camera, RenderOptions, leaf_weights
    tree = load_tree_arrays(d, args.input)
    opt = RenderOptions(step_size=args.step_size, sigma_thresh=args.sigma_thresh, stop_thresh=args.stop_thresh)
    cams = []
    for m in poses:
        c = Camera(args.width, args.height, fx, fy)
        c.set_c2w(m)
        cams.append(c)
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
