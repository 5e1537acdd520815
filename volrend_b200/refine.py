"""Refine a PlenOctree ``.npz`` where the fit still misses: split the leaves that carry the most residual error.

    python -m volrend_b200.refine tree.npz out.npz pose.txt [pose.txt ...] --targets img.png [img.png ...]
                                  --fraction F [--max-depth 23] [-i intrinsics.txt] [-r]
                                  [--width 800] [--height 800] [--fx F] [--fy F]
                                  [--step_size S] [--sigma_thresh S] [--stop_thresh S] [--background B] [--batch 16]

The score of a leaf is its residual error: every shaded sample of every pixel adds its compositing weight
T * (1 - att) times the pixel's error to its leaf, computed on the GPU by the march itself (``vr_tree_leaf_error``, see
:func:`volrend_b200.leaf_error`); the CLI's pixel error is the squared RGB error of the render against the targets.
The rewrite is host numpy.  DESIGN.md section 19 states the rules:

* candidates are the leaf slots of nodes reachable from the root whose depth (root's slots = 1, as
  ``vr_tree_info.max_depth``) is below ``max_depth`` (capped at 23, the deepest leaf ``vr_tree_create`` accepts) and
  whose score is finite and > 0;
* the ``ceil(fraction * n_candidates)`` candidates with the highest scores are split, ties broken by the lower slot;
* every existing node keeps its index (free and unreachable ones included), so every existing slot keeps its number;
  one new node per split slot is appended, in increasing order of the split slot; the split slot links to it and its
  8 leaves copy the split slot's data row, so the field does not change (the split slot's own row stays as it was).

Refine and fit first, then prune and compress: compressed input is refused.
"""
from __future__ import annotations

import argparse
import math
import os
import sys

import numpy as np

from .compress import DROPPED_KEYS, _write_npz
from .prune import N, _structure, add_view_arguments, load_tree_arrays, view_setup

MAX_TREE_DEPTH = 23            # kMaxTreeDepth: the deepest leaf level vr_tree_create accepts
MAX_NODES = 0xFFFFFFFF // 8    # the slot map holds node * 8 + octant in a u32 with 0xffffffff reserved


def check_capacity(n_nodes: int) -> None:
    """Raises ValueError when a tree of ``n_nodes`` nodes cannot be addressed by the int32 child links or the device's
    slot map."""
    if n_nodes > MAX_NODES:
        raise ValueError(f"{n_nodes} nodes: more than the {MAX_NODES} the int32 links and the u32 slot map can address")


def refine_plan(child, scores, fraction: float, max_depth: int = MAX_TREE_DEPTH):
    """(child2, src) of the tree ``child`` int32 [cap, 2, 2, 2] refined by the per-slot ``scores`` (``capacity * 8``
    floats, slot = node * 8 + octant, as :func:`leaf_error` returns them): the ``ceil(fraction * n_candidates)``
    highest-scoring candidate leaves are split (module docstring).  ``src`` (int64, ``capacity2 * 8``) is the source
    slot of every output slot, so that every per-slot array is expanded with one gather, ``x2 = x.reshape(cap * 8,
    ...)[src]``.  With nothing to split, ``child2`` is ``child`` and ``src`` the identity."""
    fraction = float(fraction)
    if not (0.0 <= fraction <= 1.0):
        raise ValueError(f"fraction {fraction} must be in [0, 1]")
    max_depth = int(max_depth)
    if max_depth < 1:
        raise ValueError(f"max_depth {max_depth} must be >= 1")
    max_depth = min(max_depth, MAX_TREE_DEPTH)
    child = np.asarray(child)
    if child.ndim != 4 or child.shape[1:] != (N, N, N) or child.shape[0] < 1:
        raise ValueError(f"child must have shape [capacity, 2, 2, 2], not {child.shape}")
    cap = child.shape[0]
    s = np.asarray(scores, np.float32).reshape(-1)
    if s.size != cap * 8:
        raise ValueError(f"scores have {s.size} elements, the tree {cap * 8} slots")
    levels, target = _structure(child)
    slots = np.concatenate([np.zeros(0, np.int64)] + [(nodes[:, None] * 8 + np.arange(8)).reshape(-1)
                                                      for nodes in levels[:max_depth - 1]])   # depth < max_depth
    slots = slots[(target[slots] < 0) & np.isfinite(s[slots]) & (s[slots] > 0)]
    n_split = math.ceil(fraction * slots.size)
    src = np.arange(cap * 8, dtype=np.int64)
    if n_split == 0:
        return child, src
    split = np.sort(slots[np.lexsort((slots, -s[slots].astype(np.float64)))[:n_split]])
    cap2 = cap + n_split
    check_capacity(cap2)
    new_nodes = cap + np.arange(n_split, dtype=np.int64)
    child2 = np.concatenate([child.reshape(cap, 8).astype(np.int32), np.zeros((n_split, 8), np.int32)])
    child2.reshape(-1)[split] = (new_nodes - split // 8).astype(np.int32)
    return child2.reshape(cap2, N, N, N), np.concatenate([src, np.repeat(split, 8)])


def refine_npz(z, scores, fraction: float, max_depth: int = MAX_TREE_DEPTH) -> dict:
    """The refined form of the tree dict ``z`` (``N3Tree`` npz keys): ``child`` from :func:`refine_plan`, ``data``
    gathered by its ``src`` in the source's dtype, the training-time keys ``compress_npz`` drops dropped, every other
    key (``extra_data`` included) passed through.  Compressed input (``quant_map``) is refused: refine and fit first,
    then prune and compress."""
    keys = list(z.files if hasattr(z, "files") else z)
    if "quant_map" in keys or "quant_colors" in keys:
        raise ValueError("the tree is compressed (quant_map): refine the uncompressed tree, then prune and compress")
    for k in ("child", "data"):
        if k not in keys:
            raise ValueError(f"the tree has no '{k}' array")
    data = np.asarray(z["data"])
    if data.ndim != 5 or data.shape[:4] != np.asarray(z["child"]).shape:
        raise ValueError(f"data has shape {data.shape}, not [capacity, 2, 2, 2, data_dim]")
    child, src = refine_plan(z["child"], scores, fraction, max_depth)
    dd = data.shape[-1]
    out = {k: z[k] for k in keys if k not in ("child", "data") and k not in DROPPED_KEYS}
    out["child"] = child
    out["data"] = data.reshape(-1, dd)[src].reshape(-1, N, N, N, dd)
    return out


def pixel_error(render, target):
    """The pixel error the CLIs and the coarse-to-fine fit score leaves with: the squared RGB error of a float render
    ``[..., 4]`` against background-composited RGB targets ``[..., 3]``, summed over the channels."""
    return (render[..., :3] - target).square().sum(-1)


def leaf_scores(tree, cams, targets, options, batch: int, out=None):
    """Residual error of every leaf slot of ``tree`` over the views ``cams`` (targets as :func:`finetune`'s),
    rendered and scored in batches of ``batch`` views: a float32 CUDA tensor [capacity, 2, 2, 2], accumulated into
    ``out`` when given."""
    import torch
    from .finetune import _target_rgb
    from .host import leaf_error, render_batch
    dev = torch.device("cuda", tree._device)
    H, W = cams[0].height, cams[0].width
    for v0 in range(0, len(cams), batch):
        vc = cams[v0:v0 + batch]
        fo = torch.empty((len(vc), H, W, 4), dtype=torch.float32, device=dev)
        render_batch(tree, vc, options, None, float_out=fo)
        tgt = torch.stack([_target_rgb(targets[v], options.background_brightness, dev)
                           for v in range(v0, v0 + len(vc))])
        if tuple(tgt.shape) != (len(vc), H, W, 3):
            raise ValueError(f"targets are {tuple(tgt.shape[1:3])}, the views {H}x{W}")
        out = leaf_error(tree, vc, options, pixel_error(fo, tgt).contiguous(), out=out)
    return out


# ---------------------------------------------------------------------------------------------------------- CLI
def _parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog="python -m volrend_b200.refine",
                                 description="Split the leaves of a PlenOctree npz that carry the most residual error "
                                             "against images of the given poses (compositing weight x squared RGB "
                                             "error, summed on the GPU).")
    ap.add_argument("input", help="npz file storing octree data (uncompressed)")
    ap.add_argument("output", help="where to write the refined npz")
    add_view_arguments(ap)
    ap.add_argument("--targets", nargs="+", required=True,
                    help="one PNG per pose, or one .npy [views, height, width, 3|4] (uint8 or float in [0, 1])")
    ap.add_argument("--background", type=float, default=1.0,
                    help="background brightness: renders and the compositing of RGBA targets")
    ap.add_argument("--fraction", type=float, required=True,
                    help="share of the candidate leaves (positive score, above --max-depth) to split, in [0, 1]")
    ap.add_argument("--max-depth", type=int, default=MAX_TREE_DEPTH,
                    help="leaves at this depth (root's slots = 1) or deeper are not split (at most 23)")
    ap.add_argument("--batch", type=int, default=16, help="views per render and error launch")
    return ap


def main(argv=None) -> int:
    from .finetune import read_targets
    ap = _parser()
    args = ap.parse_args(argv)
    if not (0.0 <= args.fraction <= 1.0):
        ap.error(f"--fraction {args.fraction} must be in [0, 1]")
    if args.max_depth < 1:
        ap.error(f"--max-depth {args.max_depth} < 1")
    if args.batch < 1:
        ap.error(f"--batch {args.batch} < 1")
    if os.path.abspath(args.input) == os.path.abspath(args.output):
        ap.error("the output would overwrite the input")
    for p in [args.input] + args.targets:
        if not os.path.exists(p):
            ap.error(f"'{p}' does not exist")
    poses, fx, fy = view_setup(ap, args)
    try:
        targets = read_targets(args.targets, len(poses), args.width, args.height)
    except ValueError as e:
        ap.error(str(e))
    with np.load(args.input) as z:
        d = {k: z[k] for k in z.files}
    if "quant_map" in d or "quant_colors" in d:
        ap.error(f"{args.input} is compressed: refine the uncompressed tree first, then prune and compress")

    from .host import Camera, RenderOptions
    tree = load_tree_arrays(d, args.input)
    opt = RenderOptions(step_size=args.step_size, sigma_thresh=args.sigma_thresh, stop_thresh=args.stop_thresh,
                        background_brightness=args.background)
    cams = []
    for m in poses:
        c = Camera(args.width, args.height, fx, fy)
        c.set_c2w(m)
        cams.append(c)
    scores = leaf_scores(tree, cams, targets, opt, args.batch).cpu().numpy().reshape(-1)
    tree.free_cuda()
    out = refine_npz(d, scores, args.fraction, args.max_depth)
    n0, n1 = np.asarray(d["child"]).shape[0], out["child"].shape[0]
    print(f"views {len(cams)}: leaves with a positive score {int((scores > 0).sum())}, split {n1 - n0}; "
          f"nodes {n0} -> {n1}")
    _write_npz(args.output, out)
    return 0


if __name__ == "__main__":
    sys.exit(main())
