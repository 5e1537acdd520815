"""Fine-tune a PlenOctree's leaf values against training images: gradient descent on the MSE of the rendered colours.

    python -m volrend_b200.finetune tree.npz out.npz pose.txt [pose.txt ...] --targets img.png [img.png ...]
                                    [-i intrinsics.txt] [-r] [--width 800] [--height 800] [--fx F] [--fy F]
                                    [--step_size S] [--sigma_thresh S] [--stop_thresh S] [--background B]
                                    [--steps 100] [--lr 1e-2] [--batch 4] [--seed 0] [--holdout K]
                                    [--refine-every K] [--refine-fraction 0.1] [--max-depth 23]
                                    [--tv-sigma 0] [--tv-color 0]

The fit uses the march's own samples: the renders are ``render_batch``'s float output and the gradients come from the
same samples on the GPU (``vr_tree_leaf_grads``, see :func:`volrend_b200.leaf_grads`; formulas in DESIGN.md section
18), so a lower loss is a better picture in the viewer.  An fp32 master copy of the data lives on the device; each step
renders a batch of views, takes the MSE on RGB against the targets, back-propagates it to the leaves, takes one Adam
step on the master and writes it, rounded to fp16, into the device tree (``N3Tree.update_data``).  The structure
changes only with ``--refine-every K``: every K steps the leaves that carry the most residual error are split
(coarse-to-fine, :mod:`volrend_b200.refine`, DESIGN.md section 19).  ``--tv-sigma`` / ``--tv-color`` add a
total-variation prior between neighbouring leaves to the gradient (:func:`volrend_b200.leaf_tv`, DESIGN.md section 20),
which keeps the many small leaves of a refined tree from fitting each training ray on its own.  Columns the device does not keep (coefficients of a basis size without its own kernel beyond the first, and
SG / ASG lobes) get no gradient and keep their values.

Targets are one PNG per pose or one ``.npy`` of shape [V, H, W, 3 | 4], uint8 or float in [0, 1].  RGBA targets are
composited onto the background brightness, as NeRF-synthetic images are used.  With ``--holdout K`` the last K poses
are not trained on; the PSNR on them is printed before and after.

Compressed trees (``quant_map``) are refused: fine-tune first, then prune and compress.
"""
from __future__ import annotations

import argparse
import math
import sys

import numpy as np

from .compress import _write_npz, carried_keys, check_uncompressed
from .views import add_view_arguments, open_inputs, target_batch

_ADVICE = "fine-tune the uncompressed tree first, then prune and compress"


def finetune(tree, cams, targets, options, *, steps: int, lr: float, batch: int, seed: int, on_step=None,
             refine_every: int = 0, refine_fraction: float = 0.1, max_depth: int = 23, on_refine=None,
             tv_sigma: float = 0.0, tv_color: float = 0.0):
    """Fits the leaf data of ``tree`` (an ``N3Tree`` loaded with ``load_cuda(slot_map=True)`` that still holds its host
    data) to ``targets``: a sequence of one image per camera in ``cams`` ([H, W, 3 | 4], uint8 or float, indexed
    lazily, so it may read files on demand).  Each of ``steps`` steps takes the next ``batch`` views of a shuffle seeded
    with ``seed`` (reshuffled after every pass), renders them with ``options``, back-propagates the MSE on RGB and takes
    one ``torch.optim.Adam`` step (learning rate ``lr``) on an fp32 master copy of the data, which is then written into
    the device tree.  ``on_step(step, loss)`` is called after every step.  Returns ``(master, losses)``: the fp32 data
    ``[capacity, 2, 2, 2, data_dim]`` on the device and the loss of every step.  The tree's host data is dropped.

    Coarse-to-fine: with ``refine_every = K > 0``, before every step ``s = K, 2K, ... < steps`` the leaves are scored
    over all of ``cams`` (:func:`volrend_b200.refine.leaf_scores`, batches of ``batch`` views) and split by
    :func:`volrend_b200.refine_plan` (``refine_fraction``, ``max_depth``); the master and both Adam moments are
    gathered by its ``src`` (a new slot starts with its parent's value and moments, the step count carries on), the
    device tree is re-created with the slot map from ``master.half()`` and ``on_refine(step, n_split, nodes_before,
    nodes_after)`` is called.  ``tree`` (``child_``, ``capacity``) then describes the refined tree.

    Total variation: with ``tv_sigma`` or ``tv_color`` > 0, every step adds the gradient of the TV prior of the master
    (:func:`volrend_b200.leaf_tv`, weights ``tv_sigma`` for sigma and ``tv_color`` for the colour coefficients) to the
    image gradient before the Adam step.  The neighbour table (:func:`volrend_b200.leaf_neighbors`) is built before
    the first step and again after every refinement that splits leaves.  ``losses`` and ``on_step`` stay the MSE."""
    import torch
    from .host import leaf_grads, leaf_neighbors, leaf_tv, render_batch
    from .refine import leaf_scores, refine_plan
    if steps < 0 or batch < 1:
        raise ValueError(f"steps {steps} must be >= 0 and batch {batch} >= 1")
    if refine_every < 0:
        raise ValueError(f"refine_every {refine_every} must be >= 0")
    for name, w in (("tv_sigma", tv_sigma), ("tv_color", tv_color)):
        if not (float(w) >= 0.0) or math.isinf(float(w)):
            raise ValueError(f"{name} {w} must be finite and >= 0")
    tv = tv_sigma > 0 or tv_color > 0
    if len(targets) != len(cams):
        raise ValueError(f"{len(targets)} targets for {len(cams)} views")
    if not cams:
        raise ValueError("no views to fit")
    if tree.data_ is None:
        raise ValueError("the tree holds no host data to start from")
    dev = torch.device("cuda", tree._device)
    H, W = cams[0].height, cams[0].width
    master = torch.tensor(np.asarray(tree.data_, np.float32), device=dev).requires_grad_(True)
    opt = torch.optim.Adam([master], lr=lr)
    gen = np.random.default_rng(seed)
    order, pos = gen.permutation(len(cams)), 0
    nb = min(batch, len(cams))
    fo = torch.empty((nb, H, W, 4), dtype=torch.float32, device=dev)
    dpix = torch.zeros((nb, H, W, 4), dtype=torch.float32, device=dev)
    grad = torch.zeros_like(master)
    nbr = leaf_neighbors(tree) if tv and steps > 0 else None
    tv_energy = torch.zeros(1, dtype=torch.float64, device=dev) if tv else None
    losses = []
    for step in range(steps):
        if refine_every > 0 and step > 0 and step % refine_every == 0:
            scores = leaf_scores(tree, cams, targets, options, batch).cpu().numpy().reshape(-1)
            child, src = refine_plan(tree.child_, scores, refine_fraction, max_depth)
            n0, n1 = tree.capacity, child.shape[0]
            if n1 > n0:
                master, opt = _gather_fit(master, opt, lr, torch.from_numpy(src).to(dev))
                grad = torch.zeros_like(master)
                tree.child_, tree.capacity = np.ascontiguousarray(child), n1
                tree.quant_ = None
                tree.data_ = master.detach().half().cpu().numpy()
                tree.load_cuda(slot_map=True)
                tree.clear_cpu_memory()
                if tv:
                    nbr = leaf_neighbors(tree)
            if on_refine is not None:
                on_refine(step, n1 - n0, n0, n1)
        if pos + nb > len(cams):
            order, pos = gen.permutation(len(cams)), 0
        views = order[pos:pos + nb]
        pos += nb
        tgt = target_batch(targets, views, options.background_brightness, dev, H, W)
        vc = [cams[int(v)] for v in views]
        render_batch(tree, vc, options, None, float_out=fo)
        diff = fo[..., :3] - tgt
        loss = diff.square().mean()
        dpix[..., :3] = diff * (2.0 / diff.numel())
        grad.zero_()
        leaf_grads(tree, vc, options, dpix, out=grad)
        if tv:
            leaf_tv(tree, nbr, master.detach(), tv_sigma, tv_color, out=grad, energy=tv_energy)
        master.grad = grad
        opt.step()
        tree.update_data(master.detach())
        losses.append(float(loss))
        if on_step is not None:
            on_step(step, losses[-1])
    return master.detach(), losses


def _gather_fit(master, opt, lr, src):
    """The fp32 master copy and a new Adam over it with every per-slot tensor (value, both moments) gathered by the
    source slot index ``src`` (``refine_plan``); the step count carries over."""
    import torch
    dd = master.shape[-1]
    take = lambda x: x.detach().reshape(-1, dd)[src].reshape(-1, 2, 2, 2, dd)
    new = take(master).requires_grad_(True)
    opt2 = torch.optim.Adam([new], lr=lr)
    st = opt.state.get(master)
    if st:
        opt2.state[new] = {"step": st["step"].clone(), "exp_avg": take(st["exp_avg"]),
                           "exp_avg_sq": take(st["exp_avg_sq"])}
    return new, opt2


def finetune_npz(z, data, *, child=None) -> dict:
    """The tree dict ``z`` (``N3Tree`` npz keys) with ``data`` (the fitted leaf values, [capacity, 2, 2, 2, data_dim],
    numpy or torch) written in the source's dtype; keys as :func:`volrend_b200.prune_npz` (the training-time keys
    ``compress_npz`` drops are dropped, every other key passes through).  ``child``: the structure of a fit with
    refinement (``N3Tree.child_`` after :func:`finetune`), written with ``data`` of its capacity; without it the
    structure is ``z``'s.  Compressed input (``quant_map``) is refused."""
    check_uncompressed(z, _ADVICE)
    src = np.asarray(z["data"])
    d = data.detach().cpu().numpy() if hasattr(data, "detach") else np.asarray(data)
    shape = src.shape if child is None else np.asarray(child).shape + src.shape[-1:]
    if d.shape != shape:
        raise ValueError(f"data has shape {d.shape}, the tree's {shape}")
    out = {k: z[k] for k in carried_keys(z, ("data",))}
    out["data"] = d.astype(src.dtype)
    if child is not None:
        out["child"] = np.asarray(child, np.int32)
    return out


# ---------------------------------------------------------------------------------------------------------- CLI
def _parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog="python -m volrend_b200.finetune",
                                 description="Fine-tune the leaf values of a PlenOctree npz against images of the given "
                                             "poses (MSE on the rendered colours, Adam on the GPU).")
    ap.add_argument("input", help="npz file storing octree data (uncompressed)")
    ap.add_argument("output", help="where to write the fine-tuned npz")
    add_view_arguments(ap, targets=True)
    ap.add_argument("--steps", type=int, default=100, help="optimiser steps")
    ap.add_argument("--lr", type=float, default=1e-2, help="Adam learning rate")
    ap.add_argument("--batch", type=int, default=4, help="views per step")
    ap.add_argument("--seed", type=int, default=0, help="seed of the view shuffle")
    ap.add_argument("--holdout", type=int, default=0, help="the last K poses are held out: PSNR before and after")
    ap.add_argument("--refine-every", type=int, default=0,
                    help="every K steps, split the leaves with the most residual error (0: never; the structure stays)")
    ap.add_argument("--refine-fraction", type=float, default=0.1,
                    help="share of the candidate leaves split at each refinement, in [0, 1]")
    ap.add_argument("--max-depth", type=int, default=23,
                    help="leaves at this depth (root's slots = 1) or deeper are not split (at most 23)")
    ap.add_argument("--tv-sigma", type=float, default=0.0,
                    help="weight of the total-variation prior on sigma between neighbouring leaves (0: none)")
    ap.add_argument("--tv-color", type=float, default=0.0,
                    help="weight of the total-variation prior on the colour coefficients (0: none)")
    return ap


def _psnr(tree, cams, targets, idx, options) -> float:
    import torch
    from .host import render_batch
    dev = torch.device("cuda", tree._device)
    se, n = 0.0, 0
    for v in idx:
        H, W = cams[v].height, cams[v].width
        fo = torch.empty((1, H, W, 4), dtype=torch.float32, device=dev)
        render_batch(tree, [cams[v]], options, None, float_out=fo)
        d = fo[..., :3] - target_batch(targets, [v], options.background_brightness, dev, H, W)
        se += float(d.square().sum())
        n += d.numel()
    return -10.0 * math.log10(max(se / n, 1e-30))


def main(argv=None) -> int:
    ap = _parser()
    args = ap.parse_args(argv)
    if args.steps < 0:
        ap.error(f"--steps {args.steps} < 0")
    if args.batch < 1:
        ap.error(f"--batch {args.batch} < 1")
    if not (args.lr > 0) or math.isinf(args.lr):
        ap.error(f"--lr {args.lr} must be a positive number")
    if args.refine_every < 0:
        ap.error(f"--refine-every {args.refine_every} < 0")
    if not (0.0 <= args.refine_fraction <= 1.0):
        ap.error(f"--refine-fraction {args.refine_fraction} must be in [0, 1]")
    if args.max_depth < 1:
        ap.error(f"--max-depth {args.max_depth} < 1")
    for flag, w in (("--tv-sigma", args.tv_sigma), ("--tv-color", args.tv_color)):
        if not (w >= 0.0) or math.isinf(w):
            ap.error(f"{flag} {w} must be a finite number >= 0")
    tree, cams, targets, d, opt = open_inputs(ap, args, _ADVICE, holdout=args.holdout)
    n_train = len(cams) - args.holdout
    held = list(range(n_train, len(cams)))
    if held:
        print(f"held-out PSNR before: {_psnr(tree, cams, targets, held, opt):.3f} dB")
    master, _ = finetune(tree, cams[:n_train], targets[:n_train], opt,
                         steps=args.steps, lr=args.lr, batch=args.batch, seed=args.seed,
                         on_step=lambda s, l: print(f"step {s}: loss {l:.6g}"),
                         refine_every=args.refine_every, refine_fraction=args.refine_fraction,
                         max_depth=args.max_depth, tv_sigma=args.tv_sigma, tv_color=args.tv_color,
                         on_refine=lambda s, n, a, b: print(f"refine before step {s}: split {n}, nodes {a} -> {b}"))
    if held:
        print(f"held-out PSNR after: {_psnr(tree, cams, targets, held, opt):.3f} dB")
    out = finetune_npz(d, master, child=tree.child_ if args.refine_every > 0 else None)
    tree.free_cuda()
    _write_npz(args.output, out)
    return 0


if __name__ == "__main__":
    sys.exit(main())
