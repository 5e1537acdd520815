"""Build PlenOctrees from voxel cells on the GPU: dense, sparse and multi-resolution grids into N3Tree arrays.

    python -m volrend_b200.build IN OUT --format SH9|RGBA|SG9|... [--center x y z] [--radius r]
                                 [--sigma-thresh s] [--merge] [--extra lobes.npy]
    python -m volrend_b200.build --uniform L OUT --format ... [--init-sigma s]

A cell ``(L, i, j, k)`` (``1 <= L <= 23``, ``0 <= i, j, k < 2^L``, ``i`` along x) is the cube ``[i, i+1) x [j, j+1) x
[k, k+1) * 2^-L`` of the tree's unit cube, and its row is laid out like a row of ``N3Tree::data_`` (colour coefficients
channel-major, sigma last).  The tree of a set of non-overlapping cells is the smallest one in which every cell is a
leaf slot: listed slots hold their rows bit for bit, every other slot +0; nodes are numbered breadth first, the nodes of
a level in Morton order, so the arrays depend only on the set of cells.  ``merge`` collapses, bottom-up, every node whose
8 slots are leaves with bitwise-equal rows (unlisted slots read +0) into a leaf of its parent; the root stays.  The
build runs in ``vr_tree_build`` (volrend_b200/csrc/vr_build.cu); DESIGN.md section 21 states it.

``IN`` is a dense ``.npy`` grid ``[R, R, R, data_dim]`` (R a power of two; ``--sigma-thresh`` keeps only cells with
sigma above it) or an ``.npz`` with ``cells`` int [n, 4] and ``rows`` [n, data_dim].  ``--uniform L`` writes a full
level-L tree whose rows are +0 but for sigma (``--init-sigma``): a start for ``python -m volrend_b200.finetune
--refine-every K``.
"""
from __future__ import annotations

import argparse
import ctypes as C
import sys

import numpy as np

from . import _capi
from ._capi import check, lib
from .host import DataFormat, _stream_ptr
from .prune import N, _structure
from .refine import MAX_TREE_DEPTH

_OCT = np.array([[(o >> 2) & 1, (o >> 1) & 1, o & 1] for o in range(8)], np.int64)   # octant -> (x, y, z)


def _device_input(x, name: str, dev):
    """``x`` (numpy or a CUDA tensor) as a contiguous CUDA tensor on ``dev`` (numpy: the current device)."""
    import torch
    if isinstance(x, np.ndarray):
        return torch.from_numpy(np.ascontiguousarray(x)).to(dev if dev is not None else "cuda")
    if not isinstance(x, torch.Tensor) or not x.is_cuda:
        raise TypeError(f"{name} must be a numpy array or a CUDA tensor")
    if dev is not None and x.device != dev:
        raise ValueError(f"{name} live on {x.device}, the other input on {dev}")
    return x.contiguous()


def build_arrays(cells, rows, *, merge: bool = False, stream=None):
    """``(child, data)`` of the tree of ``cells`` (int [n, 4]: level, i, j, k) and ``rows`` ([n, data_dim], fp16, or
    fp32 rounded with ``.half()``): CUDA tensors int32 ``[n_nodes, 2, 2, 2]`` and fp16 ``[n_nodes, 2, 2, 2,
    data_dim]`` on the inputs' device (numpy inputs: the current device), written on ``stream`` (default: the current
    stream).  Raises ``ValueError`` for the cells ``vr_tree_build`` refuses (a level outside [1, 23], a coordinate
    outside [0, 2^level), duplicate or overlapping cells, more than ``refine.MAX_NODES`` nodes)."""
    import torch
    if not torch.cuda.is_available():
        raise _capi.VolrendError(_capi.VR_ENODEVICE, "no CUDA device: volrend_b200 has no CPU fallback")
    c = _device_input(cells, "cells", None)
    r = _device_input(rows, "rows", c.device)
    if c.ndim != 2 or c.shape[1] != 4 or c.dtype.is_floating_point or c.dtype.is_complex or c.dtype == torch.bool:
        raise ValueError(f"cells must be an integer array of shape [n, 4], not {c.dtype} {tuple(c.shape)}")
    if r.ndim != 2 or r.shape[0] != c.shape[0] or r.shape[1] < 1 or r.dtype not in (torch.float16, torch.float32):
        raise ValueError(f"rows must be a float16 or float32 array of shape [{c.shape[0]}, data_dim], "
                         f"not {r.dtype} {tuple(r.shape)}")
    n, dd = int(c.shape[0]), int(r.shape[1])
    if c.dtype != torch.int32:
        if n and (int(c.min()) < -2 ** 31 or int(c.max()) >= 2 ** 31):
            raise ValueError("a cell's level or coordinate is outside the int32 range")
        c = c.to(torch.int32)
    r = r.half().contiguous()
    flags = _capi.VR_BUILD_MERGE if merge else 0
    n_nodes = C.c_int64()

    def call(child, data, cap):
        with torch.cuda.device(c.device):
            rc = lib().vr_tree_build(c.data_ptr() if n else None, r.data_ptr() if n else None, n, dd, flags,
                                     child, data, cap, C.byref(n_nodes), _stream_ptr(stream))
        if rc == _capi.VR_EINVAL:
            raise ValueError(lib().vr_last_error().decode("utf-8", "replace"))
        check(rc)

    call(None, None, 0)
    nn = int(n_nodes.value)
    child = torch.empty((nn, N, N, N), dtype=torch.int32, device=c.device)
    data = torch.empty((nn, N, N, N, dd), dtype=torch.float16, device=c.device)
    call(child.data_ptr(), data.data_ptr(), nn)
    if stream is not None and isinstance(stream, torch.cuda.Stream):
        for t in (c, r, child, data):
            t.record_stream(stream)
    return child, data


def grid_cells(grid, sigma_thresh=None):
    """``(cells, rows)`` of a dense grid ``[R, R, R, data_dim]`` (a torch tensor, or numpy, which is moved to the current
    CUDA device; R a power of two in [2, 2^23], ``grid[i, j, k]`` the cell at x index i): the level-log2(R) cells and
    their rows rounded to fp16, as tensors int32 [n, 4] and fp16 [n, data_dim] on the grid's device, in x-major order.  With ``sigma_thresh``, only the cells whose fp16 sigma is
    greater than it (compared as float32, as the march compares sigma with ``sigma_thresh``) are kept; the filter runs on
    the device, so empty space costs no cells."""
    import torch
    g = torch.from_numpy(np.ascontiguousarray(grid)).to("cuda") if isinstance(grid, np.ndarray) else grid
    if not isinstance(g, torch.Tensor):
        raise TypeError("grid must be a numpy array or a torch tensor")
    if g.ndim != 4 or not (g.shape[0] == g.shape[1] == g.shape[2]) or g.shape[3] < 1:
        raise ValueError(f"grid must have shape [R, R, R, data_dim], not {tuple(g.shape)}")
    if g.dtype not in (torch.float16, torch.float32):
        raise ValueError(f"grid must be float16 or float32, not {g.dtype}")
    R = int(g.shape[0])
    L = R.bit_length() - 1
    if R < 2 or R != 1 << L or L > MAX_TREE_DEPTH:
        raise ValueError(f"grid size {R} is not a power of two in [2, 2^{MAX_TREE_DEPTH}]")
    rows = g.half().reshape(-1, g.shape[3])
    if sigma_thresh is None:
        idx = torch.arange(rows.shape[0], device=g.device, dtype=torch.int64)
    else:
        idx = torch.nonzero(rows[:, -1].float() > float(np.float32(sigma_thresh))).reshape(-1)
        rows = rows[idx]
    cells = torch.empty((idx.shape[0], 4), dtype=torch.int32, device=g.device)
    cells[:, 0] = L
    cells[:, 1] = (idx >> (2 * L)).to(torch.int32)
    cells[:, 2] = ((idx >> L) & (R - 1)).to(torch.int32)
    cells[:, 3] = (idx & (R - 1)).to(torch.int32)
    return cells, rows.contiguous()


def leaf_cells(child, data):
    """``(cells, rows)`` of the leaves reachable from the root of the tree ``child`` int32 [cap, 2, 2, 2] / ``data``
    fp16 [cap, 2, 2, 2, data_dim]: numpy int32 [n, 4] and fp16 [n, data_dim], breadth first.  Building them without
    merge gives the tree's canonical arrays.  Raises ValueError for links outside [1, capacity) and nodes reached
    twice (``prune._structure``)."""
    child = np.asarray(child)
    data = np.asarray(data)
    if child.ndim != 4 or child.shape[1:] != (N, N, N) or child.shape[0] < 1:
        raise ValueError(f"child must have shape [capacity, 2, 2, 2], not {child.shape}")
    cap = child.shape[0]
    if data.ndim != 5 or data.shape[:4] != child.shape or data.dtype.itemsize != 2:
        raise ValueError(f"data must be a half-precision [capacity, 2, 2, 2, data_dim] array, not {data.dtype} {data.shape}")
    levels, target = _structure(child)
    if len(levels) > MAX_TREE_DEPTH:
        raise ValueError(f"the tree has leaves at depth {len(levels)}: deeper than {MAX_TREE_DEPTH}")
    dd = data.shape[-1]
    flat = np.ascontiguousarray(data).view(np.uint16).reshape(cap * 8, dd)
    coord = np.zeros((cap, 3), np.int64)            # integer corner of each reachable node at its own level
    cells, rows = [], []
    for depth, nodes in enumerate(levels, start=1):
        slots = (nodes[:, None] * 8 + np.arange(8)).reshape(-1)
        xyz = (coord[nodes][:, None, :] * 2 + _OCT[None]).reshape(-1, 3)
        t = target[slots]
        leaf = t < 0
        coord[t[~leaf]] = xyz[~leaf]
        cells.append(np.concatenate([np.full((int(leaf.sum()), 1), depth, np.int64), xyz[leaf]], 1))
        rows.append(flat[slots[leaf]])
    return (np.concatenate(cells).astype(np.int32),
            np.concatenate(rows).view(np.float16).reshape(-1, dd))


def _format(data_format: str, data_dim: int) -> DataFormat:
    f = DataFormat()
    f.parse(data_format)
    if f.to_string() != data_format:
        raise ValueError(f"unknown data format {data_format!r}")
    need = 4 if f.format == DataFormat.RGBA else 3 * f.basis_dim + 1
    if f.format != DataFormat.RGBA and f.basis_dim < 1:
        raise ValueError(f"data format {data_format!r} has no basis functions")
    if data_dim < need:
        raise ValueError(f"rows have {data_dim} values: {data_format} needs at least {need}")
    return f


def build_npz(cells, rows, *, data_format: str, center=0.0, radius=1.0, extra=None, merge: bool = False,
              backend=None) -> dict:
    """The tree of ``cells`` / ``rows`` (:func:`build_arrays`) as the arrays of an N3Tree npz, in the form
    ``synth.SynthTree.npz_dict`` writes: ``data_dim``, ``data_format``, ``invradius3 = 1 / (2 radius)``, ``offset =
    0.5 - center * invradius3`` (``center`` and ``radius`` scalars or 3 values; the world box is center +- radius),
    ``child``, ``data`` and, for SG / ASG, ``extra_data`` (``extra``: [basis, 4] / [basis, 11] lobes).  ``backend``
    replaces the device build (``backend(cells, rows, merge)`` -> host ``(child, data)``; the tests pass the oracle)."""
    dd = int(rows.shape[1]) if getattr(rows, "ndim", 0) == 2 else -1
    if dd < 1:
        raise ValueError("rows must have shape [n, data_dim]")
    f = _format(data_format, dd)
    c3 = np.broadcast_to(np.asarray(center, np.float64), (3,)).astype(np.float64)
    r3 = np.broadcast_to(np.asarray(radius, np.float64), (3,)).astype(np.float64)
    if not (np.isfinite(c3).all() and np.isfinite(r3).all() and (r3 > 0).all()):
        raise ValueError(f"center {c3.tolist()} must be finite and radius {r3.tolist()} finite and > 0")
    lobes = {DataFormat.SG: 4, DataFormat.ASG: 11}.get(f.format)
    if lobes is None and extra is not None:
        raise ValueError(f"{data_format} trees have no extra data")
    if lobes is not None:
        ex = None if extra is None else np.asarray(extra, np.float32)
        if ex is None or ex.shape != (f.basis_dim, lobes):
            raise ValueError(f"{data_format} needs extra data of shape [{f.basis_dim}, {lobes}]")
    if backend is None:
        child, data = (t.cpu().numpy() for t in build_arrays(cells, rows, merge=merge))
    else:
        child, data = backend(cells, rows, merge)
    inv = (1.0 / (2.0 * r3)).astype(np.float32)
    out = dict(data_dim=np.int64(dd), data_format=np.array(data_format),
               invradius3=inv, offset=(0.5 - c3 * inv.astype(np.float64)).astype(np.float32),
               child=np.asarray(child, np.int32), data=np.asarray(data, np.float16))
    if lobes is not None:
        out["extra_data"] = ex
    return out


def uniform_cells(level: int, data_dim: int, init_sigma: float):
    """Cells and rows of a full level-``level`` tree whose rows are +0 but for sigma = ``init_sigma``."""
    import torch
    R = 1 << level
    grid = torch.zeros((R, R, R, data_dim), dtype=torch.float16, device="cuda")
    grid[..., -1] = float(init_sigma)
    return grid_cells(grid)


# ---------------------------------------------------------------------------------------------------------- CLI
def _parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog="python -m volrend_b200.build",
                                 description="Build a PlenOctree npz from voxel cells on the GPU: a dense .npy grid, an "
                                             ".npz of cells and rows, or a uniform tree.")
    ap.add_argument("paths", nargs="+", metavar="IN OUT",
                    help="input (.npy dense grid [R, R, R, data_dim] or .npz with 'cells' and 'rows') and output npz; "
                         "with --uniform only the output")
    ap.add_argument("--format", required=True, help="data format of the rows: RGBA, SH<n>, SG<n> or ASG<n>")
    ap.add_argument("--center", type=float, nargs=3, default=[0.0, 0.0, 0.0], help="world centre of the tree's box")
    ap.add_argument("--radius", type=float, default=1.0, help="half the edge of the tree's box, in world units")
    ap.add_argument("--sigma-thresh", type=float, default=None,
                    help="dense grids: keep only the cells with sigma above this")
    ap.add_argument("--merge", action="store_true", help="collapse nodes whose 8 leaves hold bitwise-equal rows")
    ap.add_argument("--extra", default=None, help="SG / ASG: .npy of the lobes ([basis, 4] / [basis, 11])")
    ap.add_argument("--uniform", type=int, default=None, metavar="L",
                    help="instead of IN, write a full level-L tree of constant rows")
    ap.add_argument("--init-sigma", type=float, default=None, help="--uniform: sigma of every leaf (default 0.1)")
    return ap


def main(argv=None) -> int:
    ap = _parser()
    args = ap.parse_args(argv)
    if args.uniform is None:
        if len(args.paths) != 2:
            ap.error("expected IN and OUT")
        if args.init_sigma is not None:
            ap.error("--init-sigma needs --uniform")
    else:
        if len(args.paths) != 1:
            ap.error("--uniform takes only OUT")
        if not 1 <= args.uniform <= 10:
            ap.error(f"--uniform {args.uniform} outside [1, 10]: the tree has 8^L leaves, at most 2^31 - 1 cells")
        if args.sigma_thresh is not None or args.merge:
            ap.error("--sigma-thresh and --merge do not apply to --uniform")
    if not (args.radius > 0 and np.isfinite(args.radius)):
        ap.error(f"--radius {args.radius} must be finite and > 0")
    if not np.isfinite(args.center).all():
        ap.error("--center must be finite")
    if args.sigma_thresh is not None and np.isnan(args.sigma_thresh):
        ap.error("--sigma-thresh is NaN")
    f = DataFormat()
    f.parse(args.format)
    if f.to_string() != args.format or (f.format != DataFormat.RGBA and f.basis_dim < 1):
        ap.error(f"unknown --format {args.format!r}")
    out_path = args.paths[-1]
    if not out_path.endswith(".npz"):
        ap.error(f"output {out_path} must end in .npz")
    extra = np.load(args.extra) if args.extra is not None else None
    if args.uniform is not None:
        dd = 4 if f.format == DataFormat.RGBA else 3 * f.basis_dim + 1
        init = 0.1 if args.init_sigma is None else args.init_sigma
        cells, rows = uniform_cells(args.uniform, dd, init)
    else:
        src = args.paths[0]
        if src.endswith(".npy"):
            cells, rows = grid_cells(np.load(src), args.sigma_thresh)
        elif src.endswith(".npz"):
            if args.sigma_thresh is not None:
                ap.error("--sigma-thresh applies to dense .npy grids")
            with np.load(src) as z:
                if "cells" not in z.files or "rows" not in z.files:
                    ap.error(f"{src} has no 'cells' and 'rows' arrays")
                cells, rows = z["cells"], z["rows"]
        else:
            ap.error(f"input {src} must be a .npy grid or an .npz of cells and rows")
    try:
        d = build_npz(cells, rows, data_format=args.format, center=args.center, radius=args.radius, extra=extra,
                      merge=args.merge)
    except ValueError as e:
        print(f"error: {e}", file=sys.stderr)
        return 1
    from .compress import _write_npz
    n_nodes = d["child"].shape[0]
    print(f"cells read {int(cells.shape[0])}; nodes written {n_nodes}, leaves {int((d['child'] == 0).sum())}")
    _write_npz(out_path, d)
    return 0


if __name__ == "__main__":
    sys.exit(main())
