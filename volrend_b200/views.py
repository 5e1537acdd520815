"""Views, targets and tree files of the tools that march views over a tree (``prune``, ``refine``, ``finetune``):
volrend_headless's pose and intrinsics files, the tools' shared command-line options, training targets, and the
opening every one of their command lines runs (:func:`open_inputs`)."""
from __future__ import annotations

import argparse
import os

import numpy as np

from .compress import check_uncompressed


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


def cameras(poses, width: int, height: int, fx: float, fy: float) -> list:
    """One ``Camera`` of the given size and focal lengths per camera-to-world matrix of ``poses`` (row-major 3x4 or
    4x4)."""
    from .host import Camera
    cams = []
    for m in poses:
        c = Camera(width, height, fx, fy)
        c.set_c2w(m)
        cams.append(c)
    return cams


def add_view_arguments(ap: argparse.ArgumentParser, targets: bool = False) -> None:
    """The camera, pose and march options of the tools that run views over a tree: volrend_headless's pose files, -i,
    -r and image size, and the step and thresholds.  ``targets``: also the training images and the background
    brightness they are composited onto (refine, finetune)."""
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
    if targets:
        ap.add_argument("--targets", nargs="+", required=True,
                        help="one PNG per pose, or one .npy [views, height, width, 3|4] (uint8 or float in [0, 1])")
        ap.add_argument("--background", type=float, default=1.0,
                        help="background brightness: renders and the compositing of RGBA targets")


def view_setup(ap: argparse.ArgumentParser, args) -> list:
    """The cameras of add_view_arguments' values (ap.error on a bad one)."""
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
    return cameras(poses, args.width, args.height, fx, fy)


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


class _PngTargets:
    """One PNG per view, decoded when indexed."""

    def __init__(self, paths):
        self.paths = list(paths)

    def __len__(self):
        return len(self.paths)

    def __getitem__(self, i):
        if isinstance(i, slice):
            return _PngTargets(self.paths[i])
        from PIL import Image
        with Image.open(self.paths[i]) as im:
            return np.asarray(im.convert("RGBA" if im.mode in ("RGBA", "LA", "P") else "RGB"))


def read_targets(paths, n_views: int, width: int, height: int):
    """The targets of the CLI: one ``.npy`` [V, H, W, 3 | 4] (memory-mapped) or one PNG per view.  Raises ValueError
    when their number or size does not match the views."""
    if len(paths) == 1 and paths[0].endswith(".npy"):
        t = np.load(paths[0], mmap_mode="r")
        if t.ndim != 4 or t.shape[-1] not in (3, 4):
            raise ValueError(f"{paths[0]} has shape {t.shape}, not [views, height, width, 3 | 4]")
        if t.dtype != np.uint8 and not np.issubdtype(t.dtype, np.floating):
            raise ValueError(f"{paths[0]} holds {t.dtype}, not uint8 or float")
        n, size = t.shape[0], (t.shape[1], t.shape[2])
        if n == n_views and size != (height, width):
            raise ValueError(f"targets are {size[1]}x{size[0]}, the views {width}x{height}")
    else:
        if any(not p.lower().endswith(".png") for p in paths):
            raise ValueError("targets are one .npy file or one .png per pose")
        from PIL import Image
        t, n = _PngTargets(paths), len(paths)
        for p in paths:
            with Image.open(p) as im:
                if im.size != (width, height):
                    raise ValueError(f"{p} is {im.size[0]}x{im.size[1]}, the views {width}x{height}")
    if n != n_views:
        raise ValueError(f"{n} targets for {n_views} poses")
    return t


def target_rgb(img, background: float, device):
    """[H, W, 3 | 4] uint8 or float -> float32 RGB on ``device``; alpha composited onto ``background``."""
    import torch
    t = img if isinstance(img, torch.Tensor) else torch.from_numpy(np.array(img))   # (a copy: targets may be read-only)
    t = t.to(device=device)
    t = t.float() / 255.0 if t.dtype == torch.uint8 else t.float()
    if t.shape[-1] == 4:
        a = t[..., 3:4]
        t = t[..., :3] * a + background * (1.0 - a)
    return t


def target_batch(targets, idx, background: float, device, H: int, W: int):
    """The targets of the views ``idx`` as one float32 RGB tensor [len(idx), H, W, 3] on ``device``
    (:func:`target_rgb`).  Raises ValueError when they are not of the views' size H x W."""
    import torch
    tgt = torch.stack([target_rgb(targets[int(v)], background, device) for v in idx])
    if tuple(tgt.shape) != (len(idx), H, W, 3):
        raise ValueError(f"targets are {tuple(tgt.shape[1:3])}, the views {H}x{W}")
    return tgt


def pixel_error(render, target):
    """The pixel error the CLIs and the coarse-to-fine fit score leaves with: the squared RGB error of a float render
    ``[..., 4]`` against background-composited RGB targets ``[..., 3]``, summed over the channels."""
    return (render[..., :3] - target).square().sum(-1)


def open_inputs(ap: argparse.ArgumentParser, args, advice: str, holdout: int = 0):
    """The opening of the tools' command lines, after their own flag checks: ``(tree, cams, targets, d, options)``.
    In this order, each failure an ``ap.error`` raised before the device is touched: the output must not be the input;
    the input and the targets (when the tool takes them, ``add_view_arguments(targets=True)``) must exist; the views
    (:func:`view_setup`), of which at least one must remain after the last ``holdout`` are held out; the targets
    (:func:`read_targets`); the input read into the dict ``d``, which must hold an uncompressed tree (``advice`` says
    in which order to run the tools instead).  Then the tree goes on the device with the slot map, and ``options``
    are the march flags' RenderOptions, with the background brightness 1.0 of a tool without ``--background``."""
    if os.path.abspath(args.input) == os.path.abspath(args.output):
        ap.error("the output would overwrite the input")
    targets = getattr(args, "targets", None)
    for p in [args.input] + (targets or []):
        if not os.path.exists(p):
            ap.error(f"'{p}' does not exist")
    cams = view_setup(ap, args)
    if not 0 <= holdout < len(cams):
        ap.error(f"--holdout {holdout} must leave at least one of the {len(cams)} poses to train on")
    if targets is not None:
        try:
            targets = read_targets(targets, len(cams), args.width, args.height)
        except ValueError as e:
            ap.error(str(e))
    with np.load(args.input) as z:
        d = {k: z[k] for k in z.files}
    try:
        check_uncompressed(d, advice)
    except ValueError as e:
        ap.error(f"{args.input}: {e}")

    from .host import RenderOptions
    tree = load_tree_arrays(d, args.input)
    options = RenderOptions(step_size=args.step_size, sigma_thresh=args.sigma_thresh, stop_thresh=args.stop_thresh,
                            background_brightness=getattr(args, "background", 1.0))
    return tree, cams, targets, d, options
