"""Compress a PlenOctree ``.npz``: median-cut colour quantisation on the GPU into the ``quant_colors`` /
``quant_map`` / ``sigma`` / ``data_retained`` format that ``N3Tree`` (and the reference loader) decode, then deflate.

    python -m volrend_b200.compress tree.npz [more.npz ...] [--bits 16] [--retain 1] [--sigma_thresh 2.0]
                                    [--out_dir min_alt] [--overwrite] [--noquant]

The quantisation runs in ``vr_tree_compress`` (volrend_b200/csrc/vr_quant.cu); DESIGN.md section 12 states the
algorithm bit for bit.  Codebooks always have 65536 rows, whatever ``--bits`` is, because that is the stride the
loaders read them with.  ``--noquant`` only drops the training-time keys and deflates; it needs no GPU.
"""
from __future__ import annotations

import argparse
import ctypes as C
import os
import sys
import tempfile

import numpy as np

from . import _capi
from ._capi import VolrendError, check, lib
from .host import _stream_ptr

ROWS = 65536
# training-time keys the compressed file does not keep (each only when present)
DROPPED_KEYS = ("parent_depth", "geom_resize_fact", "n_free", "n_internal", "depth_limit")


def carried_keys(z, replaced=()) -> list:
    """The keys of the tree dict ``z`` (``N3Tree`` npz keys) that a rewrite of it carries over unchanged: all but the
    ``replaced`` ones and DROPPED_KEYS."""
    return [k for k in (z.files if hasattr(z, "files") else z) if k not in replaced and k not in DROPPED_KEYS]


def check_uncompressed(z, advice: str) -> None:
    """Raises ValueError unless the tree dict ``z`` holds the uncompressed ``child`` and ``data`` arrays that pruning,
    refinement and fine-tuning rewrite; ``advice`` says in which order to run the tools instead."""
    keys = z.files if hasattr(z, "files") else z
    if "quant_map" in keys or "quant_colors" in keys:
        raise ValueError(f"the tree is already compressed (quant_map): {advice}")
    for k in ("child", "data"):
        if k not in keys:
            raise ValueError(f"the tree has no '{k}' array")


def compress_device(data, data_dim: int, sigma_thresh: float = 2.0, retain: int = 1, bits: int = 16, stream=None):
    """``vr_tree_compress`` on a CUDA tensor ``data`` (fp16 or int16 bits, [n_child, data_dim] or any shape with
    that many elements).  Returns device int16 tensors (fp16 bits) ``(quant_colors [n_quant, 65536, 3], quant_map
    [n_quant, n_child], sigma [n_child], data_retained [retain, n_child, 3] or None)`` and the kept count.  Raises
    ``ValueError`` for the inputs the compressor rejects."""
    import torch
    if not data.is_cuda or data.element_size() != 2 or not data.is_contiguous():
        raise ValueError("data must be a contiguous CUDA tensor of 2-byte elements (fp16 bits)")
    if data_dim <= 0 or data.numel() % data_dim != 0:
        raise ValueError(f"data has {data.numel()} elements, not a multiple of data_dim {data_dim}")
    n_child = data.numel() // data_dim
    B = (data_dim - 1) // 3
    nq, dev = max(B - retain, 1), data.device
    colors = torch.empty((nq, ROWS, 3), dtype=torch.int16, device=dev)
    qmap = torch.empty((nq, n_child), dtype=torch.int16, device=dev)
    sigma = torch.empty(n_child, dtype=torch.int16, device=dev)
    retained = torch.empty((retain, n_child, 3), dtype=torch.int16, device=dev) if retain > 0 else None
    kept = C.c_int64()
    rc = lib().vr_tree_compress(data.data_ptr(), n_child, int(data_dim), float(sigma_thresh), int(retain), int(bits),
                                colors.data_ptr(), qmap.data_ptr(), sigma.data_ptr(),
                                retained.data_ptr() if retained is not None else None, C.byref(kept), _stream_ptr(stream))
    if rc == _capi.VR_EINVAL:
        raise ValueError(lib().vr_last_error().decode("utf-8", "replace"))
    check(rc)
    return (colors, qmap, sigma, retained), int(kept.value)


def compress_arrays(data: np.ndarray, data_dim: int, sigma_thresh: float, retain: int, bits: int):
    """Host arrays in and out: data u16 [n_child, data_dim] (fp16 bits) -> (quant_colors u16 [n_quant, 65536, 3],
    quant_map u16 [n_quant, n_child], sigma u16 [n_child], data_retained u16 [retain, n_child, 3] or None, n_kept)."""
    import torch
    if not torch.cuda.is_available():
        raise VolrendError(_capi.VR_ENODEVICE, "no CUDA device: volrend_b200 has no CPU fallback")
    d = torch.from_numpy(np.ascontiguousarray(data).view(np.int16)).to("cuda")
    outs, kept = compress_device(d, data_dim, sigma_thresh, retain, bits)
    host = [None if t is None else t.cpu().numpy().view(np.uint16) for t in outs]
    return host[0], host[1], host[2], host[3], kept


def _check_args(bits: int, retain: int, data_dim: int, data: np.ndarray) -> None:
    if not 1 <= bits <= 16:
        raise ValueError(f"bits {bits} outside [1, 16]")
    if retain < 0:
        raise ValueError(f"retain {retain} < 0")
    B = (data_dim - 1) // 3
    if data_dim < 4 or data_dim != 3 * B + 1:
        raise ValueError(f"data_dim {data_dim} is not 3 * basis_dim + 1")
    if B - retain < 1:
        raise ValueError(f"retain {retain} leaves no basis function to quantise (the tree has {B}); "
                         "use --noquant for RGBA trees")
    if data.shape[-1] != data_dim:
        raise ValueError(f"data has {data.shape[-1]} channels, data_dim says {data_dim}")


def compress_npz(z, *, bits: int = 16, sigma_thresh: float = 2.0, retain: int = 1, backend=None) -> dict:
    """The compressed form of the tree dict ``z`` (``N3Tree`` npz keys): ``data`` and the training-time keys are
    dropped, every other key passes through, and ``quant_colors`` fp16 [n_quant, 65536, 3], ``quant_map`` u16
    [n_quant, cap, N, N, N], ``sigma`` fp16 [cap, N, N, N] and, when ``retain > 0``, ``data_retained`` fp16
    [retain, cap, N, N, N, 3] are added.  ``backend`` replaces the device call (same signature as
    ``compress_arrays``; the tests pass the numpy oracle)."""
    z = {k: z[k] for k in (z.files if hasattr(z, "files") else z)}
    data = np.asarray(z["data"])
    data_dim = int(np.asarray(z["data_dim"]).reshape(-1)[0])
    _check_args(bits, retain, data_dim, data)
    if data.dtype.itemsize != 2:
        raise ValueError("data must be stored in half precision")
    shape = data.shape[:-1]
    flat = np.ascontiguousarray(data).view(np.uint16).reshape(-1, data_dim)
    colors, qmap, sigma, retained, _ = (backend or compress_arrays)(flat, data_dim, sigma_thresh, retain, bits)
    out = {k: z[k] for k in carried_keys(z, ("data",))}
    out["quant_colors"] = colors.view(np.float16).reshape(-1, ROWS, 3)
    out["quant_map"] = qmap.reshape((-1,) + shape)
    out["sigma"] = sigma.view(np.float16).reshape(shape)
    if retain > 0:
        out["data_retained"] = retained.view(np.float16).reshape((retain,) + shape + (3,))
    return out


def _write_npz(path: str, d: dict) -> None:
    """np.savez_compressed to ``path`` through a temporary file, so a failure leaves no partial output.  The file gets
    the permissions a plain ``open(path, "w")`` would give it (0666 less the umask)."""
    fd, tmp = tempfile.mkstemp(suffix=".npz.tmp", dir=os.path.dirname(path) or ".")
    try:
        with os.fdopen(fd, "wb") as f:
            np.savez_compressed(f, **d)
        umask = os.umask(0)
        os.umask(umask)
        os.chmod(tmp, 0o666 & ~umask)
        os.replace(tmp, path)
    except BaseException:
        os.unlink(tmp)
        raise


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog="python -m volrend_b200.compress",
                                 description="Compress PlenOctree npz files: median-cut colour quantisation on the GPU "
                                             "+ deflate.  The output opens in volrend as before.")
    ap.add_argument("input", nargs="+", help="input npz file(s)")
    ap.add_argument("--noquant", action="store_true", help="no quantisation: only drop training keys and deflate")
    ap.add_argument("--bits", type=int, default=16, help="median-cut levels: 2^bits colours per codebook (1..16)")
    ap.add_argument("--out_dir", default="min_alt", help="where to write the compressed npz files")
    ap.add_argument("--overwrite", action="store_true", help="overwrite existing compressed files")
    ap.add_argument("--weighted", action="store_true", help="weighted median cut (not supported)")
    ap.add_argument("--sigma_thresh", type=float, default=2.0, help="voxels with sigma <= this are dropped")
    ap.add_argument("--retain", type=int, default=1,
                    help="keep the first RETAIN basis functions unquantised (lego looks better with 4)")
    args = ap.parse_args(argv)
    if args.weighted:
        ap.error("--weighted is not supported: the weighted median cut is not implemented")
    if not args.noquant and not 1 <= args.bits <= 16:
        ap.error(f"--bits {args.bits} outside [1, 16]")
    if not args.noquant and args.retain < 0:
        ap.error(f"--retain {args.retain} < 0")
    os.makedirs(args.out_dir, exist_ok=True)
    print("Quantization disabled, only applying deflate" if args.noquant else "Quantization enabled")
    failed = 0
    for fname in args.input:
        out = os.path.join(args.out_dir, os.path.basename(fname))
        print("Compressing", fname, "to", out)
        if not args.overwrite and os.path.exists(out):
            print(" > skip")
            continue
        with np.load(fname) as z:
            if not args.noquant and "quant_colors" in z.files:
                print(" > skip since source already compressed")
                continue
            d = {k: z[k] for k in z.files}
        try:
            if args.noquant:
                d = {k: d[k] for k in carried_keys(d)}
            else:
                d = compress_npz(d, bits=args.bits, sigma_thresh=args.sigma_thresh, retain=args.retain)
        except (ValueError, VolrendError) as e:
            print(f" > error: {e}", file=sys.stderr)
            failed += 1
            continue
        _write_npz(out, d)
        mb = 1024.0 * 1024.0
        print(f" > Size {os.path.getsize(fname) / mb:.2f} MB -> {os.path.getsize(out) / mb:.2f} MB")
    return 1 if failed else 0


if __name__ == "__main__":
    sys.exit(main())
