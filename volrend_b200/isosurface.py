"""Extract surface meshes from trees on the GPU: marching cubes over sigma into closed, coloured meshes, OBJ export.

    python -m volrend_b200.isosurface TREE.npz OUT.obj --level S [--depth L] [--no-color] [--basis-minmax A B]

The surface is the level set ``sigma = level`` of the tree's leaf sigma sampled at the centres of a level-L grid
(``(i + 0.5) / 2^L`` of the unit cube, padded with 0 outside it, so every surface closes at the tree's bounds).  Leaves
deeper than L are point-sampled at those centres.  A lattice edge whose endpoints lie on either side of the level
(inside: sigma > level) holds one vertex, at the linear interpolation; the triangles come from a generated table that
keeps inside 6-connected, so the mesh is a closed, consistently oriented 2-manifold with outward normals.  Vertices are
in world coordinates, so the mesh lines up with the rendered volume.  The extraction runs in ``vr_tree_isosurface``
(volrend_b200/csrc/vr_iso.cu); DESIGN.md section 23 states it bit for bit.
"""
from __future__ import annotations

import argparse
import ctypes as C
import sys

import numpy as np

from . import _capi
from ._capi import check, lib
from .host import N3Tree, RenderOptions, _stream_ptr
from .mesh import Mesh

MAX_DEPTH = 11


def default_depth(tree: N3Tree) -> int:
    """The tree's deepest leaf level, clamped to [1, 10]."""
    return min(max(int(tree.info()["max_depth"]), 1), 10)


def isosurface_arrays(tree: N3Tree, level: float, *, depth=None, color: bool = True, options=None, stream=None):
    """``(vert, faces)``: CUDA tensors float32 ``[n, 9]`` (position, colour, normal) and int32 ``[m, 3]`` (uint32 vertex
    indices) of the isosurface ``sigma = level`` of ``tree`` on its level-``depth`` lattice (``None``: the tree's
    deepest level, clamped to [1, 10]).  ``color``: each vertex takes the colour ``N3Tree.eval`` gives its edge's inside
    endpoint seen along -normal (``options``' ``basis_minmax``); otherwise white.  Written on ``stream`` (default: the
    current stream); the count synchronises it once.  Raises ``ValueError`` for a level that is not finite and > 0 or a
    depth outside [1, 11] and :class:`VolrendError` for the trees and sizes the library refuses."""
    import torch
    if not tree.is_cuda_loaded():
        tree.load_cuda()
    d = default_depth(tree) if depth is None else int(depth)
    if not 1 <= d <= MAX_DEPTH:
        raise ValueError(f"depth {d} outside [1, {MAX_DEPTH}]")
    lv = float(np.float32(level))
    if not (np.isfinite(lv) and lv > 0):
        raise ValueError(f"level {level} must be finite and > 0")
    flags = _capi.VR_ISO_COLOR if color else 0
    o = (options if options is not None else RenderOptions())._as_c()
    nv, nf = C.c_int64(), C.c_int64()
    with torch.cuda.device(tree._device):
        sp = _stream_ptr(stream)
        check(lib().vr_tree_isosurface(tree._handle, d, lv, C.byref(o), flags, None, 0, None, 0, C.byref(nv),
                                       C.byref(nf), sp))
        vert = torch.empty((nv.value, 9), dtype=torch.float32, device=f"cuda:{tree._device}")
        faces = torch.empty((nf.value, 3), dtype=torch.int32, device=f"cuda:{tree._device}")
        if stream is not None and isinstance(stream, torch.cuda.Stream):
            stream.wait_stream(torch.cuda.current_stream())
            vert.record_stream(stream)
            faces.record_stream(stream)
        if nv.value:
            check(lib().vr_tree_isosurface(tree._handle, d, lv, C.byref(o), flags, vert.data_ptr(), nv.value,
                                           faces.data_ptr(), nf.value, C.byref(nv), C.byref(nf), sp))
    return vert, faces


def extract_mesh(tree: N3Tree, level: float, *, depth=None, color: bool = True, options=None, stream=None) -> Mesh:
    """:func:`isosurface_arrays` as a host :class:`Mesh` (triangles, named ``"isosurface"``) that can be appended to
    ``VolumeRenderer.meshes`` as it is."""
    import torch
    vert, faces = isosurface_arrays(tree, level, depth=depth, color=color, options=options, stream=stream)
    if stream is not None:
        stream.synchronize()
    else:
        torch.cuda.current_stream().synchronize()
    m = Mesh(0, 0, 3)
    m.vert = vert.cpu().numpy().reshape(-1)
    m.faces = faces.cpu().numpy().view(np.uint32).reshape(-1)
    m.name = "isosurface"
    return m


def write_obj(mesh: Mesh, path: str) -> None:
    """Writes a triangle mesh as OBJ: ``v x y z r g b``, ``vn nx ny nz`` and ``f a//a b//b c//c`` (1-based), every
    float with ``%.9g`` so that float32 values read back unchanged (``Mesh.load_basic_obj``)."""
    v = np.asarray(mesh.vert, np.float32).reshape(-1, 9)
    f = np.asarray(mesh.faces, np.uint32).reshape(-1, 3).astype(np.int64) + 1
    with open(path, "w") as out:
        out.write("# isosurface: %d vertices, %d faces\n" % (v.shape[0], f.shape[0]))
        vals = v.astype(np.float64)
        out.write("".join("v %.9g %.9g %.9g %.9g %.9g %.9g\n" % tuple(r) for r in vals[:, :6]))
        out.write("".join("vn %.9g %.9g %.9g\n" % tuple(r) for r in vals[:, 6:9]))
        out.write("".join("f %d//%d %d//%d %d//%d\n" % (a, a, b, b, c, c) for a, b, c in f))


# ---------------------------------------------------------------------------------------------------------- CLI
def _parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog="python -m volrend_b200.isosurface",
                                 description="Extract the isosurface sigma = LEVEL of a PlenOctree as an OBJ mesh.")
    ap.add_argument("tree", help="tree .npz (any file N3Tree.open loads, compressed trees included)")
    ap.add_argument("out", help="output .obj")
    ap.add_argument("--level", type=float, required=True, help="iso-level of sigma (finite, > 0)")
    ap.add_argument("--depth", type=int, default=None,
                    help=f"lattice level L in [1, {MAX_DEPTH}] (2^L samples per axis); default the tree's depth, at most 10")
    ap.add_argument("--no-color", action="store_true", help="white vertices instead of the leaves' colours")
    ap.add_argument("--basis-minmax", type=int, nargs=2, default=None, metavar=("A", "B"),
                    help="basis functions summed for the colours (default: all)")
    return ap


def main(argv=None) -> int:
    ap = _parser()
    args = ap.parse_args(argv)
    if not (np.isfinite(args.level) and args.level > 0):
        ap.error(f"--level {args.level} must be finite and > 0")
    if args.depth is not None and not 1 <= args.depth <= MAX_DEPTH:
        ap.error(f"--depth {args.depth} outside [1, {MAX_DEPTH}]")
    if not args.tree.endswith(".npz"):
        ap.error(f"tree {args.tree} must be an .npz file")
    if not args.out.endswith(".obj"):
        ap.error(f"output {args.out} must end in .obj")
    if args.no_color and args.basis_minmax is not None:
        ap.error("--basis-minmax has no effect with --no-color")
    import os
    if not os.path.exists(args.tree):
        ap.error(f"tree {args.tree} does not exist")
    tree = N3Tree(args.tree)
    opt = RenderOptions()
    if args.basis_minmax is not None:
        opt.basis_minmax = list(args.basis_minmax)
    try:
        m = extract_mesh(tree, args.level, depth=args.depth, color=not args.no_color, options=opt)
    except _capi.VolrendError as e:
        print(f"error: {e}", file=sys.stderr)
        return 1
    write_obj(m, args.out)
    print(f"vertices {m.n_verts}; faces {m.faces.size // 3}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
