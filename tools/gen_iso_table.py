"""Generate the marching-cubes triangle table of vr_tree_isosurface (DESIGN.md section 23) from its rule.

    python tools/gen_iso_table.py            # rewrite volrend_b200/csrc/vr_iso_table.h, print the largest entry
    python tools/gen_iso_table.py --check    # exit 1 when the committed header differs from the generator's output

Conventions.  Corner c of a cube (0..7) sits at offset (c & 1, (c >> 1) & 1, (c >> 2) & 1) along (x, y, z); the case
index of a cube is the sum of 1 << c over its inside corners.  Edge e (0..11) runs along axis d = e // 4 from corner
edge_corner(e) (bit d clear) to that corner + (1 << d).

The rule, per case:
  1. Each of the 6 faces is walked through its 4 corners counter-clockwise as seen from outside the cube.  Every
     maximal cyclic run of inside corners (not all 4) gives one directed segment, from the edge that enters the run
     to the edge that leaves it.  An ambiguous face (two inside corners on a diagonal) therefore gets two segments,
     each cutting off one inside corner: inside is 6-connected, and a face's segments depend on its 4 corners only, so
     the two cubes that share a face draw the same segments there.
  2. Every crossing edge ends one segment and starts another (the two faces that share an edge walk it in opposite
     directions), so the segments chain into closed loops.  Loops are listed by their smallest edge.
  3. A loop of n edges becomes n - 2 triangles fanned from one of its vertices: the smallest edge from which no fan
     diagonal joins two edges of one cube face.  (Such a diagonal could be drawn by the neighbour across that face too;
     the generator asserts that every loop has such a vertex.)
  4. The walk of step 1 winds every loop so that right-hand-rule normals point from inside to outside (checked here
     on the single-corner cases).
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "volrend_b200", "csrc", "vr_iso_table.h")


def corner_xyz(c: int):
    return (c & 1, (c >> 1) & 1, (c >> 2) & 1)


def corner_of(x: int, y: int, z: int) -> int:
    return x | (y << 1) | (z << 2)


def _others(d: int):
    """The two other axes in cyclic order: (a1, a2, d) is right-handed."""
    return (d + 1) % 3, (d + 2) % 3


def edge_corner(e: int) -> int:
    """Lower corner of edge e."""
    d, m = divmod(e, 4)
    a1, a2 = sorted(_others(d))
    xyz = [0, 0, 0]
    xyz[a1], xyz[a2] = m & 1, m >> 1
    return corner_of(*xyz)


def edge_axis(e: int) -> int:
    return e // 4


def edge_between(c0: int, c1: int) -> int:
    diff = c0 ^ c1
    assert diff in (1, 2, 4), (c0, c1)
    d = diff.bit_length() - 1
    lo = min(c0, c1)
    for e in range(4 * d, 4 * d + 4):
        if edge_corner(e) == lo:
            return e
    raise AssertionError


def face_corners(d: int, s: int):
    """The 4 corners of face (axis d, side s) counter-clockwise as seen from outside the cube."""
    a1, a2 = _others(d)
    out = []
    for p, q in ((0, 0), (1, 0), (1, 1), (0, 1)):       # counter-clockwise seen from +d
        xyz = [0, 0, 0]
        xyz[d], xyz[a1], xyz[a2] = s, p, q
        out.append(corner_of(*xyz))
    return out if s == 1 else out[::-1]


FACES = [(d, s) for d in range(3) for s in range(2)]


def face_edges(d: int, s: int):
    q = face_corners(d, s)
    return {edge_between(q[k], q[(k + 1) % 4]) for k in range(4)}


EDGE_FACES = [[f for f in range(6) if e in face_edges(*FACES[f])] for e in range(12)]


def face_segments(case: int, d: int, s: int):
    """Directed segments (edge in, edge out) of the case on face (d, s), step 1 of the rule."""
    q = face_corners(d, s)
    inside = [(case >> c) & 1 for c in q]
    if all(inside) or not any(inside):
        return []
    segs = []
    for k in range(4):
        if inside[k] and not inside[k - 1]:                      # a run starts at k
            j = k
            while inside[(j + 1) % 4]:
                j = (j + 1) % 4
            segs.append((edge_between(q[k - 1], q[k]), edge_between(q[j], q[(j + 1) % 4])))
    return segs


def case_loops(case: int):
    nxt = {}
    for d, s in FACES:
        for a, b in face_segments(case, d, s):
            assert a not in nxt, (case, a)
            nxt[a] = b
    loops, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        loop, e = [], start
        while e not in seen:
            seen.add(e)
            loop.append(e)
            e = nxt[e]
        assert e == start, (case, loop)
        loops.append(loop)
    return loops


def _shares_face(a: int, b: int) -> bool:
    return bool(set(EDGE_FACES[a]) & set(EDGE_FACES[b]))


def fan(loop):
    """Step 3: triangles of one loop, fanned from the smallest admissible vertex."""
    n = len(loop)
    for v in sorted(loop):
        r = loop.index(v)
        ring = loop[r:] + loop[:r]
        if all(not _shares_face(ring[0], ring[k]) for k in range(2, n - 1)):
            return [(ring[0], ring[k], ring[k + 1]) for k in range(1, n - 1)]
    raise AssertionError(f"no admissible fan vertex for loop {loop}")


def build_table():
    """-> list of 256 triangle lists (edge triples)."""
    return [[t for loop in case_loops(c) for t in fan(loop)] for c in range(256)]


def _check_winding(table):
    mid = lambda e: np.array(corner_xyz(edge_corner(e)), float) + 0.5 * np.eye(3)[edge_axis(e)]
    for c in range(8):
        for case, sign in ((1 << c, 1.0), (255 ^ (1 << c), -1.0)):
            (a, b, d), = table[case]
            n = np.cross(mid(b) - mid(a), mid(d) - mid(a))
            out = np.full(3, 0.5) - np.array(corner_xyz(c), float)      # from corner c towards the cube's centre
            assert sign * float(n @ out) > 0, (case, n)


def render_header(table) -> str:
    max_tri = max(len(t) for t in table)
    lines = ["// vr_iso_table.h -- marching-cubes triangle table of vr_tree_isosurface (DESIGN.md section 23).",
             "// GENERATED by tools/gen_iso_table.py from the rule stated there; do not edit.",
             "//   corner c: offset (c & 1, (c >> 1) & 1, (c >> 2) & 1) along (x, y, z); case = sum of 1 << c, c inside",
             "//   edge e: along axis e / 4 from corner kIsoEdgeCorner[e] to kIsoEdgeCorner[e] + (1 << (e / 4))",
             "#pragma once",
             "#include <stdint.h>",
             "",
             "namespace vrb {",
             "",
             f"constexpr int kIsoMaxTris = {max_tri};   // the largest entry",
             "",
             "__device__ __constant__ const uint8_t kIsoEdgeCorner[12] = {" +
             ", ".join(str(edge_corner(e)) for e in range(12)) + "};",
             "",
             "// triangles of each case",
             "__device__ __constant__ const uint8_t kIsoTriCount[256] = {"]
    for r in range(0, 256, 32):
        lines.append("    " + ", ".join(str(len(table[c])) for c in range(r, min(r + 32, 256))) + ",")
    lines.append("};")
    lines.append("")
    lines.append(f"// edges of the triangles of each case, 3 per triangle, in order")
    lines.append(f"__device__ __constant__ const uint8_t kIsoTris[256][3 * kIsoMaxTris] = {{")
    for c in range(256):
        flat = [e for t in table[c] for e in t]
        flat += [0] * (3 * max_tri - len(flat))
        lines.append("    {" + ", ".join(str(e) for e in flat) + "},")
    lines.append("};")
    lines.append("")
    lines.append("}  // namespace vrb")
    return "\n".join(lines) + "\n"


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--check", action="store_true", help="compare with the committed header instead of writing it")
    args = ap.parse_args(argv)
    table = build_table()
    _check_winding(table)
    text = render_header(table)
    print(f"largest entry: {max(len(t) for t in table)} triangles")
    if args.check:
        with open(HEADER) as f:
            same = f.read() == text
        print("header up to date" if same else f"{HEADER} differs from the generator's output")
        return 0 if same else 1
    with open(HEADER, "w") as f:
        f.write(text)
    return 0


if __name__ == "__main__":
    sys.exit(main())
