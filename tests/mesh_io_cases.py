"""Inputs of the drawlist / OBJ loader goldens (tests/golden/ref/mesh_*.npz, written by
``tools/make_golden.py --mesh``): drawlist ``.npz`` bytes and OBJ texts generated from seeds, plus the reference's
sample OBJ files.  Each golden holds its input and the reference's meshes (:func:`record`)."""
from __future__ import annotations

import io
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_DIR = os.path.join(ROOT, "tests", "golden", "ref")
F1E6 = np.float32(1e-6)


def _npz(compressed: bool, **arrays) -> bytes:
    b = io.BytesIO()
    (np.savez_compressed if compressed else np.savez)(b, **arrays)
    return b.getvalue()


def _points(rng, n, lo=-1.0, hi=1.0):
    return rng.uniform(lo, hi, size=(n, 3))


def normals_edge_points():
    """Vertices and faces that exercise the normal sum: degenerate and repeated-index faces, -0 contributions, norms
    at and just above float(1e-6), isolated vertices."""
    pts = [[0, 0, 0], [0, 1, 0], [0, 0, float(F1E6)],                                   # norm float(1e-6)
           [0, 0, 0], [0, 1, 0], [0, 0, float(np.nextafter(F1E6, np.float32(1)))],      # just above
           [0, 0, 0], [0, 1, 0], [0, 0, 2e-6],
           [-0.0, -1, 0], [0, -0.0, 1], [1, 0, -0.0],                                    # signed zeros
           [1, 1, 1], [1, 1, 1], [2, 2, 2],                                              # degenerate
           [5, 5, 5]]                                                                     # isolated
    faces = [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 9, 9, 10, 10, 11, 10, 0, 0, 0, 11, 9, 1]
    return np.asarray(pts, np.float64), np.asarray(faces, np.int64)


def _signed_grid(rng, n):
    return rng.choice(np.asarray([-1.0, -0.0, 0.0, 1.0, 0.5]), size=(n, 3))


def drawlist_cases() -> dict:
    """name -> (drawlist bytes, default_visible, needs_normals)."""
    rng = np.random.default_rng(20261015)
    out = {}
    out["dl_presets"] = (_npz(
        False,
        box="cube", box__color=np.asarray([0.1, 0.7, 0.3], np.float32), box__scale=np.float32(0.25),
        box__translation=np.asarray([0.5, -0.25, 1.0]), box__rotation=np.asarray([0.3, -1.2, 0.4], np.float32),
        ball="sphere", ball__rings=np.int32(9), ball__sectors=np.int64(12), ball__color=np.asarray([0.2, 0.4, 0.9]),
        ball__unlit=np.uint8(1), ball__visible=np.int64(0),
        seg="line", seg__a=np.asarray([0.1, 0.2, 0.3], np.float16), seg__b=np.asarray([-1, 2, 0.5], np.float32),
        cloud="points", cloud__points=_points(rng, 50).astype(np.float32), cloud__vert_color=rng.uniform(0, 1, 150),
        path="lines", path__points=_points(rng, 7), path__color=np.asarray([1, 0, 0], np.float64),
        pairs="lines", pairs__points=_points(rng, 6).astype(np.float16), pairs__segs=np.asarray([0, 1, 2, 3, 4, 5], np.int8),
        pairs16="lines", pairs16__points=_points(rng, 4), pairs16__segs=np.asarray([3, 0, 1, 2], np.int16),
        lat="points", lat__points=np.zeros(0, np.float32),
        fr="camerafrustum", fr__focal_length=np.float64(500.5), fr__image_width=np.int32(640),
        fr__image_height=np.float16(480), fr__z=np.float32(0.4), fr__color=np.asarray([0, 1, 1], np.float32),
    ), True, False)
    tiny_int_bits = np.asarray(6, np.int32).view(np.float32)            # a float32 read as its int32 bits
    out["dl_quirks"] = (_npz(
        True,
        Zeta="cube", alpha="Cube", _under="SPHERE", b2="sPhErE", b2__rings=tiny_int_bits, b2__sectors=np.int16(5),
        b2__color=np.asarray([0.25, 0.5, 0.75], np.float16),
        cameras="camerafrustum", cameras_image_width=np.int64(800), cameras__focal_length=np.float32(300),
        bad="points", bad__points=_points(rng, 5), bad__vert_color=np.ones(12),
        shape4="cube", shape4__color=np.asarray([0.9, 0.8, 0.7, 0.6], np.float32),
        shape31="cube", shape31__translation=np.asarray([[1.0], [2.0], [3.0]]),
        vis="cube", vis__visible=np.float32(1.0), vis__unlit=np.bool_(True), vis__scale=np.float64(2.5),
        strscale="cube", strscale__scale=np.asarray("abc"),
        many__parts__here=np.int32(1),
        fs0="mesh", fs0__points=_points(rng, 3), fs0__face_size=np.int32(0),
        fs2="mesh", fs2__points=_points(rng, 5), fs2__face_size=np.int8(2), fs2__faces=np.asarray([0, 1, 2], np.int32),
        notype__color=np.asarray([1, 1, 1], np.float32),
        ints3="cube", ints3__color=np.asarray([1, 2, 3], np.int32),
    ), True, True)
    pts, faces = normals_edge_points()
    soup = _signed_grid(rng, 3 * 40 + 2)
    grid = _signed_grid(rng, 30)
    gf = rng.integers(0, 30, size=3 * 80)
    out["dl_normals"] = (_npz(
        False,
        edge="mesh", edge__points=pts, edge__faces=faces.astype(np.int32),
        soup="mesh", soup__points=soup.astype(np.float32),
        grid="mesh", grid__points=grid, grid__faces=gf.astype(np.int64), grid__vert_color=rng.uniform(0, 1, 90),
        odd="mesh", odd__points=_points(rng, 12), odd__faces=rng.integers(0, 12, size=3 * 9 + 2).astype(np.int16),
        pts="mesh", pts__points=_points(rng, 8), pts__face_size=np.int64(1),
        lin="mesh", lin__points=_points(rng, 8), lin__face_size=np.int32(2), lin__faces=np.asarray([0, 7, 3, 4], np.uint32),
        big="mesh", big__points=_points(rng, 3000, -3, 3).astype(np.float32),
        big__faces=rng.integers(0, 3000, size=3 * 9000).astype(np.int32),
    ), False, True)
    # the layout scripts/extract_cams_drawlist.py writes, for 100 training cameras
    n = 100
    ang = rng.uniform(0, 2 * np.pi, n)
    t = np.stack([4 * np.cos(ang), 4 * np.sin(ang), rng.uniform(-1, 3, n)], 1)
    r = rng.normal(size=(n, 3)) * rng.uniform(0, 3, (n, 1))
    r[:3] = [[0, 0, 0], [1e-4, 0, 0], [0, 0, np.pi]]
    hW = 400
    out["dl_cams100"] = (_npz(
        True,
        cameras="camerafrustum", cameras__t=t, cameras__r=r, cameras__focal_length=hW / np.tan(0.5 * 0.6911112070083618),
        cameras_image_width=hW * 2, cameras_image_height=hW * 2, cameras_z=-0.25,
        cameras_color=np.array([1.0, 0.5, 0.0]),
        traj="camerafrustum", traj__t=t[:20].astype(np.float32), traj__r=r[:20].astype(np.float16),
        traj__connect=np.int8(1), traj__z=np.float64(-0.1), traj__color=np.asarray([0, 0.5, 1], np.float32),
        one="camerafrustum", one__t=np.asarray([1.0, 2.0, 3.0]), one__r=np.asarray([0.0, 0.5, 0.0]), one__connect=np.int32(1),
    ), True, False)
    dt = {}
    for i, ft in enumerate([np.float16, np.float32, np.float64]):
        dt[f"f{i}"] = "cube"
        dt[f"f{i}__scale"] = ft(0.3 + i)
        dt[f"f{i}__translation"] = np.asarray([0.1, -0.2, 0.3 * i], ft)
        dt[f"f{i}__rotation"] = np.asarray([0.7, 0.1, -0.5], ft)
        dt[f"f{i}__color"] = np.asarray([0.2, 0.3, 0.4], ft)
    for i, it in enumerate([np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64]):
        dt[f"i{i}"] = "sphere"
        dt[f"i{i}__rings"] = it(4 + i)
        dt[f"i{i}__sectors"] = np.asarray([5 + i, 99], it)
        dt[f"i{i}__visible"] = it(i % 2)
        dt[f"i{i}__unlit"] = it((i + 1) % 2)
        dt[f"l{i}"] = "lines"
        dt[f"l{i}__points"] = _points(rng, 5)
        dt[f"l{i}__segs"] = np.asarray([4, 0, 1, 3], it)
    out["dl_dtypes"] = (_npz(True, **dt), True, False)
    return out


def obj_cases() -> dict:
    """name -> (OBJ text, needs_normals)."""
    rng = np.random.default_rng(7)
    out = {}

    def fmt(x):
        return f"{x:.6f}"

    v = _points(rng, 40)
    lines = ["# plain: positions only", "o plain"] + [f"v {' '.join(fmt(x) for x in p)}" for p in v]
    tri = rng.integers(1, 41, size=(60, 3))
    lines += [f"f {a} {b} {c}" for a, b, c in tri]
    out["obj_plain"] = ("\n".join(lines) + "\n", True)

    v = _points(rng, 12)
    L = ["mtllib missing.mtl", "o forms", "s off", "usemtl none"]
    for i, p in enumerate(v):
        col = f" {rng.uniform():.3f} {rng.uniform():.3f} {rng.uniform():.3f}" if i % 3 else ""
        L.append(f"v {fmt(p[0])} {fmt(p[1])}   {fmt(p[2])}{col}")
    L += [f"vt {rng.uniform():.4f} {rng.uniform():.4f}" for _ in range(5)]
    L += [f"vn {fmt(a)} {fmt(b)} {fmt(c)}" for a, b, c in _points(rng, 12)]
    L += ["f 1 2 3", "f 4/1 5/2 6/3", "f 7//1 8//2 9//3", "f 10/1/1 11/2/2 12/3/3", "f -1 -2 -3",
          "f -4/-1/-1 -5/-2/-2 -6/-3/-3", "l 1 2 3", "g grp",
          # quads: one each way
          "f 1 2 3 4", "f 5 6 7 8", "f 2 4 6 8 ", "\tf 9 10 11 12"]
    # convex pentagon and hexagon (planar, on a circle) appended as new vertices 13..23
    for n in (5, 6):
        base = len([x for x in L if x.startswith("v ")])
        for k in range(n):
            a = 2 * np.pi * k / n
            L.append(f"v {fmt(np.cos(a))} {fmt(np.sin(a))} {fmt(0.25 * n)}")
        L.append("f " + " ".join(str(base + k + 1) for k in range(n)))
    L.append("vn 0 0 1")
    for k in range(11):
        L.append("vn 0 1 0")
    L.append("f 1 2")
    L.append("# end")
    out["obj_forms"] = ("\r\n".join(L) + "\r\n", False)

    v = _points(rng, 6)
    L = [f"v {' '.join(f'{x:.9e}' for x in p)}" for p in v]
    L += ["v 1 2 3 0.5", "v -.5 +.25 1e-3", "v 1E+2 -0 .0", "v 0.000000001234567 123456789012 3.25e-7 0.1 0.2 0.3",
          "f 1 2 3 4", "f 5 6 1", "f 7 8 9", "f 10 1 2", "f 1 1 2"]
    out["obj_numbers"] = ("\n".join(L), True)
    out["obj_fail"] = ("v 0 0 0\nv 1 0 0\nv 0 1 0\nf 0 1 2\n", False)
    # the reference's sample meshes, stored in their goldens (only make_golden.py reads them from the reference)
    for name in ("legoman", "teapot-tri"):
        path = os.path.join(os.environ.get("VOLREND_REF", "/root/reference"), "sample_obj", name + ".obj")
        if os.path.exists(path):
            with open(path, "rb") as f:
                out["obj_" + name.replace("-", "_")] = (f.read().decode("latin-1"), name == "legoman")
    return out


def record(kind: str, data: bytes, meshes: list, default_visible: bool = True, needs_normals: bool = False) -> dict:
    """One golden: the input and every field of the reference's meshes."""
    rec = dict(kind=np.asarray(kind), input=np.frombuffer(data, np.uint8), default_visible=np.bool_(default_visible),
               needs_normals=np.bool_(needs_normals), n=np.int32(len(meshes)))
    for i, m in enumerate(meshes):
        rec[f"m{i}_vert"] = m["vert"]
        rec[f"m{i}_faces"] = m["faces"]
        rec[f"m{i}_name"] = np.frombuffer(m["name"], np.uint8)
        rec[f"m{i}_f7"] = np.concatenate([[m["scale"]], m["translation"], m["rotation"]]).astype(np.float32)
        rec[f"m{i}_i3"] = np.asarray([m["face_size"], m["visible"], m["unlit"]], np.int32)
    return rec


def golden_files() -> list:
    return sorted(f for f in os.listdir(GOLDEN_DIR) if f.startswith("mesh_") and f.endswith(".npz"))


def load_golden(fname: str):
    """(kind, input bytes, default_visible, needs_normals, [mesh dicts as record() stored them])."""
    z = np.load(os.path.join(GOLDEN_DIR, fname))
    meshes = []
    for i in range(int(z["n"])):
        f7, i3 = z[f"m{i}_f7"], z[f"m{i}_i3"]
        meshes.append(dict(vert=z[f"m{i}_vert"], faces=z[f"m{i}_faces"], name=z[f"m{i}_name"].tobytes(),
                           scale=f7[0], translation=f7[1:4], rotation=f7[4:7], face_size=int(i3[0]),
                           visible=bool(i3[1]), unlit=bool(i3[2])))
    return str(z["kind"]), z["input"].tobytes(), bool(z["default_visible"]), bool(z["needs_normals"]), meshes


def as_record(m) -> dict:
    """A product Mesh in the form the goldens store."""
    return dict(vert=np.asarray(m.vert, np.float32).reshape(-1), faces=np.asarray(m.faces, np.uint32).reshape(-1),
                name=m.name.encode("utf-8"), scale=np.float32(m.scale),
                translation=np.asarray(m.translation, np.float32).reshape(3),
                rotation=np.asarray(m.rotation, np.float32).reshape(3), face_size=int(m.face_size),
                visible=bool(m.visible), unlit=bool(m.unlit))


def mismatches(got: list, want: list) -> list:
    """Fields that differ, byte for byte (NaNs and signed zeros included)."""
    bad = []
    if len(got) != len(want):
        return [f"{len(got)} meshes, want {len(want)}"]
    for i, (g, w) in enumerate(zip(got, want)):
        for k in w:
            a, b = g[k], w[k]
            if isinstance(b, np.ndarray) or isinstance(b, np.floating):
                a, b = np.asarray(a), np.asarray(b)
                if a.dtype != b.dtype or a.shape != b.shape or a.tobytes() != b.tobytes():
                    bad.append(f"mesh {i} ({w['name']!r}) {k}")
            elif a != b:
                bad.append(f"mesh {i} ({w['name']!r}) {k}: {a!r} != {b!r}")
    return bad
