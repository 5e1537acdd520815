"""Scenes for the mesh rasterizer's float64 reference (oracle/raster_ref64.py): the frame sizes, tile and small/large
boundaries, near-plane and guard-band cases, fill-rule, line, point, shading, incoming-depth and invalid-vertex edges
where rasterizers go wrong.  ``scene(name, small)`` builds one; ``small`` shrinks the scenes whose size is not the
point, for the CPU comparison with oracle/mesh_oracle.py."""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np

from oracle import raster_ref64 as rr

F = np.float32


@dataclass
class Scene:
    W: int
    H: int
    fx: float
    fy: float
    c2w: np.ndarray                 # 12 float32, column-major 3x4
    meshes: list                    # volrend_b200.Mesh
    depth0: np.ndarray = None
    rgba0: np.ndarray = None
    amb_max: float = 0.03
    ids: bool = False               # unlit colours encode the primitive: the winner is checked by colour
    extra: dict = field(default_factory=dict)

    def __post_init__(self):
        if self.depth0 is None:
            self.depth0 = np.full((self.H, self.W), 1e9, F)
        if self.rgba0 is None:
            self.rgba0 = np.full((self.H, self.W, 4), 7, np.uint8)


def c2w_look(eye, target, up=(0.0, 0.0, 1.0), scale=1.0):
    """Column-major 3x4 camera-to-world looking from eye at target (camera looks down -z), rotation times scale."""
    e, t, u = (np.asarray(v, np.float64) for v in (eye, target, up))
    back = e - t
    back /= np.linalg.norm(back)
    right = np.cross(u, back)
    right /= np.linalg.norm(right)
    upv = np.cross(back, right)
    return np.concatenate([right * scale, upv * scale, back * scale, e]).astype(F)


IDENT = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], F)     # camera at the origin looking down -z, +y up


def camera(s: Scene):
    from volrend_b200 import Camera
    c = Camera(s.W, s.H, s.fx, s.fy)
    c.transform = np.ascontiguousarray(np.asarray(s.c2w, F).reshape(4, 3))
    return c


def ref_spec(m):
    faces = np.asarray(m.faces, np.uint32)
    return dict(vert=np.asarray(m.vert, F), faces=faces if faces.size else None, face_size=m.face_size,
                unlit=bool(m.unlit), rotation=m.rotation, translation=m.translation, scale=m.scale)


def oracle_spec(m):
    faces = np.asarray(m.faces, np.uint32)
    return dict(vert=np.asarray(m.vert, F), faces=faces if faces.size else None, face_size=m.face_size,
                unlit=int(m.unlit), model=m.model_matrix().T.reshape(16))


def reference(s: Scene):
    return rr.draw(s.W, s.H, s.fx, s.fy, s.c2w, [ref_spec(m) for m in s.meshes], s.rgba0, s.depth0)


def prim_offsets(meshes):
    n = [(np.asarray(m.faces).size or np.asarray(m.vert).size // 9) // m.face_size for m in meshes]
    return np.concatenate([[0], np.cumsum(n)]).astype(np.int64)


def code_rgb(code):
    return np.stack([code & 255, (code >> 8) & 255, code >> 16], -1).astype(F) / F(255)


def decode(rgba):
    r = rgba.astype(np.int64)
    return r[..., 0] + 256 * r[..., 1] + 65536 * r[..., 2] - 1


def soup(prims, unlit=True, normals=None, colours=None):
    """A non-indexed mesh of primitives ``prims`` [n, face_size, 3]."""
    from volrend_b200 import Mesh
    prims = np.asarray(prims, np.float64)
    n, fsz = prims.shape[:2]
    m = Mesh(n * fsz, 0, fsz, unlit=unlit)
    v = m.vert.reshape(-1, 9)
    v[:, :3] = prims.reshape(-1, 3)
    v[:, 3:6] = 0.5 if colours is None else np.asarray(colours, F).reshape(-1, 3)
    v[:, 6:9] = (0, 0, 1) if normals is None else np.asarray(normals, F).reshape(-1, 3)
    return m


def id_code(meshes):
    """Expands every mesh to consecutive vertices, unlit, with each primitive's colour encoding its global index + 1
    (the winner is then read back from the 8-bit colour)."""
    from volrend_b200 import Mesh
    out, code = [], 1
    for m in meshes:
        v = np.asarray(m.vert, F).reshape(-1, 9)
        f = np.asarray(m.faces, np.uint32)
        idx = f.astype(np.int64) if f.size else np.arange(v.shape[0] - v.shape[0] % m.face_size)
        e = Mesh(idx.size, 0, m.face_size, unlit=True)
        ev = e.vert.reshape(-1, 9)
        ok = idx < v.shape[0]
        ev[ok] = v[idx[ok]]
        ev[~ok, :3] = np.nan                      # an out-of-range index draws nothing; so does a NaN vertex
        n = idx.size // m.face_size
        ev[:, 3:6] = np.repeat(code_rgb(np.arange(code, code + n)), m.face_size, 0)
        code += n
        e.rotation, e.translation, e.scale = m.rotation.copy(), m.translation.copy(), m.scale
        out.append(e)
    return out


def win_xyz(wx, wy, D, f, W, H):
    """Camera-space point (= world point under IDENT) at camera depth D projecting to window (wx, wy)."""
    return np.stack([(np.asarray(wx, np.float64) - W / 2) * D / f, (H / 2 - np.asarray(wy, np.float64)) * D / f,
                     np.full(np.shape(wx), -float(D))], -1)


def _tri_soup(rng, n, spread=1.0, size=0.5, centre=(0, 0, 0)):
    c = rng.uniform(-spread, spread, (n, 1, 3)) + np.asarray(centre)
    return c + rng.uniform(-size, size, (n, 3, 3))


def _lit(m, rng, unit=True):
    v = m.vert.reshape(-1, 9)
    v[:, 3:6] = rng.uniform(0.2, 1.0, (v.shape[0], 3))
    nn = rng.standard_normal((v.shape[0], 3))
    v[:, 6:9] = nn / np.linalg.norm(nn, axis=1, keepdims=True) if unit else nn
    m.unlit = False
    return m


# ---------------------------------------------------------------------------------------------------------- scenes
def _frame(W, H, small):
    rng = np.random.default_rng(W * 7 + H)
    f = max(0.9 * max(W, H), 40.0)
    tris = soup(_tri_soup(rng, 40, 0.9, 0.6))
    return Scene(W, H, f, f, c2w_look((2.6, -2.0, 1.4), (0, 0, 0)), id_code([tris]), ids=True)


def _strip(W, H, small):
    """A 32768-pixel side (kRasterMaxSide): triangles that run its whole length, so the packed box coordinates
    reach their largest value."""
    rng = np.random.default_rng(W + 3 * H)
    f, D = 64.0, 2.0
    prims = []
    for i in range(16):
        wx = rng.uniform(-0.05, 1.05, 3) * W
        wy = rng.uniform(-0.05, 1.05, 3) * H
        if i < 4:                        # one end beyond the last pixel
            (wx if W > H else wy)[0] = max(W, H) + 0.7
        prims.append(win_xyz(wx, wy, D * rng.uniform(0.8, 1.2), f, W, H))
    return Scene(W, H, f, f, IDENT, id_code([soup(prims)]), ids=True, amb_max=0.08)


def _split16(small):
    """Triangles of one shape at offsets that give 16x16 and 16x17 pixel boxes (kSmallPixels = 256)."""
    W, H, f, D = 160, 96, 64.0, 2.0
    prims = []
    for i in range(16):
        x0, y0 = 6 + 36 * (i % 4) + 0.05, 6 + 22 * (i // 4) + (0.05 if i % 2 == 0 else 0.3)
        shape = [(0, 0), (15.9, 3.1), (4.2, 16.4)] if i % 4 < 2 else [(15.9, 0), (0, 8.3), (9.7, 16.4)]
        pts = [(x0 + a, y0 + b) for a, b in shape]
        prims.append(win_xyz([p[0] for p in pts], [p[1] for p in pts], D, f, W, H))
    return Scene(W, H, f, f, IDENT, id_code([soup(prims)]), ids=True)


def _tile_borders(small):
    W, H, f, D = 200, 136, 64.0, 2.0
    prims = []
    for i, (a, b) in enumerate([(31, 64), (32, 65), (33, 63), (63, 128), (64, 127), (65, 129), (95, 160), (96, 161)]):
        x0, x1 = a + 0.5 - 0.3, b + 0.5 + 0.3      # boxes from pixel a to pixel b
        y0, y1 = (31 + 0.2 + (i % 3), 96 + 0.8 - (i % 3))
        quad = [(x0, y0), (x1, y0), (x1, y1), (x0, y1)]
        D_i = D + 0.25 * i
        for t in ((0, 1, 2), (0, 2, 3)):
            prims.append(win_xyz([quad[k][0] for k in t], [quad[k][1] for k in t], D_i, f, W, H))
    return Scene(W, H, f, f, IDENT, id_code([soup(prims)]), ids=True)


def _quads(small):
    """Frame-filling, tilted, interpenetrating quads: the winner flips along their intersection lines."""
    rng = np.random.default_rng(17)
    W, H, n = (192, 108, 30) if small else (480, 270, 300)
    f = 0.8 * W
    prims = []
    for _ in range(n):
        z = rng.uniform(-6, -3)
        nrm = rng.normal(size=3) * [0.4, 0.4, 1]
        nrm /= np.linalg.norm(nrm)
        xs, ys = np.array([-5, 5, 5, -5.0]), np.array([-4, -4, 4, 4.0])
        zs = z - (nrm[0] * xs + nrm[1] * ys) / nrm[2]
        q = np.stack([xs, ys, zs], -1)
        prims += [q[[0, 1, 2]], q[[0, 2, 3]]]
    return Scene(W, H, f, f, IDENT, id_code([soup(prims)]), ids=True, amb_max=0.06)


def _cube_inside(small):
    from volrend_b200 import Mesh
    rng = np.random.default_rng(2)
    out = []
    for s in (3.0, 0.015):     # a room, and a box whose walls lie between 1e-3 and 1e-2 from the camera
        c = Mesh.Cube((0.8, 0.6, 0.3))
        c.scale = s
        c.rotation[:] = (0.2, -0.1, 0.3)
        c.translation[:] = (0.1 * s, -0.05 * s, 0.02 * s)
        out.append(c)
    lit = out[0]
    _lit(lit, rng)
    return Scene(96, 72, 60.0, 60.0, c2w_look((0, 0, 0), (1, 0.3, 0.2)), [out[0]], extra=dict(small_box=out[1]))


def _cube_inside_near(small):
    s = _cube_inside(small)
    return Scene(s.W, s.H, s.fx, s.fy, s.c2w, id_code([s.extra["small_box"]]), ids=True)


def _horizon(small):
    from volrend_b200 import Mesh
    q = Mesh(4, 2, 3)
    v = q.vert.reshape(-1, 9)
    v[:, :3] = [(-1e4, -1, 0), (1e4, -1, 0), (1e4, 1e4, 0), (-1e4, 1e4, 0)]
    v[:, 3:6] = [(1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 0)]
    v[:, 6:9] = (0, 0, 1)
    q.faces[:] = (0, 1, 2, 0, 2, 3)
    return Scene(160, 120, 100.0, 100.0, c2w_look((0, 0, 0.3), (0, 5, 0.1)), [q], amb_max=0.06)


def _near_tris(small):
    W, H, f = 128, 96, 64.0
    n1 = float(F(1e-3))
    prims = [
        [(-1, -0.5, -2), (1, -0.5, -2), (0, -0.5, 1)],            # one vertex behind the camera
        [(-0.5, 0.3, -1.5), (0.4, 0.6, 2), (0.8, -0.2, 3)],       # two behind
        [(0.3, 0.2, -1.2), (0.6, -0.1, -0.9), (0, 0, -n1)],       # a vertex at d = 1e-3f
        [(-0.7, 0.1, -1.0), (-0.2, 0.5, -1.3), (0.1, 0.2, 0.0)],  # a vertex at d = 0
        [(-0.3, -0.3, -3), (0.3, -0.3, -3), (0, 0.4, 0)],         # d = 0 on the axis
    ]
    return Scene(W, H, f, f, IDENT, id_code([soup(prims)]), ids=True)


def _near_lines(small):
    rng = np.random.default_rng(4)
    segs = [[(-1, -0.5, -2), (0.5, 0.2, 1.0)], [(0.5, 0.5, -1), (-0.3, -0.1, 0.5)], [(0.2, -0.4, -3), (0.1, 0.3, 0)],
            [(-0.4, 0.1, 0.002), (0.9, -0.2, -0.5)]]
    segs += [[tuple(rng.uniform(-1, 1, 3) + (0, 0, -1.5)), tuple(rng.uniform(-1, 1, 3) + (0, 0, 0.5))] for _ in range(12)]
    return Scene(128, 96, 64.0, 64.0, IDENT, id_code([soup(segs)]), ids=True, amb_max=0.25)


def _near_points(small):
    W, H, f = 64, 48, 32.0
    pts = []
    for i, d in enumerate([2e-3, 1.2e-3, 1.05e-3, 0.95e-3, 0.8e-3, 0.0, -1.0]):
        pts.append([((i - 3) * 5 * d / f, (i % 3 - 1) * 5 * d / f, -d)])
    return Scene(W, H, f, f, IDENT, id_code([soup(pts)]), ids=True)


def _guard(small):
    """Vertices projecting to 2^20 +- a few pixels and to 1e8 pixels from the centre; edges cross the frame."""
    W, H, f, D = 256, 192, 128.0, 4.0
    prims, segs = [], []
    for k, r in enumerate([2.0 ** 20 - 3, 2.0 ** 20 + 3, 1e8]):
        for ang in (0.3 + k, 2.1 + k, 4.0 + k):
            far = (W / 2 + r * math.cos(ang), H / 2 + r * math.sin(ang))
            a = (W / 2 + 40 * math.cos(ang + 2.5), H / 2 + 40 * math.sin(ang + 2.5))
            b = (W / 2 + 50 * math.cos(ang - 2.2), H / 2 + 30 * math.sin(ang - 2.2))
            dz = D * (1 + 0.1 * k)
            prims.append(win_xyz([a[0], b[0], far[0]], [a[1], b[1], far[1]], dz, f, W, H))
            segs.append(win_xyz([b[0], far[0]], [b[1], far[1]], dz * 0.5, f, W, H))
    return Scene(W, H, f, f, IDENT, id_code([soup(prims), soup(segs)]), ids=True, amb_max=0.15)


def _grazing(small):
    """A jittered 48x48 grid surface seen at about 80 degrees, one colour per triangle."""
    rng = np.random.default_rng(8)
    n = 48
    g = np.stack(np.meshgrid(np.linspace(-2, 2, n + 1), np.linspace(-2, 2, n + 1), indexing="xy"), -1)
    g = g + rng.uniform(-0.3, 0.3, g.shape) * (4 / n)
    z = 0.02 * rng.standard_normal(g.shape[:2])
    P = np.concatenate([g, z[..., None]], -1)
    prims = []
    for i in range(n):
        for j in range(n):
            a, b, c, d = P[i, j], P[i, j + 1], P[i + 1, j + 1], P[i + 1, j]
            prims += [[a, b, c], [a, c, d]]
    el = math.radians(10)
    eye = (0, -6 * math.cos(el), 6 * math.sin(el))
    W, H = (96, 64) if small else (320, 200)
    return Scene(W, H, 0.9 * W, 0.9 * W, c2w_look(eye, (0, 0, 0)), id_code([soup(prims)]), ids=True, amb_max=0.10)


def _sphere(small):
    from volrend_b200 import Mesh
    s = Mesh.Sphere(24, 40) if small else Mesh.Sphere(120, 200)
    W = 96 if small else 320
    return Scene(W, W * 3 // 4, 0.8 * W, 0.8 * W, c2w_look((2.2, -1.7, 1.1), (0, 0, 0)), id_code([s]), ids=True,
                 amb_max=0.05 if small else 0.25)


def _subpixel(small):
    rng = np.random.default_rng(9)
    W, H, f, D = 96, 64, 64.0, 2.0
    n = 300 if small else 1000
    c = np.stack([rng.uniform(2, W - 2, n), rng.uniform(2, H - 2, n)], -1)
    pts = c[:, None, :] + rng.uniform(-0.7, 0.7, (n, 3, 2))
    prims = [win_xyz(p[:, 0], p[:, 1], D * rng.uniform(0.8, 1.2), f, W, H) for p in pts]
    return Scene(W, H, f, f, IDENT, id_code([soup(prims)]), ids=True, amb_max=0.9)


def _needles(small):
    rng = np.random.default_rng(10)
    W, H, f, D = 256, 256, 128.0, 2.0
    prims = []
    for i in range(24):
        a = rng.uniform(0, math.pi)
        c = rng.uniform(60, 196, 2)
        u, n = np.array([math.cos(a), math.sin(a)]), np.array([-math.sin(a), math.cos(a)])
        p = [c - 100 * u, c + 100 * u, c + 100 * u + 0.3 * n]
        prims.append(win_xyz([q[0] for q in p], [q[1] for q in p], D + 0.01 * i, f, W, H))
    return Scene(W, H, f, f, IDENT, id_code([soup(prims)]), ids=True, amb_max=0.9)


def _collinear(small):
    """Triangles whose plane passes through the eye: a segment on screen, a triangle in 3-D."""
    rng = np.random.default_rng(11)
    prims = []
    for _ in range(12):
        a, b = rng.uniform(-1, 1, 3) + (0, 0, -3), rng.uniform(-1, 1, 3) + (0, 0, -3)
        prims.append([a, b, a * rng.uniform(0.5, 2)])        # the third vertex on the eye ray through a
    prims.append([(-1, -1, -2), (1, 1, -2), (2, 2, -2)])     # collinear in 3-D as well
    return Scene(96, 64, 64.0, 64.0, IDENT, id_code([soup(prims)]), ids=True, amb_max=1.0)


def _lines(small):
    W, H, f, D = 96, 64, 64.0, 2.0
    segs = []
    for y in (10.5, 11.0, 12.3):
        segs.append(((5.25, y), (60.7, y)))          # horizontal, on a centre row, on a row boundary
    for x in (20.5, 21.0):
        segs.append(((x, 3.4), (x, 50.6)))           # vertical
    segs += [((30.5, 20.5), (50.5, 40.5)), ((70.5, 55.5), (50.5, 35.5)), ((40.5, 60.5), (60.5, 40.5))]   # 45 degrees
    segs += [((5.5, 30.5), (25.5, 36.5)), ((8.5, 40.5), (14.5, 60.5))]       # endpoints on pixel centres
    segs += [((80.2, 10.3), (80.7, 10.6)), ((82.4, 20.5), (82.4, 20.9)), ((85.1, 30.5), (85.6, 30.5))]  # short
    prims = [win_xyz([a[0], b[0]], [a[1], b[1]], D, f, W, H) for a, b in segs]
    # a perspective line (varying depth)
    prims.append(np.array([[-1.0, -0.3, -1.5], [1.2, 0.4, -5.0]]))
    return Scene(W, H, f, f, IDENT, id_code([soup(prims)]), ids=True, amb_max=0.6)


def _points(small):
    W, H, f, D = 64, 48, 32.0, 2.0
    c = [(10.5, 10.5), (20.0, 10.0), (30.5, 12.0), (40.25, 20.75),      # footprint boundaries through centres
         (0.0, 24.0), (63.9, 24.0), (32.0, 0.3), (32.0, 47.8),          # partly outside each edge
         (0.5, 0.5), (63.5, 0.0), (-1.0, 47.0), (64.5, 48.5)]           # and each corner
    prims = [win_xyz([x], [y], D, f, W, H) for x, y in c]
    return Scene(W, H, f, f, IDENT, id_code([soup(prims)]), ids=True, amb_max=0.6)


def _lit_scene(small, cam_scale=1.0, unit=True, rot=(0.4, -0.3, 0.8), fy_ratio=1.0, scale=1.3):
    from volrend_b200 import Mesh
    rng = np.random.default_rng(12)
    s = Mesh.Sphere(16, 24, (0.9, 0.7, 0.4))
    s.scale, s.rotation[:], s.translation[:] = scale, rot, (0.1, -0.2, 0.05)
    if not unit:
        v = s.vert.reshape(-1, 9)
        v[:, 6:9] *= rng.uniform(0.3, 3.0, (v.shape[0], 1))
    tris = _lit(soup(_tri_soup(rng, 12, 0.9, 0.5), unlit=False), rng, unit)
    W = 96
    return Scene(W, 72, 80.0, 80.0 * fy_ratio, c2w_look((3.0, -2.2, 1.6), (0, 0, 0), scale=cam_scale), [s, tris],
                 amb_max=0.06)


def _specular(small):
    """A lit quad facing the camera so that the reflected light direction passes through the view: a highlight."""
    from volrend_b200 import Mesh
    q = Mesh(4, 2, 3)
    v = q.vert.reshape(-1, 9)
    v[:, :3] = [(-2, -2, 0), (2, -2, 0), (2, 2, 0), (-2, 2, 0)]
    v[:, 3:6] = (0.6, 0.6, 0.6)
    v[:, 6:9] = (0, 0, 1)
    q.faces[:] = (0, 1, 2, 0, 2, 3)
    L = np.array([0.5, 0.2, 1.0]) / np.linalg.norm([0.5, 0.2, 1.0])
    return Scene(96, 96, 60.0, 60.0, c2w_look(L * 3, (0, 0, 0), up=(0, 1, 0)), [q], amb_max=0.05)


def _depth_in(kind):
    def make(small):
        s = _frame(64, 48, small)
        rng = np.random.default_rng(13)
        s.depth0 = {"zero": np.zeros((48, 64), F), "random": rng.uniform(0.5, 6, (48, 64)).astype(F),
                    "huge": np.full((48, 64), 1e9, F)}[kind]
        s.rgba0 = rng.integers(0, 256, (48, 64, 4)).astype(np.uint8)
        return s
    return make


def _invalid(small):
    rng = np.random.default_rng(14)
    prims = _tri_soup(rng, 20, 0.9, 0.5)
    prims[3, 1, 0] = np.nan
    prims[7, 2, 2] = np.inf
    s = _frame(64, 48, small)
    return Scene(64, 48, s.fx, s.fy, s.c2w, id_code([soup(prims)]), ids=True, extra=dict(invalid=(3, 7)))


# ------------------------------------------------------------------------------ exact scenes (fractions.Fraction)
# Fronto-parallel primitives under IDENT with power-of-two focal length and depth: every window coordinate is exact,
# so ownership follows from the rules alone, with no ambiguity: the top-left rule for triangles, [start, end) along
# the major axis for lines, [x - 2, x + 2) for points.
EXACT_F, EXACT_D = 64.0, 2.0


def _exact_scene(W, H, prims):
    return Scene(W, H, EXACT_F, EXACT_F, IDENT, id_code([soup(p) for p in prims]), ids=True)


def _fill_grid(small):
    """A grid of triangles whose vertices lie on pixel centres and pixel edges, in both diagonal directions."""
    W, H = 48, 40
    xs = [2.0, 7.5, 13.0, 20.5, 26.5, 33.0, 40.5, 45.0]
    ys = [1.5, 6.0, 13.5, 19.0, 26.0, 31.5, 38.0]
    prims = []
    for j in range(len(ys) - 1):
        for i in range(len(xs) - 1):
            a, b, c, d = (xs[i], ys[j]), (xs[i + 1], ys[j]), (xs[i + 1], ys[j + 1]), (xs[i], ys[j + 1])
            tris = [(a, b, c), (a, c, d)] if (i + j) % 2 else [(a, b, d), (b, c, d)]
            for t in tris:
                prims.append(win_xyz([p[0] for p in t], [p[1] for p in t], EXACT_D, EXACT_F, W, H))
    return _exact_scene(W, H, [prims])


def _lines_exact(small):
    W, H = 64, 48
    segs = [((3.5, 4.5), (20.5, 4.5)), ((20.5, 6.5), (3.5, 6.5)), ((30.5, 2.5), (30.5, 20.5)),
            ((40.5, 3.5), (50.5, 13.5)), ((5.5, 30.5), (17.5, 34.5)), ((33.5, 40.5), (36.5, 28.5)),
            ((45.0, 30.0), (60.0, 35.0)), ((50.5, 20.5), (51.25, 20.5))]
    return _exact_scene(W, H, [[win_xyz([a[0], b[0]], [a[1], b[1]], EXACT_D, EXACT_F, W, H) for a, b in segs]])


def _points_exact(small):
    W, H = 40, 32
    c = [(6.5, 6.5), (16.0, 6.0), (26.5, 7.0), (35.0, 10.5), (1.0, 20.0), (39.5, 22.0), (12.0, 0.5), (22.0, 31.5)]
    return _exact_scene(W, H, [[win_xyz([x], [y], EXACT_D, EXACT_F, W, H) for x, y in c]])


EXACT = {"fill_grid": _fill_grid, "lines_exact": _lines_exact, "points_exact": _points_exact}


def exact_owner(s: Scene):
    """Per pixel, the global index of the primitive that owns its centre under the rules, in exact arithmetic
    (-1: none).  Fails if two primitives claim one pixel."""
    from fractions import Fraction as Q
    own = np.full((s.H, s.W), -1, np.int64)
    g = 0
    for m in s.meshes:
        v = np.asarray(m.vert, F).reshape(-1, 9)
        fsz = m.face_size
        for k in range(v.shape[0] // fsz):
            P = [(Q(s.W, 2) + Q(float(p[0])) * Q(EXACT_F) / Q(EXACT_D),
                  Q(s.H, 2) - Q(float(p[1])) * Q(EXACT_F) / Q(EXACT_D)) for p in v[k * fsz:(k + 1) * fsz, :3]]
            x0, x1 = max(int(min(p[0] for p in P)) - 3, 0), min(int(max(p[0] for p in P)) + 3, s.W - 1)
            y0, y1 = max(int(min(p[1] for p in P)) - 3, 0), min(int(max(p[1] for p in P)) + 3, s.H - 1)
            for py in range(y0, y1 + 1):
                for px in range(x0, x1 + 1):
                    c = (Q(2 * px + 1, 2), Q(2 * py + 1, 2))
                    if fsz == 3:
                        a, b, d = P
                        area = (b[0] - a[0]) * (d[1] - a[1]) - (d[0] - a[0]) * (b[1] - a[1])
                        if area < 0:
                            b, d = d, b
                        ok = True
                        for e0, e1 in ((b, d), (d, a), (a, b)):
                            dx, dy = e1[0] - e0[0], e1[1] - e0[1]
                            e = dx * (c[1] - e0[1]) - dy * (c[0] - e0[0])
                            ok &= e > 0 or (e == 0 and (dy < 0 or (dy == 0 and dx < 0)))
                    elif fsz == 2:
                        a, b = P
                        ax = 0 if abs(b[0] - a[0]) >= abs(b[1] - a[1]) else 1
                        lo, hi = sorted((a, b), key=lambda p: p[ax])
                        t = (c[ax] - lo[ax]) / (hi[ax] - lo[ax])
                        minor = lo[1 - ax] + t * (hi[1 - ax] - lo[1 - ax])
                        ok = lo[ax] <= c[ax] < hi[ax] and math.floor(minor) == (py, px)[ax]
                    else:
                        ok = all(P[0][i] - 2 <= c[i] < P[0][i] + 2 for i in (0, 1))
                    if ok:
                        assert own[py, px] < 0, (px, py)
                        own[py, px] = g
            g += 1
    return own


SCENES = {
    "frame_1x1": lambda s: _frame(1, 1, s),
    "frame_1x97": lambda s: _frame(1, 97, s),
    "frame_97x1": lambda s: _frame(97, 1, s),
    "frame_33x31": lambda s: _frame(33, 31, s),
    "frame_1920x1080": lambda s: _frame(1920, 1080, s),
    "frame_32768x8": lambda s: _strip(32768, 8, s),
    "frame_8x32768": lambda s: _strip(8, 32768, s),
    "split_16": _split16,
    "tile_borders": _tile_borders,
    "quads": _quads,
    "cube_inside": _cube_inside,
    "cube_inside_near": _cube_inside_near,
    "horizon": _horizon,
    "near_tris": _near_tris,
    "near_lines": _near_lines,
    "near_points": _near_points,
    "guard_band": _guard,
    "grazing": _grazing,
    "sphere": _sphere,
    "subpixel": _subpixel,
    "needles": _needles,
    "collinear": _collinear,
    "lines": _lines,
    "points": _points,
    "lit_scaled": lambda s: _lit_scene(s, scale=2.1),
    "lit_nonunit_normals": lambda s: _lit_scene(s, unit=False),
    "rot_below_1e-3": lambda s: _lit_scene(s, rot=(0.99e-3, 0, 0)),
    "rot_above_1e-3": lambda s: _lit_scene(s, rot=(1.01e-3, 0, 0)),
    "fx_ne_fy": lambda s: _lit_scene(s, fy_ratio=0.6),
    "specular": _specular,
    "camera_scaled": lambda s: _lit_scene(s, cam_scale=1.25),
    "depth_zero": _depth_in("zero"),
    "depth_random": _depth_in("random"),
    "depth_1e9": _depth_in("huge"),
    "invalid_vertices": _invalid,
}

# scenes listed as adversarial: their band may cover more than 3 % of what they draw
ADVERSARIAL = {"frame_32768x8", "frame_8x32768", "guard_band", "near_lines", "grazing", "sphere", "subpixel", "needles",
               "collinear", "lines", "points", "quads", "horizon"}


def scene(name, small=False) -> Scene:
    return SCENES[name](small)


def compare(s: Scene, ref, rgba, depth, winner=None):
    """Checks a drawn frame against the reference; returns the ambiguous fraction of the covered pixels.
    ``winner``: global primitive index per pixel (-1: none), if the caller can tell; for id-coded scenes it is
    decoded from the colour."""
    un = ~ref["ambiguous"]
    cov = depth.view(np.uint32) != s.depth0.view(np.uint32)
    bad = (cov != ref["covered"]) & un
    assert not bad.any(), f"coverage differs at {bad.sum()} unambiguous pixels, first {np.argwhere(bad)[:5].tolist()}"
    kept = ~cov
    assert np.array_equal(rgba[kept], s.rgba0[kept]), "a pixel the depth test kept changed colour"
    both = cov & un
    off = prim_offsets(s.meshes)
    gref = np.where(ref["mesh"] >= 0, off[np.maximum(ref["mesh"], 0)] + ref["prim"], -1)
    if winner is None and s.ids:
        winner = np.where(cov, decode(rgba), -1)
    if winner is not None:
        bad = (winner != gref) & both
        assert not bad.any(), f"winner differs at {bad.sum()} pixels, first {np.argwhere(bad)[:5].tolist()}"
    dd = np.abs(depth.astype(np.float64) - ref["depth"])
    bad = both & ~(dd <= ref["depth_tol"])
    assert not bad.any(), f"depth differs at {bad.sum()} pixels, worst {dd[bad].max()}"
    want = rr.to_u8(ref["rgba"]).astype(np.int64)
    dc = np.abs(rgba.astype(np.int64) - want).max(-1)
    bad = both & (dc > ref["rgba_tol"])
    assert not bad.any(), (f"colour differs at {bad.sum()} pixels, first {np.argwhere(bad)[:3].tolist()}, "
                           f"got {rgba[bad][:3].tolist()} want {want[bad][:3].tolist()}")
    n = max(int((ref["covered"] | ref["ambiguous"]).sum()), 1)
    return float(ref["ambiguous"].sum()) / n
