"""Float64 ray-cast reference of what the reference's GL mesh pass draws, test infrastructure only.

It is written from the reference's sources (paths relative to the reference's root), not from the rasterizer:

* camera: c2w from the pose, K with -fy and CLIP_NEAR = 1e-3, w2c = affineInverse(c2w) (src/camera.cpp:58-65);
* vertex shader: FragPos = MV * aPos, Normal = normalize(mat3(M) * aNormal) per vertex (src/mesh.cpp:98-119);
* fragment shader: the fixed three-light Phong model, the interpolated normal used without renormalizing, viewDir =
  normalize(camPos - FragPos) with FragPos in camera space, Depth = length(FragPos) (src/mesh.cpp:121-160);
* Mesh::draw: model = angleAxis rotation (identity below 1e-3 rad) * scale, translation in column 3, and
  camPos = -transpose(mat3(V)) * V[3] (src/mesh.cpp:366-396);

plus the rules DESIGN.md section 8 fixes where GL leaves a choice: row 0 is the top row, coverage is sampled at
pixel centres (x + 0.5, y + 0.5) with the top-left rule, a line draws one pixel per major-axis pixel centre in
[start, end), a point the 4x4 pixels whose centres lie in [x - 2, x + 2), and the depth test is LESS against the
incoming depth with the earlier-drawn primitive winning a tie.

Nothing is rasterized.  Each pixel casts the camera-space ray through its window point; a triangle covers the pixel
when the ray meets it at camera depth >= 1e-3, which is GL's near-clipped triangle, so there is no clipping code
(the guard band does not change on-screen coverage and is ignored).  The barycentrics of the hit point are the
perspective-correct weights.  A line is solved, per major-axis pixel centre, for the point of the segment that
projects there.  All of it is float64 on the float32 inputs.

The rasterizer snaps window coordinates to 8 sub-pixel bits and projects in float32, so a decision that close
calls can go either way.  Each primitive gets a band delta = 4 * (2^-9 + ulp_f32(largest |window coordinate| of
its near-clipped vertices, at most 2^20)) pixels, and a pixel is *ambiguous* when its centre lies within delta of
one of the primitive's projected edges (lines: the minor coordinate within delta of a pixel boundary, or the
major-axis centre within delta of an end; points: a footprint boundary within delta of the centre), or when two
candidate depths, or a candidate depth and the incoming depth, differ by less than the depth tolerance
1e-5 * d + (change of d over delta).  The colour tolerance is 1 LSB plus the colour's change over delta.
"""
from __future__ import annotations

import math

import numpy as np

NEAR = 1e-3
_BAND_CAP = 2.0 ** 20


def camera_f64(c2w12):
    """V = affineInverse(c2w) (4x4, float64) and camPos = -transpose(mat3(V)) * V[3] (mesh.cpp:376)."""
    c = np.asarray(c2w12, np.float32).astype(np.float64).reshape(4, 3).T      # 3x4, columns of glm::mat4x3
    R, t = c[:, :3], c[:, 3]
    Ri = np.linalg.inv(R)
    V = np.eye(4)
    V[:3, :3], V[:3, 3] = Ri, -Ri @ t
    cam_pos = -V[:3, :3].T @ V[:3, 3]
    return V, cam_pos


def model_f64(rotation, translation, scale):
    """Mesh::draw's transform_ (mesh.cpp:368-381) in float64: glm::angleAxis -> mat4_cast, * scale, translation."""
    r = np.asarray(rotation, np.float32).astype(np.float64).reshape(3)
    M = np.eye(4)
    norm = math.sqrt(float(r @ r))
    if not norm < 1e-3:
        x, y, z = r / norm
        s = math.sin(0.5 * norm)
        w, x, y, z = math.cos(0.5 * norm), x * s, y * s, z * s
        M[:3, :3] = [[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]]
    M[:3, :3] *= float(np.float32(scale))
    M[:3, 3] = np.asarray(translation, np.float32).astype(np.float64).reshape(3)
    return M


def _band(win_xy):
    m = float(np.max(np.abs(win_xy))) if np.size(win_xy) else 0.0
    m = min(m, _BAND_CAP)
    return 4.0 * (2.0 ** -9 + float(np.spacing(np.float32(m))))


def _unit(v):
    n = np.sqrt((v * v).sum(-1, keepdims=True))
    return np.where(n > 0, v / np.where(n > 0, n, 1.0), v)


_L1 = _unit(np.array([0.5, 0.2, 1.0]))
_L2 = _unit(np.array([-0.5, -1.0, -0.5]))


def shade(unlit, col, nrm, frag, cam_pos):
    """The fragment shader (mesh.cpp:130-159) in float64: (..., 4) RGBA before clamping."""
    if unlit:
        return np.concatenate([col, np.ones(col.shape[:-1] + (1,))], -1)
    diffuse = 0.7 * np.maximum((nrm * _L1).sum(-1), 0.0)
    diffuse2 = 0.2 * np.maximum((nrm * _L2).sum(-1), 0.0)
    view = _unit(cam_pos - frag)
    inc = -_L1
    refl = inc - 2.0 * (nrm * inc).sum(-1, keepdims=True) * nrm          # GLSL reflect(I, N)
    spec = np.maximum((view * refl).sum(-1), 0.0) ** 32
    tot = 0.3 + diffuse + diffuse2 + 0.6 * spec
    return np.concatenate([tot[..., None] * col, tot[..., None]], -1)


def _seg_dist(px, py, a, b):
    """Distance from points (px, py) to the segment a-b (window space)."""
    dx, dy = b[0] - a[0], b[1] - a[1]
    ll = dx * dx + dy * dy
    if ll == 0:
        return np.hypot(px - a[0], py - a[1])
    s = np.clip(((px - a[0]) * dx + (py - a[1]) * dy) / ll, 0.0, 1.0)
    return np.hypot(px - (a[0] + s * dx), py - (a[1] + s * dy))


class _Frame:
    def __init__(self, W, H, fx, fy, c2w12, depth_in):
        self.W, self.H = int(W), int(H)
        self.fx, self.fy = float(np.float32(fx)), float(np.float32(fy))
        self.cx, self.cy = 0.5 * self.W, 0.5 * self.H
        self.V, self.cam_pos = camera_f64(c2w12)
        n = self.W * self.H
        self.din = np.asarray(depth_in, np.float32).astype(np.float64).reshape(n)
        self.d1 = np.full(n, np.inf)
        self.t1 = np.zeros(n)
        self.id1 = np.full(n, -1, np.int64)
        self.d2 = np.full(n, np.inf)
        self.t2 = np.zeros(n)
        self.amin = np.full(n, np.inf)
        self.col = np.zeros((n, 4))
        self.ctol = np.zeros(n)

    def project(self, q):
        d = -q[..., 2]
        return np.stack([self.cx + self.fx * q[..., 0] / d, self.cy - self.fy * q[..., 1] / d], -1)

    def ray(self, wx, wy):
        return np.stack([(wx - self.cx) / self.fx, (self.cy - wy) / self.fy, -np.ones(np.shape(wx))], -1)

    def submit(self, pix, amb, depth, dtol, gid, colour_fn):
        """Candidates of one primitive at distinct flat pixel indices ``pix``.  ``colour_fn(mask)`` returns the
        colour and colour tolerance of the candidates selected by ``mask``; it runs only where one takes the lead."""
        am = amb | ~np.isfinite(depth)
        if am.any():
            dm = np.where(np.isfinite(depth[am]), depth[am] - dtol[am], 0.0)
            np.minimum.at(self.amin, pix[am], dm)
        ok = ~am
        if not ok.any():
            return
        p, dc, tc = pix[ok], depth[ok], dtol[ok]
        lead = dc < self.d1[p]
        second = ~lead & (dc < self.d2[p])
        pl = p[lead]
        self.d2[pl], self.t2[pl] = self.d1[pl], self.t1[pl]
        self.d1[pl], self.t1[pl], self.id1[pl] = dc[lead], tc[lead], gid
        if lead.any():
            sel = np.zeros(pix.shape, bool)
            sel[np.flatnonzero(ok)[lead]] = True
            c, ct = colour_fn(sel)
            self.col[pl], self.ctol[pl] = c, ct
        ps = p[second]
        self.d2[ps], self.t2[ps] = dc[second], tc[second]

    def result(self, rgba_in):
        n = self.W * self.H
        win = (self.id1 >= 0) & (self.d1 < self.din)
        amb = (self.id1 >= 0) & (np.abs(self.d1 - self.din) < self.t1)
        with np.errstate(invalid="ignore"):
            amb |= win & (self.d2 - self.d1 < self.t1 + self.t2)
        amb |= self.amin < np.where(win, self.d1 + self.t1, self.din)
        rgba0 = np.asarray(rgba_in, np.uint8).reshape(n, 4)
        colour = np.where(win[:, None], self.col, rgba0 / 255.0)
        gid = np.where(win, self.id1, -1)
        sh = (self.H, self.W)
        return dict(covered=win.reshape(sh), ambiguous=amb.reshape(sh),
                    mesh=np.where(gid >= 0, gid >> 32, -1).reshape(sh),
                    prim=np.where(gid >= 0, gid & 0xffffffff, -1).reshape(sh),
                    depth=np.where(win, self.d1, self.din).reshape(sh),
                    depth_tol=np.where(win, self.t1, 0.0).reshape(sh),
                    rgba=colour.reshape(sh + (4,)), rgba_tol=np.where(win, self.ctol, 0.0).reshape(sh))


def _clip_poly(q):
    """Sutherland-Hodgman against d >= NEAR, float64; only to size the band and bound the pixel box."""
    d = -q[:, 2] - NEAR
    out = []
    n = len(q)
    for v in range(n):
        u = v - 1
        if (d[v] >= 0) != (d[u] >= 0):
            out.append(q[u] + (q[v] - q[u]) * (d[u] / (d[u] - d[v])))
        if d[v] >= 0:
            out.append(q[v])
    return np.array(out)


def _pixel_range(lo, hi, n):
    """Pixels whose centre lies in [lo, hi], clamped to [0, n)."""
    a = max(int(math.ceil(lo - 0.5)) if math.isfinite(lo) else 0, 0)
    b = min(int(math.floor(hi - 0.5)) if math.isfinite(hi) else n - 1, n - 1)
    return a, b


def _triangle(fr, gid, q, col, nrm, unlit):
    poly = _clip_poly(q)
    if len(poly) < 3:
        return
    win = fr.project(poly)
    delta = _band(win)
    x0, x1 = _pixel_range(win[:, 0].min() - delta, win[:, 0].max() + delta, fr.W)
    y0, y1 = _pixel_range(win[:, 1].min() - delta, win[:, 1].max() + delta, fr.H)
    if x0 > x1 or y0 > y1:
        return
    py, px = np.mgrid[y0:y1 + 1, x0:x1 + 1]
    px, py = px.reshape(-1), py.reshape(-1)
    wx, wy = px + 0.5, py + 0.5
    edge = np.full(px.shape, np.inf)
    for k in range(len(win)):
        edge = np.minimum(edge, _seg_dist(wx, wy, win[k - 1], win[k]))
    nv = np.cross(q[1] - q[0], q[2] - q[0])
    nn = nv @ nv
    c0 = nv @ q[0]
    ed = [np.cross(nv, q[2] - q[1]), np.cross(nv, q[0] - q[2])]

    def hit(wx, wy):
        r = fr.ray(wx, wy)
        with np.errstate(divide="ignore", invalid="ignore"):
            t = c0 / (r @ nv)
            h = t[:, None] * r
            b0 = ((h - q[1]) @ ed[0]) / nn
            b1 = ((h - q[2]) @ ed[1]) / nn
        b = np.stack([b0, b1, 1.0 - b0 - b1], -1)
        return t, h, b

    t, h, b = hit(wx, wy)
    inside = np.isfinite(t) & (t >= NEAR) & (b >= 0).all(-1)
    amb = edge < delta
    keep = inside | amb
    if not keep.any():
        return
    px, py, wx, wy, t, h, b, amb = px[keep], py[keep], wx[keep], wy[keep], t[keep], h[keep], b[keep], amb[keep]
    depth = np.where(t >= NEAR, np.sqrt((h * h).sum(-1)), np.nan)
    offs = [(delta, 0.0), (-delta, 0.0), (0.0, delta), (0.0, -delta)]
    var = np.zeros(depth.shape)
    for ox, oy in offs:
        t2, h2, _ = hit(wx + ox, wy + oy)
        with np.errstate(invalid="ignore"):
            var = np.fmax(var, np.abs(np.sqrt((h2 * h2).sum(-1)) - depth))
    dtol = 1e-5 * depth + var

    def colour(sel):
        c = np.clip(shade(unlit, b[sel] @ col, b[sel] @ nrm, h[sel], fr.cam_pos), 0, 1)
        dc = np.zeros(c.shape)
        for ox, oy in offs:
            _, h2, b2 = hit(wx[sel] + ox, wy[sel] + oy)
            c2 = np.clip(shade(unlit, b2 @ col, b2 @ nrm, h2, fr.cam_pos), 0, 1)
            dc = np.fmax(dc, np.abs(c2 - c))
        return c, 1.0 + 255.0 * dc.max(-1)

    fr.submit(py * fr.W + px, amb, depth, dtol, gid, colour)


def _line(fr, gid, q, col, nrm, unlit):
    qa, qb = q
    da, db = -qa[2], -qb[2]
    t_lo, t_hi = 0.0, 1.0
    if da < NEAR and db < NEAR:
        return
    if da < NEAR:
        t_lo = (NEAR - da) / (db - da)
    elif db < NEAR:
        t_hi = (NEAR - da) / (db - da)
    ends = np.stack([qa + t_lo * (qb - qa), qa + t_hi * (qb - qa)])
    win = fr.project(ends)
    delta = _band(win)
    dx, dy = win[1] - win[0]
    if abs(dx) < delta and abs(dy) < delta:
        return          # zero length after snapping, or a sub-band dot: the rasterizer may draw or drop it
    majors = [abs(dx) >= abs(dy)] if abs(abs(dx) - abs(dy)) >= delta else [True, False]
    qd = qb - qa
    sets = []
    for xm in majors:
        a, n_ax = (0, fr.W) if xm else (1, fr.H)
        lo, hi = sorted(win[:, a])
        m0, m1 = _pixel_range(lo - delta, hi + delta, n_ax)
        if m0 > m1:
            sets.append({})
            continue
        c = np.arange(m0, m1 + 1) + 0.5

        def solve(c):
            # the segment point whose projected major coordinate is c: linear in the segment parameter
            if xm:
                num, den = fr.fx * qa[0] + (c - fr.cx) * qa[2], fr.fx * qd[0] + (c - fr.cx) * qd[2]
            else:
                num, den = fr.fy * qa[1] - (c - fr.cy) * qa[2], fr.fy * qd[1] - (c - fr.cy) * qd[2]
            with np.errstate(divide="ignore", invalid="ignore"):
                s = -num / den
            return s, qa + s[:, None] * qd

        s, p = solve(c)
        minor = fr.project(p)[:, 1 - a]
        # the position error is a blend of the ends' errors: the band shrinks away from an end far off screen
        u = np.clip((c - win[0, a]) / (win[1, a] - win[0, a]), 0.0, 1.0)
        band = (1.0 - u) * _band(win[0]) + u * _band(win[1])
        amb_end = (np.abs(c - lo) < band) | (np.abs(c - hi) < band)
        in_range = (c >= lo) & (c < hi)
        depth = np.sqrt((p * p).sum(-1))
        var = np.zeros(depth.shape)
        for o in (delta, -delta):
            _, p2 = solve(c + o)
            var = np.fmax(var, np.abs(np.sqrt((p2 * p2).sum(-1)) - depth))
        out = {}
        for i in range(len(c)):
            if not (in_range[i] or amb_end[i]) or not math.isfinite(minor[i]):
                continue
            cells = {int(math.floor(minor[i] - band[i])), int(math.floor(minor[i] + band[i]))}
            amb = amb_end[i] or len(cells) > 1
            for nidx in cells:
                pxy = (m0 + i, nidx) if xm else (nidx, m0 + i)
                if not (0 <= pxy[0] < fr.W and 0 <= pxy[1] < fr.H):
                    continue
                out[pxy] = (amb, s[i], depth[i], 1e-5 * depth[i] + var[i], c[i])
        sets.append(out)
    if len(sets) == 2:     # the major axis itself is within the band: pixels the two rules disagree on are ambiguous
        merged = dict(sets[0])
        for k, v in sets[1].items():
            if k not in merged or merged[k][0] != v[0]:
                merged[k] = (True,) + v[1:]
        for k in set(sets[0]) - set(sets[1]):
            merged[k] = (True,) + merged[k][1:]
        sets = [merged]
    out = sets[0]
    if not out:
        return
    keys = list(out)
    pix = np.array([y * fr.W + x for x, y in keys], np.int64)
    amb = np.array([out[k][0] for k in keys])
    s = np.array([out[k][1] for k in keys])
    depth = np.array([out[k][2] for k in keys])
    dtol = np.array([out[k][3] for k in keys])
    xm0 = majors[0]

    def colour(sel):
        def at(sv):
            w = np.stack([1.0 - sv, sv], -1)
            return np.clip(shade(unlit, w @ col, w @ nrm, qa + sv[:, None] * qd, fr.cam_pos), 0, 1)
        cs = np.array([out[k][4] for k in keys])[sel]
        c = at(s[sel])
        dc = np.zeros(c.shape)
        for o in (delta, -delta):
            cc = cs + o
            if xm0:
                num, den = fr.fx * qa[0] + (cc - fr.cx) * qa[2], fr.fx * qd[0] + (cc - fr.cx) * qd[2]
            else:
                num, den = fr.fy * qa[1] - (cc - fr.cy) * qa[2], fr.fy * qd[1] - (cc - fr.cy) * qd[2]
            dc = np.fmax(dc, np.abs(at(-num / den) - c))
        return c, 1.0 + 255.0 * dc.max(-1)

    fr.submit(pix, amb, depth, dtol, gid, colour)


def _point(fr, gid, q, col, nrm, unlit):
    q = q[0]
    if not -q[2] >= NEAR:
        return
    w = fr.project(q[None])[0]
    delta = _band(w)
    axes = []
    for a, n in ((0, fr.W), (1, fr.H)):
        lo, hi = w[a] - 2.0, w[a] + 2.0
        i0, i1 = _pixel_range(lo - delta, hi + delta, n)
        idx = np.arange(i0, i1 + 1)
        c = idx + 0.5
        axes.append((idx, (np.abs(c - lo) < delta) | (np.abs(c - hi) < delta), (c >= lo) & (c < hi)))
    (ix, ax, inx), (iy, ay, iny) = axes
    if ix.size == 0 or iy.size == 0:
        return
    amb = (ax[None, :] | ay[:, None]).reshape(-1)
    keep = ((inx[None, :] & iny[:, None]).reshape(-1)) | amb
    pix = (iy[:, None] * fr.W + ix[None, :]).reshape(-1)[keep]
    amb = amb[keep]
    d = float(np.sqrt(q @ q))
    depth = np.full(pix.shape, d)

    def colour(sel):
        c = np.clip(shade(unlit, col[0][None], nrm[0][None], q[None], fr.cam_pos), 0, 1)
        return np.repeat(c, int(sel.sum()), 0), np.ones(int(sel.sum()))

    fr.submit(pix, amb, depth, 1e-5 * depth, gid, colour)


def draw(W, H, fx, fy, c2w12, meshes, rgba_in, depth_in):
    """What GL draws over ``rgba_in`` (uint8 [H,W,4]) and ``depth_in`` (float32 [H,W]), per pixel.

    ``meshes``: dicts with vert (n*9 float32: position, colour, normal), faces (uint32, or None for consecutive
    vertices), face_size (1, 2, 3), unlit, and either rotation / translation / scale (the model is then built here
    from the reference's formulas) or model (16 float32, column-major).

    Returns a dict of [H,W] arrays: covered, ambiguous, mesh and prim (the winner; -1: the incoming pixel stays),
    depth, depth_tol, rgba (float, [H,W,4], clamped to [0, 1]) and rgba_tol (in 8-bit steps)."""
    fr = _Frame(W, H, fx, fy, c2w12, depth_in)
    for mi, m in enumerate(meshes):
        vert = np.asarray(m["vert"], np.float32).reshape(-1, 9).astype(np.float64)
        fsz = int(m["face_size"])
        faces = m.get("faces")
        nv = vert.shape[0]
        faces = np.arange(nv - nv % fsz) if faces is None or len(faces) == 0 else \
            np.asarray(faces, np.uint32).astype(np.int64).reshape(-1)
        if "rotation" in m:
            M = model_f64(m["rotation"], m["translation"], m["scale"])
        else:
            M = np.asarray(m["model"], np.float32).astype(np.float64).reshape(4, 4).T
        MV = fr.V @ M
        q = vert[:, :3] @ MV[:3, :3].T + MV[:3, 3]
        nrm = _unit(vert[:, 6:9] @ M[:3, :3].T)
        col = vert[:, 3:6]
        fn = {1: _point, 2: _line, 3: _triangle}[fsz]
        with np.errstate(over="ignore", invalid="ignore"):
            ok_v = np.isfinite(q).all(-1)
        for lp in range(faces.size // fsz):
            idx = faces[lp * fsz:(lp + 1) * fsz]
            if (idx >= nv).any() or not ok_v[idx].all():
                continue
            fn(fr, (mi << 32) | lp, q[idx], col[idx], nrm[idx], bool(m.get("unlit")))
    return fr.result(rgba_in)


def to_u8(rgba):
    """The 8-bit colour GL stores for float colours in [0, 1]."""
    return np.rint(np.clip(rgba, 0, 1) * 255).astype(np.uint8)
