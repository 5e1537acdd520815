"""numpy restatement of the mesh rasterizer (volrend_b200/csrc/vr_raster.cu), test infrastructure only.

It follows the reference's GL mesh pass (paths relative to the reference's root): vertex shader
src/mesh.cpp:98-119, fragment shader :121-160, draw :366-396, camera matrices src/camera.cpp:58-66
(K with -fy, CLIP_NEAR = 1e-3, infinite far plane; w2c = affineInverse(c2w)), GL state main.cpp:628,778-780
(depth test LESS, point size 4, line width 1, no face culling) -- with the rasterization rules DESIGN.md
section 8 fixes where GL leaves them to the implementation:

* window coordinates snapped to 8 sub-pixel bits; coverage from 64-bit integer edge functions with a
  top-left fill rule, sampled at pixel centres (x + 0.5, y + 0.5); row 0 = window y in [0, 1) = top row;
* near-plane clipping at d = 1e-3 plus guard-band planes at |window - centre| = 2^20 px (Sutherland-Hodgman,
  triangles re-fanned around the first vertex, new vertices interpolated from the inside vertex);
* lines: one pixel per column (x-major) or row (y-major) whose centre lies in [start, end); points: 4x4;
* z-buffer key (ray distance bits, 1 + 8 * primitive + sub-triangle): the earliest-drawn fragment wins ties;
* perspective-correct attributes, the fixed three-light Phong shader with the reference's quirks
  (normal not renormalized, viewDir = normalize(camPos_world - FragPos_camera)), RGBA8 = rint(clamp * 255),
  depth = length(camera-space position).

Every float operation is an individually rounded float32 operation in the same order as the kernel, so
coverage, depth and the winning primitive agree bit for bit.
"""
from __future__ import annotations

import numpy as np

F = np.float32
NEAR = F(1e-3)
GUARD = F(1048576.0)
MAX_WIN = F(4194304.0)


def _w2c(c2w12) -> np.ndarray:
    """affineInverse(c2w) in double, in the operation order vr_draw_meshes uses: rows of a 3x4."""
    c = [float(v) for v in np.asarray(c2w12, np.float32).reshape(12)]
    R = [[c[3 * k + r] for k in range(3)] for r in range(3)]
    det = R[0][0] * (R[1][1] * R[2][2] - R[1][2] * R[2][1]) + R[0][1] * (R[1][2] * R[2][0] - R[1][0] * R[2][2]) + \
        R[0][2] * (R[1][0] * R[2][1] - R[1][1] * R[2][0])
    inv = [[(R[1][1] * R[2][2] - R[1][2] * R[2][1]) / det, (R[0][2] * R[2][1] - R[0][1] * R[2][2]) / det,
            (R[0][1] * R[1][2] - R[0][2] * R[1][1]) / det],
           [(R[1][2] * R[2][0] - R[1][0] * R[2][2]) / det, (R[0][0] * R[2][2] - R[0][2] * R[2][0]) / det,
            (R[0][2] * R[1][0] - R[0][0] * R[1][2]) / det],
           [(R[1][0] * R[2][1] - R[1][1] * R[2][0]) / det, (R[0][1] * R[2][0] - R[0][0] * R[2][1]) / det,
            (R[0][0] * R[1][1] - R[0][1] * R[1][0]) / det]]
    V = [[inv[r][0], inv[r][1], inv[r][2], -((inv[r][0] * c[9] + inv[r][1] * c[10]) + inv[r][2] * c[11])]
         for r in range(3)]
    return V


def _model_view(V, model16) -> np.ndarray:
    M = [float(v) for v in np.asarray(model16, np.float32).reshape(16)]   # column-major
    mv = np.zeros(12, np.float32)
    for k in range(4):
        for r in range(3):
            mv[3 * k + r] = F(((V[r][0] * M[4 * k] + V[r][1] * M[4 * k + 1]) + V[r][2] * M[4 * k + 2]) +
                              V[r][3] * M[4 * k + 3])
    return mv


def _plane(i, q, fx, fy):
    d = -q[2]
    if i == 0:
        return d - NEAR
    if i == 1:
        return GUARD * d - fx * q[0]
    if i == 2:
        return GUARD * d + fx * q[0]
    if i == 3:
        return GUARD * d - fy * q[1]
    return GUARD * d + fy * q[1]


def _lerp(qi, wi, di, qo, wo, do):
    t = di / (di - do)
    return [qi[k] + t * (qo[k] - qi[k]) for k in range(3)], [wi[k] + t * (wo[k] - wi[k]) for k in range(3)]


def _clip(qs, fsz, fx, fy):
    """qs: list of camera-space vertices (lists of np.float32).  Returns the clipped polygon [(q, w)]."""
    P = [(list(qs[j]), [F(1) if i == j else F(0) for i in range(3)]) for j in range(fsz)]
    for pl in range(5):
        dist = [_plane(pl, q, fx, fy) for q, _ in P]
        ins = [bool(d >= 0) for d in dist]
        if all(ins):
            continue
        if not any(ins) or fsz == 1:
            return []
        if fsz == 2:
            o = 1 if ins[0] else 0
            i = 1 - o
            P[o] = _lerp(P[i][0], P[i][1], dist[i], P[o][0], P[o][1], dist[o])
            continue
        out = []
        n = len(P)
        for v in range(n):
            u = n - 1 if v == 0 else v - 1
            if ins[v] != ins[u]:
                a, b = (v, u) if ins[v] else (u, v)
                out.append(_lerp(P[a][0], P[a][1], dist[a], P[b][0], P[b][1], dist[b]))
            if ins[v]:
                out.append(P[v])
        P = out
    return P


def _floor_div(a, b):
    return a // b


def _ceil_div(a, b):
    return -((-a) // b)


def _make_sub(kind, P, s, W, H, fx, fy):
    verts = [P[0]] if kind == 1 else ([P[0], P[1]] if kind == 2 else [P[0], P[s + 1], P[s + 2]])
    cx, cy = F(0.5) * F(W), F(0.5) * F(H)
    S = dict(kind=kind, q=[], w=[], d=[], X=[], Y=[])
    for q, w in verts:
        d = -q[2]
        xw = cx + (fx * q[0]) / d
        yw = cy - (fy * q[1]) / d
        if not (abs(xw) <= MAX_WIN) or not (abs(yw) <= MAX_WIN):
            return None
        S["q"].append(q); S["w"].append(w); S["d"].append(d)
        S["X"].append(int(np.rint(xw * F(256)))); S["Y"].append(int(np.rint(yw * F(256))))

    def swap(a, b):
        for k in ("q", "w", "d", "X", "Y"):
            S[k][a], S[k][b] = S[k][b], S[k][a]
    X, Y = S["X"], S["Y"]
    if kind == 3:
        A = (X[1] - X[0]) * (Y[2] - Y[0]) - (X[2] - X[0]) * (Y[1] - Y[0])
        if A == 0:
            return None
        if A < 0:
            swap(1, 2)
            A = -A
        S["A"] = A
        xlo, xhi = _ceil_div(min(X) - 128, 256), _floor_div(max(X) - 128, 256)
        ylo, yhi = _ceil_div(min(Y) - 128, 256), _floor_div(max(Y) - 128, 256)
    elif kind == 2:
        dX, dY = X[1] - X[0], Y[1] - Y[0]
        if dX == 0 and dY == 0:
            return None
        xm = abs(dX) >= abs(dY)
        if (xm and dX < 0) or (not xm and dY < 0):
            swap(0, 1)
        S["xmajor"] = xm
        M0, N0 = (X, Y) if xm else (Y, X)
        S["A"] = M0[1] - M0[0]
        mlo, mhi = _ceil_div(M0[0] - 128, 256), _ceil_div(M0[1] - 128, 256) - 1
        nlo, nhi = _floor_div(min(N0), 256), _floor_div(max(N0), 256)
        xlo, xhi, ylo, yhi = (mlo, mhi, nlo, nhi) if xm else (nlo, nhi, mlo, mhi)
    else:
        S["ox"], S["oy"] = _ceil_div(X[0] - 640, 256), _ceil_div(Y[0] - 640, 256)
        xlo, xhi, ylo, yhi = S["ox"], S["ox"] + 3, S["oy"], S["oy"] + 3
    S["bbox"] = (max(xlo, 0), min(xhi, W - 1), max(ylo, 0), min(yhi, H - 1))
    return S


def _edge_in(e, dx, dy):
    return (e > 0) | ((e == 0) & ((dy < 0) | ((dy == 0) & (dx < 0))))


def _cover_and_weights(S, px, py):
    """px, py: int64 pixel arrays.  Returns (covered mask, lam list of float32 arrays)."""
    PX, PY = px * 256 + 128, py * 256 + 128
    X, Y, d, k = S["X"], S["Y"], S["d"], S["kind"]
    if k == 3:
        E = [(X[2] - X[1]) * (PY - Y[1]) - (Y[2] - Y[1]) * (PX - X[1]),
             (X[0] - X[2]) * (PY - Y[2]) - (Y[0] - Y[2]) * (PX - X[2]),
             (X[1] - X[0]) * (PY - Y[0]) - (Y[1] - Y[0]) * (PX - X[0])]
        cov = _edge_in(E[0], X[2] - X[1], Y[2] - Y[1]) & _edge_in(E[1], X[0] - X[2], Y[0] - Y[2]) & \
            _edge_in(E[2], X[1] - X[0], Y[1] - Y[0])
        Ad = np.float64(S["A"])
        r = [(E[j].astype(np.float64) / Ad).astype(np.float32) / d[j] for j in range(3)]
        s = (r[0] + r[1]) + r[2]
        return cov, [r[j] / s for j in range(3)]
    if k == 2:
        xm = S["xmajor"]
        M0, N0 = (X, Y) if xm else (Y, X)
        P = PX if xm else PY
        n = N0[0] + np.floor_divide((P - M0[0]) * (N0[1] - N0[0]), S["A"])
        cov = (P >= M0[0]) & (P < M0[1]) & (np.floor_divide(n, 256) == (py if xm else px))
        t = ((P - M0[0]).astype(np.float64) / np.float64(S["A"])).astype(np.float32)
        r0, r1 = (F(1) - t) / d[0], t / d[1]
        s = r0 + r1
        return cov, [r0 / s, r1 / s]
    cov = (px >= S["ox"]) & (px <= S["ox"] + 3) & (py >= S["oy"]) & (py <= S["oy"] + 3)
    return cov, [np.ones(px.shape, np.float32)]


def _dot(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def _normalize(v):
    ln = np.sqrt(_dot(v, v))
    safe = np.where(ln > 0, ln, F(1)).astype(np.float32)
    return [np.where(ln > 0, v[k] / safe, v[k]).astype(np.float32) for k in range(3)]


def _u8(v):
    return np.rint(np.fmin(np.fmax(v, F(0)), F(1)) * F(255)).astype(np.uint8)


def draw_meshes(W, H, fx, fy, c2w12, meshes, rgba, depth):
    # shading is evaluated over whole bounding boxes; uncovered pixels (weights outside [0, 1]) may overflow
    with np.errstate(over="ignore", invalid="ignore"):
        return _draw_meshes(W, H, fx, fy, c2w12, meshes, rgba, depth)


def _draw_meshes(W, H, fx, fy, c2w12, meshes, rgba, depth):
    """Rasterizes ``meshes`` (dicts: vert (n*9 float32), faces (uint32 or None), face_size, unlit, model
    (16 float32, column-major)) over copies of ``rgba`` (uint8 [H,W,4]) and ``depth`` (float32 [H,W]).
    Returns (rgba, depth, winner) with winner = the winning z-buffer sequence number per pixel (0: none)."""
    fx, fy = F(fx), F(fy)
    c = np.asarray(c2w12, np.float32).reshape(12)
    V = _w2c(c)
    # camPos = -transpose(mat3(V)) * V[3] (mesh.cpp:376), in double as vr_draw_meshes_batch does
    cam_pos = [F(-((V[0][k] * V[0][3] + V[1][k] * V[1][3]) + V[2][k] * V[2][3])) for k in range(3)]
    rgba = np.array(rgba, np.uint8, copy=True)
    depth = np.array(depth, np.float32, copy=True)
    key = (depth.view(np.uint32).astype(np.uint64) << np.uint64(32))
    win = np.zeros((H, W), np.int64)
    L1, L2 = _normalize([F(0.5), F(0.2), F(1)]), _normalize([F(-0.5), F(-1), F(-0.5)])
    base = 0
    for m in meshes:
        vert = np.asarray(m["vert"], np.float32).reshape(-1, 9)
        fsz = int(m["face_size"])
        faces = m.get("faces")
        faces = None if faces is None or len(faces) == 0 else np.asarray(faces, np.uint32).reshape(-1)
        n_verts = vert.shape[0]
        n_prims = (faces.size // fsz) if faces is not None else n_verts // fsz
        if n_prims == 0:
            continue
        mv = _model_view(V, m["model"])
        M = np.asarray(m["model"], np.float32).reshape(16)
        m3 = [M[4 * k + r] for k in range(3) for r in range(3)]
        p = vert[:, :3]
        q_all = np.stack([((mv[k] * p[:, 0] + mv[3 + k] * p[:, 1]) + mv[6 + k] * p[:, 2]) + mv[9 + k]
                          for k in range(3)], 1)
        n = vert[:, 6:9]
        nw = _normalize([(m3[k] * n[:, 0] + m3[3 + k] * n[:, 1]) + m3[6 + k] * n[:, 2] for k in range(3)])
        nw = np.stack(nw, 1)
        for lp in range(n_prims):
            g = base + lp
            idx = [int(faces[lp * fsz + j]) if faces is not None else lp * fsz + j for j in range(fsz)]
            if any(i >= n_verts for i in idx):
                continue
            P = _clip([list(q_all[i]) for i in idx], fsz, fx, fy)
            nsub = (len(P) - 2 if len(P) >= 3 else 0) if fsz == 3 else (1 if P else 0)
            for s in range(nsub):
                S = _make_sub(fsz, P, s, W, H, fx, fy)
                if S is None:
                    continue
                x0, x1, y0, y1 = S["bbox"]
                if x0 > x1 or y0 > y1:
                    continue
                py, px = np.mgrid[y0:y1 + 1, x0:x1 + 1].astype(np.int64)
                cov, lam = _cover_and_weights(S, px, py)
                Pp = []
                for k in range(3):
                    acc = lam[0] * S["q"][0][k]
                    for j in range(1, fsz):
                        acc = acc + lam[j] * S["q"][j][k]
                    Pp.append(acc.astype(np.float32))
                dist = np.sqrt(_dot(Pp, Pp)).astype(np.float32)
                ok = cov & (dist <= F(3.4e38))
                seq = np.uint64(g * 8 + s + 1)
                kk = (dist.view(np.uint32).astype(np.uint64) << np.uint64(32)) | seq
                cur = key[y0:y1 + 1, x0:x1 + 1]
                better = ok & (kk < cur)
                if not better.any():
                    continue
                om = []
                for i in range(3):
                    acc = lam[0] * S["w"][0][i]
                    for j in range(1, fsz):
                        acc = acc + lam[j] * S["w"][j][i]
                    om.append(acc.astype(np.float32))
                col, nrm = [None] * 3, [None] * 3
                for i in range(fsz):
                    for k in range(3):
                        cv, nv = om[i] * vert[idx[i], 3 + k], om[i] * nw[idx[i], k]
                        col[k] = cv if i == 0 else col[k] + cv
                        nrm[k] = nv if i == 0 else nrm[k] + nv
                if m.get("unlit"):
                    out = col + [np.ones_like(col[0])]
                else:
                    diffuse = F(0.7) * np.fmax(_dot(L1, nrm), F(0))
                    diffuse2 = F(0.2) * np.fmax(_dot(L2, nrm), F(0))
                    Vd = _normalize([cam_pos[k] - Pp[k] for k in range(3)])
                    I = [-L1[0], -L1[1], -L1[2]]
                    dni2 = F(2) * _dot(nrm, I)
                    R = [I[k] - dni2 * nrm[k] for k in range(3)]
                    sp = np.fmax(_dot(Vd, R), F(0))
                    for _ in range(5):
                        sp = sp * sp
                    tot = ((F(0.3) + diffuse) + diffuse2) + F(0.6) * sp
                    out = [tot * col[0], tot * col[1], tot * col[2], tot]
                sub_rgba = rgba[y0:y1 + 1, x0:x1 + 1]
                for ch in range(4):
                    sub_rgba[..., ch] = np.where(better, _u8(np.asarray(out[ch], np.float32)), sub_rgba[..., ch])
                depth[y0:y1 + 1, x0:x1 + 1] = np.where(better, dist, depth[y0:y1 + 1, x0:x1 + 1])
                win[y0:y1 + 1, x0:x1 + 1] = np.where(better, int(seq), win[y0:y1 + 1, x0:x1 + 1])
                key[y0:y1 + 1, x0:x1 + 1] = np.where(better, kk, cur)
        base += n_prims
    return rgba, depth, win


def coverage(W, H, fx, fy, c2w12, mesh) -> np.ndarray:
    """Per pixel, how many sub-primitives of one mesh cover it (the fill-rule checks count to exactly 1)."""
    fx, fy = F(fx), F(fy)
    V = _w2c(c2w12)
    mv = _model_view(V, mesh["model"])
    vert = np.asarray(mesh["vert"], np.float32).reshape(-1, 9)
    fsz = int(mesh["face_size"])
    faces = mesh.get("faces")
    faces = np.arange(vert.shape[0], dtype=np.uint32) if faces is None or len(faces) == 0 else \
        np.asarray(faces, np.uint32).reshape(-1)
    p = vert[:, :3]
    q_all = np.stack([((mv[k] * p[:, 0] + mv[3 + k] * p[:, 1]) + mv[6 + k] * p[:, 2]) + mv[9 + k] for k in range(3)], 1)
    cnt = np.zeros((H, W), np.int64)
    for lp in range(faces.size // fsz):
        idx = [int(faces[lp * fsz + j]) for j in range(fsz)]
        P = _clip([list(q_all[i]) for i in idx], fsz, fx, fy)
        nsub = (len(P) - 2 if len(P) >= 3 else 0) if fsz == 3 else (1 if P else 0)
        for s in range(nsub):
            S = _make_sub(fsz, P, s, W, H, fx, fy)
            if S is None:
                continue
            x0, x1, y0, y1 = S["bbox"]
            if x0 > x1 or y0 > y1:
                continue
            py, px = np.mgrid[y0:y1 + 1, x0:x1 + 1].astype(np.int64)
            cov, _ = _cover_and_weights(S, px, py)
            cnt[y0:y1 + 1, x0:x1 + 1] += cov
    return cnt
