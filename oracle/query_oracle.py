"""numpy restatement of query_single_from_root (n3tree_query.hpp:13-48) over the original ``child`` / ``data``
arrays, for world points mapped as retrieve_cursor_lumisphere_kernel maps them (volrend.cu:180-182, one fused
multiply-add per axis).  TEST INFRASTRUCTURE ONLY: the CPU tests check it against the reference goldens, the GPU
tests check vr_tree_query against both."""
from __future__ import annotations

import numpy as np

HI = np.float32(1.0) - np.float32(1e-6)


def fma32(a, b, c) -> np.ndarray:
    """float32 a * b + c rounded once (what FFMA computes).  The product is exact in float64; the float64 sum is
    rounded, so the one case where rounding it again to float32 can differ from rounding once -- the float64 sum
    lands exactly halfway between two float32 values -- is settled by the sign of the sum's rounding error."""
    a, b, c = (np.asarray(v, np.float32) for v in (a, b, c))
    s = a.astype(np.float64) * b.astype(np.float64)
    cd = c.astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        r = s + cd
        bb = r - s
        err = (s - (r - bb)) + (cd - bb)                 # s + c = r + err exactly (TwoSum)
        f = r.astype(np.float32)
        fd = f.astype(np.float64)
        # r exactly halfway between f and its neighbour nb on r's side: the exact sum lies on nb's side iff err does
        nb = np.nextafter(f, np.where(r > fd, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))
        tie = (r != fd) & (r == (fd + nb.astype(np.float64)) / 2)
        toward = np.sign(err) == np.sign(r - fd)
        g = np.where(tie & toward & (err != 0), nb, f)
    return np.where(np.isfinite(r), g, f).astype(np.float32)


def tree_space(offset, scale, xyz) -> np.ndarray:
    """offset + scale * xyz (fused), clamped with the reference's min / max: NaN ends at 1 - 1e-6."""
    p = fma32(np.asarray(scale, np.float32)[None, :], np.asarray(xyz, np.float32), np.asarray(offset, np.float32)[None, :])
    with np.errstate(invalid="ignore"):
        p = np.where(p < HI, p, HI)          # min(NaN, hi) = hi, as fminf
        p = np.where(p > 0, p, np.float32(0.0))
    return p.astype(np.float32)


def query(child, data, offset, scale, xyz):
    """-> (data rows fp16 [n, data_dim], cube_sz float32 [n], local float32 [n, 3]) for world points xyz [n, 3]."""
    child = np.asarray(child, np.int32).reshape(-1)
    dd = int(np.asarray(data).shape[-1])
    data = np.asarray(data).view(np.uint16).reshape(-1, dd)
    x = tree_space(offset, scale, xyz)
    n = x.shape[0]
    rows = np.zeros((n, dd), np.uint16)
    cube = np.zeros(n, np.float32)
    local = np.zeros((n, 3), np.float32)
    node = np.zeros(n, np.int64)
    cs = np.float32(2.0)
    act = np.arange(n)
    for _ in range(64):
        if act.size == 0:
            break
        xa = x[act] * np.float32(2.0)
        u = np.floor(xa)
        xa = (xa - u).astype(np.float32)
        x[act] = xa
        sub = node[act] * 8 + (u[:, 0] * 4 + u[:, 1] * 2 + u[:, 2]).astype(np.int64)
        skip = child[sub]
        leaf = skip == 0
        done = act[leaf]
        rows[done] = data[sub[leaf]]
        cube[done] = cs
        local[done] = xa[leaf]
        node[act[~leaf]] += skip[~leaf]
        act = act[~leaf]
        cs = np.float32(cs * 2)
    assert act.size == 0, "descent did not end"
    return rows.view(np.float16), cube, local
