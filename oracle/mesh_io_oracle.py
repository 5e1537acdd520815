"""numpy restatement of the reference's estimate_normals (src/mesh.cpp:63-97).  TEST INFRASTRUCTURE ONLY.

float32 throughout, exact indices, each vertex's cross products accumulated in face order from +0.f (np.add.at
applies repeated indices one after another, in index order), and the norm threshold compared in double.  A face
with an index >= n_verts contributes nothing (the product's deliberate deviation; the reference reads out of
bounds), and so do the reference's float-rounded offsets above vertex 1 864 135 (here indices are exact)."""
from __future__ import annotations

import numpy as np

VERT_SZ = 9


def estimate_normals(vert: np.ndarray, faces: np.ndarray) -> np.ndarray:
    """A copy of ``vert`` (n_verts * 9 float32) with floats 6..8 of each vertex replaced by the estimated normal.
    ``faces`` empty: consecutive vertex triples (n_verts // 3 faces); otherwise len(faces) // 3 triangles."""
    out = np.array(vert, np.float32).reshape(-1, VERT_SZ)
    nv = out.shape[0]
    faces = np.asarray(faces, np.uint32).reshape(-1)
    if faces.size:
        f = faces[:faces.size // 3 * 3].reshape(-1, 3).astype(np.int64)
        f = f[(f < nv).all(1)]
    else:
        f = np.arange(nv // 3 * 3, dtype=np.int64).reshape(-1, 3)
    p = out[:, :3]
    a = p[f[:, 1]] - p[f[:, 0]]
    b = p[f[:, 2]] - p[f[:, 0]]
    cross = np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1],
                      a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                      a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1).astype(np.float32)
    acc = np.zeros((nv, 3), np.float32)
    # corners in face order: face 0's three corners, then face 1's, ...
    np.add.at(acc, f.reshape(-1), np.repeat(cross, 3, axis=0))
    norm = np.sqrt((acc[:, 0] * acc[:, 0] + acc[:, 1] * acc[:, 1]) + acc[:, 2] * acc[:, 2]).astype(np.float32)
    big = norm.astype(np.float64) > 1e-6
    acc[big] = acc[big] / norm[big, None]
    out[:, 6:9] = acc
    return out.reshape(-1)
