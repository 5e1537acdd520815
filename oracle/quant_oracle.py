"""numpy restatement of the tree compressor (volrend_b200/csrc/vr_quant.cu, DESIGN.md section 12).  TEST
INFRASTRUCTURE ONLY.

Median cut per point set: each level, every bucket picks the axis with the largest fp32 ``hi - lo`` (lowest axis on a
tie), is stably sorted by that axis (one ``np.lexsort`` over (segment, value) for the whole level) and splits at
floor(n / 2).  Values compare as fp16 with -0 == +0.  Bucket means are exact: the sum of 2^-24 multiples is a Python
int, converted with ``float(int)`` (round to nearest even), divided by n in double, scaled and rounded once to fp16.
``compress_arrays`` has the signature of the device path in ``volrend_b200.compress`` so tests can swap them."""
from __future__ import annotations

import numpy as np

ROWS = 65536


def okey(h: np.ndarray) -> np.ndarray:
    """16-bit key whose order is the fp16 order, -0 folded onto +0."""
    h = np.asarray(h, np.uint16).astype(np.int64)
    h = np.where(h == 0x8000, 0, h)
    return np.where(h & 0x8000, ~h & 0xFFFF, h | 0x8000)


def okey_inv(k: np.ndarray) -> np.ndarray:
    k = np.asarray(k, np.int64)
    return np.where(k & 0x8000, k & 0x7FFF, ~k & 0xFFFF).astype(np.uint16)


def mult24(h: np.ndarray) -> np.ndarray:
    """fp16 bits -> the value as an exact int64 multiple of 2^-24."""
    h = np.asarray(h, np.uint16).astype(np.int64)
    e, f = (h >> 10) & 31, h & 1023
    m = np.where(e == 0, f, (1024 + f) << np.maximum(e - 1, 0))
    return np.where(h & 0x8000, -m, m)


def bucket_sizes(M: int, level: int) -> np.ndarray:
    """Sizes of the 2^level buckets: bucket b splits into 2b (floor(n/2) points) and 2b+1 (the rest)."""
    s = np.array([M], np.int64)
    for _ in range(level):
        s = np.stack([s // 2, s - s // 2], 1).reshape(-1)
    return s


def median_cut(px: np.ndarray, py: np.ndarray, pz: np.ndarray, bits: int):
    """One point set (fp16 bits, set order) -> (codebook u16 [65536, 3], bucket id u16 [M] per point in set order)."""
    if not 1 <= bits <= 16:
        raise ValueError(f"bits {bits} outside [1, 16]")
    K = np.stack([okey(px), okey(py), okey(pz)])          # [3, M]
    M = K.shape[1]
    order = np.arange(M)                                   # order[p] = point at position p
    for L in range(bits):
        sizes = bucket_sizes(M, L)
        seg = np.repeat(np.arange(sizes.size), sizes)
        if M == 0:
            break
        kc = K[:, order]
        starts = np.concatenate([[0], np.cumsum(sizes)[:-1]])
        ne = sizes > 0
        lo = np.minimum.reduceat(kc, starts[ne], axis=1)
        hi = np.maximum.reduceat(kc, starts[ne], axis=1)
        f = lambda k: okey_inv(k).view(np.float16).astype(np.float32)
        r = f(hi) - f(lo)                                  # [3, nonempty] fp32, rounded to nearest
        axis = np.zeros(sizes.size, np.int64)
        axis[ne] = np.argmax(r, axis=0)                    # first maximum: ties keep the lowest axis
        key = kc[axis[seg], np.arange(M)]
        order = order[np.lexsort((key, seg))]              # stable: equal keys keep their current order
    sizes = bucket_sizes(M, bits)
    bucket = np.empty(M, np.uint16)
    bucket[order] = np.repeat(np.arange(sizes.size), sizes).astype(np.uint16)
    colors = np.zeros((ROWS, 3), np.uint16)
    if M:
        ne = np.nonzero(sizes)[0]
        starts = np.concatenate([[0], np.cumsum(sizes)[:-1]])[ne]
        for a, p in enumerate((px, py, pz)):
            m = mult24(np.asarray(p)[order])
            hi = np.add.reduceat(m >> 20, starts)
            lo = np.add.reduceat(m & 0xFFFFF, starts)
            mean = [float(int(h) * (1 << 20) + int(l)) / int(n) * 2.0 ** -24 for h, l, n in zip(hi, lo, sizes[ne])]
            colors[ne, a] = np.array(mean, np.float64).astype(np.float16).view(np.uint16)
    return colors, bucket


def kept_mask(sigma: np.ndarray, sigma_thresh: float) -> np.ndarray:
    """sigma (fp16 bits) > fp16_rn(sigma_thresh), compared as fp16.  The threshold reaches the C-ABI as a float, so it
    is rounded to float first and then to fp16, as torch rounds a Python scalar against an fp16 tensor."""
    thr = np.float16(np.float32(sigma_thresh))
    return np.asarray(sigma, np.uint16).view(np.float16) > thr


def compress_arrays(data: np.ndarray, data_dim: int, sigma_thresh: float, retain: int, bits: int):
    """data: u16 [n_child, data_dim] (fp16 bits) -> (quant_colors u16 [n_quant, 65536, 3], quant_map u16
    [n_quant, n_child], sigma u16 [n_child], data_retained u16 [retain, n_child, 3] or None, n_kept)."""
    B = (data_dim - 1) // 3
    if not 1 <= bits <= 16:
        raise ValueError(f"bits {bits} outside [1, 16]")
    if retain < 0:
        raise ValueError(f"retain {retain} < 0")
    if data_dim < 4 or data_dim != 3 * B + 1:
        raise ValueError(f"data_dim {data_dim} is not 3 * basis_dim + 1")
    nq = B - retain
    if nq < 1:
        raise ValueError(f"retain {retain} leaves no basis function to quantise (the tree has {B})")
    data = np.asarray(data, np.uint16).reshape(-1, data_dim)
    n_child = data.shape[0]
    keep = kept_mask(data[:, -1], sigma_thresh)
    kd = data[keep]
    q = np.concatenate([kd[:, k * B + retain:(k + 1) * B] for k in range(3)], 1)
    if ((q & 0x7C00) == 0x7C00).any():
        raise ValueError("a quantised coefficient of a kept voxel is Inf or NaN")
    sigma = np.where(keep, data[:, -1], 0).astype(np.uint16)
    retained = None
    if retain:
        retained = np.zeros((retain, n_child, 3), np.uint16)
        for j in range(retain):
            for k in range(3):
                retained[j, keep, k] = kd[:, k * B + j]
    colors = np.zeros((nq, ROWS, 3), np.uint16)
    qmap = np.zeros((nq, n_child), np.uint16)
    for i, j in enumerate(range(retain, B)):
        colors[i], qmap[i, keep] = median_cut(kd[:, j], kd[:, B + j], kd[:, 2 * B + j], bits)
    return colors, qmap, sigma, retained, int(keep.sum())
