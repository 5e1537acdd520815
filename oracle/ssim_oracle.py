"""Float64 restatement of the per-view SSIM of ``vr_image_ssim`` and of its gradient (DESIGN.md section 22).

JaxNeRF's ``compute_ssim``: an 11-tap Gaussian (sigma 1.5, normalised) applied separably with valid filtering to x, y,
x^2, y^2 and xy of each of channels 0..2; clipped variances and covariance; C1 = 0.01^2, C2 = 0.03^2 (max_val 1); the
per-view value is the mean over the channels and the valid pixels.  The gradient is the analytic one, with respect to
x, with the clip rules stated in DESIGN.md section 22.  Plain numpy, written from the definition alone.
"""
from __future__ import annotations

import numpy as np

C1 = 0.01 ** 2
C2 = 0.03 ** 2
TAPS = 11


def gaussian() -> np.ndarray:
    i = np.arange(TAPS, dtype=np.float64)
    f = np.exp(-0.5 * ((i - 5) / 1.5) ** 2)
    return f / f.sum()


def _valid(a: np.ndarray, axis: int) -> np.ndarray:
    """sum_t f_t a[i + t] along ``axis``: n -> n - 10."""
    f = gaussian()
    a = np.moveaxis(a, axis, -1)
    n = a.shape[-1] - (TAPS - 1)
    out = sum(f[t] * a[..., t:t + n] for t in range(TAPS))
    return np.moveaxis(out, -1, axis)


def _full_t(a: np.ndarray, axis: int) -> np.ndarray:
    """The transpose of _valid: out[p] = sum_t f_t a[p - t], n -> n + 10."""
    f = gaussian()
    a = np.moveaxis(a, axis, -1)
    out = np.zeros(a.shape[:-1] + (a.shape[-1] + TAPS - 1,))
    for t in range(TAPS):
        out[..., t:t + a.shape[-1]] += f[t] * a
    return np.moveaxis(out, -1, axis)


def _filt(a: np.ndarray) -> np.ndarray:
    """Valid 2-D filter of [..., H, W] planes."""
    return _valid(_valid(a, -2), -1)


def _planes(img) -> np.ndarray:
    """[V, H, W, C] (C 3 or 4) -> float64 RGB planes [V, 3, H, W]."""
    a = np.asarray(img, np.float64)
    if a.ndim != 4 or a.shape[-1] not in (3, 4):
        raise ValueError(f"images must be [V, H, W, 3 | 4], not {a.shape}")
    if a.shape[1] < TAPS or a.shape[2] < TAPS:
        raise ValueError(f"images are {a.shape[2]}x{a.shape[1]}: SSIM needs at least 11x11")
    return np.moveaxis(a[..., :3], -1, 1)


def ssim_maps(x, y, grad: bool = False):
    """The SSIM map [V, 3, H-10, W-10] of x against y and, with ``grad``, the partials (a, b, c) = (ds/dmu_x total,
    ds/dE[x^2], ds/dE[xy]) of every output pixel."""
    xp, yp = _planes(x), _planes(y)
    mx, my = _filt(xp), _filt(yp)
    return from_moments(mx, my, _filt(xp * xp), _filt(yp * yp), _filt(xp * yp), grad, _flat(xp), _flat(yp))


def _flat(a: np.ndarray) -> np.ndarray:
    """Whether each 11x11 window of [..., H, W] planes holds a single value."""
    def span(v, axis, op):
        v = np.moveaxis(v, axis, -1)
        n = v.shape[-1] - (TAPS - 1)
        out = v[..., :n]
        for t in range(1, TAPS):
            out = op(out, v[..., t:t + n])
        return np.moveaxis(out, -1, axis)
    return span(span(a, -2, np.minimum), -1, np.minimum) == span(span(a, -2, np.maximum), -1, np.maximum)


def from_moments(mx, my, exx, eyy, exy, grad: bool = False, flat_x=False, flat_y=False):
    """SSIM s of output pixels from their filtered moments and, with ``grad``, (a, b, c) as ssim_maps.  ``flat_x`` /
    ``flat_y``: windows whose x / y holds one value; their variance and the covariance are exactly 0 (as in exact
    arithmetic; rounding would leave them a few ulps either side of 0 and pick the covariance clip at random)."""
    mx, my, exx, eyy, exy = (np.asarray(v, np.float64) for v in (mx, my, exx, eyy, exy))
    vx = np.where(flat_x, 0.0, exx - mx * mx)
    vy = np.where(flat_y, 0.0, eyy - my * my)
    sxx, syy = np.maximum(vx, 0.0), np.maximum(vy, 0.0)
    sxy0 = np.where(np.logical_or(flat_x, flat_y), 0.0, exy - mx * my)
    pr = sxx * syy
    rt = np.sqrt(pr)
    clip = np.abs(sxy0) > rt
    sxy = np.where(clip, np.sign(sxy0) * rt, sxy0)
    A, B = 2 * mx * my + C1, 2 * sxy + C2
    C, D = mx * mx + my * my + C1, sxx + syy + C2
    s = A * B / (C * D)
    if not grad:
        return s
    ds_dsxy = 2 * A / (C * D)
    with np.errstate(divide="ignore", invalid="ignore"):
        dsxy_dsxx = np.where(clip & (pr > 0), np.sign(sxy0) * syy / (2 * np.where(pr > 0, rt, 1.0)), 0.0)
    ds_dsxx = -s / D + ds_dsxy * dsxy_dsxx
    c = np.where(clip, 0.0, ds_dsxy)
    b = np.where(vx >= 0, ds_dsxx, 0.0)
    direct = 2 * my * B / (C * D) - s * 2 * mx / C
    a = direct - 2 * mx * b - my * c
    return s, (a, b, c)


def ssim(x, y) -> np.ndarray:
    """Per-view SSIM, float64 [V]."""
    return ssim_maps(x, y).mean(axis=(1, 2, 3))


def ssim_grad(x, y):
    """(ssim [V], dssim_v/dx [V, H, W, 3]) in float64."""
    s, (a, b, c) = ssim_maps(x, y, grad=True)
    xp, yp = _planes(x), _planes(y)
    ft = lambda m: _full_t(_full_t(m, -2), -1)
    n = 3 * s.shape[2] * s.shape[3]
    d = (ft(a) + 2 * xp * ft(b) + yp * ft(c)) / n
    return s.mean(axis=(1, 2, 3)), np.moveaxis(d, 1, -1)
