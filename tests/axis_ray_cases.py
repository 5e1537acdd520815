"""Axis-ray cases of the leaf passes and a plain float64 reference of the composite on them.

Every view is a 2x2 frame whose pixel (1, 1) (``TILE``) runs exactly along the camera's -back axis, one of the six
tree axes: its direction components are exactly 0 and +-1, so the leaves it crosses and the length of every crossing
follow from the tree alone.  ``walk`` walks the octree along that line in float64 from ``child`` and the box
transform, applying the renderer's rules as documented (DESIGN.md 4, 17-18): the t range is the render box shrunk by
1e-6 at both ends (held in fp32, as the renderer keeps it); a sample at t finds the leaf containing the point, moves on
by the distance to the leaf's far face plus ``step_size``, is shaded iff its fp16 sigma > ``sigma_thresh``, and the ray
ends when t reaches tmax or the transmittance falls below ``stop_thresh``.  No march arithmetic and nothing of the C
oracles is used.  ``reference`` then composites those samples in torch float64 from the data rows and gets every
entry's gradient by autograd.

The shading direction is the view direction turned by a non-zero ``rot_dirs`` (Rodrigues), so that no SH basis value
is 0 and every coefficient gets a gradient while the ray itself stays on the axis.

Exactness.  Camera centres, cross-axis offsets, cell faces and the step are dyadic; with power-of-two box scales every
fp32 t, position and cell length of the march is then exact, so the sample lists agree exactly and the values differ
only by fp32 rounding of the composite.  Cameras outside the box look along +axis only: the first point of a -axis ray
from outside is 1 - 1e-6, beyond the lookup's clamp, and the clamped distance is not dyadic.  The cross-axis offsets
are odd multiples of 2^-24, strictly inside a cell at every level down to 23.  The
non-power-of-two box (``exact=False``) keeps the sample list but not the lengths, and is compared by tolerance only.

Step size.  The renderer's rule keeps the sample list analytic for axis rays with any step: the sample after a face is
the point ``step_size`` past it (a point on a face belongs to the cell above it, whichever way the ray runs).  But the
default step, 1e-4, is not dyadic: the fp32 t then carries a rounding of up to ulp(t) ~ 1e-7 at every sample, a
relative error up to 1e-5 on the lengths of small cells, above the weights pass's tolerance.  So the cases use the
dyadic step 2^-12 (``STEP``) and the default 1e-4 is left out.  A step of 0 is used on +axis rays only: a -axis ray
reaches each face exactly, and the point on the face lies in the cell it has just crossed, at distance 0 from that
cell's exit, so with no step it never moves on.
"""
from __future__ import annotations

import math
import zlib
from dataclasses import dataclass, field

import numpy as np

import edge_cases as ec
from volrend_b200 import synth

TILE = (1, 1, 1, 1)
SH_KERNELS = (4, 9, 16, 25)
ROT = [0.45, -0.7, 0.3]     # rot_dirs of every case: a generic shading direction
STEP = 2.0 ** -12           # step_size of every case that does not set one
SHRINK = 1e-6
ONE_M = float(np.float32(1.0 - 1e-6))   # the point clamp of the leaf lookup

# the SH constants of the reference's basis (real spherical harmonics, degrees 0..4)
C0 = 0.28209479177387814
C1 = 0.4886025119029199
C2 = [1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396]
C3 = [-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
      1.445305721320277, -0.5900435899266435]
C4 = [2.5033429417967046, -1.7701307697799304, 0.9461746957575601, -0.6690465435572892, 0.10578554691520431,
      -0.6690465435572892, 0.47308734787878004, -1.7701307697799304, 0.6258357354491761]


def f32(x) -> float:
    return float(np.float32(x))


# ------------------------------------------------------------------------------------------------------ trees
def full_child(depth: int) -> np.ndarray:
    """int32 [cap, 8] of a full octree with leaves at level ``depth`` (root's octants are level 1), breadth first."""
    levels, child, nxt, i = [0], [], 1, 0
    while i < len(levels):
        row = np.zeros(8, np.int32)
        if levels[i] + 1 < depth:
            for o in range(8):
                row[o] = nxt - i
                levels.append(levels[i] + 1)
                nxt += 1
        child.append(row)
        i += 1
    return np.array(child, np.int32)


def fill(child, fmt: str, basis: int, rng, kappa: float, pad: int = 0):
    """fp16 data [cap*8, data_dim] of every slot: leaves get sigma kappa * U(0.3, 1) per world unit and random colour,
    internal slots 0; ``pad`` zero columns between the colour coefficients and sigma."""
    n = child.shape[0] * 8
    dd = 4 if fmt == "RGBA" else 3 * basis + 1 + pad
    d = np.zeros((n, dd), np.float32)
    d[:, -1] = kappa * rng.uniform(0.3, 1.0, n)
    if fmt == "RGBA":
        d[:, :3] = rng.uniform(0.05, 0.95, (n, 3))
    else:
        co = rng.standard_normal((n, 3 * basis)) * 0.6
        co[:, 0::basis] *= 2.0
        d[:, :3 * basis] = co
    d[child.reshape(-1) != 0] = 0.0
    return d.astype(np.float16), dd


def make_tree(child, fmt: str, basis: int, seed: int, kappa: float = 1.5, pad: int = 0, offset=(0.5, 0.5, 0.5),
              scale=(0.5, 0.5, 0.5)) -> synth.SynthTree:
    rng = np.random.default_rng(seed)
    data, dd = fill(child, fmt, basis, rng, kappa, pad)
    cap = child.shape[0]
    name = "RGBA" if fmt == "RGBA" else f"{fmt}{basis}"
    depth = _depth(child)
    return synth.SynthTree(child=child.reshape(cap, 2, 2, 2), data=data.reshape(cap, 2, 2, 2, dd),
                           offset=np.array(offset, np.float32), invradius3=np.array(scale, np.float32), data_dim=dd,
                           data_format=name, depth=depth, extra=ec._extra(fmt, basis, rng))


def _depth(child) -> int:
    child = child.reshape(-1, 8)
    lv = np.zeros(child.shape[0], np.int64)
    for n in range(child.shape[0]):
        for o in np.flatnonzero(child[n]):
            lv[n + child[n, o]] = lv[n] + 1
    return int(lv.max()) + 1


def set_sigma(st, fn, seed):
    """Replaces the sigma of every leaf slot by fn(rng, n) (fp16)."""
    d = st.data.reshape(-1, st.data_dim).copy()
    leaf = st.child.reshape(-1) == 0
    d[leaf, -1] = np.asarray(fn(np.random.default_rng(seed), int(leaf.sum())), np.float16)
    st.data = d.reshape(st.data.shape)
    return st


# ------------------------------------------------------------------------------------------------------ views
@dataclass
class AxisView:
    origin: np.ndarray      # tree-space camera centre, float64 (the fp32 value the renderer computes)
    axis: int               # 0, 1, 2
    sign: int               # +1 / -1: the ray runs along sign * e_axis
    pose: np.ndarray        # row-major 3x4 camera-to-world, float32


def axis_view(st, origin_tree, axis: int, sign: int, exact: bool = True) -> AxisView:
    """The view whose axis pixel starts at tree point ``origin_tree`` and runs along ``sign * e_axis``."""
    scale = st.invradius3.astype(np.float64)
    off = st.offset.astype(np.float64)
    cw = np.float32((np.asarray(origin_tree, np.float64) - off) / scale)
    # the box transform fmaf(scale, world, offset) of the renderer, in fp32
    cen = np.array([f32(float(np.float32(scale[i])) * float(cw[i]) + float(np.float32(off[i]))) for i in range(3)])
    if exact:
        assert np.array_equal(cen, np.asarray(origin_tree, np.float64)), (origin_tree, cen)
    back = np.zeros(3)
    back[axis] = -sign
    right = np.zeros(3)
    right[(axis + 1) % 3] = 1.0
    up = np.cross(back, right)
    pose = np.zeros((3, 4), np.float32)
    pose[:, 0], pose[:, 1], pose[:, 2], pose[:, 3] = right, up, back, cw
    return AxisView(cen, axis, sign, pose)


def cross_offsets(rng, n, lo=0.05, hi=0.95):
    """n odd multiples of 2^-24 in (lo, hi): inside a cell at every level down to 23."""
    k = rng.integers(int(lo * 2 ** 23), int(hi * 2 ** 23), n)
    return (2 * k + 1) / 2.0 ** 24


def box_views(st, rng, n_per=2, signs=(1, -1), exact=True, lo=0.05, hi=0.95):
    """Views along all six directions (``signs``) from inside the box (dyadic centres), and along +axis from outside."""
    views = []
    for axis in range(3):
        for sign in signs:
            for _ in range(n_per):
                o = cross_offsets(rng, 3, lo, hi)
                if sign > 0:
                    p = o.copy()
                    p[axis] = -0.25
                    views.append(axis_view(st, p, axis, sign, exact))
                p = o.copy()
                p[axis] = (2 * rng.integers(int(0.2 * 2 ** 12), int(0.8 * 2 ** 12)) + 1) / 2.0 ** 13
                views.append(axis_view(st, p, axis, sign, exact))
    return views


def chain_views(st, levels: int, signs=(1, -1)):
    """Rays through the chain's deepest node along all six directions, from outside the box and from a coarse leaf
    before the chain's point; the cross-axis offsets (1 or 3 times 2^-24) stay inside the deepest node's cell."""
    P = np.zeros(3)
    for lv in range(levels - 1):
        o = (5 * lv + 3) % 8
        P += np.array([(o >> 2) & 1, (o >> 1) & 1, o & 1]) * 2.0 ** -(lv + 1)
    views = []
    for axis in range(3):
        for sign in signs:
            for start, off in (("out", (1, 3, 1)), ("in", (3, 1, 3))):
                if start == "out" and sign < 0:
                    continue
                p = P + np.array(off) / 2.0 ** 24
                if start == "out":
                    p[axis] = -0.5
                else:
                    mid = P[axis] / 2 if sign > 0 else (P[axis] + 1) / 2
                    p[axis] = math.floor(mid * 2 ** 13) / 2 ** 13 + 2.0 ** -14
                views.append(axis_view(st, p, axis, sign))
    return views


# ------------------------------------------------------------------------------------------------------ cases
@dataclass
class Case:
    name: str
    st: synth.SynthTree
    views: list
    opts: dict = field(default_factory=dict)      # RenderOptions / make_options fields
    exact: bool = True
    expect: tuple = ()          # "stopped", "skipped", "negative"

    def options(self):
        o = dict(step_size=STEP, rot_dirs=list(ROT))
        o.update(self.opts)
        return o

    def dpix(self):
        return np.random.default_rng(zlib.crc32(self.name.encode())).uniform(-1, 1, (len(self.views), 4)).astype(np.float32)

    def err(self):
        return np.random.default_rng(zlib.crc32(self.name.encode()) + 1).uniform(0.1, 1.0, len(self.views)).astype(np.float32)


def _cases():
    out = []

    def add(name, st, views=None, seed=0, **kw):
        out.append(Case(name, st, views if views is not None else box_views(st, np.random.default_rng(seed + 99)), **kw))

    # root-only and full trees of depth 1..4, every kernel basis, RGBA, SG, ASG, bases without a kernel
    add("root_sh4", make_tree(full_child(1), "SH", 4, 1), seed=1)
    add("full2_sh9_bg06", make_tree(full_child(2), "SH", 9, 2), seed=2, opts=dict(background_brightness=0.6))
    add("full3_sh16_stop0", make_tree(full_child(3), "SH", 16, 3), seed=3, opts=dict(stop_thresh=0.0))
    add("full4_sh25_minmax", make_tree(full_child(4), "SH", 25, 4, kappa=1.0), seed=4,
        opts=dict(basis_minmax=[2, 17]))
    add("full3_sh1_bg0", make_tree(full_child(3), "SH", 1, 5), seed=5, opts=dict(background_brightness=0.0))
    add("full3_rgba_bg0", make_tree(full_child(3), "RGBA", -1, 6), seed=6, opts=dict(background_brightness=0.0))
    add("full2_sg9", make_tree(full_child(2), "SG", 9, 7), seed=7)
    add("full3_asg4", make_tree(full_child(3), "ASG", 4, 8), seed=8)
    add("full3_sh2_nokernel", make_tree(full_child(3), "SH", 2, 9), seed=9)
    add("full2_sh36_nokernel", make_tree(full_child(2), "SH", 36, 10), seed=10)
    add("full3_sh4_padded", make_tree(full_child(3), "SH", 4, 11, pad=3), seed=11)
    st = make_tree(full_child(3), "SH", 9, 12)
    add("full3_sh9_step0", st, box_views(st, np.random.default_rng(12), signs=(1,)), opts=dict(step_size=0.0))
    # early stop: sigma high enough that most rays stop, stop_thresh far from every T the rays reach
    add("full3_sh9_stops", make_tree(full_child(3), "SH", 9, 13, kappa=6.0), seed=13,
        opts=dict(stop_thresh=0.2), expect=("stopped",))
    add("full2_rgba_stops_bg06", make_tree(full_child(2), "RGBA", -1, 14, kappa=6.0), seed=14,
        opts=dict(stop_thresh=0.2, background_brightness=0.6), expect=("stopped",))
    # sigma_thresh above some leaves' sigma: skipped samples
    add("full3_sh4_skip", set_sigma(make_tree(full_child(3), "SH", 4, 15), lambda r, n: np.where(
        r.random(n) < 0.3, r.uniform(0.0, 0.4, n), r.uniform(0.6, 1.6, n)), 15), seed=15,
        opts=dict(sigma_thresh=0.5), expect=("skipped",))
    # negative sigma_thresh with sigma <= 0 leaves (weights <= 0) and skipped ones below the threshold
    add("full3_sh9_negative", set_sigma(make_tree(full_child(3), "SH", 9, 16), lambda r, n: r.choice(
        [-2.0, -0.5, -0.25, -0.0, 0.0, 0.5, 0.75, 1.0, 1.25], n), 16), seed=16,
        opts=dict(sigma_thresh=-1.0), expect=("skipped", "negative"))
    # fp16 edge values of sigma (NaN, +-inf, subnormals, max) under a negative threshold
    st = make_tree(full_child(3), "SH", 4, 17)
    d = st.data.reshape(-1, st.data_dim).view(np.uint16).copy()
    leaf = np.flatnonzero(st.child.reshape(-1) == 0)
    d[leaf, -1] = ec.SIGMA_BITS[np.arange(leaf.size) % len(ec.SIGMA_BITS)]
    st.data = d.view(np.float16).reshape(st.data.shape)
    add("full3_sh4_sigma_bits", st, seed=17, opts=dict(sigma_thresh=-1.0), expect=("skipped", "stopped"))
    # mixed depths (leaves at every level 1..6)
    for i, (fmt, basis, kw) in enumerate([("SH", 16, {}), ("SH", 9, dict(background_brightness=0.6)),
                                          ("RGBA", -1, dict(stop_thresh=0.0)), ("SG", 9, {}), ("ASG", 4, {})]):
        m = ec.mixed_tree(6, basis, fmt, 300 + i)
        st = make_tree(m.child.reshape(-1, 8), fmt, basis, 300 + i)
        add(f"mixed_{st.data_format.lower()}", st, seed=300 + i, opts=kw)
    # render_bbox with planes inside cells (the rays start inside it)
    bb = [0.15, 0.2, 0.1, 0.85, 0.8, 0.9]
    st = make_tree(full_child(3), "SH", 16, 20)
    add("full3_sh16_bbox", st, box_views(st, np.random.default_rng(20), lo=0.25, hi=0.75),
        opts=dict(render_bbox=bb))
    # chains to level 22 and 23 along the rays
    st = ec.varied_chain(22)
    add("chain22_step0", st, chain_views(st, 22, signs=(1,)), opts=dict(step_size=0.0))
    st = ec.varied_chain(23)
    add("chain23", st, chain_views(st, 23))
    # power-of-two anisotropic box (lengths stay exact) and a non-power-of-two one (tolerance only)
    st = make_tree(full_child(3), "SH", 9, 30, offset=(0.375, 0.5, 0.25), scale=(0.25, 0.5, 1.0))
    add("aniso_pow2_sh9", st, seed=30)
    m = ec.mixed_tree(5, 16, "SH", 31)
    st = make_tree(m.child.reshape(-1, 8), "SH", 16, 31, offset=(0.4132, 0.5378, 0.4719),
                   scale=(0.2917, 0.4311, 0.3779))
    add("aniso_odd_sh16", st, box_views(st, np.random.default_rng(31), exact=False), exact=False)
    return out


CASES = {c.name: c for c in _cases()}


# ------------------------------------------------------------------------------------------------------ sample list
@dataclass
class Ray:
    slots: list            # every sample's leaf slot, in order
    dts: list              # every sample's delta t (tree units)
    depths: list           # every sample's leaf level
    shaded: list           # bools
    stopped: bool
    hit: bool
    delta_scale: float


def walk(st, view: AxisView, opts: dict) -> Ray:
    """The ordered samples of the axis ray of ``view`` (float64 walk of ``child``), see the module docstring."""
    child = st.child.reshape(-1, 8)
    sig = st.data.reshape(-1, st.data_dim)[:, -1].astype(np.float64)
    bbox = [f32(v) for v in opts.get("render_bbox", [0, 0, 0, 1, 1, 1])]
    step = f32(opts.get("step_size", 1e-4))
    sthr = f32(opts.get("sigma_thresh", 1e-2))
    stop = f32(opts.get("stop_thresh", 1e-2))
    c, a, s = view.origin, view.axis, view.sign
    delta_scale = 1.0 / f32(st.invradius3[a])
    for b in range(3):      # the cross-axis slabs only keep the ray when its offset is inside them
        if b != a:
            assert bbox[b] + SHRINK + 1e-5 < c[b] < bbox[b + 3] - SHRINK - 1e-5, (c, b)
    t1, t2 = (bbox[a] + SHRINK - c[a]) * s, (bbox[a + 3] - SHRINK - c[a]) * s
    tmin, tmax = f32(max(0.0, min(t1, t2))), f32(min(1e4, max(t1, t2)))
    r = Ray([], [], [], [], False, not (tmax < 0 or tmin > tmax), delta_scale)
    if not r.hit:
        return r
    t, T = tmin, 1.0
    while t < tmax:
        assert len(r.slots) < 4096, "the ray does not advance"
        p = np.clip(c + s * t * np.eye(3)[a], 0.0, ONE_M)
        node, lv = 0, 0
        while True:
            lv += 1
            k = np.floor(p * 2.0)
            p = p * 2.0 - k
            slot = node * 8 + int(k[0]) * 4 + int(k[1]) * 2 + int(k[2])
            if child[node, slot - node * 8] == 0:
                break
            node += int(child[node, slot - node * 8])
        dt = ((1.0 - p[a]) if s > 0 else p[a]) / 2.0 ** lv + step
        sh = bool(sig[slot] > sthr)
        r.slots.append(slot)
        r.dts.append(dt)
        r.depths.append(lv)
        r.shaded.append(sh)
        if sh:
            T *= math.exp(-dt * delta_scale * sig[slot])
            if stop > 0:    # the fp32 transmittance must be far from the threshold, so that both ends agree
                assert T == 0 or abs(T / stop - 1) > 1e-3, (T, stop)
            if T < stop:
                r.stopped = True
                break
        t += dt
    return r


# ------------------------------------------------------------------------------------------------------ basis
def rodrigues(aa, v):
    aa, v = np.asarray(aa, np.float64), np.asarray(v, np.float64)
    th = np.linalg.norm(aa)
    if th < 1e-6:
        return v
    k = aa / th
    return v * math.cos(th) + np.cross(k, v) * math.sin(th) + k * np.dot(k, v) * (1 - math.cos(th))


def sh_basis(d, n):
    x, y, z = d
    xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
    b = [C0, -C1 * y, C1 * z, -C1 * x,
         C2[0] * xy, C2[1] * yz, C2[2] * (2 * zz - xx - yy), C2[3] * xz, C2[4] * (xx - yy),
         C3[0] * y * (3 * xx - yy), C3[1] * xy * z, C3[2] * y * (4 * zz - xx - yy), C3[3] * z * (2 * zz - 3 * xx - 3 * yy),
         C3[4] * x * (4 * zz - xx - yy), C3[5] * z * (xx - yy), C3[6] * x * (xx - 3 * yy),
         C4[0] * xy * (xx - yy), C4[1] * yz * (3 * xx - yy), C4[2] * xy * (7 * zz - 1), C4[3] * yz * (7 * zz - 3),
         C4[4] * (zz * (35 * zz - 30) + 3), C4[5] * xz * (7 * zz - 3), C4[6] * (xx - yy) * (7 * zz - 1),
         C4[7] * xz * (xx - 3 * yy), C4[8] * (xx * (xx - 3 * yy) - yy * (3 * xx - yy))]
    return np.array(b[:n])


def basis(st, vdir):
    """(B over every coefficient the format has, number of coefficients the device keeps) for shading direction
    ``vdir``; B is None for RGBA."""
    fmt = st.data_format.rstrip("0123456789")
    if fmt == "RGBA":
        return None, 0
    bd = int(st.data_format[len(fmt):])
    ex = None if st.extra is None else np.asarray(st.extra, np.float64)
    if fmt == "SG":
        B = np.array([math.exp(ex[i, 0] * (np.dot(vdir, ex[i, 1:4]) - 1)) / bd for i in range(bd)])
    elif fmt == "ASG":
        B = np.array([np.dot(vdir, ex[i, 8:11]) * math.exp(-ex[i, 0] * np.dot(vdir, ex[i, 2:5]) ** 2
                                                             - ex[i, 1] * np.dot(vdir, ex[i, 5:8]) ** 2) / bd
                      for i in range(bd)])
    else:
        B = np.zeros(bd)
        B[:min(bd, 25)] = sh_basis(vdir, min(bd, 25))
    return B, (bd if bd in SH_KERNELS else 1)


# ------------------------------------------------------------------------------------------------------ reference
MUTANTS = ("stop_K_bg", "no_T_bg", "dcol_is_col", "grad_outside_minmax", "stop_dalpha")


@dataclass
class Ref:
    pix: np.ndarray        # [V, 4]
    grad: np.ndarray       # [n_slots, data_dim]
    A: np.ndarray          # sum over rays of |per-ray gradient|
    wmax: np.ndarray       # [n_slots], -inf where nothing is shaded
    err: np.ndarray        # [n_slots] sum of w * err
    err_abs: np.ndarray    # [n_slots] sum of |w * err|
    counters: dict         # samples, shaded, rays_hit
    rays: list
    unreached: np.ndarray  # [n_slots, data_dim] entries no ray can move: unshaded slots, columns the device does
                           # not keep or between the coefficients and sigma, coefficients outside basis_minmax


def reference(case: Case, mutant: str | None = None, rays=None) -> Ref:
    """Float64 composite of every view's axis ray, its gradient by autograd and the per-leaf outputs.  ``mutant``
    applies one deliberate error to the derivative (value unchanged) to show that the comparisons catch it.  ``rays``:
    sample lists to use instead of the walk's (one per view)."""
    import torch
    st, opts = case.st, case.options()
    dd = st.data_dim
    data = torch.from_numpy(st.data.reshape(-1, dd).astype(np.float64))
    n_slots = data.shape[0]
    bg = f32(opts.get("background_brightness", 1.0))
    mm = opts.get("basis_minmax", [0, 24])
    dpix, errv = case.dpix().astype(np.float64), case.err().astype(np.float64)
    G, A = np.zeros((n_slots, dd)), np.zeros((n_slots, dd))
    wmax = np.full(n_slots, -np.inf)
    es, ea = np.zeros(n_slots), np.zeros(n_slots)
    pix = np.zeros((len(case.views), 4))
    cnt = dict(samples=0, shaded=0, rays_hit=0)
    rays = [walk(st, view, opts) for view in case.views] if rays is None else rays
    for v, (view, ray) in enumerate(zip(case.views, rays)):
        cnt["samples"] += len(ray.slots)
        cnt["shaded"] += int(sum(ray.shaded))
        cnt["rays_hit"] += int(ray.hit)
        vdir = rodrigues([f32(x) for x in opts["rot_dirs"]], -view.pose[:, 2].astype(np.float64))
        Bfull, nk = basis(st, vdir)
        idx = [s for s, sh in zip(ray.slots, ray.shaded) if sh]
        dts = [dt for dt, sh in zip(ray.dts, ray.shaded) if sh]
        if not idx:
            pix[v] = [bg, bg, bg, 0.0]
            continue
        X = data[idx].clone().requires_grad_(True)
        one = torch.ones((), dtype=torch.float64)
        T, S, ws = one, torch.zeros(3, dtype=torch.float64), []
        if Bfull is not None:
            Bm = Bfull.copy()
            Bm[:max(mm[0], 0)] = 0
            Bm[max(mm[1] + 1, 0):] = 0
        for i in range(len(idx)):
            sg = X[i, dd - 1]
            dl = dts[i] * ray.delta_scale
            att = torch.exp(-dl * sg)
            w = T * (1 - att)
            ws.append(float(w.detach()))
            if Bfull is None:
                col = X[i, :3]
            else:
                bd = len(Bfull)
                K = torch.stack([X[i, c * bd:c * bd + nk] for c in range(3)])     # [3, nk]
                x = K @ torch.from_numpy(Bm[:nk])
                if mutant == "grad_outside_minmax":
                    x = x + (K - K.detach()) @ torch.from_numpy(Bfull[:nk] - Bm[:nk])
                col = torch.sigmoid(x)
                if mutant == "dcol_is_col":
                    col = col.detach() + (x - x.detach()) * col.detach()
            S = S + w * col
            T = T * att
        if ray.stopped:
            s = 1 / (1 - T)
            rgb = S * s
            alpha = one
            if mutant == "stop_K_bg":     # the transmittance term of the stopped pixel with K_c = bg, not pix_c
                sd = s.detach()
                rgb = S * sd + sd * bg * (T - T.detach())
            if mutant == "stop_dalpha":
                alpha = one + (1 - T) - (1 - T).detach()
        else:
            Tb = T.detach() if mutant == "no_T_bg" else T
            rgb = S + Tb * bg
            alpha = 1 - T
        p4 = torch.cat([rgb, alpha.reshape(1)])
        pix[v] = p4.detach().numpy()
        (g,) = torch.autograd.grad((p4 * torch.from_numpy(dpix[v])).sum(), X)
        g = g.numpy()
        gr = np.zeros((n_slots, dd))
        np.add.at(gr, idx, g)
        G += gr
        A += np.abs(gr)
        for s_, w in zip(idx, ws):
            wmax[s_] = max(wmax[s_], w)
            es[s_] += w * errv[v]
            ea[s_] += abs(w * errv[v])
    unreached = np.ones((n_slots, dd), bool)
    shaded = np.isfinite(wmax)
    if st.data_format == "RGBA":
        unreached[shaded, :4] = False
    else:
        bd = int(st.data_format.lstrip("SHAG"))
        nk = bd if bd in SH_KERNELS or not st.data_format.startswith("SH") else 1
        for c in range(3):
            for k in range(max(mm[0], 0), min(nk, mm[1] + 1)):
                unreached[shaded, c * bd + k] = False
        unreached[shaded, dd - 1] = False
    return Ref(pix, G, A, wmax, es, ea, cnt, rays, unreached)


def summary(case: Case, ref: Ref) -> dict:
    """What the case's sample lists cover: rays with at least two shaded leaves, stopped rays, skipped samples."""
    return dict(rays=len(ref.rays), two_shaded=sum(sum(r.shaded) >= 2 for r in ref.rays),
                stopped=sum(r.stopped for r in ref.rays), skipped=sum(len(r.shaded) - sum(r.shaded) for r in ref.rays),
                negative=int((ref.wmax[np.isfinite(ref.wmax)] <= 0).sum()))
