"""CPU: the point-query oracle (oracle/query_oracle.py) against the reference's query_single_from_root goldens
(tests/golden/ref/query_*.npz), the query cases themselves, and the argument checks of N3Tree.query / eval."""
from fractions import Fraction

import numpy as np
import pytest

from oracle import query_oracle as qo
from query_cases import QUERY_TREES, SETS, all_points, golden_path, query_tree


def _tree(name):
    from volrend_b200 import N3Tree
    t = N3Tree()
    t.load_npz(query_tree(name))
    return t


@pytest.mark.parametrize("name", QUERY_TREES)
def test_oracle_matches_reference_golden(name):
    z = np.load(golden_path(name))
    t = _tree(name)
    pts, lab = all_points(name, query_tree(name))
    assert np.array_equal(pts.view(np.uint32), z["points"].view(np.uint32)) and np.array_equal(lab, z["set"])
    data, cube, local = qo.query(t.child_, t.data_, t.offset, t.scale, pts)
    assert np.array_equal(data.view(np.uint16), z["data"])
    assert np.array_equal(cube.view(np.uint32), z["cube"].view(np.uint32))
    assert np.array_equal(local.view(np.uint32), z["local"].view(np.uint32))


def test_cases_cover_every_set_and_the_chain_depth():
    for name in QUERY_TREES:
        _, lab = all_points(name, query_tree(name))
        assert sorted(set(lab.tolist())) == list(range(len(SETS)))
    z = np.load(golden_path("chain"))
    assert float(z["cube"].max()) == 2.0 ** 23
    nf = np.load(golden_path("lego_sh16"))
    pts = nf["points"][nf["set"] == SETS.index("nonfinite")]
    assert np.isnan(pts).any() and np.isinf(pts).any()


def test_nan_clamps_to_upper_bound():
    p = qo.tree_space(np.zeros(3, np.float32), np.ones(3, np.float32),
                      np.array([[np.nan, np.inf, -np.inf]], np.float32))
    assert p[0, 0] == qo.HI and p[0, 1] == qo.HI and p[0, 2] == 0


def _rne32(v: Fraction) -> np.float32:
    """The float32 nearest to the rational v, ties to even (v finite, in the normal range)."""
    f = np.float32(float(v))
    cands = [np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))]
    dist = [abs(Fraction(float(c)) - v) for c in cands]
    best = min(dist)
    ties = [c for c, d in zip(cands, dist) if d == best]
    return ties[0] if len(ties) == 1 else next(c for c in ties if int(c.view(np.uint32)) % 2 == 0)


def test_fma32_rounds_once():
    f32 = np.float32
    a = b = f32(1 + 2 ** -12)
    # a*b - 1 = 2^-11 + 2^-24 exactly: representable, where a rounded product would lose 2^-24
    assert qo.fma32(a, b, f32(-1)) == f32(2 ** -11 + 2 ** -24)
    # a*b = 1 + 2^-11 + 2^-24 lies halfway between two float32: ties to even, and a tiny addend decides the tie
    assert qo.fma32(a, b, f32(0)) == f32(1 + 2 ** -11)
    assert qo.fma32(a, b, f32(2 ** -60)) == f32(1 + 2 ** -11 + 2 ** -23)
    assert qo.fma32(a, b, f32(-2 ** -60)) == f32(1 + 2 ** -11)
    rng = np.random.default_rng(0)
    x, y = (rng.standard_normal(3000).astype(np.float32) for _ in range(2))
    w = (rng.standard_normal(3000) * 10.0 ** rng.integers(-9, 3, 3000)).astype(np.float32)
    # addends that put the exact sum on or next to a float32 midpoint
    w[:1000] = (-(x[:1000].astype(np.float64) * y[:1000].astype(np.float64))).astype(np.float32)
    got = qo.fma32(x, y, w)
    for i in range(3000):
        v = Fraction(float(x[i])) * Fraction(float(y[i])) + Fraction(float(w[i]))
        if v == 0:
            assert got[i] == 0, i
            continue
        assert got[i].view(np.uint32) == _rne32(v).view(np.uint32), (i, x[i], y[i], w[i])


def test_argument_checks():
    from volrend_b200 import N3Tree
    with pytest.raises(RuntimeError, match="no data"):
        N3Tree().query(np.zeros((1, 3), np.float32))
    t = _tree("cfg1_sh1")
    with pytest.raises(ValueError, match="shape"):
        t.query(np.zeros((4, 2), np.float32))
    with pytest.raises(ValueError, match="shape"):
        t.query(np.zeros(3, np.float32))
    with pytest.raises(TypeError, match="float32"):
        t.query(np.zeros((4, 3), np.float64))
    with pytest.raises(TypeError):
        t.query([[0.0, 0.0, 0.0]])
    with pytest.raises(ValueError, match="shape"):
        t.eval(np.zeros((4, 3), np.float32), np.zeros((5, 3), np.float32))


def _has_gpu() -> bool:
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.mark.skipif(_has_gpu(), reason="a device is present: the GPU tests run these calls")
def test_nan_and_empty_points_reach_the_device_call():
    """NaN points and n = 0 pass the argument checks: without a device the call then fails in the C-ABI."""
    from volrend_b200 import VolrendError, _capi
    t = _tree("cfg1_sh1")
    for pts in (np.full((2, 3), np.nan, np.float32), np.zeros((0, 3), np.float32)):
        with pytest.raises(VolrendError) as e:
            t.query(pts)
        assert e.value.code == _capi.VR_ENODEVICE
