"""`-m "not gpu"`: the two algebraic rewrites the sm_90a march uses instead of the reference's
literal operations (vr_march.cuh: cell_delta_t) are bit-for-bit identities in fp32.  Checked here
in numpy float32 on dense random inputs plus the edge values; the GPU parity tests then check the
kernel that uses them against the reference kernel's golden vectors."""
import numpy as np

F = np.float32


def _rz_to_f32(v64):
    """Round float64 values (exactly representable sums) toward zero to float32."""
    r = v64.astype(F)                       # round to nearest
    too_big = np.abs(r.astype(np.float64)) > np.abs(v64)
    return np.where(too_big, np.nextafter(r, F(0)), r).astype(F)


def test_exit_distance_without_max():
    # reference (rt_core.cuh:37-49): t1 = -p*inv; t2 = t1 + inv; max(t1, t2)
    # kernel: t1 + max(inv, 0)            (inv finite and non-zero, 0 <= p <= 1)
    rng = np.random.default_rng(0)
    n = 2_000_000
    mag = np.exp(rng.uniform(np.log(0.5), np.log(1e17), n))
    inv = (mag * rng.choice([-1.0, 1.0], n)).astype(F)
    p = rng.random(n).astype(F)
    p[:1000] = 0.0
    p[1000:2000] = 1.0
    p[2000:3000] = np.nextafter(F(1), F(0))
    p[3000:4000] = np.nextafter(F(0), F(1))
    t1 = (inv * -p).astype(F)
    ref = np.maximum(t1, (inv + t1).astype(F))
    new = (np.maximum(inv, F(0)) + t1).astype(F)
    assert np.array_equal(ref.view(np.uint32) & 0x7fffffff == 0, new.view(np.uint32) & 0x7fffffff == 0)
    nz = ref != 0
    assert np.array_equal(ref[nz].view(np.uint32), new[nz].view(np.uint32))
    # where both are zero only the sign of zero may differ; the next operation is
    # min(...) * 2^-depth + step_size with step_size > 0, which maps -0 and +0 to the same value


def test_in_cell_coordinate_with_rz_fma():
    # reference (n3tree_query.hpp:28-33 unrolled): f = x*2^d - floor(x*2^d), position x in [0, 1-1e-6]
    # kernel: X = x*2^24 (exact), cube = 2^(d-24);  fl = RZ(X*cube + 2^23);  f = fma(X, cube, 2^23 - fl)
    rng = np.random.default_rng(1)
    for depth in (1, 2, 5, 10, 11, 17, 23):
        x = rng.random(300_000).astype(F)
        x = np.minimum(x, F(1.0) - F(1e-6))
        x[:100] = 0.0
        x[100:200] = F(1.0) - F(1e-6)
        x[200:300] = np.nextafter(F(0), F(1))          # denormal-scale positions
        x[300:400] = (np.arange(100) / 2.0 ** depth).astype(F)  # exactly on cell boundaries
        X = (x * F(16777216.0)).astype(F)
        assert np.array_equal(X.astype(np.float64), x.astype(np.float64) * 16777216.0)  # exact scaling
        v = X.astype(np.float64) * 2.0 ** (depth - 24)                                  # exact product
        ref = (v - np.floor(v)).astype(F)              # exact difference, representable in fp32
        fl = _rz_to_f32(v + 8388608.0)
        neg = (F(8388608.0) - fl).astype(F)
        new = (v + neg.astype(np.float64)).astype(F)   # fma: exact product, one rounding
        assert np.array_equal(fl.astype(np.float64) - 8388608.0, np.floor(v))
        assert np.array_equal(ref.view(np.uint32), new.view(np.uint32))


def test_leaf_word_exponent_field():
    # leaf entry of a wide table: 0x80000000 | (103 + depth) << 23 | sigma (vr_tree.cu: build_wide_kernel)
    for depth in range(1, 24):
        w = np.uint32(0x80000000 | ((103 + depth) << 23) | 0x3c00)
        cb = np.uint32(w & np.uint32(0x7f800000))
        cube = cb.view(F)
        icube = np.uint32(np.uint32(0x73000000) - cb).view(F)
        assert float(cube) == 2.0 ** (depth - 24)
        assert float(icube) == 2.0 ** (-depth)
        assert int(w >> np.uint32(23)) - (256 + 103) == depth
