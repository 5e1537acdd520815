"""`-m "not gpu"`: the CPU restatements of the leaf passes (orc_leaf_grads, orc_leaf_weights, orc_leaf_error) and
orc_render's float output against the float64 autograd reference of tests/axis_ray_cases.py, on axis rays whose
samples are known without running any march code, entry by entry.  Mutants of the reference (each a deliberate error
in the derivation, the value unchanged) show that the same comparison rejects a subtly wrong derivative."""
import numpy as np
import pytest

import axis_ray_cases as ac
from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)

RTOL, ATOL = 1e-4, 1e-7          # gradients: |g - g64| <= RTOL * A + ATOL
PIX_TOL = 1e-5
W_RTOL, W_ATOL = 1e-6, 1e-7      # weights
E_RTOL, E_ATOL = 1e-5, 1e-7      # error sums, relative to the sum of |terms|


def oracle(case):
    """The C restatements over every view of the case: grad, A, float pixels, weights, error sums, counters."""
    from oracle import binding as ob
    from oracle import error_binding as eb
    from oracle import grads_binding as gb
    from oracle import weights_binding as wb
    st = case.st
    ot = ob.OracleTree.from_synth(st)
    opt = ob.make_options(**case.options())
    n = st.capacity * 8
    G, A = np.zeros((n, st.data_dim)), np.zeros((n, st.data_dim))
    W = np.full(n, -np.inf, np.float32)
    E = np.zeros(n)
    pix = np.zeros((len(case.views), 4), np.float32)
    cnt = dict(samples=0, shaded=0, rays_hit=0)
    dpix, err = case.dpix(), case.err()
    for v, view in enumerate(case.views):
        cam = ob.make_camera(2, 2, 1.0, 1.0, ob_colmajor(view.pose))
        _, _, rgba = gb.leaf_grads(ot, cam, opt, dpix[v].reshape(1, 1, 4), tile=ac.TILE, grad=G, A=A, nthreads=1)
        f, _, _ = ob.render(ot, cam, opt, tile=ac.TILE, want_u8=False, nthreads=1)
        assert np.array_equal(rgba.view(np.uint32), f.view(np.uint32))
        pix[v] = f[0, 0]
        _, _, c = wb.leaf_weights(ot, cam, opt, tile=ac.TILE, weights=W, want_alpha=False, nthreads=1)
        s, _, _, c2 = eb.leaf_error(ot, cam, opt, err[v].reshape(1, 1), tile=ac.TILE, nthreads=1)
        assert c == c2
        E += s
        for k in cnt:
            cnt[k] += c[k]
    return G, A, pix, W, E, cnt


def ob_colmajor(pose):
    from volrend_b200 import synth
    return synth.c2w_to_colmajor12(pose)


def grad_bad(g, ref):
    return np.abs(g - ref.grad) > RTOL * ref.A + ATOL


@pytest.mark.parametrize("name", list(ac.CASES))
def test_oracles_match_reference(name):
    case = ac.CASES[name]
    ref = ac.reference(case)
    s = ac.summary(case, ref)
    assert s["two_shaded"] >= 0.6 * s["rays"], s
    for what in case.expect:
        assert s[what] > 0, (what, s)
    G, A, pix, W, E, cnt = oracle(case)
    assert cnt == ref.counters, (cnt, ref.counters)
    np.testing.assert_allclose(pix, ref.pix, rtol=0, atol=PIX_TOL)
    bad = grad_bad(G, ref)
    assert not bad.any(), (int(bad.sum()), np.argwhere(bad)[:5].tolist())
    assert not G[ref.unreached].any() and not ref.grad[ref.unreached].any()
    touched = np.isfinite(ref.wmax)
    assert np.array_equal(np.isfinite(W), touched)
    np.testing.assert_allclose(W[touched], ref.wmax[touched], rtol=W_RTOL, atol=W_ATOL)
    assert (np.abs(E - ref.err) <= E_RTOL * ref.err_abs + E_ATOL).all()
    assert not E[~touched].any()


def test_reference_reproduces_closed_form():
    """The two-leaf ray of test_grads_cpu: pixel to 1e-12, gradient to the accuracy of its double central
    differences."""
    import test_grads_cpu as tg
    for fmt in ("SH1", "RGBA"):
        for case_kind in ("runs_out", "stops_early"):
            rows = {0: [0.75, -1.5, 2.0, 2.0], 4: [-0.5, 0.25, 1.25, 3.0 if case_kind == "runs_out" else 10.0]}
            if fmt == "RGBA":
                rows = {o: [abs(v) / 2.5 for v in r[:3]] + [r[3]] for o, r in rows.items()}
            _, data = tg._root_tree(rows, fmt)
            rows64 = {o: data.reshape(8, 4)[o].astype(np.float64) for o in rows}
            from volrend_b200 import synth
            st = synth.SynthTree(child=np.zeros((1, 2, 2, 2), np.int32), data=data, offset=np.zeros(3, np.float32),
                                 invradius3=np.ones(3, np.float32), data_dim=4, data_format=fmt, depth=1)
            g = np.array([0.7, -1.3, 0.4, 2.1])
            bg, stop = 0.6, (0.0 if case_kind == "runs_out" else 0.01)
            view = ac.axis_view(st, [-1.0, 0.25, 0.25], 0, 1)
            case = ac.Case("closed", st, [view], dict(step_size=0.0, stop_thresh=stop, background_brightness=bg,
                                                      rot_dirs=[0, 0, 0]))
            case.dpix = lambda: g[None].astype(np.float32)
            ray = ac.Ray([0, 4], [0.5, 0.5], [1, 1], [True, True], case_kind == "stops_early", True, 1.0)
            ref = ac.reference(case, rays=[ray])
            want = tg._closed_form(rows64, fmt, g.astype(np.float32).astype(np.float64), bg, stop)
            np.testing.assert_allclose(ref.grad[[0, 4]], want, rtol=1e-7, atol=1e-9)
            # the pixel itself, from the same formula as the closed form
            bg = float(np.float32(bg))      # the option as the renderer holds it
            T, S = 1.0, np.zeros(3)
            for o in (0, 4):
                att = np.exp(-0.5 * rows64[o][3])
                col = rows64[o][:3] if fmt == "RGBA" else 1 / (1 + np.exp(-ac.C0 * rows64[o][:3]))
                S, T = S + T * (1 - att) * col, T * att
            want_pix = np.append(S / (1 - T), 1.0) if case_kind == "stops_early" else np.append(S + T * bg, 1 - T)
            np.testing.assert_allclose(ref.pix[0], want_pix, rtol=0, atol=1e-12)


# the cases each mutant is tried on: each needs a stopped ray, a restricted basis_minmax or a sigmoid basis
MUTANT_CASES = ["full3_sh9_stops", "full2_rgba_stops_bg06", "full4_sh25_minmax", "full2_sh9_bg06", "mixed_sh16"]


@pytest.mark.parametrize("mutant", ac.MUTANTS)
def test_mutant_is_rejected(mutant):
    rejected = []
    for name in MUTANT_CASES:
        case = ac.CASES[name]
        ref = ac.reference(case, mutant=mutant)
        G = oracle(case)[0]
        n = int(grad_bad(G, ref).sum())
        if n:
            rejected.append((name, n))
    print(f"mutant {mutant}: rejected by {rejected}")
    assert rejected, f"mutant {mutant} passes every comparison"
