"""`-m "not gpu"`: the lumisphere probe disc (enable_probe) without a device -- the CPU restatement
(oracle/probe_oracle.c) against the reference's own launch_renderer output (tests/golden/ref/probe_*.npz, made on an
H100 by tools/make_golden.py --probe), its disc mask against the reference's predicate, and the C-ABI's argument
checks."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import ROOT
from oracle import binding as ob
from oracle import probe_oracle as po
from probe_cases import PROBE_CASES, H, W, focal, golden_path, probe_case
from volrend_b200 import synth


def _oracle(name, want_mask_only=False):
    st, pose, optkw, probe, disp, comp = probe_case(name)
    t = ob.OracleTree.from_synth(st)
    cam = ob.make_camera(W, H, focal(), focal(), synth.c2w_to_colmajor12(pose))
    opt = ob.make_options(**optkw)
    if want_mask_only:
        return po.overlay(t, cam, opt, probe, disp)
    rin, din = comp if comp is not None else (None, None)
    return po.render(t, cam, opt, probe, disp, rgba_in=rin, depth_in=din)


def test_probe_goldens_present():
    for name in PROBE_CASES:
        assert os.path.exists(golden_path(name)), name


@pytest.mark.parametrize("name", list(PROBE_CASES))
def test_oracle_matches_reference_probe_golden(built, name):
    """Disc pixels: the oracle's bytes equal the reference's, except where a colour's truncation sits on an integer
    boundary and the glibc / libdevice expf ulp decides it (then by one).  Elsewhere the reference frame with the
    probe equals the one without it, byte for byte."""
    z = np.load(golden_path(name), allow_pickle=False)
    ref, ref_off = z["ref_u8"], z["ref_u8_off"]
    f, u, mask = _oracle(name)
    assert np.array_equal(ref[~mask], ref_off[~mask])
    d = np.abs(u[mask].astype(int) - ref[mask].astype(int))
    assert d.max(initial=0) <= 1
    assert int((d > 0).any(-1).sum()) <= max(2, int(mask.sum()) // 2000)
    assert (u[mask][:, 3] == 255).all() and (f[mask][:, 3] == 1.0).all()
    # the march part, as the march oracle's golden test bounds it
    assert np.abs(u[~mask].astype(int) - ref[~mask].astype(int)).max(initial=0) <= 1
    if name.startswith("sh16_d") or name == "sh16_centre":
        sizes = {"sh16_d0": 0, "sh16_d1": 0, "sh16_dmax": 0, "sh16_dneg": 0}
        if name in sizes:
            assert mask.sum() == sizes[name]
        else:
            assert mask.sum() > 0


def _predicate(disp: int, w: int, h: int) -> np.ndarray:
    """volrend.cu:100-110 in numpy: int32 wrapping adds, float32 divisions, c = fma(a, a, b*b) <= 1."""
    y, x = np.mgrid[0:h, 0:w].astype(np.int64)
    wrap = lambda v: ((np.asarray(v, np.int64) + 2 ** 31) % 2 ** 32 - 2 ** 31)   # noqa: E731
    cand = (y < wrap(disp + 5)) & (x >= wrap(w - disp - 5))
    xx, yy = wrap(x + 5 - w + disp).astype(np.float32), (y - 5).astype(np.float32)
    hs = np.float32(disp) * np.float32(0.5)
    with np.errstate(divide="ignore", invalid="ignore"):
        a = (xx / hs).astype(np.float32) - np.float32(1)
        b = (yy / hs).astype(np.float32) - np.float32(1)
    c = (a.astype(np.float64) * a + (b * b).astype(np.float64)).astype(np.float32)   # a*a is exact in double
    return cand & (c <= 1)


@pytest.mark.parametrize("disp", [100, 37, 1, 0, -3, -4, 500, 2 ** 31 - 6, 2 ** 31 - 1, -2 ** 31])
def test_mask_matches_reference_predicate(built, disp):
    st, pose, optkw, probe, _, _ = probe_case("sh16_centre")
    t = ob.OracleTree.from_synth(st)
    cam = ob.make_camera(W, H, focal(), focal(), synth.c2w_to_colmajor12(pose))
    mask = po.overlay(t, cam, ob.make_options(**optkw), probe, disp)
    assert np.array_equal(mask, _predicate(disp, W, H))
    if 2 <= disp <= 500:
        assert mask.sum() > 0
    # the candidate corner never leaves the top-right (S + 5)^2 square
    assert not mask[min(max(disp + 5, 0), H):].any() if 0 <= disp < H else True


def test_golden_disc_changes_lie_in_the_mask(built):
    for name in PROBE_CASES:
        z = np.load(golden_path(name), allow_pickle=False)
        changed = (z["ref_u8"] != z["ref_u8_off"]).any(-1)
        mask = _oracle(name, want_mask_only=True)
        assert not (changed & ~mask).any(), name
        if mask.any():
            assert changed.any(), name


def test_header_and_binding_declare_vr_draw_probe(built):
    from volrend_b200 import _capi
    txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "volrend_b200.h")).read(), flags=re.S)
    m = re.search(r"int\s+vr_draw_probe\s*\(([^)]*)\)", txt)
    assert m is not None
    assert len(m.group(1).split(",")) == len(_capi.SYMBOLS["vr_draw_probe"][1]) == 11


def test_draw_probe_argument_checks(built):
    """Malformed calls are refused before any device work."""
    from volrend_b200 import _capi, lib
    cam = (_capi.vr_camera * 2)()
    opt = _capi.vr_options()
    xyz = (C.c_float * 3)(0.0, 0.0, 1.0)
    buf = C.c_void_p(0x1000)   # never dereferenced: every call below fails its checks first
    L = lib()
    assert L.vr_draw_probe(None, cam, -1, C.byref(opt), xyz, 100, None, buf, None, 0, None) == _capi.VR_EINVAL
    assert L.vr_draw_probe(None, cam, 1, C.byref(opt), None, 100, None, buf, None, 0, None) == _capi.VR_EINVAL
    assert L.vr_draw_probe(None, cam, 1, C.byref(opt), xyz, 100, None, None, None, 0, None) == _capi.VR_EINVAL
    assert b"no output" in L.vr_last_error()
    # the surface form: one view, no tile, no linear or float output
    assert L.vr_draw_probe(None, cam, 2, C.byref(opt), xyz, 100, None, None, None, 7, None) == _capi.VR_EINVAL
    r = _capi.vr_rect(0, 0, 4, 4)
    assert L.vr_draw_probe(None, cam, 1, C.byref(opt), xyz, 100, C.byref(r), None, None, 7, None) == _capi.VR_EINVAL
    assert L.vr_draw_probe(None, cam, 1, C.byref(opt), xyz, 100, None, buf, None, 7, None) == _capi.VR_EINVAL
    # a null tree
    assert L.vr_draw_probe(None, cam, 1, C.byref(opt), xyz, 100, None, buf, None, 0, None) == _capi.VR_EINVAL
    assert L.vr_draw_probe(None, cam, 0, C.byref(opt), xyz, 100, None, buf, None, 0, None) == _capi.VR_OK
