"""`-m "not gpu"`: the C-ABI library loads here and exports every symbol the header declares;
without a device every entry point fails loudly (no CPU fallback)."""
import ctypes as C
import os
import re

import pytest

from conftest import ROOT


def header_functions():
    txt = open(os.path.join(ROOT, "include", "volrend_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(vr_[a-z_0-9]+)\s*\(", txt)))


def test_header_and_binding_agree(built):
    from volrend_b200 import _capi
    assert header_functions() == sorted(_capi.SYMBOLS)


def test_library_exports_every_declared_symbol(built):
    from volrend_b200 import LIB_PATH
    h = C.CDLL(LIB_PATH)
    for name in header_functions():
        assert getattr(h, name) is not None, name


def test_version_and_kernel_variants(built):
    from volrend_b200 import lib
    l = lib()
    assert b"sm_90a" in l.vr_version()
    assert l.vr_set_variant(9) != 0 and b"variant" in l.vr_last_error()
    for v in (8, 1, 2, 3, 4, 5, 6, 19, 3 + 16 * 64, 3 + 16 * 65):   # no kernel behind these ids
        assert l.vr_set_variant(v) != 0, v
    assert l.vr_set_variant(300) != 0
    assert l.vr_set_variant(-1) != 0
    assert l.vr_set_variant(0) == 0 and l.vr_get_variant() == 0
    # product kernels: shading queue (7) for >= 4 basis functions, inline shading (3 + 16*193) for every basis size
    for kbd in (4, 9, 16, 25):
        assert l.vr_variant_supported(kbd, 7) == 1 and l.vr_variant_supported(kbd, 3 + 16 * 193) == 1
    for kbd in (-1, 1):
        assert l.vr_variant_supported(kbd, 7) == 0 and l.vr_variant_supported(kbd, 3 + 16 * 193) == 1
    assert l.vr_variant_supported(16, 0) == 1 and l.vr_variant_supported(5, 0) == 0
    assert l.vr_set_variant(7) == 0 and l.vr_get_variant() == 7 and l.vr_set_variant(0) == 0


def test_default_options_match_reference_defaults(built):
    # include/volrend/render_options.hpp:14-32
    from volrend_b200 import _capi, lib
    o = _capi.vr_options()
    lib().vr_default_options(C.byref(o))
    assert abs(o.step_size - 1e-4) < 1e-10 and abs(o.sigma_thresh - 1e-2) < 1e-9 and abs(o.stop_thresh - 1e-2) < 1e-9
    assert o.background_brightness == 1.0
    assert list(o.render_bbox) == [0, 0, 0, 1, 1, 1]
    assert list(o.basis_minmax) == [0, 24]


def test_no_cpu_fallback(built):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from volrend_b200 import _capi, lib
    d = _capi.vr_tree_desc()
    h = C.c_void_p()
    rc = lib().vr_tree_create(C.byref(d), C.byref(h))
    assert rc == _capi.VR_ENODEVICE
    assert b"no CPU fallback" in lib().vr_last_error()
    # the multi-GPU entry points fail the same way, and reject nonsense before touching a device
    mg = C.c_void_p()
    devs = (C.c_int * 2)(0, 1)
    assert lib().vr_mg_create(C.byref(d), devs, 2, C.byref(mg)) == _capi.VR_ENODEVICE and not mg.value
    assert b"no CPU fallback" in lib().vr_mg_last_error(None)
    assert lib().vr_mg_create(C.byref(d), devs, 0, C.byref(mg)) == _capi.VR_EINVAL
    assert lib().vr_mg_device_count(None) == 0 and lib().vr_mg_device(None, 0) == -1 and not lib().vr_mg_tree(None, 0)
    ms = C.c_float(0)
    assert lib().vr_mg_render(None, None, 0, None, 0, 8, 0, None, None, C.byref(ms)) == _capi.VR_EINVAL
    lib().vr_mg_destroy(None)                       # no-op
    assert lib().vr_band_rows(1080, 8, 8, 0) == 136 and lib().vr_band_rows(1080, 8, 8, 7) == 128
    assert sum(lib().vr_band_rows(92, 8, 3, p) for p in range(3)) == 92


def test_product_never_imports_oracle():
    """The oracle is test infrastructure: nothing under volrend_b200/ may reference it."""
    pkg = os.path.join(ROOT, "volrend_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".hpp", ".cpp")):
                txt = open(os.path.join(dp, f), errors="replace").read()
                assert "march_oracle" not in txt and "liboracle" not in txt and "from oracle" not in txt \
                    and "import oracle" not in txt, os.path.join(dp, f)
