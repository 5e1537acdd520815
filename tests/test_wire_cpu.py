"""`-m "not gpu"`: the grid-wireframe oracle against the reference's stored gen_wireframe output, the argument checks
of vr_tree_wireframe without a device, and the Python layer's refusal of grids a mesh cannot index."""
import ctypes as C
import glob
import os

import numpy as np
import pytest

from conftest import ROOT
from oracle import wire_oracle as wo
from wire_cases import WIRE_CASES, golden_name, matches, wire_tree

GOLDEN = os.path.join(ROOT, "tests", "golden", "ref")


def test_every_case_has_a_golden():
    have = {os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "wire_*.npz"))}
    assert {golden_name(n, d) for n, d in WIRE_CASES} <= have


@pytest.mark.parametrize("name,max_depth", WIRE_CASES)
def test_oracle_matches_reference(name, max_depth):
    st = wire_tree(name)
    v = wo.wireframe(st.child, st.offset, st.invradius3, max_depth)
    rec = np.load(os.path.join(GOLDEN, golden_name(name, max_depth) + ".npz"))
    assert matches(rec, v)
    if "sample" in rec:
        assert np.array_equal(v.reshape(-1, 9)[rec["sample_idx"]].view(np.uint32), rec["sample"].view(np.uint32))


def test_vertex_order_is_twelve_distinct_edges():
    sel = wo.SEL.reshape(12, 2, 3)
    assert np.all(np.abs(sel[:, 0] - sel[:, 1]).sum(1) == 1)          # each segment runs along one axis
    assert np.all(sel[:, 1] >= sel[:, 0])                             # from its low end to its high end
    assert len({tuple(e.reshape(-1)) for e in sel}) == 12


def test_cut_semantics():
    """max_depth <= 0: the root's 8 cells; beyond the tree's depth: every leaf, each once."""
    st = wire_tree("sh4_d5")
    for d in (-5, 0):
        corner, level = wo.cells(st.child, d)
        assert corner.shape[0] == 8 and np.all(level == 1)
    corner, level = wo.cells(st.child, 100)
    assert corner.shape[0] == int((st.child == 0).sum())
    vol = (np.float64(0.5) ** level) ** 3
    assert abs(vol.sum() - 1.0) < 1e-12                               # the leaves tile the unit cube


def test_no_device_errors(built):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from volrend_b200 import _capi, lib
    n = C.c_int64(-7)
    assert lib().vr_tree_wireframe(None, 3, None, 0, C.byref(n), None) == _capi.VR_EINVAL
    fake = C.create_string_buffer(64)           # never dereferenced: the device check comes first
    assert lib().vr_tree_wireframe(C.addressof(fake), 3, None, 0, None, None) == _capi.VR_EINVAL
    assert lib().vr_tree_wireframe(C.addressof(fake), 3, None, 0, C.byref(n), None) == _capi.VR_ENODEVICE
    assert b"no CPU fallback" in lib().vr_last_error()
    assert n.value == -7


class _FakeTree:
    def __init__(self, n_verts):
        self.n_verts = n_verts
        self.calls = 0

    def is_cuda_loaded(self):
        return True

    def wireframe_vertex_count(self, max_depth):
        self.calls += 1
        return self.n_verts


def test_grid_mesh_refuses_int32_vertex_counts():
    from volrend_b200 import VolumeRenderer
    vr = VolumeRenderer()
    vr._tree = _FakeTree(2 ** 31)
    assert vr._grid_mesh() is None                  # show_grid off: nothing asked of the tree
    assert vr._tree.calls == 0
    vr.options.show_grid = True
    with pytest.raises(ValueError, match="vertices"):
        vr._grid_mesh()
    vr.clear()
    assert vr._grid_mesh() is None                  # no tree, no grid
