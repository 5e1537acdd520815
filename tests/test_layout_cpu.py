"""CPU: the layout transforms of tests/layout_cases.py describe the same tree (query oracle, march oracle), have the
shape they claim (link signs, free nodes, out-of-range links), and prune._structure accepts them and refuses the
malformed trees with the messages vr_tree_create uses."""
import numpy as np
import pytest

import edge_cases as ec
import layout_cases as lc
from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)
from oracle import query_oracle as qo
from volrend_b200 import prune

CASES = [(t, lay) for t in ec.TREES for lay in lc.LAYOUTS if not (t == "quant_mixed" and lay == "wide")]
IDS = [f"{t}-{lay}" for t, lay in CASES]
ORACLE_VIEWS = {"default": ["px", "inside"], "chain": ["deep", "face"], "aniso_ndc": ["ndc", "odd"]}


def _relaid(name, layout):
    st, npz = ec.edge_tree(name)
    return st, lc.relayout(st, layout, npz, seed=7)


def _rows(st, r, rows):
    """Rows of the relaid tree cut back to the canonical tree's columns (the wide layout's extra columns dropped)."""
    if r.st.data_dim == st.data_dim:
        return rows
    return np.concatenate([rows[:, :st.data_dim - 1], rows[:, -1:]], 1)


@pytest.mark.parametrize("name,layout", CASES, ids=IDS)
def test_every_leaf_is_found_at_its_centre(name, layout):
    st, r = _relaid(name, layout)
    slots, depth, centres = lc.leaf_centres(st)
    pts = lc.centre_points(st, centres, depth)
    rows, cube, _ = qo.query(r.st.child, r.st.data, r.st.offset, r.st.invradius3, pts)
    want = st.data.reshape(-1, st.data_dim)[slots]
    assert np.array_equal(_rows(st, r, rows).view(np.uint16), want.view(np.uint16))
    assert np.array_equal(cube, (2.0 ** depth).astype(np.float32))
    # the relaid tree's own leaves are the canonical ones through the slot map, at the same centres and depths
    s2, d2, c2 = lc.leaf_centres(r.st)
    m = r.slot_map[s2]
    assert (m >= 0).all()
    order = np.argsort(m)
    assert np.array_equal(m[order], np.sort(slots))
    ref = np.argsort(slots)
    assert np.array_equal(d2[order], depth[ref]) and np.array_equal(c2[order], centres[ref])


@pytest.mark.parametrize("name,layout", CASES, ids=IDS)
def test_march_oracle_is_layout_invariant(name, layout):
    st, r = _relaid(name, layout)
    key = "chain" if name.startswith("chain") else name if name in ORACLE_VIEWS else "default"
    for v in ORACLE_VIEWS[key]:
        fr = f"{name}.{v}.default"
        f0, u0, c0 = ec.oracle_render(fr, st)
        f1, u1, c1 = ec.oracle_render(fr, r.st)
        assert np.array_equal(f0.view(np.uint32), f1.view(np.uint32)), fr
        assert np.array_equal(u0, u1) and c0 == c1, fr


@pytest.mark.parametrize("name,layout", CASES, ids=IDS)
def test_layout_has_the_shape_it_claims(name, layout):
    st, r = _relaid(name, layout)
    cap = r.st.capacity
    tgt = lc.targets(r.st.child)
    reach = np.concatenate(lc.bfs_levels(r.st.child)) if layout != "dirty" else None
    rel = r.st.child.reshape(cap, 8)
    if layout == "dirty":
        levels, _ = prune._structure(r.st.child)
        reach = np.concatenate(levels)
        assert reach.size == st.capacity and cap == st.capacity + r.n_free + lc.N_TRAIL
        free = np.setdiff1d(np.arange(cap), reach)
        ft = tgt[free][rel[free] != 0]
        assert ((ft >= cap) | (ft <= 0)).any() and (ft < 0).any() and (ft == 0).any() and (ft > cap).any()
        inside = ft[(ft > 0) & (ft < cap)]
        assert np.isin(inside, free).any() and (st.capacity == 1 or np.isin(inside, reach).any())
        assert not r.st.child[cap - lc.N_TRAIL:].any() and not r.st.data[cap - lc.N_TRAIL:].view(np.uint16).any()
        inner = r.st.data.reshape(cap * 8, -1).view(np.uint16)[(rel != 0).reshape(-1)]
        assert st.capacity == 1 or np.isin(lc.SPECIAL_BITS, inner).all()
        assert (r.slot_map.reshape(cap, 8)[free] == -1).all()
    else:
        assert reach.size == cap
    non_root = rel[1:][rel[1:] != 0]
    if layout == "reverse":
        assert (non_root < 0).all()
    if layout == "dfs":
        assert (rel >= 0).all()
        depth = np.zeros(cap, int)
        for d, nodes in enumerate(lc.bfs_levels(r.st.child)):
            depth[nodes] = d
        if st.capacity > 2 and not name.startswith("chain"):
            assert (np.diff(depth) < 0).any()          # not level-sorted
    if layout in ("shuffle", "dirty") and st.capacity > 8:
        assert (non_root < 0).any() and (non_root > 0).any()
    if layout == "wide":
        assert r.st.data_dim == st.data_dim + lc.WIDE_EXTRA


def test_chains_reversed_are_backward_links_all_the_way():
    for levels in (22, 23):
        st = ec.varied_chain(levels)
        r = lc.relayout(st, "reverse")
        ch = r.st.child.reshape(levels, 8)
        links = ch[1:][ch[1:] != 0]
        assert links.size == levels - 2 and (links < 0).all()


@pytest.mark.parametrize("layout", lc.LAYOUTS)
def test_prune_structure_accepts_every_layout(layout):
    st = ec.edge_tree("mixed_sh9")[0]
    r = lc.relayout(st, layout, seed=3)
    lv0, _ = prune._structure(st.child)
    lv1, t1 = prune._structure(r.st.child)
    assert [len(x) for x in lv0] == [len(x) for x in lv1]
    m = r.slot_map
    inner = t1 >= 0
    # a link of the relaid tree goes to the node that holds the canonical target's slots
    canon_t = lc.targets(st.child).reshape(-1)[m[inner]]
    first = m.reshape(-1, 8)[:, 0]                     # canonical slot of each new node's octant 0
    node_of = np.full(st.capacity, -1, np.int64)
    node_of[first[first >= 0] // 8] = np.flatnonzero(first >= 0)
    assert np.array_equal(node_of[canon_t], t1[inner])


@pytest.mark.parametrize("base", ["mixed_sh9", "mixed_rgba"])
def test_prune_structure_refuses_malformed_trees(base):
    st = ec.edge_tree(base)[0]
    cases = lc.malformed(st)
    assert len(cases) == 7
    for name, (bad, msg) in cases.items():
        with pytest.raises(ValueError, match=msg):
            prune._structure(bad.child)
    prune._structure(lc.relayout(st, "dirty", seed=5).st.child)    # the same defects in free nodes: accepted


def test_quantised_arrays_follow_the_nodes():
    st, npz = ec.edge_tree("quant_mixed")
    r = lc.relayout(st, "shuffle", npz, seed=2)
    from volrend_b200 import N3Tree
    host = N3Tree(gpu_decode=False)
    host.load_npz(r.npz)
    assert np.array_equal(host.data_.view(np.uint16), r.st.data.view(np.uint16))
