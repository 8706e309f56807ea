"""
CPU tests of the build rule of rt_rebuild_bvh_ploc through its numpy model (tests/ploc_model.py): the model's trees are accepted by
rt_upload_scene's record layout (rt_bvh_layout.h build_layout) and number their records the same way, every iteration merges a
pair, the depth guard fires on a geometric chain, the oracle traces the model's trees exactly like the SAH tree, and the trees
cost about what the host SAH builder's cost.  Cases: those of test_lbvh_cpu (shipped scenes, deformed versions, adversarial
soups) and duplicate triangles, whose distances all tie.
"""
import ctypes as C

import numpy as np
import pytest

from oracle.orcbind import Oracle
from raytracing_b200 import capi
from raytracing_b200.layouts import TRIANGLE_DT
from tests import lbvh_model, ploc_model
from tests.helpers import bits, scene
from tests.refit_model import records_match_nodes
from tests.test_bvh_layout import build as layout_build
from tests.test_bvh_layout import lib  # noqa: F401  (the build_layout fixture)
from tests.test_lbvh_cpu import CASES as LBVH_CASES
from tests.test_lbvh_cpu import case as lbvh_case
from tests.test_lbvh_cpu import rays_for, t_alone


def duplicates(n=300, distinct=7, seed=6):
    """n triangles that are copies of `distinct` ones: every distance within a group of copies ties."""
    rng = np.random.default_rng(seed)
    base = np.zeros(distinct, dtype=TRIANGLE_DT)
    for v in ("v1", "v2", "v3"):
        base[v]["position"][:, :3] = rng.uniform(-1, 1, (distinct, 3)).astype(np.float32)
        base[v]["normal"][:, :3] = (0, 0, 1)
    return base[rng.integers(0, distinct, n)]


def geometric_chain(n=90):
    """Triangles whose x extent grows as 1.5^k: each iteration merges the chain with the next triangle (depth n)."""
    t = np.zeros(n, dtype=TRIANGLE_DT)
    x = np.float32(1.5) ** np.arange(n, dtype=np.float32)
    for v, (px, py) in (("v1", (0, 0)), ("v2", (1, 0)), ("v3", (1, 1))):
        t[v]["position"][:, 0] = x * np.float32(px)
        t[v]["position"][:, 1] = np.float32(py)
        t[v]["normal"][:, :3] = (0, 0, 1)
    return t


def soup_case(name, make):
    """The scene dict of test_lbvh_cpu.case for the soup make(): an SAH tree over its triangles."""
    from tests.test_lbvh_cpu import SOUPS
    SOUPS[name] = make
    try:
        return lbvh_case(name)
    finally:
        del SOUPS[name]


def case(which):
    return soup_case("duplicates", duplicates) if which == "duplicates" else lbvh_case(which)


CASES = LBVH_CASES + ["duplicates"]


@pytest.mark.parametrize("which", CASES)
def test_model_tree_is_a_valid_upload_tree(lib, which):  # noqa: F811
    """build_layout accepts the model's tree; its records hold the children's boxes, its record numbering is the model's, its
    root reference and top prefix are the rule's; one triangle per leaf, every triangle once, every .w and padding word 0."""
    sc = case(which)
    tris = sc["triangles"]
    n = len(tris)
    nodes, info = ploc_model.build(tris)
    assert len(nodes) == 2 * n - 1 and not info["depth_error"]
    rc, err, wn, wt, root, depth, top_n = layout_build(lib, nodes, tris)
    assert rc == 0, err
    assert depth == info["max_depth"] <= 64
    assert top_n == min(n - 1, 1024) == info["top_n"]
    assert root == (~0 if n == 1 else 0)
    assert len(wn) == max(n - 1, 1)
    assert (wt[:, 9].view("<u4") == 1).all()
    if n > 1:
        assert records_match_nodes(nodes, wn) == n - 1
        refs = wn[:, 12:14].copy().view("<i4")
        interior = np.flatnonzero((nodes["num_primitives_axis"] >> 16) == 0)
        rec = info["record"][interior]
        second = nodes["offset"][interior].astype(np.int64)
        for s, child in enumerate((interior + 1, second)):
            inner = (nodes["num_primitives_axis"][child] >> 16) == 0
            assert np.array_equal(refs[rec[inner], s], info["record"][child[inner]])
            assert np.array_equal(refs[rec[~inner], s], ~nodes["offset"][child[~inner]].astype(np.int32))
        assert np.array_equal(wn[:, 14].view("<u4")[rec], nodes["num_primitives_axis"][interior])
        assert info["iterations"] >= int(np.ceil(np.log2(n)))
    leaf = (nodes["num_primitives_axis"] >> 16) > 0
    assert (nodes["num_primitives_axis"][leaf] == 1 << 16).all() and leaf.sum() == n
    assert np.array_equal(np.sort(nodes["offset"][leaf]), np.arange(n))
    assert not nodes["bounds_min"][:, 3].view("<u4").any() and not nodes["bounds_max"][:, 3].view("<u4").any()
    assert not nodes["padding"].any()


def test_geometric_chain_is_too_deep():
    """The 1.5^k chain: one merge per iteration, one level per triangle; the model reports the depth error, the LBVH stays
    shallow."""
    t = geometric_chain()
    _, info = ploc_model.build(t)
    assert info["iterations"] == len(t) - 1
    assert info["max_depth"] == len(t) and info["depth_error"]
    assert lbvh_model.build(t)[1]["max_depth"] <= 20
    _, info = ploc_model.build(t[:64])
    assert info["max_depth"] == 64 and not info["depth_error"]


def test_equal_distances_pair_off_in_neighbours():
    """Distances that all tie (one triangle repeated): position i pairs with i + 1 for even i, so each iteration halves the list
    (ties to the smallest j alone would merge one pair per iteration)."""
    t = duplicates(n=64, distinct=1)
    _, info = ploc_model.build(t)
    assert info["iterations"] == 6 and info["max_depth"] == 7


@pytest.mark.parametrize("which", CASES)
def test_oracle_traces_the_model_tree_like_the_sah_tree(which):
    """As test_lbvh_cpu's test of the same name, with the PLOC model's tree."""
    sc = case(which)
    nodes, _ = ploc_model.build(sc["triangles"])
    pl = {**sc, "nodes": nodes}
    rays = rays_for(sc)
    a, _ = Oracle(sc).trace(rays)
    b, _ = Oracle(pl).trace(rays)
    p = np.stack([sc["triangles"][v]["position"][:, :3] for v in ("v1", "v2", "v3")], 1)
    bad = np.flatnonzero(~np.isfinite(p).all((1, 2)))
    keep = ~(np.isin(a["primitive_id"], bad) | np.isin(b["primitive_id"], bad))
    assert keep.all() or which == "non_finite"
    assert keep.mean() > 0.9
    rays, a, b = rays[keep], a[keep], b[keep]
    assert np.array_equal(bits(a["t"]), bits(b["t"]))
    diff = np.flatnonzero(a["primitive_id"] != b["primitive_id"])
    assert diff.size <= max(10, rays.size // 100) or which == "duplicates", diff.size
    for k in diff:
        ta, tb = t_alone(sc, int(a["primitive_id"][k]), rays[k]), t_alone(sc, int(b["primitive_id"][k]), rays[k])
        assert ta is not None and tb is not None and bits(np.float32(ta)) == bits(np.float32(tb)) == bits(a["t"][k]), k
    fa, _ = Oracle(sc).trace(rays, any_hit=True)
    fb, _ = Oracle(pl).trace(rays, any_hit=True)
    assert np.array_equal(fa, fb)


@pytest.mark.parametrize("name", ["CornellBox_Dragon", "ShaderBalls"])
def test_sah_cost_is_that_of_the_host_builder(name):
    """SAH cost (C_node = C_tri = 1, areas relative to the root): at most 1.05x the host SAH tree's and below the LBVH's."""
    sc = scene(name)
    sah = ploc_model.sah_cost(sc["nodes"])
    lbvh = ploc_model.sah_cost(lbvh_model.build(sc["triangles"])[0])
    ploc = ploc_model.sah_cost(ploc_model.build(sc["triangles"])[0])
    assert ploc <= 1.05 * sah and ploc < lbvh, (sah, lbvh, ploc)


def test_rebuild_ploc_rejects_a_null_context():
    L = capi.load_library()
    n = C.c_uint64()
    assert L.rt_rebuild_bvh_ploc(None, C.byref(n)) == -1
