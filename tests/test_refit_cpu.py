"""
CPU tests of the refit rule of rt_update_triangles: the numpy model (tests/refit_model.py) against the host SAH builder's boxes
on the shipped scenes and on generated triangle soups, its comparison rule on crafted cases (signed zeros, NaN in either
operand position, a single-leaf tree), and the null-context checks of the three new entry points.
"""
import ctypes as C

import numpy as np
import pytest

from raytracing_b200 import capi, hostapi
from raytracing_b200.layouts import NODE_DT, TRIANGLE_DT
from tests.helpers import scene
from tests.refit_model import FLT_MAX, deform, levels, refit, vmax, vmin

SCENES = ["CornellBox", "ShaderBalls", "CornellBox_Dragon"]


def boxes(nodes):
    return np.concatenate([nodes["bounds_min"][:, :3], nodes["bounds_max"][:, :3]], axis=1)


def soup(n, seed):
    rng = np.random.default_rng(seed)
    t = np.zeros(n, dtype=TRIANGLE_DT)
    c = rng.uniform(-5, 5, (n, 3)).astype(np.float32)
    for v in ("v1", "v2", "v3"):
        t[v]["position"][:, :3] = c + rng.normal(0, 0.3, (n, 3)).astype(np.float32)
        t[v]["normal"][:, :3] = (0, 0, 1)
    return t


@pytest.mark.parametrize("name", SCENES)
def test_model_reproduces_shipped_scene_boxes(name):
    """With unchanged positions the refit gives the builder's boxes as float values (== : the sign of a zero may differ)."""
    sc = scene(name)
    got = refit(sc["nodes"], sc["triangles"])
    reach = np.concatenate(levels(sc["nodes"]))
    assert reach.size == len(sc["nodes"])
    assert (boxes(got) == boxes(sc["nodes"])).all()
    for f in ("offset", "num_primitives_axis", "padding"):
        assert np.array_equal(got[f], sc["nodes"][f])
    assert np.array_equal(got["bounds_min"][:, 3].view("<u4"), sc["nodes"]["bounds_min"][:, 3].view("<u4"))


@pytest.mark.parametrize("n,seed", [(1, 3), (2, 4), (37, 5), (4000, 6)])
def test_model_reproduces_host_builder_on_soups(n, seed):
    tris, nodes, _ = hostapi.build_bvh(soup(n, seed))
    assert (boxes(refit(nodes, tris)) == boxes(nodes)).all()
    # and a deformed soup refits to boxes that contain every triangle of each leaf
    moved = deform(tris, "noise", seed=seed)
    new = refit(nodes, moved)
    count = nodes["num_primitives_axis"] >> 16
    for leaf in np.flatnonzero(count > 0):
        for v in ("v1", "v2", "v3"):
            p = moved[v]["position"][nodes["offset"][leaf]: nodes["offset"][leaf] + count[leaf], :3]
            assert (p >= new["bounds_min"][leaf, :3]).all() and (p <= new["bounds_max"][leaf, :3]).all()


def test_comparison_rule_signed_zero_and_nan():
    """min(a, b) = (b < a) ? b : a: equal zeros keep the first operand, a NaN second operand never wins, a NaN first operand
    always stays."""
    z, nz, nan = np.float32(0.0), np.float32(-0.0), np.float32(np.nan)
    assert np.signbit(vmin(nz, z)) and not np.signbit(vmin(z, nz))
    assert np.signbit(vmax(nz, z)) and not np.signbit(vmax(z, nz))
    assert vmin(np.float32(1), nan) == 1 and vmax(np.float32(1), nan) == 1
    assert np.isnan(vmin(nan, np.float32(1))) and np.isnan(vmax(nan, np.float32(1)))


def two_leaf_tree(tris):
    nodes = np.zeros(3, dtype=NODE_DT)
    nodes[0]["offset"] = 2; nodes[0]["num_primitives_axis"] = 0          # interior, split axis 0
    nodes[1]["offset"] = 0; nodes[1]["num_primitives_axis"] = 1 << 16
    nodes[2]["offset"] = 1; nodes[2]["num_primitives_axis"] = 1 << 16
    return nodes


def tri(p1, p2, p3):
    t = np.zeros(1, dtype=TRIANGLE_DT)
    for v, p in zip(("v1", "v2", "v3"), (p1, p2, p3)):
        t[v]["position"][0, :3] = p
    return t


def test_crafted_leaves_and_parents():
    nan = np.nan
    # leaf 0: NaN in p1.x (first operand of Bounds3(p1, p2)): min(p1, p2) keeps NaN, then min(NaN, p3) keeps NaN, and the fold
    # min(FLT_MAX, NaN) keeps FLT_MAX.  leaf 1: NaN in p3.y (second operand): ignored.
    t = np.concatenate([tri((nan, 0, 0), (1, 1, 1), (2, 2, 2)), tri((-0.0, 1, 0), (0.0, 2, 0), (1, nan, 0))])
    nodes = refit(two_leaf_tree(t), t)
    assert nodes["bounds_min"][1, 0] == FLT_MAX and nodes["bounds_max"][1, 0] == -FLT_MAX
    assert nodes["bounds_min"][1, 1] == 0 and nodes["bounds_max"][1, 1] == 2
    assert np.signbit(nodes["bounds_min"][2, 0]) and not np.signbit(nodes["bounds_max"][2, 0])   # -0 first, +0 second
    assert nodes["bounds_min"][2, 1] == 1 and nodes["bounds_max"][2, 1] == 2
    # root = Union(first, second): x min = min(FLT_MAX, -0) = -0, x max = max(-FLT_MAX, 1) = 1 (the first child's x is empty)
    assert np.signbit(nodes["bounds_min"][0, 0]) and nodes["bounds_max"][0, 0] == 1
    assert nodes["bounds_min"][0, 1] == 0 and nodes["bounds_max"][0, 1] == 2


def test_single_leaf_tree():
    t = np.concatenate([tri((0, 0, 0), (1, 0, 0), (0, 1, 0)), tri((-1, 0, 3), (0, -2, 0), (0, 1, 1))])
    nodes = np.zeros(1, dtype=NODE_DT)
    nodes[0]["num_primitives_axis"] = 2 << 16
    got = refit(nodes, t)
    assert np.array_equal(got["bounds_min"][0, :3], [-1, -2, 0]) and np.array_equal(got["bounds_max"][0, :3], [1, 1, 3])


def test_entry_points_reject_a_null_context():
    L = capi.load_library()
    t = np.zeros(1, dtype=TRIANGLE_DT)
    assert L.rt_update_triangles(None, t.ctypes.data, 1) == -1
    assert L.rt_update_triangles_device(None, None, 1) == -1
    n = C.c_uint64()
    assert L.rt_read_bvh(None, None, None, C.byref(n)) == -1
