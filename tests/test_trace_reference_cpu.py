"""
CPU tests of the traversal against the brute force of tests/trace_reference.py, which ignores the BVH: the oracle's closest-hit and
any-hit traversal (Oracle.trace, pinned to the reference's kernels by test_oracle_vs_ref.py) meets its rules on the designed scenes
of tests/trace_cases.py and samples of the shipped ones, with every tree the kernels trace: the host SAH tree (or the caller's
chain), and the LBVH and PLOC models' trees.  Rays: camera rays, rays that start on box planes with direction components of
exactly +0 and -0, and shadow rays that end exactly on their hit (t == t_max).  Also: the float32 restatement finds the float64
intersection on every clean ray, and build_layout accepts the depth-64 chain and refuses the depth-65 one.
"""
import numpy as np
import pytest

from oracle.orcbind import Oracle
from tests import lbvh_model, ploc_model
from tests import trace_cases as T
from tests import trace_reference as R
from tests.helpers import bits
from tests.test_bvh_layout import build as layout_build
from tests.test_bvh_layout import lib  # noqa: F401  (the build_layout fixture)

TREES = ("given", "lbvh", "ploc")
_cases = {}


def case(name):
    if name not in _cases:
        _cases[name] = T.case(name)
    return _cases[name]


def tree(sc, which):
    if which == "given":
        return sc["nodes"]
    return (lbvh_model if which == "lbvh" else ploc_model).build(sc["triangles"])[0]


def rays_of(name, sc, cam):
    """-> (camera rays, rays that start on box planes)."""
    rays = Oracle(sc).generate_rays(cam, T.W, T.H)
    if name in T.SHIPPED:
        rays = T.shipped_rays(rays)
    return rays, T.designed_rays(sc, 500 if name in T.SHIPPED else 1500)


# A ray with a zero direction component that starts on a box plane meets 0 * inf = NaN in the slab test, which fminf / fmaxf drop,
# so that box is judged on the other axes alone (the reference's rule, trace_bvh.cl:75-97): such a ray can miss a hit on the
# plane.  Measured on these rays: up to 170 of 1 500 (walls), 63 of 500 (CornellBox).
PLANE_RAY_MISSES = 0.15


@pytest.mark.parametrize("which", TREES)
@pytest.mark.parametrize("name", T.DESIGNED + T.SHIPPED)
def test_oracle_meets_the_brute_force(name, which):
    """Closest hit and occlusion, and occlusion again with t_max at the closest hit's t (inclusive: still occluded) and just
    below it."""
    sc, cam = case(name)
    if which == "given" and name == "lbvh_deep":
        pytest.skip("uploaded with the LBVH model's tree")
    nodes = tree(sc, which)
    tris = sc["triangles"]
    orc = Oracle({**sc, "nodes": nodes})
    cam_rays, plane_rays = rays_of(name, sc, cam)
    rays = np.concatenate([cam_rays, plane_rays])
    ref = R.closest(tris, rays)
    cls = R.classify(tris, rays, nodes, ref)[0]
    hits, _ = orc.trace(rays)
    for part, allow in ((slice(0, len(cam_rays)), 0.0 if name in T.SHIPPED else 0.01), (slice(len(cam_rays), None), PLANE_RAY_MISSES)):
        rep = R.verdict(tris, rays[part], nodes, hits["primitive_id"][part], hits["bc"][part], hits["t"][part], (name, which),
                        ref=R.select(ref, part), cls=cls[part], allow_box=allow)
        print(name, which, "camera" if part.start == 0 else "plane", rep)
    box = cls == 3
    occ, _ = orc.trace(rays, any_hit=True)
    assert ((occ == 0) == (ref.n_accepted > 0))[~box].all(), (name, which)
    hit = np.flatnonzero(ref.prim != 0xFFFFFFFF)
    for t_max, blocked in ((ref.t[hit], True), (np.nextafter(ref.t[hit], np.float32(-1)), False)):
        shadow = rays[hit].copy()
        shadow["direction"][:, 3] = t_max
        want = R.any_hit(tris, shadow)
        assert (want == blocked).all()
        occ, _ = orc.trace(shadow, any_hit=True)
        assert ((occ == 0) == want)[~box[hit]].all(), (name, which)


@pytest.mark.parametrize("name", ["chain64", "CornellBox", "ShaderBalls"])
def test_restatement_is_an_intersection_test(name):
    """On every clean ray the float32 restatement's closest triangle is the float64 nearest one, at a t within 2^-16."""
    sc, cam = case(name)
    rays = np.concatenate(rays_of(name, sc, cam))
    ref = R.closest(sc["triangles"], rays)
    cls, p64 = R.classify(sc["triangles"], rays, sc["nodes"], ref)
    clean = cls == 0
    assert clean.sum() > 300, (name, np.bincount(cls, minlength=4))
    assert np.array_equal(ref.prim[clean], p64[clean]), name
    assert (ref.prim[clean] != 0xFFFFFFFF).any()


def test_prefilter_changes_nothing():
    sc, cam = case("ShaderBalls")
    rays = T.shipped_rays(Oracle(sc).generate_rays(cam, T.W, T.H), 300)
    a, b = R.closest(sc["triangles"], rays, prefilter=True), R.closest(sc["triangles"], rays, prefilter=False)
    assert np.array_equal(a.prim, b.prim) and np.array_equal(bits(a.t), bits(b.t)) and np.array_equal(a.n_accepted, b.n_accepted)


@pytest.mark.parametrize("name", ["chain64", "ploc64", "lbvh_deep"])
def test_a_ray_defers_depth_minus_one_entries(lib, name):  # noqa: F811
    """The chain (the caller's tree), the PLOC model's tree of the 1.5^k chain and the LBVH model's tree of the deep soup reach
    64, 64 and 43 levels; build_layout accepts them; a camera ray holds depth - 1 deferred entries under the literal rule, and the
    oracle visits exactly the nodes the stack model visits on it.  Under trace_fast's rule (a far child is deferred only when its
    box is hit too) a camera ray also holds 63 on the two depth-64 trees, and 41 on the LBVH."""
    sc, cam = case(name)
    nodes = tree(sc, {"chain64": "given", "ploc64": "ploc", "lbvh_deep": "lbvh"}[name])
    rc, err, _, _, _, dep, _ = layout_build(lib, nodes, sc["triangles"])
    assert rc == 0, err
    assert dep == {"chain64": 64, "ploc64": 64, "lbvh_deep": 43}[name]
    rays = Oracle(sc).generate_rays(cam, T.W, T.H)
    deferred = [T.deferred_entries(nodes, rays["origin"][k, :3], rays["direction"][k, :3]) for k in range(len(rays))]
    k = int(np.argmax([d for d, _ in deferred]))
    assert deferred[k][0] == dep - 1
    _, counters = Oracle({**sc, "nodes": nodes}).trace(rays[k: k + 1])
    assert counters[0] == deferred[k][1]
    fast = max(T.deferred_entries(nodes, rays["origin"][i, :3], rays["direction"][i, :3], fast=True)[0] for i in range(len(rays)))
    assert fast == {"chain64": 63, "ploc64": 63, "lbvh_deep": 41}[name]


@pytest.mark.parametrize("name", sorted(T.REACH))
def test_designed_cases_reach_their_edges(name):
    """The bounce-0 rays reach what each case is built for (trace_cases.reached / REACH)."""
    sc, cam = case(name)
    rays = Oracle(sc).generate_rays(cam, T.W, T.H)
    got = T.reached(name, sc, rays, R.closest(sc["triangles"], rays))
    print(name, got)
    assert all(got[k] >= v for k, v in T.REACH[name].items()), (name, got)
    assert name != "walls" or got["t_zero"] == 0


def test_depth_65_is_refused(lib):  # noqa: F811
    sc = T.chain(64)
    rc, err, *_ = layout_build(lib, sc["nodes"], sc["triangles"])
    assert rc == 1 and "deeper" in err
    _, info = ploc_model.build(T.geometric_chain(65)["triangles"])
    assert info["max_depth"] == 65 and info["depth_error"]
