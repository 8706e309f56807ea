"""
CPU tests of the build rule of rt_rebuild_bvh through its numpy model (tests/lbvh_model.py): the model's trees are accepted by
rt_upload_scene's record layout (rt_bvh_layout.h build_layout) and number their records the same way, stay within 62 levels,
hold one triangle per leaf in key order, and trace exactly like the SAH tree: the oracle gives bit-identical t and occlusion for
camera and random rays with either tree, and the same primitive wherever t is not tied.  Cases: the shipped scenes, deformed
versions of them, and adversarial soups (equal key points, a chain of Morton bits, NaN and inf coordinates, n = 1, 2, 3, a
planar scene).
"""
import ctypes as C

import numpy as np
import pytest

from oracle.orcbind import Oracle
from raytracing_b200 import capi, hostapi
from raytracing_b200.camera import default_camera
from raytracing_b200.layouts import NODE_DT, RAY_DT, TRIANGLE_DT
from tests import lbvh_model
from tests.helpers import bits, scene
from tests.refit_model import deform, records_match_nodes, refit
from tests.test_bvh_layout import build as layout_build
from tests.test_bvh_layout import lib  # noqa: F401  (the build_layout fixture)

SCENES = ["CornellBox", "ShaderBalls", "CornellBox_Dragon"]
KINDS = ["noise", "rigid", "scale"]


def soup_from_points(c, eps=np.float32(1e-3), seed=0):
    """Small triangles around the points c (n, 3)."""
    rng = np.random.default_rng(seed)
    n = len(c)
    t = np.zeros(n, dtype=TRIANGLE_DT)
    c = np.asarray(c, np.float32)
    d1 = (rng.standard_normal((n, 3)) * eps).astype(np.float32)
    d2 = (rng.standard_normal((n, 3)) * eps).astype(np.float32)
    for v, p in (("v1", c), ("v2", c + d1), ("v3", c + d2)):
        t[v]["position"][:, :3] = p
        t[v]["normal"][:, :3] = (0, 0, 1)
    return t


def equal_key_points(n=400, seed=1):
    """Every key point is exactly 0: p3 = -(p1 + p2) as floats."""
    rng = np.random.default_rng(seed)
    t = np.zeros(n, dtype=TRIANGLE_DT)
    p1 = rng.uniform(-1, 1, (n, 3)).astype(np.float32)
    p2 = rng.uniform(-1, 1, (n, 3)).astype(np.float32)
    for v, p in (("v1", p1), ("v2", p2), ("v3", -(p1 + p2))):
        t[v]["position"][:, :3] = p
        t[v]["normal"][:, :3] = (0, 0, 1)
    return t


def morton_chain(n=1 << 12, seed=2):
    """Key points at 2^-k of the extent on one axis at a time, so that consecutive sorted codes differ in one Morton bit after
    another, and the triangles at code 0 placed at ids 0, 1, 2, 4, 8, ... so that their ids chain too."""
    pts = np.full((n, 3), 1.0, np.float32)                      # everything else at the top corner
    chain_ids = [0] + [1 << k for k in range(int(np.log2(n - 1)) + 1) if (1 << k) < n]
    pts[chain_ids] = 0.0
    others = [i for i in range(n) if i not in set(chain_ids)]
    j = 0
    for k in range(1, 11):
        for a in range(3):
            p = np.zeros(3, np.float32); p[a] = np.float32(2.0 ** -k)
            pts[others[j]] = p; j += 1
    return soup_from_points(pts, eps=np.float32(0.0), seed=seed)


def non_finite(n=300, seed=3):
    t = soup_from_points(np.random.default_rng(seed).uniform(-3, 3, (n, 3)), eps=np.float32(0.2), seed=seed)
    bad = [(5, "v1", 0, np.nan), (17, "v2", 1, np.inf), (40, "v3", 2, -np.inf), (41, "v1", 1, np.nan), (41, "v2", 1, np.nan),
           (99, "v1", 0, np.inf), (99, "v2", 0, np.inf), (99, "v3", 0, np.inf)]
    for i, v, a, x in bad:
        t[v]["position"][i, a] = x
    return t


def planar(n=500, seed=4):
    c = np.random.default_rng(seed).uniform(-2, 2, (n, 3)).astype(np.float32)
    t = soup_from_points(c, eps=np.float32(0.05), seed=seed)
    for v in ("v1", "v2", "v3"):
        t[v]["position"][:, 2] = 0.5
    return t


def tiny(n, seed=5):
    return soup_from_points(np.random.default_rng(seed).uniform(-1, 1, (n, 3)), eps=np.float32(0.5), seed=seed)


SOUPS = {"equal_key_points": equal_key_points, "morton_chain": morton_chain, "non_finite": non_finite, "planar": planar,
         "n1": lambda: tiny(1), "n2": lambda: tiny(2), "n3": lambda: tiny(3)}


def finite_copy(t):
    t = t.copy()
    for v in ("v1", "v2", "v3"):
        p = t[v]["position"]
        p[~np.isfinite(p)] = 0.0
    return t


def case(which):
    """-> (scene dict with the SAH tree over the case's triangles, in leaf order)."""
    if which in SOUPS:
        raw = SOUPS[which]()
        tris, nodes, _ = hostapi.build_bvh(finite_copy(raw))      # an SAH tree over the same triangles ...
        # ... the builder reorders: carry the non-finite coordinates along by matching each reordered triangle to its source
        src = {bytes(r): i for i, r in enumerate(finite_copy(raw).view(np.uint8).reshape(len(raw), -1))}
        perm = np.array([src[bytes(r)] for r in tris.view(np.uint8).reshape(len(tris), -1)])
        tris = raw[perm]
        nodes = refit(nodes, tris)
        return {**scene("CornellBox"), "triangles": tris, "nodes": nodes, "emissive": np.zeros(0, "<u4")}
    name, _, kind = which.partition(":")
    sc = scene(name)
    if kind:
        t = deform(sc["triangles"], kind, seed=13)
        sc = {**sc, "triangles": t, "nodes": refit(sc["nodes"], t)}
    return sc


CASES = SCENES + ["%s:%s" % (s, k) for s in SCENES for k in KINDS] + list(SOUPS)


@pytest.mark.parametrize("which", CASES)
def test_model_tree_is_a_valid_upload_tree(lib, which):  # noqa: F811
    """build_layout accepts the model's tree; its records hold the children's boxes, its record numbering is the model's, its
    root reference and top prefix are the rule's; one triangle per leaf, leaves in key order, every .w and padding word 0."""
    sc = case(which)
    tris = sc["triangles"]
    n = len(tris)
    nodes, info = lbvh_model.build(tris)
    assert len(nodes) == 2 * n - 1
    rc, err, wn, wt, root, depth, top_n = layout_build(lib, nodes, tris)
    assert rc == 0, err
    assert depth == info["max_depth"] <= 62
    assert top_n == min(n - 1, 1024) == info["top_n"]
    assert root == (~0 if n == 1 else 0)
    assert len(wn) == max(n - 1, 1)
    assert (wt[:, 9].view("<u4") == 1).all()                     # end-of-leaf flags
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
    leaf = (nodes["num_primitives_axis"] >> 16) > 0
    assert (nodes["num_primitives_axis"][leaf] == 1 << 16).all() and leaf.sum() == n
    ids = (info["keys"] & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    assert np.array_equal(nodes["offset"][leaf], ids)            # preorder visits the leaves in key order
    assert not nodes["bounds_min"][:, 3].view("<u4").any() and not nodes["bounds_max"][:, 3].view("<u4").any()
    assert not nodes["padding"].any()


def test_adversarial_depths():
    """The chained soup reaches deep into the key bits; equal key points split by id alone (axis 0 everywhere)."""
    _, info = lbvh_model.build(morton_chain())
    assert info["max_depth"] >= 35
    nodes, info = lbvh_model.build(equal_key_points())
    assert not (info["keys"] >> np.uint64(32)).any()
    assert (nodes["num_primitives_axis"] == 0).sum() == len(nodes) // 2


def test_key_rule_on_crafted_points():
    """Quantization: the box is that of the finite key points; non-finite components give 0; an axis without spread gives 0."""
    s = np.array([[0, 5, np.nan], [3, 5, np.inf], [1.5, 5, 1.0], [np.inf, 5, 2.0]], np.float32)
    q = lbvh_model.quantize(s)
    assert q[:, 0].tolist() == [0, 1023, 512, 0]
    assert q[:, 1].tolist() == [0, 0, 0, 0]
    assert q[:, 2].tolist() == [0, 0, 0, 1023]
    code = lbvh_model.morton(np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1], [1023, 1023, 1023]], np.uint32))
    assert code.tolist() == [4, 2, 1, (1 << 30) - 1]


def rays_for(sc, n_random=3000, seed=11):
    """Camera rays and random rays from inside the finite box of the geometry."""
    cam = default_camera(48, 32)
    rays = [Oracle(sc).generate_rays(cam, 48, 32)]
    p = np.concatenate([sc["triangles"][v]["position"][:, :3] for v in ("v1", "v2", "v3")])
    p = p[np.isfinite(p).all(1)]
    lo, hi = p.min(0), p.max(0)
    rng = np.random.default_rng(seed)
    r = np.zeros(n_random, dtype=RAY_DT)
    r["origin"][:, :3] = rng.uniform(lo, hi, (n_random, 3)).astype(np.float32)
    d = rng.standard_normal((n_random, 3)).astype(np.float32)
    r["direction"][:, :3] = d / np.linalg.norm(d, axis=1, keepdims=True).astype(np.float32)
    r["direction"][:, 3] = rays[0]["direction"][0, 3]
    rays.append(r)
    return np.concatenate(rays)


def t_alone(sc, i, ray):
    """t of ray against triangle i of sc alone (a single-leaf tree)."""
    t = sc["triangles"][i: i + 1]
    nodes = np.zeros(1, dtype=NODE_DT); nodes[0]["num_primitives_axis"] = 1 << 16
    hit, _ = Oracle({**sc, "triangles": t, "nodes": refit(nodes, t)}).trace(ray[None])
    return hit["t"][0] if hit["primitive_id"][0] == 0 else None


@pytest.mark.parametrize("which", CASES)
def test_oracle_traces_the_model_tree_like_the_sah_tree(which):
    """Closest hit: bit-identical t; the same primitive unless the other tree's primitive hits the ray at the same t.  Any hit:
    identical occlusion flags.  A triangle with a non-finite coordinate can report a hit at t = NaN, after which the traversal
    keeps whatever it meets in its own order, with any tree: rays whose closest hit is such a triangle in either tree are left
    out (in the non_finite soup only)."""
    sc = case(which)
    nodes, _ = lbvh_model.build(sc["triangles"])
    lb = {**sc, "nodes": nodes}
    rays = rays_for(sc)
    a, _ = Oracle(sc).trace(rays)
    b, _ = Oracle(lb).trace(rays)
    p = np.stack([sc["triangles"][v]["position"][:, :3] for v in ("v1", "v2", "v3")], 1)
    bad = np.flatnonzero(~np.isfinite(p).all((1, 2)))
    keep = ~(np.isin(a["primitive_id"], bad) | np.isin(b["primitive_id"], bad))
    assert keep.all() or which == "non_finite"
    assert keep.mean() > 0.9
    rays, a, b = rays[keep], a[keep], b[keep]
    assert np.array_equal(bits(a["t"]), bits(b["t"]))
    diff = np.flatnonzero(a["primitive_id"] != b["primitive_id"])
    assert diff.size <= max(10, rays.size // 100), diff.size
    for k in diff:
        ta, tb = t_alone(sc, int(a["primitive_id"][k]), rays[k]), t_alone(sc, int(b["primitive_id"][k]), rays[k])
        assert ta is not None and tb is not None and bits(np.float32(ta)) == bits(np.float32(tb)) == bits(a["t"][k]), k
    fa, _ = Oracle(sc).trace(rays, any_hit=True)
    fb, _ = Oracle(lb).trace(rays, any_hit=True)
    assert np.array_equal(fa, fb)


def test_rebuild_rejects_a_null_context():
    L = capi.load_library()
    n = C.c_uint64()
    assert L.rt_rebuild_bvh(None, C.byref(n)) == -1
