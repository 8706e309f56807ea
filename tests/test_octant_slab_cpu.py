"""raytracing_b200/csrc/rt_octant.h on the host: the octant-ordered interior records take the same decisions as the pairwise
slab test of trace_fast wherever their guards pass, the guards reject the inputs where the two can differ, and a walk of
CornellBox's tree through the eight tables returns the oracle's hits."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from oracle.orcbind import Oracle
from raytracing_b200.camera import default_camera
from raytracing_b200.layouts import NODE_DT, RAY_DT, TRIANGLE_DT
from tests.helpers import scene

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
FLT_MAX = np.float32(3.4028234663852886e38)


@pytest.fixture(scope="module")
def lib():
    so = os.path.join(tempfile.gettempdir(), f"liboctant_slab_host_{os.getpid()}.so")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-I" + os.path.join(REPO, "include"),
                    "-I" + os.path.join(REPO, "raytracing_b200", "csrc"), "-o", so, os.path.join(HERE, "octant_slab_host.cpp"),
                    os.path.join(HERE, "bvh_layout_host.cpp")], check=True)
    L = C.CDLL(so)
    L.octant_compare.argtypes = [C.c_uint64] + [C.c_void_p] * 7
    L.octant_walk.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_int, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                              C.c_void_p, C.c_void_p]
    L.octant_walk.restype = C.c_uint64
    L.octant_order.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
    L.bvh_layout_build.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int),
                                   C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.c_char_p, C.c_int]
    yield L
    os.remove(so)


def compare(L, recs, o, inv, t_max):
    recs, o, inv, t_max = (np.ascontiguousarray(x, "<f4") for x in (recs, o, inv, t_max))
    n = len(recs)
    ray_ok, rec_ok, differs = (np.zeros(n, np.uint8) for _ in range(3))
    L.octant_compare(n, recs.ctypes.data, o.ctypes.data, inv.ctypes.data, t_max.ctypes.data, ray_ok.ctypes.data, rec_ok.ctypes.data, differs.ctypes.data)
    return ray_ok.astype(bool), rec_ok.astype(bool), differs


def records(rng, n, flat=0.2):
    """n canonical records: two boxes with min <= max (a share of the axes flat: min == max), any split axis, child refs."""
    lo = rng.uniform(-2, 2, (n, 2, 3)).astype("<f4")
    ext = rng.uniform(0, 2, (n, 2, 3)).astype("<f4") * (rng.random((n, 2, 3)) >= flat)
    hi = (lo + ext).astype("<f4")
    rec = np.zeros((n, 16), "<f4")
    rec[:, 0:3], rec[:, 3:6], rec[:, 6:9], rec[:, 9:12] = lo[:, 0], hi[:, 0], lo[:, 1], hi[:, 1]
    rec[:, 12:15] = np.stack([rng.integers(0, 1000, n), ~rng.integers(0, 1000, n), rng.integers(0, 3, n)], 1).astype("<i4").view("<f4")
    return rec


def test_ordered_step_equals_pairwise_step_on_random_cases(lib):
    rng = np.random.default_rng(20261016)
    n = 1_200_000
    rec = records(rng, n)
    o = rng.uniform(-3, 3, (n, 3)).astype("<f4")
    d = rng.normal(size=(n, 3)).astype("<f4")
    third = n // 3                      # a third of the origins exactly on a plane of one of the boxes, a third with extreme directions
    k = rng.integers(0, 12, third); o[np.arange(third), k % 3] = rec[np.arange(third), k]
    d[third:2 * third] *= (10.0 ** rng.uniform(-44, 38, (third, 3))).astype("<f4")
    d[d == 0] = np.float32(1e-3)
    with np.errstate(over="ignore"):
        inv = (np.float32(1) / d).astype("<f4")
    t_max = np.where(rng.random(n) < 0.5, np.float32(1e30), rng.uniform(0, 5, n)).astype("<f4")
    ray_ok, rec_ok, differs = compare(lib, rec, o, inv, t_max)
    assert rec_ok.all() and ray_ok.sum() > 0.9 * n and (~ray_ok).sum() > 1000      # 1/denormal overflows: the guard sees it
    assert np.array_equal(ray_ok, np.isfinite(inv).all(1) & (inv != 0).all(1))
    assert not (differs[ray_ok] & 3).any()          # same hit decisions, child references and interval bounds
    for s in range(8):                              # every octant and every split axis took part
        sel = ray_ok & ((inv[:, 0] < 0) + 2 * (inv[:, 1] < 0) + 4 * (inv[:, 2] < 0) == s)
        assert all((sel & (rec[:, 14].view("<u4") == a)).sum() > 1000 for a in range(3))


def test_adversarial_cases(lib):
    planes = np.array([0.0, -0.0, 1.0, -1.0, 1e-45, -1e-45, 1e-38, 3e38, -3e38, 0.5, 0.50000006, 2.0], "<f4")
    invs = np.array([1.0, -1.0, 1e-38, -1e-38, 3e38, -3e38, 1e-45, -1e-45, 7.0, -0.3], "<f4")
    rng = np.random.default_rng(5)
    n = 400_000
    lo = rng.choice(planes, (n, 2, 3)); hi = rng.choice(planes, (n, 2, 3))
    lo, hi = np.minimum(lo, hi), np.maximum(lo, hi)
    rec = np.zeros((n, 16), "<f4")
    rec[:, 0:3], rec[:, 3:6], rec[:, 6:9], rec[:, 9:12] = lo[:, 0], hi[:, 0], lo[:, 1], hi[:, 1]
    rec[:, 12:15] = np.stack([np.arange(n), ~np.arange(n), rng.integers(0, 3, n)], 1).astype("<i4").view("<f4")
    o = rng.choice(planes, (n, 3)); inv = rng.choice(invs, (n, 3))
    t_max = rng.choice(np.array([0.0, 1e-30, 1.0, 1e30, np.inf], "<f4"), n)
    ray_ok, rec_ok, differs = compare(lib, rec, o, inv, t_max)
    assert ray_ok.all() and rec_ok.all()
    assert not (differs & 3).any()                  # products that overflow to +-inf or underflow to +-0 included
    # the one thing that may differ is the sign of a zero bound (rt_octant.h): a box with min = +0, max = -0 seen from o = +0
    rec = np.zeros((1, 16), "<f4"); rec[0, 0:3] = (0.0, -1, -1); rec[0, 3:6] = (-0.0, 1, 1); rec[0, 6:9] = -1; rec[0, 9:12] = 1
    one = np.ones((1, 3), "<f4")
    ray_ok, rec_ok, differs = compare(lib, rec, np.zeros((1, 3), "<f4"), one, np.array([1e30], "<f4"))
    assert ray_ok[0] and rec_ok[0] and differs[0] == 4


def test_guards_reject_what_could_differ(lib):
    f = np.float32
    rec = np.zeros((1, 16), "<f4"); rec[0, 0:3] = 0; rec[0, 3:6] = (1, 0, 1); rec[0, 6:9] = (0, 0, 0); rec[0, 9:12] = (1, 1, 1)
    rec[0, 12:15] = np.array([1, 2, 1], "<i4").view("<f4")
    # a ray in the plane y = 0 of a flat box, direction component 0: 0 * inf = NaN, dropped by fminf/fmaxf and kept by a selection
    o = np.array([[0.5, 0.0, -1.0]], "<f4"); d = np.array([[0.0, 0.0, 1.0]], "<f4")
    with np.errstate(divide="ignore"):
        inv = (f(1) / d).astype("<f4")
    ray_ok, rec_ok, differs = compare(lib, rec, o, inv, np.array([1e30], "<f4"))
    assert not ray_ok[0] and rec_ok[0] and differs[0] & 1
    for bad in (np.inf, -np.inf, np.nan, 0.0, -0.0):
        for k in range(3):
            inv = np.array([[1.0, -2.0, 3.0]], "<f4"); inv[0, k] = bad
            assert not compare(lib, rec, o, inv, np.array([1.0], "<f4"))[0][0], (bad, k)
    with np.errstate(over="ignore"):
        for tiny in (1e-45, 1e-39, -2e-39):         # denormal direction components whose reciprocal overflows
            assert not compare(lib, rec, o, (f(1) / np.array([[tiny, 1, 1]], "<f4")).astype("<f4"), np.array([1.0], "<f4"))[0][0]
    assert compare(lib, rec, o, np.array([[FLT_MAX, -FLT_MAX, 1e-45]], "<f4"), np.array([1.0], "<f4"))[0][0]
    ok_inv = np.array([[1.0, -2.0, 3.0]], "<f4")
    for k in range(12):
        for bad in (np.nan, np.inf, -np.inf):
            r = rec.copy(); r[0, k] = bad
            assert not compare(lib, r, o, ok_inv, np.array([1.0], "<f4"))[1][0], (k, bad)
    r = rec.copy(); r[0, 0], r[0, 3] = 1.0, 0.5       # min > max
    assert not compare(lib, r, o, ok_inv, np.array([1.0], "<f4"))[1][0]
    r = rec.copy(); r[0, 14] = np.array([3], "<u4").view("<f4")[0]
    assert not compare(lib, r, o, ok_inv, np.array([1.0], "<f4"))[1][0]
    assert compare(lib, rec, o, ok_inv, np.array([1.0], "<f4"))[1][0]


def test_ordered_record_layout(lib):
    rec = np.arange(16, dtype="<f4"); rec[12:15] = np.array([7, ~5, 1], "<i4").view("<f4")
    for s in range(8):
        out = np.zeros(16, "<f4")
        lib.octant_order(rec.ctypes.data, s, out.ctypes.data)
        swap = (s >> 1) & 1
        for c in range(2):
            box = rec[6 * (c ^ swap): 6 * (c ^ swap) + 6]
            for k in range(3):
                neg = (s >> k) & 1
                assert out[6 * c + k] == box[3 + k if neg else k] and out[6 * c + 3 + k] == box[k if neg else 3 + k]
        refs = out[12:14].view("<i4")
        assert (refs[0], refs[1]) == ((~5, 7) if swap else (7, ~5))


def cornell_rays(orc, w, h, seed):
    """The primary rays of a w x h CornellBox frame, and from every primary hit point a seeded random direction (the continuation
    rays of a diffuse bounce start on the walls — flat boxes — like these) plus a few axis-parallel ones."""
    cam = default_camera(w, h)
    rays = orc.generate_rays(cam, w, h)
    hits, _ = orc.trace(rays)
    ok = hits["primitive_id"] != 0xFFFFFFFF
    p = (rays["origin"][ok, :3] + rays["direction"][ok, :3] * hits["t"][ok, None]).astype("<f4")
    rng = np.random.default_rng(seed)
    d = rng.normal(size=p.shape).astype("<f4"); d /= np.linalg.norm(d, axis=1, keepdims=True).astype("<f4")
    axis = rng.random(len(d)) < 0.02
    d[axis] = np.eye(3, dtype="<f4")[rng.integers(0, 3, axis.sum())] * rng.choice(np.array([-1, 1], "<f4"), axis.sum())[:, None]
    sec = np.zeros(len(p), RAY_DT)
    sec["origin"][:, :3] = p; sec["direction"][:, :3] = d; sec["direction"][:, 3] = 1e30
    return np.concatenate([rays, sec])


def test_walk_of_cornellbox_through_the_tables_matches_the_oracle(lib):
    sc = scene("CornellBox")
    nodes = np.ascontiguousarray(sc["nodes"], NODE_DT); tris = np.ascontiguousarray(sc["triangles"], TRIANGLE_DT)
    wn = np.zeros((len(nodes), 16), "<f4"); wt = np.zeros((len(tris), 12), "<f4")
    root, depth, top, nrec = C.c_int(), C.c_int(), C.c_uint32(), C.c_uint64()
    err = C.create_string_buffer(256)
    assert lib.bvh_layout_build(nodes.ctypes.data, len(nodes), tris.ctypes.data, len(tris), wn.ctypes.data, wt.ctypes.data,
                                C.byref(root), C.byref(depth), C.byref(top), C.byref(nrec), err, 256) == 0, err.value
    # the staging budget of the octant mode: canonical records + triangles + 8 tables + the flag word, 40 KB
    assert (nrec.value * 9 * 64 + len(tris) * 48 + 16) <= 40 * 1024
    orc = Oracle(sc)
    rays = cornell_rays(orc, 96, 54, 11)
    want, _ = orc.trace(rays)
    o = np.ascontiguousarray(rays["origin"][:, :3]); d = np.ascontiguousarray(rays["direction"][:, :3]); t_max = np.ascontiguousarray(rays["direction"][:, 3])
    root_box = np.concatenate([nodes["bounds_min"][0, :3], nodes["bounds_max"][0, :3]]).astype("<f4")
    for use_tables in (1, 0):
        prim = np.zeros(len(rays), "<u4"); uvt = np.zeros((len(rays), 3), "<f4")
        walked = lib.octant_walk(wn.ctypes.data, nrec.value, wt.ctypes.data, root.value, root_box.ctypes.data, len(rays), o.ctypes.data, d.ctypes.data,
                                 t_max.ctypes.data, use_tables, prim.ctypes.data, uvt.ctypes.data)
        with np.errstate(divide="ignore"):
            finite = np.isfinite(np.float32(1) / d).all(1)
        assert walked == (finite.sum() if use_tables else 0) and 0 < (~finite).sum() < 0.05 * len(rays)
        assert np.array_equal(prim, want["primitive_id"])
        hit = prim != 0xFFFFFFFF
        assert hit.sum() > 0.5 * len(rays)
        assert np.array_equal(uvt[hit, :2].view("<u4"), want["bc"][hit].view("<u4")) and np.array_equal(uvt[hit, 2].view("<u4"), want["t"][hit].view("<u4"))


def test_rays_outside_the_guard_are_rare_on_the_bench_frame():
    """The rays the ordered path hands to the pairwise traversal, counted on the frame bench.py renders (CornellBox 1920x1080 x 8
    bounces, the oracle's per-bounce dump of the extension rays): fewer than 1 in 10^4 at every bounce.  (The count is 0 of
    11.98 M: even image sizes put no pixel centre on an axis and no sampled direction has a zero or denormal component.)"""
    w, h, mb = 1920, 1080, 8
    orc = Oracle(scene("CornellBox")); cam = default_camera(w, h)
    total = 0
    for bounce in range(mb + 1):
        rays = np.zeros(w * h, RAY_DT); work = np.zeros((w * h, 2), np.uint32); n = C.c_uint32(0)
        orc.lib.orc_set_dump(bounce, rays.ctypes.data_as(C.c_void_p), work.ctypes.data_as(C.c_void_p), C.byref(n))
        try:
            orc.render(cam, w, h, mb, want_hits=False)
        finally:
            orc.lib.orc_set_dump(-1, None, None, None)
        assert n.value > 0
        with np.errstate(divide="ignore", over="ignore"):
            inv = np.float32(1) / rays["direction"][: n.value, :3]
        outside = ~(np.isfinite(inv).all(1) & (inv != 0).all(1))
        assert outside.sum() <= n.value * 1e-4, bounce
        total += n.value
    assert total > 11_000_000
