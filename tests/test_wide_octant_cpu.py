"""The 4-wide octant tables of raytracing_b200/csrc/rt_octant.h on the host: the tables equal a plain restatement of the collapse
(tools/wide_bvh_model.cpp), a walk of them returns the oracle's closest and any hits bit for bit on the rays of bounces 0-3, they
fit the room the staging reserves for them, and the nesting guard rejects a tree whose collapsed child does not contain its
children."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from oracle.orcbind import Oracle
from raytracing_b200 import hostapi
from raytracing_b200.camera import default_camera
from raytracing_b200.layouts import HIT_DT, NODE_DT, RAY_DT, TRIANGLE_DT
from tests.helpers import scene
from tests.scenes_extra import closed_cornell, many_lights_scene, single_leaf_scene, textured_cornell

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
NONE = 0xFFFFFFFF


@pytest.fixture(scope="module")
def lib():
    so = os.path.join(tempfile.gettempdir(), f"libwide_octant_host_{os.getpid()}.so")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-I" + os.path.join(REPO, "include"),
                    "-I" + os.path.join(REPO, "raytracing_b200", "csrc"), "-o", so, os.path.join(HERE, "wide_octant_host.cpp"),
                    os.path.join(HERE, "bvh_layout_host.cpp")], check=True)
    L = C.CDLL(so)
    L.wide_tables.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32)]
    L.wide_walk.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_int, C.c_void_p, C.c_uint64] + [C.c_void_p] * 3 + [C.c_int] + [C.c_void_p] * 4
    L.bvh_layout_build.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int),
                                   C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.c_char_p, C.c_int]
    yield L
    os.remove(so)


def layout(L, sc):
    """rt_bvh_layout.h's records (n x 16 floats), triangle records and root reference of a scene."""
    nodes = np.ascontiguousarray(sc["nodes"], NODE_DT); tris = np.ascontiguousarray(sc["triangles"], TRIANGLE_DT)
    wn = np.zeros((len(nodes), 16), "<f4"); wt = np.zeros((len(tris), 12), "<f4")
    root, depth, top, nrec = C.c_int(), C.c_int(), C.c_uint32(), C.c_uint64()
    err = C.create_string_buffer(256)
    assert L.bvh_layout_build(nodes.ctypes.data, len(nodes), tris.ctypes.data, len(tris), wn.ctypes.data, wt.ctypes.data,
                              C.byref(root), C.byref(depth), C.byref(top), C.byref(nrec), err, 256) == 0, err.value
    n = nrec.value if root.value >= 0 else 0          # a root-leaf tree has no record to visit (stage_bvh)
    return np.ascontiguousarray(wn[:n]), wt, root.value, nodes


def tables(L, recs):
    n = len(recs)
    out = np.zeros_like(recs); tab = np.full((8, 2 * max(n, 1), 8), np.nan, "<f4"); ns = C.c_uint32(0)
    ok = L.wide_tables(recs.ctypes.data, n, out.ctypes.data, tab.ctypes.data, C.byref(ns))
    return ok, out, tab, ns.value


def restated_tables(recs):
    """The collapse restated: wide nodes = interior records at even depth, each a run of slots in record order; in octant s the
    slots follow the binary traversal's order (near child first by the sign of the split axis, an interior child replaced by its
    own two children in the same order), entry plane = box max on the axes where the octant's bit is set, else box min."""
    n = len(recs)
    ref = recs[:, 12:14].view("<i4"); axis = recs[:, 14].view("<u4")
    depth = np.full(n, -1)
    if n:
        depth[0] = 0
        todo = [0]
        while todo:
            r = todo.pop()
            for c in range(2):
                if ref[r, c] >= 0:
                    depth[ref[r, c]] = depth[r] + 1; todo.append(int(ref[r, c]))
    assert (depth >= 0).all()
    wide = [r for r in range(n) if depth[r] % 2 == 0]
    count = {r: sum(1 if ref[r, c] < 0 else 2 for c in range(2)) for r in wide}
    first, k = {}, 0
    for r in wide:
        first[r] = k; k += count[r]
    tab = np.zeros((8, k, 8), "<f4")

    def children(r, s):          # (box min, box max, ref) of record r's two children in visiting order
        sw = (s >> int(axis[r])) & 1
        return [(recs[r, 6 * c:6 * c + 3], recs[r, 6 * c + 3:6 * c + 6], int(ref[r, c])) for c in (sw, 1 - sw)]

    for s in range(8):
        neg = np.array([(s >> a) & 1 for a in range(3)], bool)
        for r in wide:
            slots = []
            for lo, hi, q in children(r, s):
                slots += [(lo, hi, q)] if q < 0 else [(l2, h2, first.get(g, g) if g >= 0 else g) for l2, h2, g in children(q, s)]
            for j, (lo, hi, q) in enumerate(slots):
                row = tab[s, first[r] + j]
                row[0:3] = np.where(neg, hi, lo); row[3:6] = np.where(neg, lo, hi)
                row[6:8] = np.array([q, count[r]], "<i4").view("<f4")
    return tab, k


SMALL = {"CornellBox": lambda: scene("CornellBox"), "textured": textured_cornell, "closed": closed_cornell, "many_lights": many_lights_scene,
         "leaf3": lambda: single_leaf_scene(3)}


@pytest.mark.parametrize("name", sorted(SMALL))
def test_tables_equal_the_restated_collapse(lib, name):
    recs, _, _, _ = layout(lib, SMALL[name]())
    ok, out, tab, n_slots = tables(lib, recs)
    want, k = restated_tables(recs)
    assert ok == 1 and n_slots == k
    assert np.array_equal(tab[:, :k].view("<u4"), want.view("<u4"))
    first = out[:, 15].view("<u4")
    assert np.array_equal(out[:, :15].view("<u4"), recs[:, :15].view("<u4"))         # only word 15 is written
    assert first[0] == 0                                                              # the root opens the table
    assert (first != NONE).sum() < len(recs) or len(recs) == 1                        # some records collapse


def bounce_rays(orc, cam, w, h, mb, bounce):
    rays = np.zeros(w * h, RAY_DT); work = np.zeros((w * h, 2), np.uint32); n = C.c_uint32(0)
    orc.lib.orc_set_dump(bounce, rays.ctypes.data_as(C.c_void_p), work.ctypes.data_as(C.c_void_p), C.byref(n))
    try:
        orc.render(cam, w, h, mb, want_hits=False)
    finally:
        orc.lib.orc_set_dump(-1, None, None, None)
    return np.ascontiguousarray(rays[: n.value])


@pytest.mark.parametrize("name", ["CornellBox", "closed", "many_lights"])
def test_walk_of_the_tables_matches_the_oracle(lib, name):
    sc = SMALL[name]()
    recs, wt, root, nodes = layout(lib, sc)
    ok, _, tab, _ = tables(lib, recs)
    assert ok == 1
    root_box = np.concatenate([nodes["bounds_min"][0, :3], nodes["bounds_max"][0, :3]]).astype("<f4")
    orc = Oracle(sc)
    w, h = 160, 90
    cams = [default_camera(w, h), default_camera(w, h, position=(0.4, -1.5, 0.7), yaw=1.8, pitch=1.45, aperture=0.03, focus_distance=2.0)]
    steps = nodes_visited = 0
    for cam in cams:
        for bounce in range(4):
            rays = bounce_rays(orc, cam, w, h, 4, bounce)
            assert len(rays) > 0
            o = np.ascontiguousarray(rays["origin"][:, :3]); d = np.ascontiguousarray(rays["direction"][:, :3])
            t_max = np.ascontiguousarray(rays["direction"][:, 3])
            for any_hit in (0, 1):
                if any_hit:     # shadow-ray lengths: up to and past the closest hit, so that some rays are not occluded
                    near, _ = orc.trace(rays)
                    rng = np.random.default_rng(bounce)
                    t_max = np.where(near["primitive_id"] != NONE, near["t"] * rng.uniform(0.3, 1.2, len(rays)), t_max).astype("<f4")
                    rays = rays.copy(); rays["direction"][:, 3] = t_max
                prim = np.zeros(len(rays), "<u4"); uvt = np.zeros((len(rays), 3), "<f4"); st = np.zeros(len(rays), np.uint8)
                counts = np.zeros(3, np.uint64)
                lib.wide_walk(tab.ctypes.data, len(recs), wt.ctypes.data, root, root_box.ctypes.data, len(rays), o.ctypes.data, d.ctypes.data,
                              t_max.ctypes.data, any_hit, prim.ctypes.data, uvt.ctypes.data, st.ctypes.data, counts.ctypes.data)
                walked = st == 1
                assert walked.sum() >= 0.999 * len(rays), (bounce, any_hit)
                assert counts[2] <= 128
                if any_hit:
                    flags, _ = orc.trace(rays, any_hit=True)
                    assert np.array_equal(np.where(prim == 0, 0, NONE)[walked], flags[walked]), (cam, bounce)
                    assert (prim[walked] == 0).any() and (prim[walked] == NONE).any()
                else:
                    want, _ = orc.trace(rays)
                    assert np.array_equal(prim[walked], want["primitive_id"][walked]), (bounce,)
                    hit = walked & (prim != NONE)
                    assert hit.sum() > 0.3 * len(rays)
                    assert np.array_equal(uvt[hit, :2].view("<u4"), want["bc"][hit].view("<u4"))
                    assert np.array_equal(uvt[hit, 2].view("<u4"), want["t"][hit].view("<u4"))
                    steps += int(counts[0]); nodes_visited += int(walked.sum())
    assert steps < 8 * nodes_visited            # a few wide steps per ray (CornellBox: about 4.5)


def subset_scene(n_tris):
    """The first n_tris triangles of ShaderBalls under a BVH of their own."""
    sc = dict(scene("ShaderBalls"))
    ordered, nodes, _ = hostapi.build_bvh(sc["triangles"][:n_tris].copy())
    sc["triangles"], sc["nodes"] = ordered, nodes
    return sc


def test_tables_fit_the_reserved_room(lib):
    """The staging reserves 8 x 64 bytes per record for the tables (rt_bvh_staging's formula is unchanged): every tree staged
    with the tables, here every subset of ShaderBalls whose staged bytes fit 40 KB, needs no more."""
    checked = 0
    for n_tris in list(range(2, 40)) + list(range(40, 160, 3)):
        recs, wt, _, _ = layout(lib, subset_scene(n_tris))
        n = len(recs)
        if n * 64 + n_tris * 48 + n * 8 * 64 + 16 > 40 * 1024:
            continue
        ok, _, _, n_slots = tables(lib, recs)
        assert ok == 1 and n_slots * 32 <= n * 64, n_tris
        checked += 1
    assert checked > 50


def hand_tree():
    """Records of a tree of depth 3: root 0 -> (1, 2), 1 -> (leaf, leaf), 2 -> (3, leaf), 3 -> (leaf, leaf); nesting everywhere."""
    boxes = {0: [(0, 0, 0, 1, 1, 1), (2, 0, 0, 4, 1, 1)], 1: [(0, 0, 0, .4, 1, 1), (.6, 0, 0, 1, 1, 1)],
             2: [(2, 0, 0, 3, 1, 1), (3.5, 0, 0, 4, 1, 1)], 3: [(2, 0, 0, 2.4, 1, 1), (2.5, 0, 0, 3, 1, 1)]}
    refs = {0: (1, 2, 0), 1: (~0, ~1, 0), 2: (3, ~2, 0), 3: (~3, ~4, 0)}
    recs = np.zeros((4, 16), "<f4")
    for r in range(4):
        recs[r, 0:6], recs[r, 6:12] = boxes[r]
        recs[r, 12:15] = np.array(refs[r], "<i4").view("<f4")
    return recs


def test_nesting_guard(lib):
    recs = hand_tree()
    ok, out, _, n_slots = tables(lib, recs)
    assert ok == 1 and n_slots == 4 + 2 and list(out[:, 15].view("<u4")) == [0, NONE, NONE, 4]
    bad = recs.copy(); bad[1, 9] = 1.5                  # a grandchild of the root sticks out of its collapsed parent's box (x)
    assert tables(lib, bad)[0] == 0
    bad = recs.copy(); bad[2, 2] = -0.5                 # likewise, on z and below
    assert tables(lib, bad)[0] == 0
    # record 3 is a wide node (depth 2): its box is tested before its children, as the binary traversal does, so a child of
    # it that sticks out is accepted
    fine = recs.copy(); fine[3, 0] = 1.9
    assert tables(lib, fine)[0] == 1
    bad = recs.copy(); bad[0, 12] = np.array([9], "<i4").view("<f4")[0]
    assert tables(lib, bad)[0] == 0                     # a reference out of range
