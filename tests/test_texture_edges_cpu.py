"""
CPU tests (-m "not gpu") of the textured-material rule at its edges (tests/texture_cases.py): texture shapes 1x1 to 2048x2048,
texture indices 253 and 254 of 255, coordinates at integers, their float32 neighbours, -1e-9, +-2^23, +-2^24, +-1e30, NaN, +-inf
and a zero weight against an infinite coordinate, every texture slot, and every emission exponent byte.

- The oracle against what the reference's own kernels (oracle/_ref) produced on the chart and ladder scenes, bit for bit
  (tests/golden/ref/texture_edges.json.xz, written by tests/golden/make_texture_edge_records.py).
- The oracle's albedo AOV against a numpy restatement from its own primary hits: the float32 lookup restated literally, the
  (texel / 255)^2.2 in float64 within 1 ulp (rt_powf's bound, tests/test_rt_math.py).  Every designed edge, shape and index is
  reached by some pixel.
- The host's per-material record (mat_rec, rt_bvh_layout.h) holds ldexp(mantissa, e - 136) bit for bit for every exponent byte,
  and the oracle's max_bounces = 0 frame of the ladder is that emission at every pixel of the untextured and per-hit variants.
"""
import ctypes as C
import json
import lzma
import os

import numpy as np
import pytest

from oracle.orcbind import Oracle
from raytracing_b200.camera import default_camera
from tests import texture_cases as T
from tests.helpers import GOLDEN, bits, digest, frame_record

REF_KEYS = ("n_ext", "n_miss", "n_shadow", "n_cont", "n_unoccluded")
# case -> (scene builder, camera(w, h), w, h, max_bounces, samples)
REF_CASES = {
    "chart_b6": (T.chart_scene, T.chart_camera, T.CHART_W, T.CHART_H, 6, 3),
    "ladder_b0": (T.ladder_scene, default_camera, T.LADDER_W, T.LADDER_H, 0, 1),
    "ladder_b3": (T.ladder_scene, default_camera, T.LADDER_W, T.LADDER_H, 3, 2),
}
_scenes = {}


def cached(build):
    if build not in _scenes:
        _scenes[build] = build()
    return _scenes[build]


def ref_records():
    with lzma.open(os.path.join(GOLDEN, "ref", "texture_edges.json.xz"), "rt") as f:
        return json.load(f)


@pytest.mark.parametrize("case", sorted(REF_CASES))
def test_oracle_matches_reference_kernels(case):
    build, cam_of, w, h, mb, n = REF_CASES[case]
    sc = cached(build)
    cam = cam_of(w, h)
    o = Oracle(sc)
    acc = np.zeros((h, w, 4), "<f4")
    recs = []
    for s in range(n):
        acc, hits, st = o.render(cam, w, h, mb, sample_idx=s, radiance=acc)
        recs.append(frame_record(st, mb, acc, hits, keys=REF_KEYS))
    want = ref_records()
    assert recs == want[case], case
    if case.startswith("chart"):
        al, _, _, _ = o.aovs(cam, cam, w, h)
        assert digest(bits(al[..., :3])) == want[case + "/albedo"]


def chart_primary(sc, w=T.CHART_W, h=T.CHART_H):
    """The oracle's primary hits and albedo AOV of the chart at sample 0."""
    cam = T.chart_camera(w, h)
    o = Oracle(sc)
    _, hits, _ = o.render(cam, w, h, 0)
    al, _, _, _ = o.aovs(cam, cam, w, h)
    return hits, al.reshape(-1, 4)


def check_albedo(sc, prim, bc, albedo):
    """albedo (n, 4) float32 against the restatement: exact where untextured, within 1 ulp of the float64 power where textured.
    -> the restatement's (textured mask, f32 texel, f64 texel, uv32)."""
    want, textured, i32, i64, uv32 = T.albedo_restatement(sc, prim, bc)
    got = albedo[:, :3]
    plain = ~textured
    assert np.array_equal(bits(got[plain]), bits(want[plain].astype(np.float32)))
    d = T.ulp_distance(got[textured], want[textured])
    assert d.max() <= 1.0, (d.max(), np.argmax(d.max(1)))
    assert (albedo[:, 3] == 0).all()
    return textured, i32, i64, uv32


def test_albedo_aov_matches_restatement():
    sc = cached(T.chart_scene)
    hits, al = chart_primary(sc)
    prim, bc = hits["primitive_id"], hits["bc"]
    textured, i32, i64, uv32 = check_albedo(sc, prim, bc, al)
    hit = prim != 0xFFFFFFFF
    tex_of = np.full(len(prim), -1)
    tex_of[hit] = (sc["materials"]["diffuse_albedo"][sc["triangles"]["mtlIndex"][prim[hit]]] >> 24).astype(np.int64)
    # every shape and index of the chart is sampled, 253 and 254 of 255 included
    for t in T.CHART_ROWS:
        assert (textured & (tex_of == t)).sum() > 50, t
    assert len(sc["textures"]) == 255 and sc["textures"]["data_start"][254] > 1 << 24
    # every coordinate edge is reached
    edge = T.edge_of_pixel(sc, prim)
    u = uv32[:, 0].astype(np.float64)
    with np.errstate(invalid="ignore"):
        frac32 = (uv32 - np.floor(uv32)).astype(np.float32)
    reach = {}
    for k in (0.0, 1.0, -1.0, 3.0):
        name = {0.0: "zero", 1.0: "one", -1.0: "minus_one", 3.0: "three"}[k]
        m = textured & (edge == name)
        below, above = np.nextafter(np.float32(k), np.float32(-np.inf)), np.nextafter(np.float32(k), np.float32(np.inf))
        reach[name] = [int((m & (uv32[:, 0] == np.float32(k))).sum())]
        if k != 0.0:          # the neighbours of 0 are subnormals no interpolation reaches; v sweeps both signs of 0 instead
            reach[name] += [int((m & (uv32[:, 0] == below)).sum()), int((m & (uv32[:, 0] == above)).sum())]
        else:
            reach[name] += [int((m & (uv32[:, 1] < 0)).sum()), int((m & (uv32[:, 1] > 0)).sum())]
    m = textured & (edge == "tiny_negative")
    reach["tiny_negative"] = int((m & (frac32[:, 0] == 1.0) & (frac32[:, 1] == 1.0)).sum())
    for name, lo in (("2^23", 2.0 ** 23), ("2^24", 2.0 ** 24), ("1e30", 1e30)):
        m = textured & (edge == name)
        reach[name] = int((m & (np.abs(u) >= lo) & (np.abs(uv32[:, 1]) >= lo)).sum())
    reach["nan"] = int((textured & (edge == "nan") & np.isnan(uv32[:, 0])).sum())
    reach["inf"] = int((textured & (edge == "inf") & np.isnan(frac32).all(1)).sum())
    zw = len(sc["materials"]) - 1          # the triangle at the camera: u = v = 0 against +-inf
    m = hit.copy(); m[hit] = sc["triangles"]["mtlIndex"][prim[hit]] == zw
    reach["zero_weight"] = int((m & np.isnan(uv32).all(1) & (bc == 0).all(1)).sum())
    for name, n in reach.items():
        assert (min(n) if isinstance(n, list) else n) > 0, (name, reach)
    # where a float64 evaluation of the lookup picks another texel: the integers' neighbours and the large magnitudes
    differ = textured & (i32 != i64)
    per_edge = {name: int((differ & (edge == name)).sum()) for name in T.EDGES}
    print("pixels whose float64 lookup picks another texel:", int(differ.sum()), per_edge, "reach:", reach)
    for name in ("one", "minus_one", "three", "2^23"):
        assert per_edge[name] > 0, (name, per_edge)


@pytest.fixture(scope="module")
def layout_lib():
    """tests/bvh_layout_host.cpp: rt_bvh_layout.h's host records in a temporary shared library."""
    import subprocess
    import tempfile
    here = os.path.dirname(os.path.abspath(__file__)); repo = os.path.dirname(here)
    with tempfile.TemporaryDirectory() as d:
        so = os.path.join(d, "libbvh_layout_host.so")
        subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-I" + os.path.join(repo, "include"),
                        "-I" + os.path.join(repo, "raytracing_b200", "csrc"), "-o", so, os.path.join(here, "bvh_layout_host.cpp")], check=True)
        L = C.CDLL(so)
    L.shade_records_build.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


def test_emission_decode_is_exact_for_every_exponent(layout_lib):
    """ldexp(mantissa, e - 136) in float64 is exactly representable in float32 for every byte (2^-136 and its multiples up to 255
    are subnormal above 2^-149); mat_rec holds it bit for bit, exponent 0 included."""
    from raytracing_b200.layouts import LIGHT_DT, MATERIAL_DT, TRIANGLE_DT
    sc = cached(T.ladder_scene)
    mats = np.ascontiguousarray(sc["materials"], MATERIAL_DT)
    tris = np.ascontiguousarray(sc["triangles"], TRIANGLE_DT); lights = np.ascontiguousarray(sc["lights"], LIGHT_DT)
    to = np.zeros((len(tris), 28), "<f4"); mo = np.zeros((len(mats), 16), "<f4"); lo = np.zeros((len(lights), 8), "<f4")
    layout_lib.shade_records_build(tris.ctypes.data, len(tris), mats.ctypes.data, len(mats), lights.ctypes.data, len(lights),
                                   to.ctypes.data, mo.ctypes.data, lo.ctypes.data)
    want = np.stack([T.emission_f64(w) for w in mats["emission"]])
    assert np.array_equal(want.astype(np.float32).astype(np.float64), want)
    assert np.array_equal(bits(mo[:, 8:11]), bits(want.astype(np.float32)))
    exps = mats["emission"] >> 24
    assert set(exps.tolist()) == set(range(256))
    assert (want[exps == 0] > 0).any() and (want[(want > 0)] < 2.0 ** -126).any()     # subnormal emission present
    # textured flag: the per-hit variants take the per-hit path
    per_hit = np.array([sc["ladder"][i][0] != "untextured" for i in range(len(mats))])
    assert np.array_equal(mo[:, 13].copy().view("<u4") != 0, per_hit)


def ladder_expected(sc, prim):
    """-> (pixels on an untextured or per-hit ladder quad, their float64 emission, their variant)."""
    hit = prim != 0xFFFFFFFF
    mtl = np.full(len(prim), -1, np.int64)
    mtl[hit] = sc["triangles"]["mtlIndex"][prim[hit]]
    keep = np.array([m >= 0 and sc["ladder"].get(int(m), ("floor",))[0] in ("untextured", "per_hit") for m in mtl])
    want = np.stack([T.emission_f64(sc["materials"]["emission"][m]) for m in mtl[keep]])
    return np.flatnonzero(keep), want, [sc["ladder"][int(m)] for m in mtl[keep]]


def test_ladder_primary_radiance_is_the_emission():
    """max_bounces = 0 with diffuse and specular 0: the oracle's radiance at a primary hit is the emission alone, on both the
    untextured and the per-hit variant, for every exponent byte (what tests/test_gpu_texture_edges.py asserts of the device)."""
    sc = cached(T.ladder_scene)
    w, h = T.LADDER_W, T.LADDER_H
    rad, hits, _ = Oracle(sc).render(default_camera(w, h), w, h, 0)
    px, want, where = ladder_expected(sc, hits["primitive_id"])
    got = rad.reshape(-1, 4)[px, :3]
    assert np.array_equal(bits(got), bits(want.astype(np.float32)))
    seen = {(v, e) for v, e in where}
    assert all((v, e) in seen for v in ("untextured", "per_hit") for e in range(256))
