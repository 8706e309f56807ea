"""
CPU tests (-m "not gpu") of the shading pass across the packed material space (tests/material_cases.py): every value of every
material byte field, the diffuse and specular channels at their edges, shading normals that are zero, flipped, scaled, grazing or
at tangent_frame's switch, and lights exactly grazing, below the horizon, on the surface, at the camera and at the mirror
direction of a roughness-0 surface.

- The oracle against what the reference's own kernels (oracle/_ref) produced on every case, bit for bit: kRandom and blue noise
  (synthetic tables), white furnace on and off, 0, 1 and 6 bounces, 2 progressive samples; per-bounce counters, the digests of the
  radiance bits and primary hits, and the bounce-0 albedo AOV (tests/golden/ref/material_edges.json.xz, written by
  tests/golden/make_material_edge_records.py).
- What each designed branch is reached by (REACH), from a numpy restatement of the primary hits and the kRandom draws.
- The host's per-material record (build_mat_rec, rt_bvh_layout.h) against the numpy decode of all 256 values of every byte field.
- Known answers in float64 (material.h:132-241 restated), without the oracle: (a) one directional light at 0 bounces, a black sky:
  L * brdf * cos_l; (b) a light of radiance 0 and a constant sky c at 1 bounce: c * bxdf / pdf of the sampled direction.  Each
  negative control (a mistake made in the restatement) is rejected by the comparison.
"""
import json
import lzma
import os

import numpy as np
import pytest

from oracle.orcbind import Oracle
from raytracing_b200.camera import default_camera
from tests import material_cases as M
from tests.helpers import GOLDEN, bits, digest, frame_record, synthetic_sampler_tables
from tests.test_rt_math import host  # noqa: F401  (fixture)
from tests.test_texture_edges_cpu import layout_lib  # noqa: F401  (fixture)

REF_KEYS = ("n_ext", "n_miss", "n_shadow", "n_cont", "n_unoccluded")
CW, CH = M.CHART_W, M.CHART_H
# scene -> (builder, camera(w, h), w, h)
SCENES = {
    "chart": (M.chart_scene, M.chart_camera, CW, CH),
    "grazing": (lambda: M.chart_scene("grazing"), M.chart_camera, CW, CH),
    "per_hit": (lambda: M.chart_scene("per_hit"), M.chart_camera, CW, CH),
    "normals": (M.normal_scene, default_camera, CW, CH),
    "lights": (M.lights_scene, default_camera, M.LIGHTS_W, M.LIGHTS_H),
    "mirror": (M.mirror_scene, M.mirror_camera, M.MIRROR_W, M.MIRROR_H),
}
# case -> (scene, max_bounces, samples, white furnace, sampler)
REF_CASES = {
    "chart_b6": ("chart", 6, 2, False, "random"), "chart_b0": ("chart", 0, 2, False, "random"),
    "chart_b1_bn": ("chart", 1, 2, False, "blue_noise"), "chart_b6_wf": ("chart", 6, 2, True, "random"),
    "grazing_b6": ("grazing", 6, 2, False, "random"), "grazing_b1_bn": ("grazing", 1, 2, False, "blue_noise"),
    "per_hit_b6": ("per_hit", 6, 2, False, "random"),
    "normals_b6": ("normals", 6, 2, False, "random"), "normals_b1_bn": ("normals", 1, 2, False, "blue_noise"),
    "normals_b6_wf": ("normals", 6, 2, True, "random"),
    "lights_b6": ("lights", 6, 2, False, "random"), "lights_b0_bn": ("lights", 0, 2, False, "blue_noise"),
    "mirror_b1": ("mirror", 1, 2, False, "random"), "mirror_b6_bn": ("mirror", 6, 2, False, "blue_noise"),
}
# scene -> {branch: least number of bounce-0 pixels of sample 0 that reach it (material_cases.reach)}
REACH = {
    "chart": {"pass_through": 5000, "delta_lobe": 500, "nan_lobe_pdf": 10, "tangent_axis_x": 20000},
    "grazing": {"pass_through": 5000, "delta_lobe": 500, "nan_lobe_pdf": 10, "n.i<0": 5000, "n.i_at_eps_clamp": 500,
                "|n.i|<1e-5": 5, "tangent_axis_y": 20000},
    "normals": {"nan_normal": 1000, "tangent_axis_y": 1000, "tangent_axis_x": 1000, "tangent_at_switch": 1000,
                "tangent_above_switch_4ulp": 500, "tangent_below_switch_4ulp": 500, "n.i<0": 500, "cos_l==0_skip": 1000},
    "lights": {"pass_through": 1000, "delta_lobe": 1000, "cos_l==0_skip": 3000, "light_at_hit": 1},
    "mirror": {"delta_lobe": 2000, "n.h==1_at_alpha_0": 200},
}
_scenes = {}


def cached(name):
    if name not in _scenes:
        build, cam, w, h = SCENES[name]
        _scenes[name] = (build(), cam(w, h), w, h)
    return _scenes[name]


def sampler_tables(sampler):
    return synthetic_sampler_tables() if sampler == "blue_noise" else None


def ref_records():
    with lzma.open(os.path.join(GOLDEN, "ref", "material_edges.json.xz"), "rt") as f:
        return json.load(f)


def oracle_records(case):
    name, mb, n, wf, sampler = REF_CASES[case]
    sc, cam, w, h = cached(name)
    o = Oracle(sc)
    acc = np.zeros((h, w, 4), "<f4")
    recs = []
    try:
        o.set_sampler_tables(sampler_tables(sampler))
        for s in range(n):
            acc, hits, st = o.render(cam, w, h, mb, sample_idx=s, white_furnace=wf, radiance=acc)
            recs.append(frame_record(st, mb, acc, hits, keys=REF_KEYS))
        al = o.aovs(cam, cam, w, h, sample_idx=n - 1)[0]
    finally:
        o.set_sampler_tables(None)
    return recs, digest(bits(al[..., :3]))


@pytest.mark.parametrize("case", sorted(REF_CASES))
def test_oracle_matches_reference_kernels(case):
    recs, albedo = oracle_records(case)
    want = ref_records()
    assert recs == want[case], case
    assert albedo == want[case + "/albedo"], case


def scene_reach(name, sample=0):
    sc, cam, w, h = cached(name)
    _, hits, _ = Oracle(sc).render(cam, w, h, 0, sample_idx=sample)
    return M.reach(sc, M.primary_view(sc, cam, w, h, hits, sample), w, h, sample)


@pytest.mark.parametrize("name", sorted(REACH))
def test_designed_branches_are_reached(name):
    got = scene_reach(name)
    print(name, got)
    for branch, least in REACH[name].items():
        assert got[branch] >= least, (name, branch, got)


def test_chart_holds_every_byte_value():
    sc = cached("chart")[0]
    m = sc["materials"]
    fields = {"roughness": m["roughness_metalness"] & 0xFF, "metalness": (m["roughness_metalness"] >> 16) & 0xFF,
              "ior": m["ior_emission_idx_transparency"] & 0xFF, "transparency": (m["ior_emission_idx_transparency"] >> 16) & 0xFF}
    for f, v in fields.items():
        assert set(v.tolist()) == set(range(256)), f
    assert len(m) == 1711
    for word in ("diffuse_albedo", "specular_albedo"):
        for s in (0, 8, 16):
            assert set(M.CHANNEL_VALUES) <= set(((m[word] >> s) & 0xFF).tolist()), (word, s)


def test_per_hit_twin_changes_no_value(host):     # noqa: F811
    """The per-hit twin's 1x1 white emission texture multiplies the (zero) emission by rt_powf(255/255, 2.2f) = 1: both facts
    hold in float32, so the twin decodes to the same values as the untextured chart."""
    one = np.float32(255.0) / np.float32(255.0)
    assert one == np.float32(1.0)
    assert host("pow", np.array([one], "<f4"), np.array([2.2], "<f4"))[0] == np.float32(1.0)
    a, b = cached("chart")[0]["materials"], cached("per_hit")[0]["materials"]
    for k in ("diffuse_albedo", "specular_albedo", "emission", "roughness_metalness"):
        assert np.array_equal(a[k], b[k])
    assert ((b["ior_emission_idx_transparency"] >> 8) & 0xFF == 0).all()
    assert np.array_equal(a["ior_emission_idx_transparency"] | 0xFF00, b["ior_emission_idx_transparency"] | 0xFF00)


def test_host_decode_matches_numpy(layout_lib):     # noqa: F811
    """build_mat_rec (rt_bvh_layout.h) holds the numpy decode of all 256 values of every byte field, bit for bit."""
    from raytracing_b200.layouts import LIGHT_DT, MATERIAL_DT, TRIANGLE_DT
    v = np.arange(256, dtype=np.uint32)
    mats = np.zeros(256, MATERIAL_DT)
    mats["diffuse_albedo"] = v | v << 8 | v << 16 | np.uint32(0xFF) << 24
    mats["specular_albedo"] = (255 - v) | v << 8 | (v ^ 0x55) << 16 | np.uint32(0xFF) << 24
    mats["roughness_metalness"] = v | 0xFF << 8 | (255 - v) << 16 | np.uint32(0xFF) << 24
    mats["ior_emission_idx_transparency"] = v | 0xFF << 8 | (v ^ 0xAA) << 16 | np.uint32(0xFF) << 24
    tris = np.zeros(1, TRIANGLE_DT); lights = np.zeros(1, LIGHT_DT)
    to = np.zeros((1, 28), "<f4"); mo = np.zeros((256, 16), "<f4"); lo = np.zeros((1, 8), "<f4")
    layout_lib.shade_records_build(tris.ctypes.data, 1, mats.ctypes.data, 256, lights.ctypes.data, 1,
                                   to.ctypes.data, mo.ctypes.data, lo.ctypes.data)
    f = np.float32
    b255 = lambda x: (x.astype(f) / f(255.0)).astype(f)
    want = np.zeros((256, 16), f)
    want[:, 0:3] = b255(v)[:, None]
    want[:, 3] = b255(v)
    want[:, 4], want[:, 5], want[:, 6] = b255(255 - v), b255(v), b255(v ^ 0x55)
    want[:, 7] = b255(255 - v)
    want[:, 11] = (v.astype(f) / f(25.5)).astype(f)
    want[:, 12] = b255(v ^ 0xAA)
    assert np.array_equal(bits(mo[:, [0, 1, 2, 3, 4, 5, 6, 7, 11, 12]]), bits(want[:, [0, 1, 2, 3, 4, 5, 6, 7, 11, 12]]))
    assert (mo[:, 13].view("<u4") == 0).all()            # untextured
    # the edges the issue names: ior byte 0 gives f0 = 1, bytes 25 and 26 straddle ior 1 (f0 about 0)
    ior = want[:, 11].astype(np.float64)
    f0 = ((ior - 1) / (ior + 1)) ** 2
    assert f0[0] == 1.0 and f0[25] < 1e-3 and f0[26] < 1e-3 and want[25, 11] < 1.0 < want[26, 11]


# ------------------------------------------------------------------------------------------------------------ known answers
# Lobes sharper than float32 resolves, left out of the comparison (byte 0, alpha = 0, is compared: D is exactly 0 off n.h == 1):
# (a) near its peak D = a2 / pi / (1 - n.h^2 (1 - a2))^2 has a relative error of about 2^-23 / a2 from the rounding of n.h in
#     float32, above 1e-4 for a2 = alpha^2 < 1.2e-3: roughness bytes 1..47.
# (b) the sampled half vector's polar angle (about alpha) is cos_theta rounded to float32, in steps of sqrt(2^-23) = 3.5e-4 rad:
#     for alpha < 1e-3 (bytes 1..8) the float32 direction is quantised at the lobe's own scale.  And where the sampled n.o is below
#     1e-2, G and max(n.o, 0) have a relative sensitivity of 1 / n.o to the rounding of the direction.
SHARP_DIRECT, SHARP_SKY, LOW_NO = 47, 8, 1e-2
TOL = 1e-4
# Byte 3 (alpha = 1.38e-4, just above the delta threshold 1e-4) gives NaN radiance in (b) by the reference's float32 arithmetic:
# alpha^2 = 1.9e-8 is below half an ulp of 1, so in GGX_D (bxdf.h:104-109) a2 - 1 == -1, and a sampled half vector with n.h == 1
# gives D = a2 / pi / 0 = inf; bxdf / pdf (material.h:93-101, hit_surface.cl:161-164) is inf / inf.
NAN_BYTE = 3


def ka_frame(kind, variant="untextured"):
    """The oracle's known-answer frame (a) or (b) of the chart: -> (view, radiance (n, 3) at the covered pixels, stats)."""
    sc = M.direct_frame_scene(variant) if kind == "direct" else M.sky_frame_scene(variant)
    cam, w, h = M.chart_camera(CW, CH), CW, CH
    rad, hits, st = Oracle(sc).render(cam, w, h, 0 if kind == "direct" else 1)
    view = M.primary_view(sc, cam, w, h, hits)
    return view, rad.reshape(-1, 4)[view["px"], :3], st


def known_answer(kind, view, control=None):
    if kind == "direct":
        return M.f64_direct(view, control=control), None
    want, *extra = M.f64_sky(view, CW, CH, control=control)
    return want, extra


def compare(kind, view, got, want, extra=None):
    """-> (number of pixels outside TOL among those compared, number compared, zero-pattern mismatches)."""
    rough_byte = np.rint(view["m"]["roughness"] * 255).astype(int)
    keep = np.ones(len(got), bool)
    if kind == "direct":
        keep &= ~((rough_byte >= 1) & (rough_byte <= SHARP_DIRECT))
    else:
        keep &= ~((rough_byte >= 1) & (rough_byte <= SHARP_SKY))
        keep &= extra[1] > 1e-6            # lobe choices within 1e-6 of the boundary may fall either way in float32
        keep &= ~(np.abs(extra[2]) < LOW_NO) | (view["m"]["transparency"] < 0.5)
    # per-cell scale: 1e-3 of the cell's largest value
    cell_max = np.zeros(view["mtl"].max() + 1)
    np.maximum.at(cell_max, view["mtl"], np.nan_to_num(np.abs(want)).max(1))
    big = np.abs(want) > 1e-3 * cell_max[view["mtl"]][:, None]
    with np.errstate(all="ignore"):
        rel = np.abs(got.astype(np.float64) - want) / np.abs(want)
    bad = keep[:, None] & big & ~(rel <= TOL)
    zero_want = np.all(want == 0, 1)
    zero_bad = int((keep & (zero_want != np.all(got == 0, 1))).sum())
    return int(bad.any(1).sum()), int((keep[:, None] & big).any(1).sum()), zero_bad


@pytest.mark.parametrize("kind", ["direct", "sky"])
def test_oracle_meets_float64_known_answer(kind):
    view, got, st = ka_frame(kind)
    want, extra = known_answer(kind, view)
    bad, n, zero_bad = compare(kind, view, got, want, extra)
    print(kind, "pixels compared", n, "outside", bad, "zero-pattern mismatches", zero_bad)
    assert n > 15000 and bad == 0 and zero_bad == 0
    if kind == "direct":          # a shadow ray exactly where the known answer is not 0
        assert st["n_shadow"][0] == int((~np.all(want == 0, 1)).sum())
    else:                         # a continuation exactly where the sampled pdf is > 0
        spawned = extra[0]
        assert st["n_cont"][0] == int(spawned.sum())
        passing = view["m"]["transparency"] < 0.5
        rough_byte = np.rint(view["m"]["roughness"] * 255).astype(int)
        nan = np.isnan(got).any(1)
        assert nan.sum() > 50 and (rough_byte[nan] == NAN_BYTE).all() and extra[3][nan].all()
        assert np.allclose(got[passing], np.array(M.SKY_C), rtol=1e-6, atol=0)


@pytest.mark.parametrize("control", M.CONTROLS)
@pytest.mark.parametrize("kind", ["direct", "sky"])
def test_negative_controls_are_rejected(kind, control):
    view, got, _ = ka_frame(kind)
    want, extra = known_answer(kind, view, control)
    bad, n, zero_bad = compare(kind, view, got, want, extra)
    print(kind, control, "outside", bad, "of", n, "zero-pattern mismatches", zero_bad)
    assert bad + zero_bad > 50, (kind, control)


def test_pass_through_le_threshold_is_indistinguishable():
    """The literal mistake `transparency <= 0.5` for `< 0.5` changes nothing: no byte b gives b / 255 == 0.5 in float32, so the
    negative control moves the threshold by one byte instead (pass_through_le_128, test_negative_controls_are_rejected)."""
    t = (np.arange(256, dtype=np.float32) / np.float32(255.0)).astype(np.float32)
    assert not (t == np.float32(0.5)).any()
    assert t[127] < 0.5 < t[128]
