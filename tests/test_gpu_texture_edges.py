"""
GPU tests (-m gpu) of the textured-material path at its edges (tests/texture_cases.py), where the kernels decode packed materials
and sample textures per hit (rt_device.cuh: unpack_material, sample_texture):

- the texture chart and a textured OBJ loaded by the host loader, under every rt_integrate schedule, the stepwise steps,
  rt_integrate_samples (per-phase and one-kernel frames) and rank 2 of a 3-way partition, 3 progressive samples of 6 bounces, bit for
  bit against the oracle: radiance, per-bounce counters, the AOVs and the stepwise arm's primary hits;
- known answers at max_bounces = 0 without the oracle: the chart's albedo AOV is the numpy restatement of
  tests/test_texture_edges_cpu.py, and the emission ladder's radiance is ldexp(mantissa, e - 136) in float64 at every covered
  pixel, on the untextured and the per-hit variant alike, subnormal exponents included;
- a 4K frame of tiled charts, where k_shade_queues sorts its continuation rays, against the oracle on a band of rows;
- the ladder's textured emitters sampled as lights (RT_OPT_EMITTER_SAMPLING) against tests/light_model.cpp;
- rt_upload_scene refuses a texture whose last texel lies at or beyond index 2^31, without launching a kernel.
"""
import ctypes as C
import mmap

import numpy as np
import pytest

from oracle.orcbind import Oracle
from raytracing_b200 import capi
from raytracing_b200.camera import default_camera
from tests import texture_cases as T
from tests.helpers import bits
from tests.test_gpu_parity import EVERY, check_stats, run_frame, schedule_ctx
from tests.test_gpu_samples import make as samples_ctx
from tests.test_gpu_schedules import sm_count
from tests.test_texture_edges_cpu import check_albedo, ladder_expected

pytestmark = pytest.mark.gpu

MB, SAMPLES = 6, 3
_scenes = {}


def chart():
    if "chart" not in _scenes:
        _scenes["chart"] = (T.chart_scene(), T.chart_camera(T.CHART_W, T.CHART_H), T.CHART_W, T.CHART_H)
    return _scenes["chart"]


def obj(tmp_path_factory):
    if "obj" not in _scenes:
        w, h = 160, 96
        _scenes["obj"] = (T.obj_scene(str(tmp_path_factory.mktemp("edges_obj"))), default_camera(w, h), w, h)
    return _scenes["obj"]


def assert_aovs(got, want, where):
    for name, g, o in zip(("albedo", "depth", "normal"), got, want):
        assert np.array_equal(bits(g), bits(o)), tuple(where) + (name,)


@pytest.mark.parametrize("case", ["chart", "obj"])
def test_every_schedule_matches_oracle(case, tmp_path_factory):
    sc, cam, w, h = chart() if case == "chart" else obj(tmp_path_factory)
    if case == "obj":
        assert len(sc["textures"]) >= 6 and (sc["materials"]["ior_emission_idx_transparency"] >> 24 != 0xFF).any()
    o = Oracle(sc)
    ctxs = {s: schedule_ctx(s, sc, cam, w, h, ((capi.OPT_AOV_ALWAYS, 1),)) for s in EVERY}
    part = schedule_ctx(None, sc, cam, w, h, rank=2, world=3)
    try:
        for c in list(ctxs.values()) + [part]:
            c.reset()
        acc = np.zeros((h, w, 4), "<f4"); pacc = np.zeros((h, w, 4), "<f4")
        for s in range(SAMPLES):
            acc, hits, ost = o.render(cam, w, h, MB, sample_idx=s, radiance=acc)
            aovs = o.aovs(cam, cam, w, h, sample_idx=s)
            stepwise = ctxs["stepwise"]          # its primary hits first: the stepwise frame then regenerates the same rays
            stepwise.generate_rays(); stepwise.intersect(0)
            dh, pix = stepwise.read_hits(0)
            prim = np.full(w * h, 0xFFFFFFFE, np.uint32); prim[pix] = dh["primitive_id"]
            bc = np.zeros((w * h, 2), np.float32); bc[pix] = dh["bc"]
            assert np.array_equal(prim, hits["primitive_id"]), (case, s)
            assert np.array_equal(bits(bc), bits(hits["bc"])), (case, s)
            for name, c in ctxs.items():
                where = (case, name, "sample %d" % s)
                run_frame(c, name, MB)
                check_stats(c.frame_stats(), ost, MB, where)
                assert np.array_equal(bits(c.read_radiance()[..., :3]), bits(acc[..., :3])), where
                assert_aovs(c.read_aovs(), aovs, where)
            pacc, _, pst = o.render(cam, w, h, MB, sample_idx=s, radiance=pacc, row_first=2, row_step=3)
            part.integrate(MB)
            check_stats(part.frame_stats(), pst, MB, (case, "rank 2 of 3", s))
            rows = np.arange(2, h, 3)
            rad = np.zeros((h, w, 4), "<f4"); part.read_radiance(rad)
            assert np.array_equal(bits(rad[rows][..., :3]), bits(pacc[rows][..., :3])), (case, "rank 2 of 3", s)
        for fk in (0, 1):                 # rt_integrate_samples: the per-phase frames, the one-kernel frames
            c = samples_ctx(sc, cam, w, h, ((capi.OPT_FRAME_KERNEL, fk),))
            c.integrate_samples(MB, SAMPLES)
            assert c.sample_count() == SAMPLES
            assert np.array_equal(bits(c.read_radiance()[..., :3]), bits(acc[..., :3])), (case, "samples", fk)
            c.destroy()
    finally:
        for c in list(ctxs.values()) + [part]:
            c.destroy()


def test_chart_albedo_is_the_restatement():
    """max_bounces = 0: the device's albedo AOV at every pixel against the numpy restatement from the device's own primary hits."""
    sc, cam, w, h = chart()
    c = schedule_ctx("stepwise", sc, cam, w, h, ((capi.OPT_AOV_ALWAYS, 1),))
    try:
        c.reset()
        c.generate_rays(); c.intersect(0)
        dh, pix = c.read_hits(0)
        prim = np.full(w * h, 0xFFFFFFFF, np.uint32); prim[pix] = dh["primitive_id"]
        bc = np.zeros((w * h, 2), np.float32); bc[pix] = dh["bc"]
        c.integrate_stepwise(0)
        al = c.read_aovs()[0].reshape(-1, 4)
        textured, _, _, uv32 = check_albedo(sc, prim, bc, al)
        assert textured.sum() > 10000 and np.isnan(uv32[textured]).any()
    finally:
        c.destroy()


@pytest.mark.parametrize("schedule", ["frame", "phase_graph", "stepwise"])
def test_ladder_radiance_is_the_emission(schedule):
    """max_bounces = 0, one sample: radiance = ldexp(mantissa, e - 136) bit for bit at every pixel of an untextured or per-hit
    quad, for all 256 exponent bytes; exponents below 10 give subnormal emission on both paths."""
    sc = T.ladder_scene()
    w, h = T.LADDER_W, T.LADDER_H
    cam = default_camera(w, h)
    c, hc = schedule_ctx(schedule, sc, cam, w, h), schedule_ctx("stepwise", sc, cam, w, h)
    try:
        c.reset(); hc.reset()
        run_frame(c, schedule, 0)
        rad = c.read_radiance().reshape(-1, 4)
        hc.generate_rays(); hc.intersect(0)              # the primary hits of sample 0, from a context of their own
        dh, pix = hc.read_hits(0)
        prim = np.full(w * h, 0xFFFFFFFF, np.uint32); prim[pix] = dh["primitive_id"]
    finally:
        c.destroy(); hc.destroy()
    px, want, where = ladder_expected(sc, prim)
    got = rad[px, :3]
    bad = np.flatnonzero((bits(got) != bits(want.astype(np.float32))).any(1))
    assert len(bad) == 0, [(where[i], got[i].tolist(), want[i].tolist()) for i in bad[:4]]
    assert {(v, e) for v, e in where} == {(v, e) for v in ("untextured", "per_hit") for e in range(256)}
    assert (want[[e < 10 for _, e in where]] < 2.0 ** -126).any()


def test_4k_sorted_shading_matches_oracle():
    """3840 x 2160 of 5 x 5 tiled charts: above 32 K local pixels per SM, so k_shade_queues sorts its continuation rays; the
    per-phase default and the one-kernel frame agree on the whole frame and a band of 18 rows equals the oracle."""
    w, h, mb, tile = 3840, 2160, 4, 5
    assert w * h > 32768 * sm_count()
    sc = T.chart_scene(tile)
    cam = T.chart_camera(w, h, tile)
    imgs = []
    for fk in (2, 1):
        c = schedule_ctx(None, sc, cam, w, h, ((capi.OPT_FRAME_KERNEL, fk),))
        assert c.local_pixel_count() > 32768 * sm_count()
        c.reset(); c.integrate(mb)
        imgs.append(c.read_radiance()); c.destroy()
    assert np.array_equal(bits(imgs[0]), bits(imgs[1]))
    row_first, row_step = 13, 120
    orad, hits, _ = Oracle(sc).render(cam, w, h, mb, row_first=row_first, row_step=row_step)
    rows = np.arange(row_first, h, row_step)
    assert len(rows) >= 17
    prim = hits["primitive_id"].reshape(h, w)[rows]
    assert (prim != 0xFFFFFFFF).mean() > 0.3                  # the charts cover most of the band
    assert np.array_equal(bits(imgs[0][rows][..., :3]), bits(orad[rows][..., :3]))


@pytest.mark.parametrize("schedule", ["frame", "phase_graph", "stepwise"])
def test_ladder_emitters_sampled_as_lights_match_model(schedule):
    """RT_OPT_EMITTER_SAMPLING on the per-hit (1x1 white emission texture) and random ladders lighting a floor: exponents 0..140,
    so the emitter table stays finite; the textured emission is looked up at the light sample's uv."""
    from tests.test_gpu_sampled_light_scenes import compare
    sc = T.ladder_scene(exponents=range(0, 141), variants=("per_hit", "random"), floor=True)
    assert len(sc["emissive"]) > 200
    compare(sc, {}, 3, "emitters", schedule, w=128, h=96)


def test_upload_refuses_texels_beyond_2_31():
    """A texture whose last texel index reaches 2^31 (data_start + width * height > 2^31) is refused with
    RT_ERR_INVALID_ARGUMENT before anything is copied: the texel array is a lazily zeroed mapping no page of which is touched.
    A texture ending exactly at 2^31 - 1 passes this check (the upload itself is not attempted here)."""
    sc = T.ladder_scene(exponents=range(2), variants=("untextured",))
    n = (1 << 31) + 64
    buf = mmap.mmap(-1, 4 * n, flags=mmap.MAP_PRIVATE | mmap.MAP_ANONYMOUS | getattr(mmap, "MAP_NORESERVE", 0))
    texels = np.frombuffer(buf, dtype="<u4")
    tex = np.zeros(1, T.TEXTURE_DT)
    tex[0] = ((1 << 31) - 8, 4, 3, 0)                   # texels 2^31 - 8 .. 2^31 + 3
    mats = sc["materials"].copy()
    mats["diffuse_albedo"][0] = T.rgb_word(10, 20, 30, 0)
    c = capi.Context(64, 48)
    try:
        a = {k: np.ascontiguousarray(sc[k]) for k in ("triangles", "nodes", "lights", "env", "emissive")}
        a["materials"] = mats
        d = capi.RtSceneDesc()
        d.triangles, d.n_triangles = a["triangles"].ctypes.data, len(a["triangles"])
        d.nodes, d.n_nodes = a["nodes"].ctypes.data, len(a["nodes"])
        d.materials, d.n_materials = a["materials"].ctypes.data, len(a["materials"])
        d.lights, d.n_lights = a["lights"].ctypes.data, len(a["lights"])
        d.textures, d.n_textures = tex.ctypes.data, 1
        d.texture_data, d.n_texture_data = texels.ctypes.data, n
        d.env_image, d.env_width, d.env_height = a["env"].ctypes.data, int(sc["env_width"]), int(sc["env_height"])
        info = np.ascontiguousarray(sc["scene_info"]).view("<u4").ravel()
        for i in range(4):
            d.scene_info[i] = int(info[i])
        rc = c.lib.rt_upload_scene(c.h, C.byref(d))
        assert rc == -1, rc                                 # RT_ERR_INVALID_ARGUMENT
        assert b"2^31" in c.lib.rt_last_error(c.h)
    finally:
        c.destroy()
        del texels
        buf.close()
