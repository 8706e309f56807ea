"""
GPU tests (-m gpu) of the shading pass across the packed material space (tests/material_cases.py): the material chart (every
value of every byte field, channel edges, a cross grid, black and white corners) at the default and a grazing pose, its per-hit
twin, the normal panel, the light placements and the mirror case.

- Every rt_integrate schedule, the stepwise steps, rt_integrate_samples (per-phase and one-kernel frames) and rank 2 of a 3-way
  partition, 2 progressive samples of 6 bounces with kRandom and with blue noise, bit for bit against the oracle: radiance,
  per-bounce counters, the AOVs and the stepwise arm's primary hits.
- The untextured chart (mat_rec) and its per-hit twin (unpack_material) give byte-identical radiance, counters and AOVs.
- The float64 known answers of tests/test_material_edges_cpu.py on the device's own frames and primary hits: (a) direct light at
  0 bounces, (b) a constant sky through the sampled direction at 1 bounce.
- Emitter sampling with an emissive panel over the chart and environment sampling under CornellBox's sky, against the light
  model (tests/light_model.cpp): bxdf_eval_sampled and mis_power's NaN -> 0 rule on every material.
- A 4K frame of tiled charts, where k_shade_queues sorts its continuation rays, against the oracle on a band of rows.
"""
import numpy as np
import pytest

from oracle.orcbind import Oracle
from raytracing_b200 import capi
from raytracing_b200.layouts import TRIANGLE_DT
from tests import material_cases as M
from tests import test_material_edges_cpu as T
from tests.helpers import bits
from tests.test_gpu_parity import EVERY, check_stats, run_frame, schedule_ctx
from tests.test_gpu_samples import make as samples_ctx
from tests.test_gpu_schedules import sm_count

pytestmark = pytest.mark.gpu

MB, SAMPLES = 6, 2


def assert_aovs(got, want, where):
    for name, g, o in zip(("albedo", "depth", "normal"), got, want):
        assert np.array_equal(bits(g), bits(o)), tuple(where) + (name,)


def with_tables(c, tables):
    if tables is not None:
        c.upload_sampler_tables(*tables); c.set_option(capi.OPT_SAMPLER, 1)
    return c


def device_hits(c, w, h):
    """Primary hits of the context's next sample through the stepwise steps: -> {'primitive_id', 'bc'} over the whole frame."""
    c.generate_rays(); c.intersect(0)
    dh, pix = c.read_hits(0)
    prim = np.full(w * h, 0xFFFFFFFF, np.uint32); prim[pix] = dh["primitive_id"]
    bc = np.zeros((w * h, 2), np.float32); bc[pix] = dh["bc"]
    return {"primitive_id": prim, "bc": bc}


@pytest.mark.parametrize("sampler", ["random", "blue_noise"])
@pytest.mark.parametrize("case", sorted(T.SCENES))
def test_every_schedule_matches_oracle(case, sampler):
    sc, cam, w, h = T.cached(case)
    tables = T.sampler_tables(sampler)
    o = Oracle(sc)
    ctxs = {s: with_tables(schedule_ctx(s, sc, cam, w, h, ((capi.OPT_AOV_ALWAYS, 1),)), tables) for s in EVERY}
    part = with_tables(schedule_ctx(None, sc, cam, w, h, rank=2, world=3), tables)
    try:
        o.set_sampler_tables(tables)
        for c in list(ctxs.values()) + [part]:
            c.reset()
        acc = np.zeros((h, w, 4), "<f4"); pacc = np.zeros((h, w, 4), "<f4")
        for s in range(SAMPLES):
            acc, hits, ost = o.render(cam, w, h, MB, sample_idx=s, radiance=acc)
            aovs = o.aovs(cam, cam, w, h, sample_idx=s)
            dh = device_hits(ctxs["stepwise"], w, h)       # the stepwise frame then regenerates the same rays
            assert np.array_equal(dh["primitive_id"], hits["primitive_id"]), (case, s)
            assert np.array_equal(bits(dh["bc"]), bits(hits["bc"])), (case, s)
            for name, c in ctxs.items():
                where = (case, sampler, name, "sample %d" % s)
                run_frame(c, name, MB)
                check_stats(c.frame_stats(), ost, MB, where)
                assert np.array_equal(bits(c.read_radiance()[..., :3]), bits(acc[..., :3])), where
                assert_aovs(c.read_aovs(), aovs, where)
            pacc, _, pst = o.render(cam, w, h, MB, sample_idx=s, radiance=pacc, row_first=2, row_step=3)
            part.integrate(MB)
            check_stats(part.frame_stats(), pst, MB, (case, sampler, "rank 2 of 3", s))
            rows = np.arange(2, h, 3)
            rad = np.zeros((h, w, 4), "<f4"); part.read_radiance(rad)
            assert np.array_equal(bits(rad[rows][..., :3]), bits(pacc[rows][..., :3])), (case, sampler, "rank 2 of 3", s)
        for fk in (0, 1):                 # rt_integrate_samples: the per-phase frames, the one-kernel frames
            c = samples_ctx(sc, cam, w, h, ((capi.OPT_FRAME_KERNEL, fk),), tables=tables)
            try:
                c.integrate_samples(MB, SAMPLES)
                assert c.sample_count() == SAMPLES
                assert np.array_equal(bits(c.read_radiance()[..., :3]), bits(acc[..., :3])), (case, sampler, "samples", fk)
            finally:
                c.destroy()
    finally:
        o.set_sampler_tables(None)
        for c in list(ctxs.values()) + [part]:
            c.destroy()


@pytest.mark.parametrize("schedule", ["frame", "phase_graph", "stepwise"])
def test_untextured_and_per_hit_paths_agree(schedule):
    """The chart through mat_rec and its per-hit twin through unpack_material: byte-identical radiance, counters and AOVs."""
    out = []
    for name in ("chart", "per_hit"):
        sc, cam, w, h = T.cached(name)
        c = schedule_ctx(schedule, sc, cam, w, h, ((capi.OPT_AOV_ALWAYS, 1),))
        try:
            c.reset()
            run_frame(c, schedule, MB); run_frame(c, schedule, MB)
            st = c.frame_stats()
            out.append((c.read_radiance(), {k: st[k][: MB + 1].copy() for k in st.dtype.names}, c.read_aovs()))
        finally:
            c.destroy()
    (ra, sa, aa), (rb, sb, ab) = out
    assert np.array_equal(bits(ra), bits(rb))
    for k in sa:
        assert np.array_equal(sa[k], sb[k]), k
    for x, y in zip(aa, ab):
        assert np.array_equal(bits(x), bits(y))


@pytest.mark.parametrize("kind", ["direct", "sky"])
def test_known_answers_on_device(kind):
    """Frames (a) and (b) of the chart on the device, against the float64 restatement from the device's own primary hits."""
    sc = M.direct_frame_scene() if kind == "direct" else M.sky_frame_scene()
    cam, w, h = M.chart_camera(T.CW, T.CH), T.CW, T.CH
    mb = 0 if kind == "direct" else 1
    c, hc = schedule_ctx(None, sc, cam, w, h), schedule_ctx("stepwise", sc, cam, w, h)
    try:
        c.reset(); hc.reset()
        c.integrate(mb)
        rad = c.read_radiance().reshape(-1, 4)
        st = c.frame_stats()
        hits = device_hits(hc, w, h)
    finally:
        c.destroy(); hc.destroy()
    view = M.primary_view(sc, cam, w, h, hits)
    got = rad[view["px"], :3]
    want, extra = T.known_answer(kind, view)
    bad, n, zero_bad = T.compare(kind, view, got, want, extra)
    assert n > 15000 and bad == 0 and zero_bad == 0, (kind, n, bad, zero_bad)
    if kind == "direct":
        assert st["n_shadow"][0] == int((~np.all(want == 0, 1)).sum())
    else:
        assert st["n_cont"][0] == int(extra[0].sum())


def emitter_panel(z=2.7, x=(-1.2, 1.2), y=(-0.6, 0.9)):
    """Two triangles on the plane z, facing -z (down onto the chart's upper rows)."""
    t = np.zeros(2, TRIANGLE_DT)
    for k, ps in enumerate(([(x[0], y[0]), (x[0], y[1]), (x[1], y[1])], [(x[0], y[0]), (x[1], y[1]), (x[1], y[0])])):
        for v, p in zip(("v1", "v2", "v3"), ps):
            t[k][v]["position"][:3] = (p[0], p[1], z)
            t[k][v]["normal"][:3] = (0.0, 0.0, -1.0)
    return t


def lit_chart():
    """The chart with an emissive panel above it (and CornellBox's lights and sky)."""
    from tests.texture_cases import finish
    base = M.chart_scene()
    mats = list(base["materials"]) + [M.material(emission=(255, 230, 200, 129), diffuse=(0, 0, 0), roughness=255)]
    panel = emitter_panel(); panel["mtlIndex"] = len(mats) - 1
    # the chart's triangles in their (leaf) order plus the panel; finish() rebuilds the tree
    sc = finish([base["triangles"], panel], mats, *M.WHITE_TEX)
    sc["tags"] = base["tags"] + [("panel", 0)]
    assert len(sc["emissive"]) == 2
    return sc


@pytest.mark.parametrize("schedule", ["frame", "phase_graph", "stepwise"])
@pytest.mark.parametrize("config", ["emitters", "env"])
def test_light_sampling_on_the_chart_matches_model(config, schedule):
    from tests.test_gpu_sampled_light_scenes import compare
    compare(lit_chart(), {}, 3, config, schedule, w=T.CW, h=T.CH)


def test_4k_sorted_shading_matches_oracle():
    """3840 x 2160 of 3 x 3 tiled charts: above 32 K local pixels per SM, so k_shade_queues sorts its continuation rays; the
    per-phase default and the one-kernel frame agree on the whole frame and a band of rows equals the oracle."""
    w, h, mb, tile = 3840, 2160, 4, 3
    assert w * h > 32768 * sm_count()
    sc = M.chart_scene(tile=tile)
    cam = M.chart_camera(w, h, tile)
    imgs = []
    for fk in (2, 1):
        c = schedule_ctx(None, sc, cam, w, h, ((capi.OPT_FRAME_KERNEL, fk),))
        try:
            assert c.local_pixel_count() > 32768 * sm_count()
            c.reset(); c.integrate(mb)
            imgs.append(c.read_radiance())
        finally:
            c.destroy()
    assert np.array_equal(bits(imgs[0]), bits(imgs[1]))
    row_first, row_step = 13, 120
    orad, hits, _ = Oracle(sc).render(cam, w, h, mb, row_first=row_first, row_step=row_step)
    rows = np.arange(row_first, h, row_step)
    assert len(rows) >= 17
    prim = hits["primitive_id"].reshape(h, w)[rows]
    assert (prim != 0xFFFFFFFF).mean() > 0.3
    assert np.array_equal(bits(imgs[0][rows][..., :3]), bits(orad[rows][..., :3]))
