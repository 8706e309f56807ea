"""
GPU tests (-m gpu) of the two-plane shadow records and the shared BSDF constants.

A shadow ray toward a directional light stores only planes sA and sC; the shadow pass takes its direction and t_max from the
light's record.  Every other shadow ray (point lights, emitter and environment samples) keeps plane sB.  evaluate_material,
sample_bxdf and bxdf_eval_sampled take their per-material constants from one derivation (rt_device.cuh derive_bsdf), and
sample_bxdf skips the Fresnel term of materials without specular.

- Radiance bits and per-bounce counters equal the oracle's on every schedule (per-phase, one-kernel frame, stepwise),
  rt_integrate_samples on the one-kernel frame and both ranks of a 2-way partition, for one directional light, several
  directional lights, a point light among directional lights, and materials with and without specular, metals and textures.
  With emitter and environment sampling on, every schedule agrees with the one-kernel frame.
"""
import numpy as np
import pytest

from oracle.orcbind import Oracle
from raytracing_b200 import capi
from raytracing_b200.camera import default_camera
from tests import material_cases as M
from tests.helpers import bits, scene

F = np.float32

W, H, MB = 64, 48, 4
SCHEDULES = {
    "frame": ((capi.OPT_FRAME_KERNEL, 1),),
    "phase_graph": ((capi.OPT_FRAME_KERNEL, 0),),
    "timed": ((capi.OPT_KERNEL_TIMING, 1),),
    "stepwise": ((capi.OPT_FRAME_KERNEL, 0),),
}


def with_lights(sc, lights):
    sc = dict(sc)
    out = np.zeros(len(lights), dtype=sc["lights"].dtype)
    for i, (kind, origin, rad) in enumerate(lights):
        out[i]["origin"][:3] = origin; out[i]["radiance"][:3] = rad; out[i]["type"] = kind
    sc["lights"] = out
    info = np.array(sc["scene_info"], copy=True); info["analytic_light_count"] = len(out)
    sc["scene_info"] = info
    return sc


def unit(d):
    d = np.asarray(d, F)
    return d / F(np.sqrt((d * d).sum(dtype=F)))


SCENES = {
    "one_directional": (lambda: scene("CornellBox"), default_camera),
    "three_directional": (lambda: with_lights(scene("CornellBox"), [(1, unit((-0.2, -0.4, 0.9)), (1.0, 0.9, 0.8)),
                                                                    (1, unit((0.5, -0.3, 0.8)), (0.5, 0.5, 1.0)),
                                                                    (1, unit((0.0, 0.0, 1.0)), (0.7, 0.7, 0.7))]), default_camera),
    "point_among_directional": (lambda: with_lights(scene("CornellBox"), [(1, unit((-0.2, -0.4, 0.9)), (1.0, 0.9, 0.8)),
                                                                          (0, (0.1, 0.2, 1.8), (3.0, 3.0, 3.0)),
                                                                          (1, unit((0.4, -0.6, 0.7)), (0.6, 0.8, 1.0))]), default_camera),
    "shader_balls": (lambda: scene("ShaderBalls"), default_camera),
    "chart_specular_metals": (lambda: with_lights(M.chart_scene(), [(1, unit((-0.3, -0.8, 0.5)), (3.0, 2.5, 2.0))]), M.chart_camera),
    "chart_textured": (lambda: with_lights(M.chart_scene("per_hit"), [(1, unit((-0.3, -0.8, 0.5)), (3.0, 2.5, 2.0)),
                                                                      (0, (0.0, -0.5, 1.5), (2.0, 2.0, 2.0))]), M.chart_camera),
}


def ctx(sc, cam, schedule, rank=0, world=1, options=()):
    c = capi.Context(W, H, rank=rank, world=world)
    c.upload_scene(sc); c.set_camera(cam)
    for k, v in SCHEDULES.get(schedule, ()) + tuple(options):
        c.set_option(k, v)
    c.reset()
    return c


def run(c, schedule, samples):
    for _ in range(samples):
        c.integrate_stepwise(MB) if schedule == "stepwise" else c.integrate(MB)


def oracle(sc, cam, samples):
    o = Oracle(sc)
    acc = np.zeros((H, W, 4), "<f4")
    stats = []
    for s in range(samples):
        acc, _, st = o.render(cam, W, H, MB, sample_idx=s, radiance=acc)
        stats.append(st)
    return acc, stats


def check_stats(st, ost, where):
    for k in ("n_ext", "n_miss", "n_shadow", "n_cont", "n_unoccluded"):
        assert np.array_equal(np.asarray(st[k][: MB + 1]), np.asarray(ost[k][: MB + 1])), (k,) + where


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SCENES))
def test_every_schedule_matches_oracle(name):
    build, camera = SCENES[name]
    sc = build(); cam = camera(W, H)
    oacc, ost = oracle(sc, cam, 2)
    for schedule in SCHEDULES:
        c = ctx(sc, cam, schedule)
        try:
            run(c, schedule, 2)
            assert np.array_equal(bits(c.read_radiance()[..., :3]), bits(oacc[..., :3])), (name, schedule)
            check_stats(c.frame_stats(), ost[-1], (name, schedule))
        finally:
            c.destroy()
    # rt_integrate_samples on the one-kernel frame: two samples in one call
    c = ctx(sc, cam, "frame")
    try:
        c.integrate_samples(MB, 2)
        assert np.array_equal(bits(c.read_radiance()[..., :3]), bits(oacc[..., :3])), (name, "integrate_samples")
    finally:
        c.destroy()
    # both ranks of a 2-way partition, per-phase and one-kernel frame
    for schedule in ("frame", "phase_graph"):
        for rank in (0, 1):
            c = ctx(sc, cam, schedule, rank=rank, world=2)
            try:
                run(c, schedule, 2)
                rad = c.read_radiance()
                assert np.array_equal(bits(rad[rank::2, :, :3]), bits(oacc[rank::2, :, :3])), (name, schedule, rank)
            finally:
                c.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("light", ("emitters", "environment", "both"))
def test_sampled_lights_agree_across_schedules(light):
    """Emitter and environment samples keep three-plane shadow records next to the two-plane ones of the directional light: every
    schedule agrees with the one-kernel frame."""
    sc = scene("CornellBox"); cam = default_camera(W, H)
    opts = (((capi.OPT_EMITTER_SAMPLING, 1),) if light in ("emitters", "both") else ()) + \
           (((capi.OPT_ENV_SAMPLING, 1),) if light in ("environment", "both") else ())
    want = ctx(sc, cam, "frame", options=opts)
    try:
        run(want, "frame", 2)
        wrad, wst = want.read_radiance(), want.frame_stats()
    finally:
        want.destroy()
    assert int(np.asarray(wst["n_shadow"][: MB + 1]).sum()) > 0
    for schedule in ("phase_graph", "timed", "stepwise"):
        c = ctx(sc, cam, schedule, options=opts)
        try:
            if schedule == "stepwise":
                c.integrate(MB); c.reset()          # the stepwise steps take the frame's last bounce from the last rt_integrate call
            run(c, schedule, 2)
            assert np.array_equal(bits(c.read_radiance()[..., :3]), bits(wrad[..., :3])), (light, schedule)
            check_stats(c.frame_stats(), wst, (light, schedule))
        finally:
            c.destroy()
