"""
GPU tests (-m gpu) of the sampled lights (RT_OPT_EMITTER_SAMPLING, RT_OPT_ENV_SAMPLING, rt_set_light_selection) on device paths the
shipped scenes never take with them on, bit for bit against the CPU model (tests/light_model.cpp), radiance and per-bounce counters:

- emitters with an emission texture (the emitter-side uv and texture lookup of a light sample) next to a transparency texture;
- five analytic lights, point and directional (the analytic sample divided by 1 - (P_e + P_v)), seen through a thin lens;
- environment images of odd sizes (7x5, 1x3, 3x1) and a sky with a few-texel sun;
- a closed box at 60 bounces, where every path ends by its sampled direction's pdf.
"""
import numpy as np
import pytest

from raytracing_b200 import capi
from raytracing_b200.camera import default_camera
from tests.helpers import bits, scene
from tests.light_model import LightModel
from tests.scenes_extra import closed_cornell, many_lights_scene, textured_cornell
from tests.test_env_sampling_cpu import SKEW
from tests.test_gpu_parity import SCHEDULES, check_stats

pytestmark = pytest.mark.gpu

CONFIGS = {"emitters": (True, False, (1.0, 1.0, 1.0)), "env": (False, True, (1.0, 1.0, 1.0)), "both": (True, True, (1.0, 1.0, 1.0)),
           "both_skewed": (True, True, SKEW)}


def set_byte(word, shift, value):
    return (int(word) & ~(0xFF << shift) | (value << shift)) & 0xFFFFFFFF


def textured_lamp_cornell():
    """textured_cornell() with the lamp's material carrying an emission texture and another material a transparency texture."""
    sc = dict(textured_cornell())
    mats = sc["materials"].copy()
    lamp = int(sc["triangles"]["mtlIndex"][sc["emissive"][0]])
    other = (lamp + 1) % len(mats)
    mats["ior_emission_idx_transparency"][lamp] = set_byte(mats["ior_emission_idx_transparency"][lamp], 8, 0)
    mats["ior_emission_idx_transparency"][other] = set_byte(mats["ior_emission_idx_transparency"][other], 24, 1)
    sc["materials"] = mats
    return sc


def sky(w, h, sun=False, seed=3):
    """An RGBA32F sky with a vertical gradient (bright zenith row 0, dim nadir) and, optionally, a few-texel sun."""
    rng = np.random.default_rng(seed)
    v = (np.arange(h) + 0.5) / h
    img = np.zeros((h, w, 4), "<f4")
    img[..., 0] = (1.2 - v)[:, None] * 0.8
    img[..., 1] = (1.2 - v)[:, None] * 0.9
    img[..., 2] = (1.3 - 0.8 * v)[:, None]
    img[..., :3] *= 1.0 + 0.2 * rng.random((h, w, 1))
    if sun:
        j, i = h // 4, int(rng.integers(0, w - 2))
        img[j:j + 2, i:i + 2, :3] = 300.0
    return img


def under_sky(name, img):
    sc = dict(scene(name))
    h, w = img.shape[:2]
    sc["env"], sc["env_width"], sc["env_height"] = img.reshape(-1), w, h
    return sc


CASES = {
    "textured_lamp": (textured_lamp_cornell, {}, 4),
    "many_lights_lens": (lambda: many_lights_scene("CornellBox"), dict(position=(0.15, -1.3, 0.9), aperture=0.04, focus_distance=1.7), 4),
    "sky_7x5": (lambda: under_sky("CornellBox", sky(7, 5)), {}, 4),
    "sky_1x3": (lambda: under_sky("CornellBox", sky(1, 3)), {}, 4),
    "sky_3x1": (lambda: under_sky("CornellBox", sky(3, 1)), {}, 4),
    "sky_sun": (lambda: under_sky("CornellBox", sky(16, 32, sun=True)), {}, 4),
}


def compare(sc, cam_kw, mb, config, schedule, w=96, h=64, samples=2):
    cam = default_camera(w, h, **cam_kw)
    em, env, wts = CONFIGS[config]
    m = LightModel(sc)
    c = capi.Context(w, h)
    try:
        c.upload_scene(sc); c.set_camera(cam)
        for k, v in SCHEDULES.get(schedule, ()):
            c.set_option(k, v)
        c.set_option(capi.OPT_EMITTER_SAMPLING, int(em)); c.set_option(capi.OPT_ENV_SAMPLING, int(env))
        c.set_light_selection(*wts)
        if schedule == "stepwise":
            c.integrate(mb)            # the stepwise steps take the last bounce from the last rt_integrate call
        c.reset()
        acc = np.zeros((h, w, 4), "<f4")
        for s in range(samples):
            _, _, ost = m.render(cam, w, h, mb, s, radiance=acc, emitters=em, env=env, weights=wts)
            c.integrate_stepwise(mb) if schedule == "stepwise" else c.integrate(mb)
            check_stats(c.frame_stats(), ost, mb, (config, schedule, s))
            assert np.array_equal(bits(c.read_radiance()[..., :3]), bits(acc[..., :3])), (config, schedule, s)
        return acc
    finally:
        c.destroy()


@pytest.mark.parametrize("schedule", ["frame", "phase_graph", "stepwise"])
@pytest.mark.parametrize("config", ["env", "both", "both_skewed"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_scene_matches_model(case, config, schedule):
    build, cam_kw, mb = CASES[case]
    compare(build(), cam_kw, mb, config, schedule)


@pytest.mark.parametrize("schedule", ["frame", "phase_graph", "stepwise"])
@pytest.mark.parametrize("config", ["emitters", "both"])
def test_closed_box_60_bounces_matches_model(config, schedule):
    compare(closed_cornell(), {}, 60, config, schedule, w=64, h=48)
