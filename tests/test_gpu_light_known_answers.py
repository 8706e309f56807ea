"""
GPU known-answer tests (-m gpu) of the sampled lights: frames of the floor-under-lamps scenes (tests/analytic_light.py) rendered by
the kernels, 32 batches of 1 024 samples per pixel through rt_integrate_samples on the one-kernel frame and on the per-phase
graph, against their float64 expectations per pixel and channel (tests/test_light_known_answers_cpu.py states the checks).  The
batch means are differences of successive accumulated radiance reads in float64; the float32 accumulation drifts by about 1e-5
relative at these counts, far below the 2e-3 bound on the global bias.
"""
import numpy as np
import pytest

from raytracing_b200 import capi
from raytracing_b200.camera import default_camera
from tests.analytic_light import CAMERA, expected_image
from tests.test_gpu_parity import SCHEDULES
from tests.test_light_known_answers_cpu import ARMS, MB, arm_scene, check_against_reference

pytestmark = pytest.mark.gpu

W, H, BATCHES, PER = 96, 64, 32, 1024
_refs = {}


def reference(arm, cam):
    key = repr(sorted(ARMS[arm][0].items()))          # the arms on one scene share its expectation
    if key not in _refs:
        k, _ = arm_scene(ARMS[arm][0])
        _refs[key] = expected_image(k, cam, W, H)
    return _refs[key]


@pytest.mark.parametrize("schedule", ["frame", "phase_graph"])
@pytest.mark.parametrize("arm", sorted(ARMS))
def test_frames_match_the_float64_expectation(arm, schedule):
    kind, em, env, wts = ARMS[arm]
    _, sc = arm_scene(kind)
    cam = default_camera(W, H, **CAMERA)
    c = capi.Context(W, H)
    try:
        c.upload_scene(sc); c.set_camera(cam)
        for k, v in SCHEDULES[schedule]:
            c.set_option(k, v)
        c.set_option(capi.OPT_EMITTER_SAMPLING, int(em)); c.set_option(capi.OPT_ENV_SAMPLING, int(env))
        c.set_light_selection(*wts)
        c.reset()
        c.integrate(MB)
        st = c.frame_stats()
        assert st["n_miss"][0] == 0 and st["n_emissive_hits"][0] == 0         # every primary ray hits the floor
        c.reset()
        bm = np.zeros((BATCHES, H, W, 3))
        prev = np.zeros((H, W, 3))
        for b in range(BATCHES):
            c.integrate_samples(MB, PER)
            cur = c.read_radiance()[..., :3].astype(np.float64)
            bm[b] = (cur - prev) / PER
            prev = cur
    finally:
        c.destroy()
    check_against_reference(bm, reference(arm, cam), "GPU %s %s" % (arm, schedule), 2e-3, 1.003)
