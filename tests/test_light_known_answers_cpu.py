"""
Known-answer tests of the sampled lights on the CPU model (tests/light_model.cpp, held bit for bit to the kernels): frames of the
floor-under-lamps scenes of tests/analytic_light.py against their float64 expectations, per pixel and channel, for every
combination of the options and weights.  Unlike the same-expectation tests, which compare two arms of the product, the reference
here is an independent closed form or quadrature, so a bias common to every arm shows too.
"""
import numpy as np
import pytest
from scipy.stats import t as student_t

from raytracing_b200.camera import default_camera
from tests.analytic_light import CAMERA, expected_image, gradient_sky, known_answer_scene
from tests.light_model import LightModel
from tests.test_env_sampling_cpu import SKEW

MB = 2
# arm: (scene kind, emitters, env, weights)
ARMS = {
    "off": (dict(sky="grad_nosun"), False, False, (1.0, 1.0, 1.0)),
    "emitters": (dict(), True, False, (1.0, 1.0, 1.0)),
    "env": (dict(sky="grad"), False, True, (1.0, 1.0, 1.0)),
    "both": (dict(sky="grad"), True, True, (1.0, 1.0, 1.0)),
    "both_skewed": (dict(sky="grad"), True, True, SKEW),
    "all_kinds": (dict(sky="grad", point=0.6), True, True, (1.0, 1.0, 1.0)),
    "ggx": (dict(floor="ggx"), True, False, (1.0, 1.0, 1.0)),
    "textured": (dict(textured=True), True, False, (1.0, 1.0, 1.0)),
    # environment images of odd sizes (w x h): rows 36 to 180 degrees tall, where p_v's sin theta must be the direction's
    "env_7x5": (dict(sky=(7, 5)), True, True, (1.0, 1.0, 1.0)),
    "env_1x3": (dict(sky=(1, 3)), False, True, (1.0, 1.0, 1.0)),
    "env_3x1": (dict(sky=(3, 1)), True, True, SKEW),
}


def arm_scene(kind, sky_size=(32, 16)):
    """(reference kind, scene) of an arm.  BSDF sampling alone meets the sun too rarely for normal batch means: the arm with both
    options off sees the gradient without it."""
    k = dict(kind)
    if k.get("sky") in ("grad", "grad_nosun"):
        k["sky"] = gradient_sky(*sky_size, sun=k["sky"] == "grad")
    elif isinstance(k.get("sky"), tuple):
        k["sky"] = gradient_sky(*k["sky"], i_sun=2)
    return k, known_answer_scene(floor=k.get("floor", "lambert"), sky=k.get("sky"), point=k.get("point", 0.0), textured=k.get("textured", False))


def check_against_reference(batch_means, ref, where, max_rel_bias, control):
    """batch_means (B, h, w, 3) against ref (h, w, 3): per pixel and channel |t| under the Bonferroni threshold (family-wise 1e-3,
    t with B - 1 degrees of freedom), mean z^2 in [0.8, 1.25], the global relative bias within 5 sigma and max_rel_bias, and the
    global check rejecting the reference scaled by `control`.  Returns the statistics it printed."""
    B = batch_means.shape[0]
    mean = batch_means.mean(0)
    se = batch_means.std(0, ddof=1) / np.sqrt(B)
    z = (mean - ref) / se
    n = z.size
    thr = student_t.isf(1e-3 / (2 * n), B - 1)
    tot = batch_means.reshape(B, -1).sum(1)
    gse = tot.std(ddof=1) / np.sqrt(B)
    bias = (tot.mean() - ref.sum()) / ref.sum()
    gz = (tot.mean() - ref.sum()) / gse
    cz = (tot.mean() - control * ref.sum()) / gse
    stats = dict(max_t=float(np.abs(z).max()), mean_z2=float(np.mean(z * z)), bias=float(bias), bias_sigma=float(gz),
                 control_sigma=float(cz), threshold=float(thr))
    print("%s: max |t| %.2f (threshold %.2f), mean z^2 %.3f, global bias %.2e (%.2f sigma, 1 sigma = %.1e); reference x %g at %.1f sigma"
          % (where, stats["max_t"], thr, stats["mean_z2"], bias, gz, gse / ref.sum(), control, cz))
    assert np.all(np.isfinite(z)), where
    assert np.abs(z).max() < thr, where
    assert 0.8 <= np.mean(z * z) <= 1.25, where
    assert abs(gz) < 5 and abs(bias) < max_rel_bias, where
    assert abs(cz) > 5, where
    return stats


@pytest.mark.parametrize("arm", sorted(ARMS))
def test_model_frames_match_the_float64_expectation(arm):
    kind, em, env, wts = ARMS[arm]
    k, sc = arm_scene(kind)
    # BSDF sampling alone meets the lamps rarely: its batch means need more samples to be near normal
    w, h, spp, B = 32, 24, 4096 if arm == "off" else 1024, 32
    cam = default_camera(w, h, **CAMERA)
    m = LightModel(sc)
    _, _, st = m.render(cam, w, h, MB, 0, emitters=em, env=env, weights=wts, model=True)
    assert st["n_miss"][0] == 0 and st["n_emissive_hits"][0] == 0           # every primary ray hits the floor
    ref = expected_image(k, cam, w, h)
    per = spp // B
    bm = np.zeros((B, h, w, 3))
    acc = np.zeros((h, w, 4), "<f4")
    prev = np.zeros((h, w, 3))
    for b in range(B):
        for s in range(b * per, (b + 1) * per):
            m.render(cam, w, h, MB, s, radiance=acc, emitters=em, env=env, weights=wts, model=True)
        cur = acc[..., :3].astype(np.float64)
        bm[b] = (cur - prev) / per
        prev = cur
    check_against_reference(bm, ref, "model %s" % arm, 1e-2, 1.02)
