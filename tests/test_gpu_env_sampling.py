"""
GPU tests (-m gpu) of environment sampling (RT_OPT_ENV_SAMPLING) and the light-kind weights (rt_set_light_selection): every schedule
against the CPU model of the rules (tests/light_model.cpp) bit for bit, the inactive cases against a context that never set them,
the same-expectation test at GPU scale, the argument checks, and the host layers.
"""
import os
import subprocess

import numpy as np
import pytest

from raytracing_b200 import capi
from raytracing_b200.camera import default_camera
from tests.helpers import bits, scene, synthetic_sampler_tables
from tests.light_model import LightModel
from tests.test_emitter_sampling_cpu import get_scene
from tests.test_env_sampling_cpu import SKEW, sun_scene, z_scores
from tests.test_gpu_parity import SCHEDULES, check_stats

pytestmark = pytest.mark.gpu

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# (emitters, env, weights): environment alone, both kinds, both kinds with skewed weights
CONFIGS = {"env": (False, True, (1.0, 1.0, 1.0)), "both": (True, True, (1.0, 1.0, 1.0)), "both_skewed": (True, True, SKEW)}


def ctx_for(sc, cam, w, h, schedule, config=None, options=(), **kw):
    c = capi.Context(w, h, **kw)
    c.upload_scene(sc); c.set_camera(cam)
    for k, v in SCHEDULES.get(schedule, ()) + tuple(options):
        c.set_option(k, v)
    if config is not None:
        em, env, wts = CONFIGS[config]
        c.set_option(capi.OPT_EMITTER_SAMPLING, int(em)); c.set_option(capi.OPT_ENV_SAMPLING, int(env))
        c.set_light_selection(*wts)
    return c


def model_kw(config):
    em, env, wts = CONFIGS[config]
    return dict(emitters=em, env=env, weights=wts)


def run(c, schedule, mb):
    if schedule == "stepwise":
        c.integrate_stepwise(mb)
    else:
        c.integrate(mb)


@pytest.mark.parametrize("config", sorted(CONFIGS))
@pytest.mark.parametrize("sampler", ["random", "blue_noise"])
@pytest.mark.parametrize("schedule", ["frame", "phase_graph", "phase_direct", "stepwise"])
@pytest.mark.parametrize("name", ["CornellBox", "ShaderBalls", "procedural"])
def test_schedules_match_model(name, schedule, sampler, config):
    sc = get_scene(name)
    w, h, mb = 96, 64, 4
    cam = default_camera(w, h)
    m = LightModel(sc)
    tables = synthetic_sampler_tables() if sampler == "blue_noise" else None
    m.set_sampler_tables(tables)
    c = ctx_for(sc, cam, w, h, schedule, config)
    if tables is not None:
        c.upload_sampler_tables(*tables); c.set_option(capi.OPT_SAMPLER, 1)
    if schedule == "stepwise":
        c.integrate(mb)            # the stepwise steps take the last bounce from the last rt_integrate call
    c.reset()
    acc = np.zeros((h, w, 4), "<f4")
    try:
        for s in range(2):
            m.render(cam, w, h, mb, s, radiance=acc, **model_kw(config))
            _, _, ost = m.render(cam, w, h, mb, s, radiance=np.zeros_like(acc), **model_kw(config))
            run(c, schedule, mb)
            check_stats(c.frame_stats(), ost, mb, (name, schedule, sampler, config, s))
            assert np.array_equal(bits(c.read_radiance()[..., :3]), bits(acc[..., :3])), (name, schedule, sampler, config, s)
    finally:
        c.destroy(); m.set_sampler_tables(None)


@pytest.mark.parametrize("schedule", ["frame", "phase_graph"])
def test_sun_sky_matches_model(schedule):
    """The synthetic sun sky: most environment samples go to a few texels."""
    sc = sun_scene("ShaderBalls")
    w, h, mb = 96, 64, 4
    cam = default_camera(w, h)
    m = LightModel(sc)
    c = ctx_for(sc, cam, w, h, schedule, "both_skewed")
    c.reset()
    acc = np.zeros((h, w, 4), "<f4")
    for s in range(2):
        m.render(cam, w, h, mb, s, radiance=acc, **model_kw("both_skewed"))
        c.integrate(mb)
        assert np.array_equal(bits(c.read_radiance()[..., :3]), bits(acc[..., :3])), s
    c.destroy()


def test_multi_sample_frame_kernel_setting_and_partitions_match_model():
    """rt_integrate_samples with RT_OPT_FRAME_KERNEL 1 (N one-kernel frames with the option on), a 3-way partition, and a multi-device
    context that lists device 0 three times."""
    sc = scene("ShaderBalls")
    w, h, mb, n = 80, 48, 3, 3
    cam = default_camera(w, h)
    m = LightModel(sc)
    acc = np.zeros((h, w, 4), "<f4")
    for s in range(n):
        m.render(cam, w, h, mb, s, radiance=acc, **model_kw("env"))
    c = ctx_for(sc, cam, w, h, "frame", "env")
    c.reset(); c.integrate_samples(mb, n)
    assert np.array_equal(bits(c.read_radiance()[..., :3]), bits(acc[..., :3]))
    c.destroy()
    for rank in range(3):
        part = np.zeros((h, w, 4), "<f4")
        for s in range(n):
            m.render(cam, w, h, mb, s, row_first=rank, row_step=3, radiance=part, **model_kw("env"))
        c = ctx_for(sc, cam, w, h, "phase_graph", "env", rank=rank, world=3)
        c.reset()
        for _ in range(n):
            c.integrate(mb)
        rows = np.arange(rank, h, 3)
        assert np.array_equal(bits(c.read_radiance()[rows][..., :3]), bits(part[rows][..., :3])), rank
        c.destroy()
    acc = np.zeros((h, w, 4), "<f4")
    for s in range(n):
        m.render(cam, w, h, mb, s, radiance=acc, **model_kw("both_skewed"))
    c = ctx_for(sc, cam, w, h, "frame", "both_skewed", devices=[0, 0, 0])
    c.reset()
    for _ in range(n):
        c.integrate(mb)
    assert np.array_equal(bits(c.read_radiance()[..., :3]), bits(acc[..., :3]))
    c.destroy()


def test_sorted_shading_pass_matches_model():
    """A 4K frame takes the sorted shading pass (k_shade_queues<true, true>); a band of rows against the model."""
    sc = scene("ShaderBalls")
    w, h, mb = 3840, 2160, 2
    cam = default_camera(w, h)
    m = LightModel(sc)
    ref = m.render(cam, w, h, mb, 0, row_first=5, row_step=173, **model_kw("both"))[0]
    c = ctx_for(sc, cam, w, h, "phase_graph", "both")
    c.reset(); c.integrate(mb)
    rows = np.arange(5, h, 173)
    assert np.array_equal(bits(c.read_radiance()[rows][..., :3]), bits(ref[rows][..., :3]))
    c.destroy()


def test_adaptive_sampling_each_pixel_matches_model_at_its_count():
    sc = scene("ShaderBalls")
    w, h, mb = 64, 48, 3
    cam = default_camera(w, h)
    c = ctx_for(sc, cam, w, h, "frame", "both")
    c.set_adaptive_sampling(0.05, 2)
    c.reset()
    for _ in range(8):
        c.integrate(mb)
    counts = c.pixel_samples()
    rad = c.read_radiance()
    c.destroy()
    assert counts.min() < counts.max()
    m = LightModel(sc)
    acc = np.zeros((h, w, 4), "<f4")
    seen = np.zeros((h, w), bool)
    for s in range(int(counts.max())):
        m.render(cam, w, h, mb, s, radiance=acc, **model_kw("both"))
        at = counts == s + 1
        assert np.array_equal(bits(rad[at][..., :3]), bits(acc[at][..., :3])), s
        seen |= at
    assert seen.all()


def test_switching_option_and_weights_between_frames():
    sc = scene("ShaderBalls")
    w, h, mb = 48, 32, 3
    cam = default_camera(w, h)
    m = LightModel(sc)
    steps = [(False, False, (1.0, 1.0, 1.0)), (False, True, (1.0, 1.0, 1.0)), (True, True, SKEW), (True, False, SKEW),
             (False, True, (2.0, 1.0, 0.25)), (False, False, (2.0, 1.0, 0.25))]
    for schedule in ("frame", "phase_graph", "stepwise"):
        c = ctx_for(sc, cam, w, h, schedule)
        c.integrate(mb)
        c.reset()
        acc = np.zeros((h, w, 4), "<f4")
        for s, (em, env, wts) in enumerate(steps):
            c.set_option(capi.OPT_EMITTER_SAMPLING, int(em)); c.set_option(capi.OPT_ENV_SAMPLING, int(env))
            c.set_light_selection(*wts)
            run(c, schedule, mb)
            m.render(cam, w, h, mb, s, radiance=acc, emitters=em, env=env, weights=wts)
            assert np.array_equal(bits(c.read_radiance()[..., :3]), bits(acc[..., :3])), (schedule, s)
        c.destroy()


def frames(sc, cam, w, h, mb, setup, schedule="phase_graph"):
    c = ctx_for(sc, cam, w, h, schedule)
    setup(c)
    c.reset(); c.integrate(mb); c.integrate(mb)
    out = (c.read_radiance().tobytes(), c.frame_stats().tobytes())
    c.destroy()
    return out


@pytest.mark.parametrize("schedule", ["frame", "phase_graph"])
def test_inactive_cases_are_byte_identical(schedule):
    """Both options off (whatever the weights), and white furnace with the option on, are byte-identical to a context that never
    set them; emitter sampling alone with the default weights is byte-identical to the emitter frames of a context that never
    called rt_set_light_selection."""
    sc = scene("CornellBox")
    w, h, mb = 64, 48, 3
    cam = default_camera(w, h)
    base = frames(sc, cam, w, h, mb, lambda c: None, schedule)

    def off(c):
        c.set_option(capi.OPT_ENV_SAMPLING, 1); c.set_light_selection(*SKEW); c.set_option(capi.OPT_ENV_SAMPLING, 0)
    assert frames(sc, cam, w, h, mb, off, schedule) == base
    wf = lambda c: c.set_option(capi.OPT_WHITE_FURNACE, 1)
    assert frames(sc, cam, w, h, mb, lambda c: (wf(c), c.set_option(capi.OPT_ENV_SAMPLING, 1)), schedule) == \
        frames(sc, cam, w, h, mb, wf, schedule)
    em = lambda c: c.set_option(capi.OPT_EMITTER_SAMPLING, 1)

    def em_default(c):
        c.set_light_selection(*SKEW); c.set_option(capi.OPT_ENV_SAMPLING, 1); em(c)
        c.set_option(capi.OPT_ENV_SAMPLING, 0); c.set_light_selection(1.0, 1.0, 1.0)
    assert frames(sc, cam, w, h, mb, em_default, schedule) == frames(sc, cam, w, h, mb, em, schedule)


def test_argument_checks():
    sc = scene("CornellBox")
    w, h = 32, 24
    cam = default_camera(w, h)
    c = ctx_for(sc, cam, w, h, "frame")
    for v in (2, 7):
        with pytest.raises(capi.RtError) as e:
            c.set_option(capi.OPT_ENV_SAMPLING, v)
        assert e.value.code == -1
    bad = [(0.0, 1.0, 1.0), (1.0, 0.0, 1.0), (1.0, 1.0, 0.0), (-1.0, 1.0, 1.0), (1.0, -0.5, 1.0), (1.0, 1.0, -2.0),
           (float("nan"), 1.0, 1.0), (1.0, float("inf"), 1.0), (1.0, 1.0, float("-inf")), (3e38, 3e38, 1.0)]
    for wts in bad:
        with pytest.raises(capi.RtError) as e:
            c.set_light_selection(*wts)
        assert e.value.code == -1, wts
    c.destroy()
    c = ctx_for(sc, cam, w, h, "frame", devices=[0, 0])
    with pytest.raises(capi.RtError) as e:
        c.set_light_selection(1.0, 0.0, 1.0)
    assert e.value.code == -1
    c.set_light_selection(*SKEW)
    c.destroy()


@pytest.mark.parametrize("name", ["ShaderBalls", "procedural", "ShaderBalls_sun"])
def test_same_expectation_at_gpu_scale(name):
    """64x64, 8192 samples per arm in 32 batches (disjoint sample indices); per 8x8 tile and channel z = (m_on - m_off) / se, with
    both kinds sampled at skewed weights against both options off (under the sun sky against environment sampling alone at the
    default weights: test_env_sampling_cpu.test_same_expectation_as_the_option_off says why)."""
    sun = name == "ShaderBalls_sun"
    sc = sun_scene("ShaderBalls") if sun else get_scene(name)
    w = h = 64
    mb, n, batches = 3, 8192, 32
    cam = default_camera(w, h)
    means = {}
    for on in (1, 0):
        c = ctx_for(sc, cam, w, h, "frame", "both_skewed" if on else ("env" if sun else None))
        c.reset()
        if not on:
            c.integrate_samples(mb, n)                 # skip the samples the other arm used
        bm = []
        prev = np.zeros((h, w, 3), np.float64) if on else c.read_radiance()[..., :3].astype(np.float64)
        for _ in range(batches):
            c.integrate_samples(mb, n // batches)
            cur = c.read_radiance()[..., :3].astype(np.float64)
            bm.append((cur - prev) / (n // batches))
            prev = cur
        means[on] = np.array(bm)
        c.destroy()
    z = z_scores(means[1], means[0], w, h, batches)
    print("%s: max |z| %.2f, mean z^2 %.2f" % (name, np.abs(z).max(), np.mean(z * z)))
    assert np.all(np.abs(z) < 5)
    assert 0.5 <= np.mean(z * z) <= 2.0


def host_render_setup(tmp_path, w, h):
    from raytracing_b200 import hostapi
    from tests.test_host import PROC_OBJ, make_env
    env_path, _ = make_env(tmp_path, w=64, h=32)
    s = hostapi.HostScene(PROC_OBJ)
    s.add_directional_light((-0.6, -1.5, 3.5), (15, 10, 5))
    r = hostapi.HostRender(s, w, h, env_path)
    return s, r, env_path


def test_host_render_setters_match_the_c_abi(tmp_path):
    """Render::SetEnvironmentSampling / SetLightSelection through hostapi: every frame equals the C ABI's with the same sequence
    (the accumulation is kept), and the options change the image."""
    from raytracing_b200 import hostapi
    w, h, mb, n = 160, 90, 5, 4
    s, r, _ = host_render_setup(tmp_path, w, h)
    r.set_max_bounces(mb)
    r.set_samples_per_frame(n)
    a = s.arrays(); a["nodes"] = r.nodes()
    cam = hostapi.default_camera(w, h)
    c = capi.Context(w, h)
    c.upload_scene(a); c.set_camera(cam)
    off = capi.Context(w, h)
    off.upload_scene(a); off.set_camera(cam)
    c.reset(); off.reset()
    try:
        with pytest.raises(hostapi.HostError):
            r.set_light_selection(1.0, 0.0, 1.0)
        for frame, (em, env, wts) in enumerate([(False, True, (1.0, 1.0, 1.0)), (True, True, SKEW), (False, True, (1.0, 1.0, 4.0))]):
            r.set_emitter_sampling(em); r.set_environment_sampling(env); r.set_light_selection(*wts)
            c.set_option(capi.OPT_EMITTER_SAMPLING, int(em)); c.set_option(capi.OPT_ENV_SAMPLING, int(env)); c.set_light_selection(*wts)
            r.render_frame()
            c.integrate_samples(mb, n); off.integrate_samples(mb, n)
            img = c.resolve()
            assert np.array_equal(bits(r.image()), bits(img)), frame
            assert not np.array_equal(bits(img), bits(off.resolve())), frame
    finally:
        r.close(); s.close(); c.destroy(); off.destroy()


def test_headless_render_env_and_lights_flags(tmp_path):
    """examples/headless_render with env=1 lights=WA,WE,WV writes the image HostRender renders with the same settings."""
    exe = str(tmp_path / "headless_render")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-I" + os.path.join(REPO, "include"), "-I" + os.path.join(REPO, "raytracing_b200", "host"),
                    os.path.join(REPO, "examples", "headless_render.cpp"), "-L" + os.path.join(REPO, "raytracing_b200"), "-l:librt_host.so",
                    "-l:librt_b200.so", "-Wl,-rpath," + os.path.join(REPO, "raytracing_b200"), "-o", exe], check=True)
    from tests.test_host import PROC_OBJ
    w, h, n = 64, 40, 4
    s, r, env_path = host_render_setup(tmp_path, w, h)
    out = str(tmp_path / "out.pfm")
    p = subprocess.run([exe, PROC_OBJ, env_path, str(w), str(h), str(n), out, "env=1", "lights=1,1,3"], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    with open(out, "rb") as f:
        assert f.readline() == b"PF\n" and f.readline() == b"%d %d\n" % (w, h) and f.readline() == b"-1.0\n"
        img = np.frombuffer(f.read(), "<f4").reshape(h, w, 3)[::-1]
    r.set_max_bounces(8); r.set_environment_sampling(True); r.set_light_selection(1, 1, 3); r.set_samples_per_frame(n)
    r.render_frame()
    want = r.image()[..., :3]
    r.close(); s.close()
    assert np.array_equal(bits(img), bits(want))
    p = subprocess.run([exe, PROC_OBJ, env_path, str(w), str(h), str(n), out, "lights=1,1"], capture_output=True, text=True)
    assert p.returncode == 2
