"""
GPU tests (-m gpu) of emitter sampling (RT_OPT_EMITTER_SAMPLING): every schedule against the CPU model of the rule
(tests/emitter_model.cpp) bit for bit, the inactive cases against the option off, the same-expectation test at GPU scale, and
the argument checks.
"""
import numpy as np
import pytest

from raytracing_b200 import capi
from raytracing_b200.camera import default_camera
from tests.emitter_model import EmitterModel
from tests.helpers import bits, scene, synthetic_sampler_tables
from tests.test_emitter_sampling_cpu import get_scene
from tests.test_gpu_parity import SCHEDULES, check_stats

pytestmark = pytest.mark.gpu

EMIT = ((capi.OPT_EMITTER_SAMPLING, 1),)


def ctx_for(sc, cam, w, h, schedule, options=(), **kw):
    c = capi.Context(w, h, **kw)
    c.upload_scene(sc); c.set_camera(cam)
    for k, v in SCHEDULES.get(schedule, ()) + tuple(options):
        c.set_option(k, v)
    return c


def run(c, schedule, mb):
    if schedule == "stepwise":
        c.integrate_stepwise(mb)
    else:
        c.integrate(mb)


@pytest.mark.parametrize("sampler", ["random", "blue_noise"])
@pytest.mark.parametrize("schedule", ["frame", "phase_graph", "phase_direct", "stepwise"])
@pytest.mark.parametrize("name", ["CornellBox", "ShaderBalls", "procedural"])
def test_schedules_match_model(name, schedule, sampler):
    sc = get_scene(name)
    w, h, mb = 96, 64, 4
    cam = default_camera(w, h)
    m = EmitterModel(sc)
    tables = synthetic_sampler_tables() if sampler == "blue_noise" else None
    m.set_sampler_tables(tables)
    c = ctx_for(sc, cam, w, h, schedule, EMIT)
    if tables is not None:
        c.upload_sampler_tables(*tables); c.set_option(capi.OPT_SAMPLER, 1)
    if schedule == "stepwise":
        c.integrate(mb)            # the stepwise steps take the last bounce from the last rt_integrate call
    c.reset()
    acc = np.zeros((h, w, 4), "<f4")
    try:
        for s in range(2):
            m.render(cam, w, h, mb, s, radiance=acc, emitters=True)
            _, _, ost = m.render(cam, w, h, mb, s, radiance=np.zeros_like(acc), emitters=True)
            run(c, schedule, mb)
            check_stats(c.frame_stats(), ost, mb, (name, schedule, sampler, s))
            assert np.array_equal(bits(c.read_radiance()[..., :3]), bits(acc[..., :3])), (name, schedule, sampler, s)
    finally:
        c.destroy(); m.set_sampler_tables(None)


@pytest.mark.parametrize("name", ["CornellBox", "ShaderBalls"])
def test_multi_sample_frame_kernel_setting_and_partitions_match_model(name):
    """rt_integrate_samples with RT_OPT_FRAME_KERNEL 1 (N one-kernel frames with the option on), a 3-way partition, and a multi-device
    context that lists device 0 three times."""
    sc = scene(name)
    w, h, mb, n = 80, 48, 3, 3
    cam = default_camera(w, h)
    m = EmitterModel(sc)
    acc = np.zeros((h, w, 4), "<f4")
    for s in range(n):
        m.render(cam, w, h, mb, s, radiance=acc, emitters=True)
    c = ctx_for(sc, cam, w, h, "frame", EMIT)
    c.reset(); c.integrate_samples(mb, n)
    assert np.array_equal(bits(c.read_radiance()[..., :3]), bits(acc[..., :3]))
    c.destroy()
    for rank in range(3):
        part = np.zeros((h, w, 4), "<f4")
        for s in range(n):
            m.render(cam, w, h, mb, s, row_first=rank, row_step=3, radiance=part, emitters=True)
        c = ctx_for(sc, cam, w, h, "phase_graph", EMIT, rank=rank, world=3)
        c.reset()
        for _ in range(n):
            c.integrate(mb)
        rows = np.arange(rank, h, 3)
        assert np.array_equal(bits(c.read_radiance()[rows][..., :3]), bits(part[rows][..., :3])), rank
        c.destroy()
    c = ctx_for(sc, cam, w, h, "frame", EMIT, devices=[0, 0, 0])
    c.reset()
    for _ in range(n):
        c.integrate(mb)
    assert np.array_equal(bits(c.read_radiance()[..., :3]), bits(acc[..., :3]))
    c.destroy()


def test_sorted_shading_pass_matches_model():
    """A 4K frame takes the sorted shading pass (k_shade_queues<true>); a band of rows against the model."""
    sc = scene("CornellBox")
    w, h, mb = 3840, 2160, 2
    cam = default_camera(w, h)
    m = EmitterModel(sc)
    ref = m.render(cam, w, h, mb, 0, row_first=5, row_step=173, emitters=True)[0]
    c = ctx_for(sc, cam, w, h, "phase_graph", EMIT)
    c.reset(); c.integrate(mb)
    rows = np.arange(5, h, 173)
    assert np.array_equal(bits(c.read_radiance()[rows][..., :3]), bits(ref[rows][..., :3]))
    c.destroy()


def test_adaptive_sampling_each_pixel_matches_model_at_its_count():
    sc = scene("CornellBox")
    w, h, mb = 64, 48, 3
    cam = default_camera(w, h)
    c = ctx_for(sc, cam, w, h, "frame", EMIT)
    c.set_adaptive_sampling(0.02, 2)
    c.reset()
    for _ in range(8):
        c.integrate(mb)
    counts = c.pixel_samples()
    rad = c.read_radiance()
    c.destroy()
    assert counts.min() < counts.max()
    m = EmitterModel(sc)
    acc = np.zeros((h, w, 4), "<f4")
    seen = np.zeros((h, w), bool)
    for s in range(int(counts.max())):
        m.render(cam, w, h, mb, s, radiance=acc, emitters=True)
        at = counts == s + 1
        assert np.array_equal(bits(rad[at][..., :3]), bits(acc[at][..., :3])), s
        seen |= at
    assert seen.all()


@pytest.mark.parametrize("case", ["no_emitters", "white_furnace"])
def test_inactive_is_byte_identical_to_off(case):
    sc = dict(scene("CornellBox"))
    if case == "no_emitters":
        sc["emissive"] = np.zeros(0, "<u4")
    w, h, mb = 64, 48, 3
    cam = default_camera(w, h)
    out = []
    for opt in (0, 1):
        c = ctx_for(sc, cam, w, h, "phase_graph", ((capi.OPT_EMITTER_SAMPLING, opt), (capi.OPT_WHITE_FURNACE, int(case == "white_furnace"))))
        c.reset(); c.integrate(mb); c.integrate(mb)
        out.append((c.read_radiance(), c.frame_stats()))
        c.destroy()
    assert out[0][0].tobytes() == out[1][0].tobytes() and out[0][1].tobytes() == out[1][1].tobytes()


def test_argument_checks_and_switching_mid_accumulation():
    sc = dict(scene("CornellBox"))
    w, h, mb = 32, 24, 3
    cam = default_camera(w, h)
    c = ctx_for(sc, cam, w, h, "frame")
    with pytest.raises(capi.RtError) as e:
        c.set_option(capi.OPT_EMITTER_SAMPLING, 2)
    assert e.value.code == -1
    bad = dict(sc); bad["emissive"] = np.array([0, 0], "<u4")
    c.upload_scene(bad)                                # permissive with the option off
    with pytest.raises(capi.RtError) as e:
        c.set_option(capi.OPT_EMITTER_SAMPLING, 1)
    assert e.value.code == -1
    c.upload_scene(sc)
    c.set_option(capi.OPT_EMITTER_SAMPLING, 1)
    for idx in ([len(sc["triangles"])], [1, 1]):
        bad = dict(sc); bad["emissive"] = np.array(idx, "<u4")
        with pytest.raises(capi.RtError) as e:
            c.upload_scene(bad)
        assert e.value.code == -1
    c.upload_scene(sc)
    # switching mid-accumulation: sample 0 off, sample 1 on, sample 2 off
    m = EmitterModel(sc)
    acc = np.zeros((h, w, 4), "<f4")
    c.set_option(capi.OPT_EMITTER_SAMPLING, 0)
    c.reset()
    for s, on in enumerate((False, True, False)):
        c.set_option(capi.OPT_EMITTER_SAMPLING, int(on))
        c.integrate(mb)
        m.render(cam, w, h, mb, s, radiance=acc, emitters=on)
        assert np.array_equal(bits(c.read_radiance()[..., :3]), bits(acc[..., :3])), s
    c.destroy()


@pytest.mark.parametrize("name", ["procedural", "CornellBox"])
def test_same_expectation_at_gpu_scale(name):
    """64x64, 8192 samples per arm in 32 batches (disjoint sample indices); per 8x8 tile and channel z = (m_on - m_off) / se."""
    sc = get_scene(name)
    w = h = 64
    mb, n, batches = 3, 8192, 32
    cam = default_camera(w, h)
    means = {}
    for on in (1, 0):
        c = ctx_for(sc, cam, w, h, "frame", ((capi.OPT_EMITTER_SAMPLING, on),))
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
    tile = lambda x: x.reshape(x.shape[0], h // 8, 8, w // 8, 8, 3).mean((2, 4))
    ton, toff = tile(means[1]), tile(means[0])
    se = lambda t: t.std(0, ddof=1) / np.sqrt(batches)
    # tiles without noise (the sky seen directly) differ only by the rounding of the float accumulations, which is about 2e-4 of
    # their value after 16 K samples: tiles whose standard error is below 3e-4 of their value are left out
    var = se(ton) ** 2 + se(toff) ** 2
    z = (ton.mean(0) - toff.mean(0)) / np.sqrt(var)
    z = z[np.isfinite(z) & (np.sqrt(var) > 3e-4 * np.abs(toff.mean(0)))]
    print("%s: max |z| %.2f, mean z^2 %.2f" % (name, np.abs(z).max(), np.mean(z * z)))
    assert np.all(np.abs(z) < 5)
    assert 0.5 <= np.mean(z * z) <= 2.0


def test_host_render_set_emitter_sampling_matches_the_c_abi(tmp_path):
    """Render::SetEmitterSampling through hostapi: the image of every frame equals the C ABI's with the same option sequence
    (on for two frames, then off: the accumulation is kept), and the option changes the image."""
    from raytracing_b200 import hostapi
    from tests.test_host import PROC_OBJ, make_env
    w, h, mb, n = 160, 90, 5, 4
    env_path, _ = make_env(tmp_path, w=64, h=32)
    s = hostapi.HostScene(PROC_OBJ)
    s.add_directional_light((-0.6, -1.5, 3.5), (15, 10, 5))
    r = hostapi.HostRender(s, w, h, env_path)
    r.set_max_bounces(mb)
    r.set_samples_per_frame(n)
    a = s.arrays(); a["nodes"] = r.nodes()
    assert len(a["emissive"]) > 0
    cam = hostapi.default_camera(w, h)
    c = capi.Context(w, h)
    c.upload_scene(a); c.set_camera(cam)
    off = capi.Context(w, h)
    off.upload_scene(a); off.set_camera(cam)
    c.reset(); off.reset()
    try:
        for frame, on in enumerate((True, True, False)):
            r.set_emitter_sampling(on)
            c.set_option(capi.OPT_EMITTER_SAMPLING, int(on))
            r.render_frame()
            c.integrate_samples(mb, n); off.integrate_samples(mb, n)
            img = c.resolve()
            assert np.array_equal(bits(r.image()), bits(img)), frame
            assert not np.array_equal(bits(img), bits(off.resolve())), frame
    finally:
        r.close(); s.close(); c.destroy(); off.destroy()
