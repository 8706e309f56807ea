"""
GPU tests (-m gpu) of the spatial denoiser (rt_set_spatial_denoiser).  Every comparison is bit for bit: the filtered resolve against
the scalar model (tests/spatial_denoise_model.c) applied to the context's own unfiltered resolve and AOVs, and end to end against the
model applied to the oracle's resolve and AOVs; everything the filter must not touch against a context with it off.
"""
import numpy as np
import pytest
import torch

from oracle.orcbind import Oracle
from raytracing_b200 import capi
from raytracing_b200.camera import default_camera
from tests import sd_model
from tests.helpers import bits, scene
from tests.test_gpu_parity import run_frame, schedule_ctx

pytestmark = pytest.mark.gpu

SIGMAS = (0.3, 0.25, 0.15)                   # colour, normal, depth
SETTINGS = [(i,) + SIGMAS for i in range(1, 6)] + [(5, 0.0, 0.25, 0.15), (5, 0.3, 0.0, 0.15), (5, 0.3, 0.25, 0.0), (3, 0.0, 0.0, 0.0)]
NOT_READY, INVALID, UNSUPPORTED = -4, -1, -5


def model_of(c, setting):
    """The model applied to context c's unfiltered resolve and its AOVs (the filter is switched off for the read and back on)."""
    c.set_spatial_denoiser(0)
    raw = c.resolve()
    _, depth, normal, _ = c.read_aovs()
    c.set_spatial_denoiser(*setting)
    return sd_model.filter_image(raw, normal, depth, *setting), raw


def assert_filtered(c, setting, where=()):
    c.set_spatial_denoiser(*setting)
    got = c.resolve()
    want, _ = model_of(c, setting)
    assert np.array_equal(bits(got), bits(want)), (setting,) + tuple(where)
    return got


def oracle_frames(name, cam, w, h, mb, n):
    """The oracle's accumulation after n samples, its resolve and the AOVs of the last sample."""
    o = Oracle(scene(name))
    acc = np.zeros((h, w, 4), "<f4")
    for s in range(n):
        acc, _, _ = o.render(cam, w, h, mb, sample_idx=s, radiance=acc, want_hits=False)
    zero_cam = np.zeros_like(np.asarray(cam))
    al, de, no, ve = o.aovs(cam, zero_cam, w, h, sample_idx=n - 1)
    return o.resolve(0, acc, al, de, no, ve, n), de, no


@pytest.mark.parametrize("schedule", ["frame", "phase_graph", "stepwise"])
@pytest.mark.parametrize("name,w,h,mb", [("CornellBox", 96, 64, 3), ("ShaderBalls", 120, 72, 4)])
def test_filter_equals_the_model(name, w, h, mb, schedule):
    """Every iteration count and each sigma dropped in turn, on every schedule: the context's own unfiltered resolve and AOVs through
    the model, and the oracle's resolve and AOVs through the model, end to end."""
    cam = default_camera(w, h)
    c = schedule_ctx(schedule, scene(name), cam, w, h)
    c.set_spatial_denoiser(*SETTINGS[0])
    c.reset()
    for _ in range(2):
        run_frame(c, schedule, mb)
    ores, odepth, onormal = oracle_frames(name, cam, w, h, mb, 2)
    for st in SETTINGS:
        got = assert_filtered(c, st, (name, schedule))
        want = sd_model.filter_image(ores, onormal, odepth, *st)
        assert np.array_equal(bits(got), bits(want)), ("oracle", st, name, schedule)
    c.destroy()


def test_resolve_async_and_device_target():
    """rt_resolve_async delivers the filtered image, twice in a row (both resolve buffers), equal to rt_resolve's."""
    name, w, h, mb = "ShaderBalls", 97, 61, 3
    c = schedule_ctx("phase_graph", scene(name), default_camera(w, h), w, h)
    st = (4,) + SIGMAS
    c.set_spatial_denoiser(*st)
    c.reset(); c.integrate(mb)
    want = assert_filtered(c, st)
    outs = [np.zeros((h, w, 4), "<f4") for _ in range(2)]
    for o in outs:
        c.resolve_async(o)
    c.resolve_wait()
    for o in outs:
        assert np.array_equal(bits(o), bits(want))
    c.destroy()


@pytest.mark.parametrize("schedule", ["frame", "phase_graph"])
def test_integrate_samples(schedule):
    """rt_integrate_samples with N = 4: the model of the context's own image, and the image of four single frames."""
    name, w, h, mb, n = "CornellBox", 96, 64, 3, 4
    sc, cam = scene(name), default_camera(w, h)
    st = (5,) + SIGMAS
    a = schedule_ctx(schedule, sc, cam, w, h); a.set_spatial_denoiser(*st); a.reset(); a.integrate_samples(mb, n)
    b = schedule_ctx(schedule, sc, cam, w, h); b.set_spatial_denoiser(*st); b.reset()
    for _ in range(n):
        b.integrate(mb)
    got = assert_filtered(a, st)
    assert np.array_equal(bits(got), bits(b.resolve()))
    a.destroy(); b.destroy()


def test_adaptive_sampling_with_stopped_pixels():
    """With adaptive sampling the filter runs on the per-pixel-count resolve and the AOVs stopped pixels kept."""
    name, w, h, mb = "CornellBox", 128, 128, 3
    c = schedule_ctx("phase_graph", scene(name), default_camera(w, h), w, h)
    st = (5,) + SIGMAS
    c.set_adaptive_sampling(0.01, 4)
    c.set_spatial_denoiser(*st)
    c.reset()
    for _ in range(16):
        c.integrate(mb)
    assert 0 < c.active_pixels() < w * h
    assert len(np.unique(c.pixel_samples())) > 1
    assert_filtered(c, st)
    # turned on after frames rendered without AOVs: not ready until a reset and a frame (the stopped pixels have no guides)
    d = schedule_ctx("phase_graph", scene(name), default_camera(w, h), w, h)
    d.set_adaptive_sampling(0.01, 4); d.reset()
    for _ in range(8):
        d.integrate(mb)
    d.set_spatial_denoiser(*st)
    d.integrate(mb)
    with pytest.raises(capi.RtError) as e:
        d.resolve()
    assert e.value.code == NOT_READY
    d.reset(); d.integrate(mb)
    assert_filtered(d, st)
    c.destroy(); d.destroy()


def test_temporal_denoiser_on():
    """Under the temporal denoiser the filter's input is the radiance alone through Reinhard."""
    name, w, h, mb = "CornellBox", 96, 64, 3
    c = schedule_ctx("phase_graph", scene(name), default_camera(w, h), w, h)
    st = (5,) + SIGMAS
    c.set_option(capi.OPT_DENOISER, 1)
    c.set_spatial_denoiser(*st)
    c.reset()
    for _ in range(3):
        c.integrate(mb)
        c.denoise(); c.copy_history()
    assert_filtered(c, st)
    c.destroy()


@pytest.mark.parametrize("w,h,iters", [(97, 61, 5), (7, 5, 5), (1, 40, 5), (40, 1, 5), (1, 1, 3), (33, 9, 2)])
def test_sizes_no_tile_divides(w, h, iters):
    c = schedule_ctx("frame", scene("ShaderBalls"), default_camera(w, h), w, h)
    st = (iters,) + SIGMAS
    c.set_spatial_denoiser(*st)
    c.reset(); c.integrate(3); c.integrate(3)
    assert_filtered(c, st, (w, h))
    c.destroy()


def test_full_1080p_frame():
    w, h = 1920, 1080
    c = schedule_ctx("phase_graph", scene("CornellBox"), default_camera(w, h), w, h)
    st = (5,) + SIGMAS
    c.set_spatial_denoiser(*st)
    c.reset(); c.integrate(8)
    assert_filtered(c, st)
    c.destroy()


def test_non_finite_pixels():
    """NaN and inf written into the device radiance: the filtered image equals the model's, and no non-finite value spreads."""
    name, w, h, mb = "ShaderBalls", 120, 72, 3
    c = schedule_ctx("phase_graph", scene(name), default_camera(w, h), w, h)
    st = (5,) + SIGMAS
    c.set_spatial_denoiser(*st)
    c.reset(); c.integrate(mb); c.integrate(mb)
    c.sync()
    ptr, _ = c.radiance_device_ptr()
    n = w * h

    class _Slab:
        __cuda_array_interface__ = {"shape": (n, 4), "typestr": "<f4", "data": (ptr, False), "version": 3, "strides": None}
    rad = torch.as_tensor(_Slab(), device="cuda")
    bad = [(5, 7), (30, 60), (31, 60), (71, 119), (0, 0), (40, 10)]
    vals = [float("nan"), float("inf"), -float("inf"), float("nan"), float("inf"), float("nan")]
    for (y, x), v in zip(bad, vals):
        rad[y * w + x, (y + x) % 3] = v
    torch.cuda.synchronize()
    got = assert_filtered(c, st)
    keep = np.ones((h, w), bool)
    for y, x in bad:
        keep[y, x] = False
    assert np.isfinite(got[keep]).all()
    c.destroy()


def test_nothing_else_changes_and_toggling_between_graph_frames():
    """Radiance, statistics, AOVs, sample counts and the AOV views equal a context with the filter off (and the AOVs forced on);
    toggling the filter between per-phase graph frames renders the same frames as fresh contexts."""
    name, w, h, mb = "ShaderBalls", 120, 72, 4
    sc, cam = scene(name), default_camera(w, h)
    on = schedule_ctx("phase_graph", sc, cam, w, h); on.set_spatial_denoiser(5, *SIGMAS); on.reset()
    off = schedule_ctx("phase_graph", sc, cam, w, h, ((capi.OPT_AOV_ALWAYS, 1),)); off.reset()
    tog = schedule_ctx("phase_graph", sc, cam, w, h); tog.reset()
    for k in range(4):
        tog.set_spatial_denoiser(*((5,) + SIGMAS if k % 2 == 0 else (0,)))
        for c in (on, off, tog):
            c.integrate(mb)
        on.resolve()
        for c in (on, tog):
            assert np.array_equal(bits(c.read_radiance()), bits(off.read_radiance())), k
            for key in ("n_ext", "n_miss", "n_shadow", "n_cont", "n_unoccluded", "n_emissive_hits"):
                assert np.array_equal(c.frame_stats()[key], off.frame_stats()[key]), (k, key)
            assert np.array_equal(c.pixel_samples(), off.pixel_samples())
        for x, y in zip(on.read_aovs(), off.read_aovs()):
            assert np.array_equal(bits(x), bits(y)), k
    # the last toggled frame ran with the filter off: no guides of that frame
    tog.set_spatial_denoiser(5, *SIGMAS)
    with pytest.raises(capi.RtError) as e:
        tog.resolve()
    assert e.value.code == NOT_READY
    tog.integrate(mb); on.integrate(mb); off.integrate(mb)
    assert np.array_equal(bits(tog.resolve()), bits(on.resolve()))
    for v in (1, 2, 3, 4):
        on.set_option(capi.OPT_AOV, v); off.set_option(capi.OPT_AOV, v)
        assert np.array_equal(bits(on.resolve()), bits(off.resolve())), v
    for c in (on, off, tog):
        c.destroy()


def test_errors_and_refused_combinations():
    name, w, h, mb = "CornellBox", 64, 48, 2
    sc, cam = scene(name), default_camera(w, h)

    def refused(code, fn, *args):
        with pytest.raises(capi.RtError) as e:
            fn(*args)
        assert e.value.code == code, (fn, args)

    c = schedule_ctx("frame", sc, cam, w, h)
    for bad in ((6, 0.3, 0.2, 0.1), (1, -0.1, 0.2, 0.1), (1, 0.3, -1.0, 0.1), (1, 0.3, 0.2, -1e-9), (1, float("nan"), 0.2, 0.1),
                (1, 0.3, float("inf"), 0.1), (1, 0.3, 0.2, float("nan")), (0, -1.0, 0.0, 0.0)):
        refused(INVALID, c.set_spatial_denoiser, *bad)
    c.set_spatial_denoiser(2, *SIGMAS)
    c.reset()
    refused(NOT_READY, c.resolve)                          # no frame has written AOVs yet
    refused(NOT_READY, c.resolve_async, np.zeros((h, w, 4), "<f4"))
    c.integrate(mb)
    assert_filtered(c, (2,) + SIGMAS)
    # the gathered resolve, in both orders
    ptr, nbytes = c.radiance_device_ptr()
    refused(UNSUPPORTED, c.resolve_gathered, ptr, w * h * 16)
    c.set_spatial_denoiser(0)
    c.resolve_gathered(ptr, w * h * 16)
    c.set_spatial_denoiser(2, *SIGMAS)
    refused(UNSUPPORTED, c.resolve_gathered, ptr, w * h * 16)
    # a partition, in both orders
    refused(UNSUPPORTED, lambda: c._ck(c.lib.rt_set_partition(c.h, 0, 2)))
    c.set_spatial_denoiser(0)
    c._ck(c.lib.rt_set_partition(c.h, 0, 2))
    refused(UNSUPPORTED, c.set_spatial_denoiser, 2, *SIGMAS)
    c.destroy()
    p = schedule_ctx("frame", sc, cam, w, h, rank=1, world=2)
    refused(UNSUPPORTED, p.set_spatial_denoiser, 1, *SIGMAS)
    p.destroy()
    # a multi-device context (one device listed twice)
    m = capi.Context(w, h, devices=[0, 0])
    refused(UNSUPPORTED, m.set_spatial_denoiser, 1, *SIGMAS)
    m.set_spatial_denoiser(0)
    m.destroy()


def test_device_rt_expf_equals_host():
    """rt_math_eval fn 10 (sm_90a, -fmad=false) equals the host rt_expf (-ffp-contract=off) bit for bit."""
    from tests.test_spatial_denoise_cpu import expf_arguments
    x = np.concatenate([expf_arguments(4321), -np.abs(np.random.default_rng(5).normal(0, 20, 1 << 18)).astype("<f4")])
    dev = capi.math_eval("exp", x)
    hst = sd_model.expf(x)
    assert np.array_equal(bits(dev), bits(hst))


def test_host_render_matches_the_c_abi(tmp_path):
    from raytracing_b200 import hostapi
    from tests.test_host import PROC_OBJ, make_env
    w, h, mb, n = 160, 90, 5, 4
    env_path, _ = make_env(tmp_path, w=64, h=32)
    s = hostapi.HostScene(PROC_OBJ)
    s.add_directional_light((-0.6, -1.5, 3.5), (15, 10, 5))
    r = hostapi.HostRender(s, w, h, env_path)
    r.set_max_bounces(mb)
    r.set_samples_per_frame(n)
    r.set_spatial_denoiser(4, *SIGMAS)
    a = s.arrays(); a["nodes"] = r.nodes()
    cam = hostapi.default_camera(w, h)
    c = capi.Context(w, h)
    c.upload_scene(a); c.set_camera(cam)
    c.set_spatial_denoiser(4, *SIGMAS)
    r.render_frame()
    c.reset(); c.integrate_samples(mb, n)
    assert np.array_equal(bits(r.image()), bits(c.resolve()))
    assert np.array_equal(bits(c.resolve()), bits(model_of(c, (4,) + SIGMAS)[0]))
    r.close(); s.close(); c.destroy()
