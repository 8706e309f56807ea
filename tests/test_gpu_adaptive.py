"""
GPU tests (-m gpu) of adaptive sampling (rt_set_adaptive_sampling).  A pixel's path for sample s depends only on (pixel, s, bounce,
camera, scene), so a pixel that stops after n samples holds exactly the radiance of n frames.  Every check is bit-exact: each
pixel's sample count against a numpy model of the stop rule, its radiance against the oracle's accumulation at that count, the
resolved image against the oracle's resolve at each pixel's count, and every schedule and call form against the others.
"""
import numpy as np
import pytest

from oracle.orcbind import Oracle
from raytracing_b200 import capi
from raytracing_b200.camera import default_camera
from tests.helpers import bits, scene, synthetic_sampler_tables
from tests.test_gpu_parity import SCHEDULES, run_frame, schedule_ctx

pytestmark = pytest.mark.gpu

EVERY = tuple(SCHEDULES) + ("stepwise",)          # frame, phase_graph, phase_direct, counted, timed, stepwise
STAT_KEYS = ("n_ext", "n_miss", "n_shadow", "n_cont", "n_unoccluded", "n_emissive_hits")
MAX_ERROR, MIN_SAMPLES = 0.01, 4          # on these scenes: a fifth to three quarters of the pixels stop within 24 samples


def luma(r):
    """rt_device.cuh's luma() in float32: (x * 0.299f + y * 0.587f) + z * 0.114f"""
    return (r[..., 0] * np.float32(0.299) + r[..., 1] * np.float32(0.587)) + r[..., 2] * np.float32(0.114)


def model(accs, max_error, min_samples):
    """The stop rule over the accumulations after samples 1..N -> (each pixel's count, pixels active at the start of each frame, pixels
    active after the last)."""
    h, w = accs[0].shape[:2]
    count = np.zeros((h, w), np.uint32)
    y_prev = np.zeros((h, w), np.float32)
    q = np.zeros((h, w), np.float64)
    active = np.ones((h, w), bool)
    n_active = []
    for n, acc in enumerate(accs, 1):
        n_active.append(int(active.sum()))
        Y = luma(acc)
        y = Y.astype(np.float64) - y_prev.astype(np.float64)
        qn = q + y * y
        m = Y.astype(np.float64) / n
        v = np.maximum(qn / n - m * m, 0.0)
        d = 1.0 + m
        e = np.sqrt(v / n) / (d * d)
        stop = (n >= min_samples) & (e <= max_error)
        q = np.where(active, qn, q); y_prev = np.where(active, Y, y_prev); count = np.where(active, np.uint32(n), count)
        active &= ~stop
    return count, n_active, int(active.sum())


def oracle_accs(sc, cam, w, h, mb, n, tables=None):
    """The oracle's accumulated radiance after each of n samples in sequence, (n, h, w, 4)."""
    o = Oracle(sc)
    acc = np.zeros((h, w, 4), dtype="<f4")
    out = []
    try:
        o.set_sampler_tables(tables)
        for s in range(n):
            acc, _, _ = o.render(cam, w, h, mb, sample_idx=s, radiance=acc, want_hits=False)
            out.append(acc.copy())
    finally:
        o.set_sampler_tables(None)
    return np.stack(out)


def at_counts(accs, count):
    """Every pixel's accumulation at its own count (count >= 1)."""
    h, w = count.shape
    yy, xx = np.mgrid[0:h, 0:w]
    return accs[count.astype(np.int64) - 1, yy, xx]


def resolve_at(acc, count):
    """k_resolve's shaded colour with per-pixel counts: radiance / count, then x / (1 + x); alpha 1."""
    hdr = acc[..., :3] / count.astype(np.float32)[..., None]
    out = np.ones(acc.shape[:2] + (4,), np.float32)
    out[..., :3] = hdr / (hdr + np.float32(1.0))
    return out


def adaptive_ctx(schedule, sc, cam, w, h, options=(), tables=None, max_error=MAX_ERROR, min_samples=MIN_SAMPLES, rank=0, world=1):
    c = schedule_ctx(schedule, sc, cam, w, h, options, rank=rank, world=world)
    if tables is not None:
        c.upload_sampler_tables(*tables); c.set_option(capi.OPT_SAMPLER, 1)
    c.set_adaptive_sampling(max_error, min_samples)
    c.reset()
    return c


def frames(c, mb, n, schedule="frame"):
    """n frames; returns the per-bounce statistics summed over them."""
    total = {k: np.zeros(capi.MAX_BOUNCES + 1, np.uint32) for k in STAT_KEYS}
    for _ in range(n):
        run_frame(c, schedule, mb)
        st = c.frame_stats()
        for k in STAT_KEYS:
            total[k] += st[k]
    return total


def assert_same(a, b, where=()):
    """Radiance bits, per-pixel counts, active count, sample count and resolved image of two contexts."""
    assert np.array_equal(bits(a.read_radiance()[..., :3]), bits(b.read_radiance()[..., :3])), tuple(where)
    assert np.array_equal(a.pixel_samples(), b.pixel_samples()), tuple(where)
    assert a.active_pixels() == b.active_pixels(), tuple(where)
    assert a.sample_count() == b.sample_count(), tuple(where)
    assert np.array_equal(bits(a.resolve()), bits(b.resolve())), tuple(where)


@pytest.mark.parametrize("sampler", ["random", "blue_noise"])
@pytest.mark.parametrize("name,w,h,mb,n", [("CornellBox", 128, 128, 3, 24), ("ShaderBalls", 200, 112, 5, 24)])
def test_every_pixel_matches_the_oracle_at_its_count(name, w, h, mb, n, sampler):
    """Every schedule: each pixel's count equals the model's, its radiance the oracle's accumulation at that count, the resolved
    image the oracle's resolve at each pixel's count, n_ext[0] of each frame the model's active count; every schedule's per-bounce
    statistics agree frame by frame."""
    sc, cam = scene(name), default_camera(w, h)
    tables = synthetic_sampler_tables() if sampler == "blue_noise" else None
    accs = oracle_accs(sc, cam, w, h, mb, n, tables)
    want_count, want_active, want_left = model(accs, MAX_ERROR, MIN_SAMPLES)
    # guards: the case exercises early stops, pixels that never stop and a spread of counts
    assert (want_count < n).mean() >= 0.2 and (want_count == n).mean() >= 0.1 and len(np.unique(want_count)) >= 3
    want_rad = at_counts(accs, want_count)
    ctxs = {s: adaptive_ctx(s, sc, cam, w, h, tables=tables) for s in EVERY}
    try:
        for f in range(n):
            stats = {}
            for s, c in ctxs.items():
                run_frame(c, s, mb)
                stats[s] = c.frame_stats()
                assert stats[s]["n_ext"][0] == want_active[f], (s, "frame %d" % f)
            for s in EVERY[1:]:
                for k in STAT_KEYS:
                    assert np.array_equal(stats[s][k][: mb + 1], stats[EVERY[0]][k][: mb + 1]), (s, k, "frame %d" % f)
        for s, c in ctxs.items():
            assert np.array_equal(c.pixel_samples(), want_count), s
            assert c.active_pixels() == want_left, s
            assert c.sample_count() == n, s
            assert np.array_equal(bits(c.read_radiance()[..., :3]), bits(want_rad[..., :3])), s
            assert np.array_equal(bits(c.resolve()), bits(resolve_at(want_rad, want_count))), s
    finally:
        for c in ctxs.values():
            c.destroy()


@pytest.mark.parametrize("fk", [0, 1, 2], ids=["phase", "frame_kernel_forced", "default"])
def test_integrate_samples_equals_frames(fk):
    """rt_integrate_samples(N) with the feature on equals N x rt_integrate: the per-phase frames, k_frame (the default at this size)
    and RT_OPT_FRAME_KERNEL 1.  Radiance, counts and summed statistics, over two calls."""
    name, w, h, mb = "CornellBox", 128, 128, 3
    sc, cam = scene(name), default_camera(w, h)
    opts = ((capi.OPT_FRAME_KERNEL, fk),)
    got = adaptive_ctx(None, sc, cam, w, h, opts)
    want = adaptive_ctx(None, sc, cam, w, h, opts)
    for n in (9, 7):
        want_stats = frames(want, mb, n)
        got.integrate_samples(mb, n)
        st = got.frame_stats()
        for k in STAT_KEYS:
            assert np.array_equal(st[k], want_stats[k]), (fk, n, k)
        assert_same(got, want, (fk, n))
    assert got.active_pixels() < w * h                                   # pixels did stop during the calls
    got.destroy(); want.destroy()


@pytest.mark.parametrize("schedule", ["frame", "phase_graph", "stepwise", "samples"])
def test_nothing_stops_is_byte_identical_to_off(schedule):
    """With min_samples above the frame count no pixel stops: radiance, statistics and the resolved image are byte-identical to the
    feature off, every pixel's count is the sample count."""
    name, w, h, mb, n = "ShaderBalls", 160, 96, 4, 6
    sc, cam = scene(name), default_camera(w, h)
    sched = "frame" if schedule == "samples" else schedule
    on = adaptive_ctx(sched, sc, cam, w, h, min_samples=1000)
    off = schedule_ctx(sched, sc, cam, w, h); off.reset()
    for f in range(n if schedule != "samples" else 1):
        for c in (on, off):
            if schedule == "samples":
                c.integrate_samples(mb, n)
            else:
                run_frame(c, schedule, mb)
        a, b = on.frame_stats(), off.frame_stats()
        for k in a.dtype.names:
            assert np.array_equal(a[k], b[k]), (schedule, f, k)
        assert on.read_radiance().tobytes() == off.read_radiance().tobytes(), (schedule, f)
        assert on.resolve().tobytes() == off.resolve().tobytes(), (schedule, f)
    assert np.array_equal(on.pixel_samples(), np.full((h, w), n, np.uint32))
    assert np.array_equal(off.pixel_samples(), np.full((h, w), n, np.uint32))
    assert on.active_pixels() == off.active_pixels() == w * h
    on.destroy(); off.destroy()


@pytest.mark.parametrize("schedule", ["frame", "phase_graph", "stepwise", "samples"])
def test_all_stopped_traces_nothing(schedule):
    """Once every pixel has stopped, further frames trace no rays and change no radiance; the sample count still advances and the
    counts stay."""
    name, w, h, mb = "CornellBox", 96, 64, 3
    sc, cam = scene(name), default_camera(w, h)
    c = adaptive_ctx("frame" if schedule == "samples" else schedule, sc, cam, w, h, max_error=1e30, min_samples=2)
    for _ in range(2):
        run_frame(c, "frame" if schedule == "samples" else schedule, mb)
    assert c.active_pixels() == 0
    rad = c.read_radiance()
    res = c.resolve()
    for _ in range(2):
        if schedule == "samples":
            c.integrate_samples(mb, 3)
        else:
            run_frame(c, schedule, mb)
        st = c.frame_stats()
        for k in STAT_KEYS:
            assert not st[k].any(), (schedule, k)
    assert c.sample_count() == (8 if schedule == "samples" else 4)
    assert c.read_radiance().tobytes() == rad.tobytes()
    assert c.resolve().tobytes() == res.tobytes()
    assert np.array_equal(c.pixel_samples(), np.full((h, w), 2, np.uint32))
    c.destroy()


def test_partition_rank_equals_single_rows():
    """Rank 1 of a 3-way rt_set_partition holds the single context's rows: radiance, counts and resolve; its active count is the
    number of its pixels still active on the single context."""
    name, w, h, mb, n = "ShaderBalls", 150, 77, 5, 10
    sc, cam = scene(name), default_camera(w, h)
    for sched in ("frame", "phase_graph"):
        one = adaptive_ctx(sched, sc, cam, w, h, max_error=0.02)
        part = adaptive_ctx(sched, sc, cam, w, h, max_error=0.02, rank=1, world=3)
        for _ in range(n):
            run_frame(one, sched, mb); run_frame(part, sched, mb)
        rows = np.arange(1, h, 3)
        assert np.array_equal(bits(part.read_radiance()[rows][..., :3]), bits(one.read_radiance()[rows][..., :3])), sched
        counts = one.pixel_samples()
        assert np.array_equal(part.pixel_samples()[rows], counts[rows]), sched
        assert np.array_equal(bits(part.resolve()[rows]), bits(one.resolve()[rows])), sched
        left = part.active_pixels()
        assert 0 < left < len(rows) * w, sched
        run_frame(one, sched, mb); run_frame(part, sched, mb)         # the active pixels are the ones whose count advances
        assert left == int((one.pixel_samples()[rows] == n + 1).sum()), sched
        assert np.array_equal(part.pixel_samples()[rows], one.pixel_samples()[rows]), sched
        one.destroy(); part.destroy()


def test_multi_device_equals_one_device():
    """A multi-device context (the node's GPUs, or one GPU listed three times) equals one device in radiance, counts, resolve and
    active count, after rt_integrate frames and an rt_integrate_samples call."""
    name, w, h, mb = "CornellBox", 128, 96, 3
    sc, cam = scene(name), default_camera(w, h)
    n_dev = capi.device_count()
    devices = list(range(n_dev)) if n_dev >= 2 else [0, 0, 0]
    one = adaptive_ctx(None, sc, cam, w, h)
    multi = capi.Context(w, h, devices=devices)
    multi.upload_scene(sc); multi.set_camera(cam)
    multi.set_adaptive_sampling(MAX_ERROR, MIN_SAMPLES); multi.reset()
    for c in (one, multi):
        frames(c, mb, 6)
        c.integrate_samples(mb, 6)
    assert_same(multi, one, ("multi", devices))
    assert 0 < one.active_pixels() < w * h
    one.destroy(); multi.destroy()


def test_setting_applies_at_reset_and_reset_reactivates():
    """The setting takes effect at the next reset (on and off); a reset makes every pixel active with a count of 0 again, and the
    frames after it equal a fresh context's."""
    name, w, h, mb = "CornellBox", 96, 64, 3
    sc, cam = scene(name), default_camera(w, h)
    off = schedule_ctx("frame", sc, cam, w, h); off.reset()
    c = schedule_ctx("frame", sc, cam, w, h); c.reset()
    c.set_adaptive_sampling(0.05, 2)              # not yet: the frames run as with the feature off
    frames(c, mb, 4); frames(off, mb, 4)
    assert c.active_pixels() == w * h and np.array_equal(c.pixel_samples(), np.full((h, w), 4, np.uint32))
    assert c.read_radiance().tobytes() == off.read_radiance().tobytes()
    c.reset()
    assert c.active_pixels() == w * h and not c.pixel_samples().any()
    fresh = adaptive_ctx("frame", sc, cam, w, h, max_error=0.05, min_samples=2)
    frames(c, mb, 5); frames(fresh, mb, 5)
    assert_same(c, fresh, ("after the setting's reset",))
    assert c.active_pixels() < w * h
    c.set_adaptive_sampling(0, 0)                # off: still on until the next reset
    frames(c, mb, 2); frames(fresh, mb, 2)
    assert_same(c, fresh, ("off requested, no reset yet",))
    c.set_adaptive_sampling(0.05, 2)
    c.reset(); fresh.reset()                     # a reset reactivates every pixel
    assert c.active_pixels() == w * h and not c.pixel_samples().any()
    frames(c, mb, 5); frames(fresh, mb, 5)
    assert_same(c, fresh, ("after a second reset",))
    c.set_adaptive_sampling(0, 0); c.reset()
    frames(c, mb, 3); off.reset(); frames(off, mb, 3)
    assert c.read_radiance().tobytes() == off.read_radiance().tobytes() and c.active_pixels() == w * h
    for x in (c, off, fresh):
        x.destroy()


def test_host_render_camera_move_matches_capi(tmp_path):
    """Render::SetAdaptiveSampling with SetSamplesPerFrame(8) (kFrame): a frame, a camera move (RequestReset), another frame — the
    image and the active count equal a capi context driven the same way."""
    from raytracing_b200 import hostapi
    from tests.test_host import PROC_OBJ, make_env
    w, h, mb, n = 160, 90, 5, 8
    env_path, _ = make_env(tmp_path, w=64, h=32)
    s = hostapi.HostScene(PROC_OBJ)
    s.add_directional_light((-0.6, -1.5, 3.5), (15, 10, 5))
    r = hostapi.HostRender(s, w, h, env_path)
    r.set_max_bounces(mb)
    r.set_samples_per_frame(n)
    r.set_adaptive_sampling(0.02, 2)
    a = s.arrays(); a["nodes"] = r.nodes()
    cam = hostapi.default_camera(w, h)
    cam2 = cam.copy(); cam2["position"][:3] = (cam["position"][0] + 0.3, cam["position"][1] - 0.2, cam["position"][2] + 0.1)
    c = capi.Context(w, h)
    c.upload_scene(a); c.set_camera(cam)
    c.set_adaptive_sampling(0.02, 2)
    for k, pos in enumerate((cam, cam2)):
        if k:
            r.set_camera(pos); c.set_camera(pos)
        r.render_frame()
        c.reset(); c.integrate_samples(mb, n)
        assert np.array_equal(bits(r.image()), bits(c.resolve())), k
        assert r.active_pixels() == c.active_pixels(), k
        assert 0 < c.active_pixels() < w * h, k
    r.close(); s.close(); c.destroy()


def test_errors_and_refused_combinations():
    """Invalid settings are RT_ERR_INVALID_ARGUMENT; the denoiser, a fused-gather target, RT_OPT_PRESENT 1 on a multi-device context
    and rt_resolve_gathered are RT_ERR_UNSUPPORTED whichever comes second.  The context renders exactly as a fresh one afterwards."""
    name, w, h, mb = "CornellBox", 96, 64, 3
    sc, cam = scene(name), default_camera(w, h)
    c = schedule_ctx("frame", sc, cam, w, h)

    def refused(code, fn, *args):
        with pytest.raises(capi.RtError) as e:
            fn(*args)
        assert e.value.code == code, (fn, args)

    for me, ms in ((-0.01, 4), (float("nan"), 4), (float("inf"), 4), (-float("inf"), 4), (0.01, 1), (0.01, 0)):
        refused(-1, c.set_adaptive_sampling, me, ms)
    # adaptive first
    c.set_adaptive_sampling(MAX_ERROR, MIN_SAMPLES)
    refused(-5, c.set_option, capi.OPT_DENOISER, 1)
    buf, stride, _ = c.gather_buffer()
    refused(-5, c.set_gather_target, buf, stride)
    refused(-5, c.resolve_gathered, buf, stride)
    c.reset()
    refused(-5, c.set_option, capi.OPT_DENOISER, 1)
    refused(-5, c.set_gather_target, buf, stride)
    # then the other order
    d = schedule_ctx("frame", sc, cam, w, h)
    d.set_option(capi.OPT_DENOISER, 1)
    refused(-5, d.set_adaptive_sampling, MAX_ERROR, MIN_SAMPLES)
    d.set_option(capi.OPT_DENOISER, 0)
    dbuf, dstride, _ = d.gather_buffer()
    d.set_gather_target(dbuf, dstride)
    refused(-5, d.set_adaptive_sampling, MAX_ERROR, MIN_SAMPLES)
    d.set_gather_target(None)
    d.set_adaptive_sampling(0, 0)                # off is always accepted
    # multi-device: RT_OPT_PRESENT 1 in both orders
    n_dev = capi.device_count()
    devices = list(range(min(n_dev, 2))) if n_dev >= 2 else [0, 0]
    m = capi.Context(w, h, devices=devices)
    m.upload_scene(sc); m.set_camera(cam)
    m.set_option(capi.OPT_PRESENT, 1)
    refused(-5, m.set_adaptive_sampling, MAX_ERROR, MIN_SAMPLES)
    m.set_option(capi.OPT_PRESENT, 0)
    m.set_adaptive_sampling(MAX_ERROR, MIN_SAMPLES)
    refused(-5, m.set_option, capi.OPT_PRESENT, 1)
    m.reset()
    frames(m, mb, 5)
    # every context still renders as a fresh one
    fresh = adaptive_ctx("frame", sc, cam, w, h)
    frames(c, mb, 5); frames(fresh, mb, 5)
    assert_same(c, fresh, ("after errors",))
    assert_same(m, fresh, ("multi after errors",))
    d.reset(); frames(d, mb, 2)
    off = schedule_ctx("frame", sc, cam, w, h); off.reset(); frames(off, mb, 2)
    assert d.read_radiance().tobytes() == off.read_radiance().tobytes()
    for x in (c, d, m, fresh, off):
        x.destroy()


def test_set_partition_reinitialises_the_state():
    """rt_set_partition with the feature on: every pixel of the new partition is active with a count of 0, and the frames that follow
    (sample indices continue from the context's sample count) hold, per pixel of the rank's rows, the oracle's accumulation of those
    samples at the model's count."""
    name, w, h, mb = "CornellBox", 96, 64, 3
    sc, cam = scene(name), default_camera(w, h)
    max_error, min_samples, before, after = 0.05, 2, 5, 8
    c = adaptive_ctx("frame", sc, cam, w, h, max_error=max_error, min_samples=min_samples)
    frames(c, mb, before)
    assert c.active_pixels() < w * h                                     # pixels stopped on the whole image
    c._ck(c.lib.rt_set_partition(c.h, 1, 3))
    rows = np.arange(1, h, 3)
    n_local = len(rows) * w
    assert c.local_pixel_count() == n_local and c.active_pixels() == n_local
    assert not c.pixel_samples()[rows].any()
    frames(c, mb, after)
    o = Oracle(sc)
    acc = np.zeros((h, w, 4), dtype="<f4")
    accs = []
    for s in range(before, before + after):
        acc, _, _ = o.render(cam, w, h, mb, sample_idx=s, radiance=acc, row_first=1, row_step=3, want_hits=False)
        accs.append(acc[rows].copy())
    accs = np.stack(accs)
    want_count, _, want_left = model(accs, max_error, min_samples)
    assert (want_count < after).any() and (want_count == after).any()
    assert np.array_equal(c.pixel_samples()[rows], want_count)
    assert c.active_pixels() == want_left
    assert c.sample_count() == before + after
    assert np.array_equal(bits(c.read_radiance()[rows][..., :3]), bits(at_counts(accs, want_count)[..., :3]))
    c.destroy()
