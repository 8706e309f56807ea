"""
GPU tests (-m gpu) of rt_integrate_samples: n_samples frames in one call.  Every check is bit-exact against n calls of
rt_integrate on a fresh context with the same options: the radiance bits, the sample count and the per-bounce statistics summed
over the frames, plus (where stated) the AOV buffers, the resolved views and the fused-gather slab.  The frames of rt_integrate's
schedule run n times with the statistics summed on the device: n one-kernel frames where RT_OPT_FRAME_KERNEL 1 forces it (or
the default selects it), n per-phase frames otherwise.  A band of rows is also compared with the CPU oracle rendering the
samples in sequence.
"""
import numpy as np
import pytest

from oracle.orcbind import Oracle
from raytracing_b200 import capi
from raytracing_b200.camera import default_camera
from tests.helpers import bits, scene, synthetic_sampler_tables
from tests.scenes_extra import closed_cornell, many_lights_scene, textured_cornell

pytestmark = pytest.mark.gpu

STAT_KEYS = ("n_ext", "n_miss", "n_shadow", "n_cont", "n_unoccluded", "n_emissive_hits")
STAGING = {"whole": ("CornellBox", ()), "l1": ("ShaderBalls", ()), "top": ("ShaderBalls", ((capi.OPT_TOP_SMEM, 100),))}


def make(sc, cam, w, h, options=(), rank=0, world=1, tables=None, start=0):
    """A reset context with the options, the blue-noise tables (if any) and `start` samples counted already (no launch)."""
    c = capi.Context(w, h, rank=rank, world=world)
    c.upload_scene(sc); c.set_camera(cam)
    if tables is not None:
        c.upload_sampler_tables(*tables); c.set_option(capi.OPT_SAMPLER, 1)
    for k, v in options:
        c.set_option(k, v)
    c.reset()
    for _ in range(start):
        c.advance_sample_count()
    return c


def frames(c, mb, n):
    """n calls of rt_integrate; returns the per-bounce statistics summed over them (uint32 arithmetic, like the counters)."""
    total = {k: np.zeros(capi.MAX_BOUNCES + 1, np.uint32) for k in STAT_KEYS}
    for _ in range(n):
        c.integrate(mb)
        st = c.frame_stats()
        for k in STAT_KEYS:
            total[k] += st[k]
    return total


def assert_same(got, want, want_stats, where):
    """Context `got` after rt_integrate_samples equals context `want` after the frames: radiance, sample count, summed statistics."""
    st = got.frame_stats()
    for k in STAT_KEYS:
        assert np.array_equal(st[k], want_stats[k]), (k,) + tuple(where)
    assert got.sample_count() == want.sample_count(), tuple(where)
    assert np.array_equal(bits(got.read_radiance()), bits(want.read_radiance())), tuple(where)


def compare(sc, cam, w, h, mb, n, options=(), rank=0, world=1, tables=None, start=0, where=()):
    """rt_integrate_samples(mb, n) against n x rt_integrate on fresh contexts; returns both contexts (caller destroys them)."""
    want = make(sc, cam, w, h, options, rank, world, tables, start)
    got = make(sc, cam, w, h, options, rank, world, tables, start)
    want_stats = frames(want, mb, n)
    got.integrate_samples(mb, n)
    assert_same(got, want, want_stats, tuple(where) + ("n=%d" % n,))
    return got, want


def oracle_rows(sc, cam, w, h, mb, n, row_first, row_step, tables=None, wf=False, start=0):
    o = Oracle(sc)
    acc = np.zeros((h, w, 4), dtype="<f4")
    try:
        o.set_sampler_tables(tables)
        for s in range(start, start + n):
            acc, _, _ = o.render(cam, w, h, mb, sample_idx=s, white_furnace=wf, radiance=acc, row_first=row_first, row_step=row_step,
                                 want_hits=False)
    finally:
        o.set_sampler_tables(None)
    return np.arange(row_first, h, row_step), acc


@pytest.mark.parametrize("n", [1, 2, 5, 17])
@pytest.mark.parametrize("staging", list(STAGING))
def test_samples_match_frames_and_oracle(staging, n):
    """CornellBox (BVH staged whole), ShaderBalls through L1 and with the top of its tree staged, for every RT_OPT_FRAME_KERNEL
    mode: modes 1 and 2 (default) run k_frame n times at this size, mode 0 the per-phase graph n times.  A band of rows equals
    the oracle's n samples in sequence."""
    name, options = STAGING[staging]
    sc = scene(name)
    w, h, mb = 120, 68, 6
    cam = default_camera(w, h)
    rows, orad = oracle_rows(sc, cam, w, h, mb, n, 2, 7)
    for fk in (0, 1, 2):
        got, want = compare(sc, cam, w, h, mb, n, options + ((capi.OPT_FRAME_KERNEL, fk),), where=(staging, "fk=%d" % fk))
        assert np.array_equal(bits(got.read_radiance()[rows][..., :3]), bits(orad[rows][..., :3])), (staging, fk, n)
        got.destroy(); want.destroy()


@pytest.mark.parametrize("threads", [32, 96, 1024])
def test_frame_threads_whole_image_and_partition(threads):
    """RT_OPT_FRAME_THREADS 32 (one warp per CTA), 96 and 1024, on the whole image and on each rank of a 3-way partition, for a
    scene staged whole and one traversed through L1."""
    w, h, mb, n = 150, 77, 5, 5
    for name in ("CornellBox", "ShaderBalls"):
        sc = scene(name); cam = default_camera(w, h)
        for world in (1, 3):
            for rank in range(world):
                got, want = compare(sc, cam, w, h, mb, n, ((capi.OPT_FRAME_KERNEL, 1), (capi.OPT_FRAME_THREADS, threads)), rank, world,
                                    where=(name, threads, "rank %d/%d" % (rank, world)))
                got.destroy(); want.destroy()


@pytest.mark.parametrize("case", ["textured", "lights_thin_lens", "white_furnace"])
def test_scene_variants(case):
    """Textured materials, five lights seen through a thin lens, and the white furnace: both schedules, against the frames and a
    band of oracle rows."""
    w, h, mb, n = 128, 80, 5, 4
    wf = case == "white_furnace"
    sc = {"textured": textured_cornell, "lights_thin_lens": many_lights_scene, "white_furnace": lambda: scene("CornellBox")}[case]()
    cam = default_camera(w, h, position=(0.15, -1.3, 0.9), aperture=0.04, focus_distance=1.7) if case == "lights_thin_lens" else default_camera(w, h)
    rows, orad = oracle_rows(sc, cam, w, h, mb, n, 1, 9, wf=wf)
    for fk in (1, 0):
        got, want = compare(sc, cam, w, h, mb, n, ((capi.OPT_FRAME_KERNEL, fk), (capi.OPT_WHITE_FURNACE, int(wf))), where=(case, fk))
        assert np.array_equal(bits(got.read_radiance()[rows][..., :3]), bits(orad[rows][..., :3])), (case, fk)
        got.destroy(); want.destroy()


@pytest.mark.parametrize("sampler,start,n", [("blue_noise", 250, 10), ("random", 65530, 10)])
def test_late_sample_indices(sampler, start, n):
    """Blue noise from sample 250 over the 256-sample wrap of its index, kRandom from 65 530 over 65 536; the resolved image uses
    the advanced sample count."""
    name, w, h, mb = "CornellBox", 96, 64, 4
    sc = scene(name); cam = default_camera(w, h)
    tables = synthetic_sampler_tables() if sampler == "blue_noise" else None
    rows, orad = oracle_rows(sc, cam, w, h, mb, n, 0, 5, tables=tables, start=start)
    for fk in (1, 0):
        got, want = compare(sc, cam, w, h, mb, n, ((capi.OPT_FRAME_KERNEL, fk),), tables=tables, start=start, where=(sampler, fk))
        assert got.sample_count() == start + n
        assert np.array_equal(bits(got.resolve()), bits(want.resolve())), (sampler, fk)
        assert np.array_equal(bits(got.read_radiance()[rows][..., :3]), bits(orad[rows][..., :3])), (sampler, fk)
        got.destroy(); want.destroy()


@pytest.mark.parametrize("mb,sampler", [(60, "blue_noise"), (255, "random")])
def test_long_paths(mb, sampler):
    """The closed Cornell box, whose paths last up to RT_MAX_BOUNCES bounces, on the forced one-kernel frame: the per-bounce
    statistics of the long paths add up over the call's frames."""
    w, h, n = 64, 48, 4
    sc = closed_cornell(); cam = default_camera(w, h)
    tables = synthetic_sampler_tables() if sampler == "blue_noise" else None
    got, want = compare(sc, cam, w, h, mb, n, ((capi.OPT_FRAME_KERNEL, 1),), tables=tables, where=("closed_cornell", mb, sampler))
    st = got.frame_stats()
    assert st["n_ext"][55] >= st["n_ext"][0] // 2, st["n_ext"][: mb + 1]        # the case still produces long paths
    got.destroy(); want.destroy()


def test_aov_views_hold_the_last_sample():
    """With an AOV view selected the AOV buffers equal those after the last of the n frames, and every resolved view is equal."""
    name, w, h, mb, n = "ShaderBalls", 128, 72, 4, 5
    sc = scene(name); cam = default_camera(w, h)
    for fk in (1, 0):
        got, want = compare(sc, cam, w, h, mb, n, ((capi.OPT_FRAME_KERNEL, fk), (capi.OPT_AOV, 3)), where=("aov", fk))
        for x, y in zip(got.read_aovs(), want.read_aovs()):
            assert np.array_equal(bits(x), bits(y)), fk
        for view in (0, 1, 2, 3, 4):
            got.set_option(capi.OPT_AOV, view); want.set_option(capi.OPT_AOV, view)
            assert np.array_equal(bits(got.resolve()), bits(want.resolve())), (fk, view)
        got.destroy(); want.destroy()


def test_after_earlier_frames_and_reset():
    """A call after two single-sample frames, then after rt_reset, then mixed with rt_integrate again."""
    name, w, h, mb = "CornellBox", 112, 63, 5
    sc = scene(name); cam = default_camera(w, h)
    for fk in (1, 0):
        opts = ((capi.OPT_FRAME_KERNEL, fk),)
        got, want = make(sc, cam, w, h, opts), make(sc, cam, w, h, opts)
        for c in (got, want):
            c.integrate(mb); c.integrate(mb)
        want_stats = frames(want, mb, 3); got.integrate_samples(mb, 3)
        assert_same(got, want, want_stats, (fk, "after frames"))
        got.reset(); want.reset()
        want_stats = frames(want, mb, 6); got.integrate_samples(mb, 6)
        assert_same(got, want, want_stats, (fk, "after reset"))
        got.integrate(mb); want.integrate(mb)
        want_stats = frames(want, mb, 2); got.integrate_samples(mb, 2)
        assert_same(got, want, want_stats, (fk, "mixed"))
        got.destroy(); want.destroy()


def test_forced_frame_kernel_call_launches():
    """With RT_OPT_FRAME_KERNEL 1, and with the default selector at this size, a call of n samples is n one-kernel frames, which
    add up their statistics, and one statistics sum at the end, whatever the BVH staging."""
    name, w, h, mb = "ShaderBalls", 96, 54, 4
    sc = scene(name); cam = default_camera(w, h)
    for staging in ((), ((capi.OPT_TOP_SMEM, 100),), ((capi.OPT_SMEM_BVH, 0),)):
        c = make(sc, cam, w, h, ((capi.OPT_FRAME_KERNEL, 1),) + staging)
        for n in (2, 5, 17, 64):
            before = c.launch_count()
            c.integrate_samples(mb, n)
            assert c.launch_count() - before == n + 1, (staging, n)
        c.destroy()
    c = make(scene("CornellBox"), default_camera(w, h), w, h)
    before = c.launch_count()
    c.integrate_samples(mb, 9)                   # default selector at this size
    assert c.launch_count() - before == 9 + 1
    c.destroy()



@pytest.mark.parametrize("fk", [1, 2, 0])
def test_taps_after_a_call_see_one_frame_at_most(fk):
    """rt_read_rays / rt_read_hits take their entry count from the frame counters: after a multi-sample call it never exceeds the
    context's pixels (the call's sums live apart, for rt_read_frame_stats only), on a whole image and on a partition rank.  The
    summed statistics are unchanged by the taps, and the next rt_integrate returns one frame's statistics again."""
    name, w, h, mb, n = "CornellBox", 96, 54, 4, 6
    sc = scene(name); cam = default_camera(w, h)
    for rank, world in ((0, 1), (1, 3)):
        where = ("taps", fk, rank, world)
        want = make(sc, cam, w, h, ((capi.OPT_FRAME_KERNEL, fk),), rank, world)
        got = make(sc, cam, w, h, ((capi.OPT_FRAME_KERNEL, fk),), rank, world)
        want_stats = frames(want, mb, n)
        got.integrate_samples(mb, n)
        local = got.local_pixel_count()
        for b in (0, 1, 2):
            rays, _ = got.read_rays(b)
            hits, _ = got.read_hits(b)
            assert len(rays) <= local and len(hits) <= local, where + (b, len(rays), len(hits), local)
        assert_same(got, want, want_stats, where)
        got.integrate(mb); want.integrate(mb)
        st, wst = got.frame_stats(), want.frame_stats()
        for k in STAT_KEYS:
            assert np.array_equal(st[k], wst[k]), (k,) + where + ("next frame",)
        assert st["n_ext"][0] == local, where
        got.destroy(); want.destroy()


@pytest.mark.parametrize("fk", [1, 2])
@pytest.mark.parametrize("present", [0, 1])
def test_multi_device_context(present, fk):
    """rt_create_multi over device 0 listed three times: the call fans out; radiance, summed statistics and the resolved image equal
    a single-device context's frames.  With RT_OPT_PRESENT 1 the ranks' kernels push the last samples' pixels into the gather
    buffer and the call signals once: the gathered image is resolved from what was pushed."""
    name, w, h, mb, n = "CornellBox", 160, 91, 5, 4
    sc = scene(name); cam = default_camera(w, h)
    one = make(sc, cam, w, h)
    many = capi.Context(w, h, devices=[0, 0, 0])
    many.upload_scene(sc); many.set_camera(cam); many.set_option(capi.OPT_FRAME_KERNEL, fk); many.set_option(capi.OPT_PRESENT, present)
    many.reset()
    for rep in range(2):
        want_stats = frames(one, mb, n)
        many.integrate_samples(mb, n)
        assert_same(many, one, want_stats, ("multi", present, fk, rep))
        assert np.array_equal(bits(many.resolve()), bits(one.resolve())), (present, fk, rep)
    one.destroy(); many.destroy()


def test_fused_gather_slab_equals_radiance():
    """rt_set_gather_target on three partition contexts: after a multi-sample call and rt_gather_wait the gather buffer, resolved
    with rt_resolve_gathered, equals the single-context image; on the one-kernel frame and on the per-phase schedule."""
    name, w, h, mb, n = "ShaderBalls", 150, 83, 5, 3
    sc = scene(name); cam = default_camera(w, h)
    for fk in (1, 2, 0):
        one = make(sc, cam, w, h)
        parts = [make(sc, cam, w, h, ((capi.OPT_FRAME_KERNEL, fk),), rank=r, world=3) for r in range(3)]
        buf, stride, _ = parts[0].gather_buffer()
        for c in parts:
            c.set_gather_target(buf, stride)
        for rep in range(2):
            frames(one, mb, n)
            for c in reversed(parts):
                c.integrate_samples(mb, n)
            parts[0].gather_wait()
            assert np.array_equal(bits(parts[0].resolve_gathered(buf, stride)), bits(one.resolve())), (fk, rep)
        for c in parts + [one]:
            c.destroy()


def test_host_render_samples_per_frame(tmp_path):
    """Render::SetSamplesPerFrame(n): one RenderFrame() gives the image of n RenderFrame() calls; with n > 1 the kFused schedule
    is refused with an error."""
    from raytracing_b200 import hostapi
    from tests.test_host import PROC_OBJ, make_env
    w, h, mb, n = 160, 90, 5, 6
    env_path, _ = make_env(tmp_path, w=64, h=32)
    imgs = []
    for per_frame in (1, n):
        s = hostapi.HostScene(PROC_OBJ)
        s.add_directional_light((-0.6, -1.5, 3.5), (15, 10, 5))
        r = hostapi.HostRender(s, w, h, env_path)
        r.set_max_bounces(mb)
        r.set_samples_per_frame(per_frame)
        for _ in range(n // per_frame):
            r.render_frame()
        imgs.append(r.image())
        if per_frame > 1:
            r.set_schedule("fused")
            with pytest.raises(hostapi.HostError):
                r.render_frame()
            with pytest.raises(hostapi.HostError):
                r.set_samples_per_frame(0)
        r.close(); s.close()
    assert np.array_equal(bits(imgs[0]), bits(imgs[1]))


def test_errors_leave_the_context_usable():
    """n_samples = 0, a sample count that would wrap, max_bounces = 256 (RT_ERR_INVALID_ARGUMENT) and the denoiser with n > 1
    (RT_ERR_UNSUPPORTED) are refused before anything is enqueued; the context then renders exactly as before."""
    name, w, h, mb = "CornellBox", 96, 54, 4
    sc = scene(name); cam = default_camera(w, h)
    for fk in (1, 0):
        opts = ((capi.OPT_FRAME_KERNEL, fk),)
        got, want = make(sc, cam, w, h, opts), make(sc, cam, w, h, opts)
        got.integrate(mb); want.integrate(mb)
        launches = got.launch_count()
        for args, code in (((mb, 0), -1), ((mb, 0xFFFFFFFF), -1), ((256, 2), -1)):
            with pytest.raises(capi.RtError) as e:
                got.integrate_samples(*args)
            assert e.value.code == code, args
        assert got.launch_count() == launches and got.sample_count() == 1
        want_stats = frames(want, mb, 3); got.integrate_samples(mb, 3)
        assert_same(got, want, want_stats, (fk, "after errors"))
        got.destroy(); want.destroy()
    c = make(sc, cam, w, h, ((capi.OPT_DENOISER, 1),))
    with pytest.raises(capi.RtError) as e:
        c.integrate_samples(mb, 2)
    assert e.value.code == -5
    assert c.sample_count() == 0
    c.integrate_samples(mb, 1)                  # one sample per call is rt_integrate, denoiser included
    assert c.sample_count() == 1
    c.destroy()
