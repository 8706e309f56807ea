"""
GPU tests (-m gpu) of the extension-ray queue layout and of bounce 0 of the per-phase frame.

The per-phase frame generates its primary rays inside the bounce-0 traversal kernel (k_trace_primary) and stores only the planes
the bounce-0 shading pass reads; the stepwise schedule still writes the whole queue with k_raygen and traces it with k_intersect.
Every check is bit for bit: the per-phase frame (graph, direct launches, counted traversal) against the stepwise schedule, on
adaptive sampling with a partial active list, AOVs (depth needs the ray origin), emitter sampling, an instanced scene, a 2-way
partition and rt_integrate_samples; against the oracle where it renders the same thing; and rt_read_rays against the packed
pixel and t_max that the queue held before the pixel moved from plane A to plane B.
"""
import numpy as np
import pytest

from oracle.orcbind import Oracle
from raytracing_b200 import capi
from raytracing_b200.camera import default_camera
from tests.helpers import bits, scene
from tests.test_gpu_parity import SCHEDULES

pytestmark = pytest.mark.gpu

W, H, MB = 96, 64, 4
STAT_KEYS = ("n_ext", "n_miss", "n_shadow", "n_cont", "n_unoccluded", "n_emissive_hits")
PHASE = ("phase_graph", "phase_direct", "counted")       # per-phase frames: bounce 0 in k_trace_primary


def flat_ctx(sc, cam, schedule, options=(), rank=0, world=1):
    c = capi.Context(W, H, rank=rank, world=world)
    c.upload_scene(sc); c.set_camera(cam)
    for k, v in ((capi.OPT_FRAME_KERNEL, 0),) + SCHEDULES.get(schedule, ()) + tuple(options):
        c.set_option(k, v)
    c.aovs_wanted = (capi.OPT_AOV_ALWAYS, 1) in tuple(options)
    return c


def render(c, schedule, frames, mb=MB, samples=0):
    """Resets c and renders `frames` frames (or one rt_integrate_samples call of `samples`); -> radiance, stats, AOVs, counts."""
    c.reset()
    if samples:
        c.integrate_samples(mb, samples)
    for _ in range(frames):
        c.integrate_stepwise(mb) if schedule == "stepwise" else c.integrate(mb)
    aovs = c.read_aovs() if c.aovs_wanted else None
    return c.read_radiance(), c.frame_stats(), aovs, c.pixel_samples()


def assert_same(got, want, mb, where):
    rad, st, aovs, counts = got
    wrad, wst, waovs, wcounts = want
    assert np.array_equal(bits(rad), bits(wrad)), where
    for k in STAT_KEYS:
        assert np.array_equal(st[k][: mb + 1], wst[k][: mb + 1]), (k,) + where
    for name, a, b in zip(("albedo", "depth", "normal", "velocity"), aovs or (), waovs or ()):
        assert np.array_equal(bits(a), bits(b)), (name,) + where
    assert np.array_equal(counts, wcounts), where


def against_stepwise(make, frames=1, samples=0, mb=MB, ref="stepwise"):
    """Every per-phase arm equals the reference schedule bit for bit: stepwise (k_raygen + k_intersect), or the one-kernel frame
    (k_frame, which stores every plane of its primary rays); returns the reference's result."""
    c = make(ref)
    want = render(c, ref, frames, mb) if not samples else None
    c.destroy()
    for s in PHASE:
        c = make(s)
        got = render(c, s, frames, mb, samples)
        c.destroy()
        if want is None:
            want = got
            continue
        assert_same(got, want, mb, (s,))
    return want


def oracle_frames(sc, cam, n, mb=MB):
    o = Oracle(sc)
    acc = np.zeros((H, W, 4), dtype="<f4")
    for s in range(n):
        acc, _, st = o.render(cam, W, H, mb, sample_idx=s, radiance=acc, want_hits=False)
    return acc, st


def test_plain_frames_match_stepwise_and_oracle():
    sc = scene("CornellBox"); cam = default_camera(W, H)
    rad, st, _, _ = against_stepwise(lambda s: flat_ctx(sc, cam, s), frames=2)
    oacc, ost = oracle_frames(sc, cam, 2)
    assert np.array_equal(bits(rad[..., :3]), bits(oacc[..., :3]))
    for k in STAT_KEYS[:5]:
        assert np.array_equal(st[k][: MB + 1], ost[k][: MB + 1]), k


def test_adaptive_partial_active_list():
    """After a few frames only part of the pixels is still active: k_trace_primary takes slot i from active[i] and counts
    n_primary = the active pixels, as k_raygen does."""
    sc = scene("CornellBox"); cam = default_camera(W, H)

    def make(s):
        c = flat_ctx(sc, cam, s)
        c.set_adaptive_sampling(0.05, 2)
        return c
    rad, st, _, counts = against_stepwise(make, frames=8)
    assert 0 < st["n_ext"][0] < W * H, st["n_ext"][0]              # the last frame traced a partial list
    assert counts.min() < counts.max()


def test_aovs_with_depth():
    """AOVs on: the bounce-0 traversal stores plane A as well, for the depth AOV; AOVs equal the stepwise schedule's."""
    sc = scene("ShaderBalls"); cam = default_camera(W, H)
    _, _, (al, de, no, ve), _ = against_stepwise(lambda s: flat_ctx(sc, cam, s, ((capi.OPT_AOV_ALWAYS, 1),)))
    assert np.isfinite(de).all() and (de < 20000.0).any() and (de > 0.0).any()


def test_emitter_sampling():
    """Against the one-kernel frame: the last bounce of a frame samples analytic lights only, and the stepwise calls do not know
    which bounce is the last."""
    sc = scene("CornellBox"); cam = default_camera(W, H)
    _, st, _, _ = against_stepwise(lambda s: flat_ctx(sc, cam, s, ((capi.OPT_EMITTER_SAMPLING, 1), (capi.OPT_AOV_ALWAYS, 1))), frames=2,
                                   ref="frame")
    assert st["n_emissive_hits"][1:MB + 1].sum() > 0


def test_instanced_scene():
    from tests.test_gpu_instancing import as_mesh, EYE
    base = scene("CornellBox")
    mats = [EYE, np.hstack([np.eye(3) * 0.5, np.array([[0.3], [0.2], [-0.1]])]).astype(np.float32)]
    cam = default_camera(W, H)

    def make(s):
        c = capi.Context(W, H)
        for k, v in SCHEDULES.get(s, ()) + ((capi.OPT_AOV_ALWAYS, 1),):
            c.set_option(k, v)
        c.upload_instanced_scene([as_mesh(base)], base)
        c.set_instances([0, 0], mats)
        c.set_camera(cam)
        c.aovs_wanted = True
        return c
    against_stepwise(make, frames=2)


def test_two_way_partition_matches_whole_image_rows():
    sc = scene("ShaderBalls"); cam = default_camera(W, H)
    whole = flat_ctx(sc, cam, "phase_graph")
    wrad = render(whole, "phase_graph", 1)[0]
    whole.destroy()
    for rank in (0, 1):
        for s in PHASE + ("stepwise",):
            c = flat_ctx(sc, cam, s, rank=rank, world=2)
            rad, st, _, _ = render(c, s, 1)
            c.destroy()
            assert st["n_ext"][0] == W * H // 2, (rank, s)
            assert np.array_equal(bits(rad[rank::2]), bits(wrad[rank::2])), (rank, s)


def test_integrate_samples_equals_frames():
    """rt_integrate_samples on the per-phase frames: the radiance of 5 stepwise frames, statistics summed over them."""
    sc = scene("CornellBox"); cam = default_camera(W, H)
    c = flat_ctx(sc, cam, "stepwise")
    c.reset()
    sums = {k: 0 for k in STAT_KEYS}
    for _ in range(5):
        c.integrate_stepwise(MB)
        st = c.frame_stats()
        for k in STAT_KEYS:
            sums[k] = sums[k] + st[k][: MB + 1].astype(np.uint64)
    want = c.read_radiance()
    c.destroy()
    for s in PHASE:
        c = flat_ctx(sc, cam, s)
        got = render(c, s, 0, samples=5)
        c.destroy()
        assert np.array_equal(bits(got[0]), bits(want)), s
        for k in STAT_KEYS:
            assert np.array_equal(got[1][k][: MB + 1].astype(np.uint64), sums[k]), (k, s)


def test_read_rays_keeps_pixel_and_t_max():
    """rt_read_rays after rt_generate_rays and after a continuation bounce: pixel indices in the order of the queue, direction.w =
    RT_MAX_RENDER_DIST (the t_max of every extension ray), origin.w = 0; rt_read_hits gives the same pixels."""
    sc = scene("CornellBox"); cam = default_camera(W, H)
    c = flat_ctx(sc, cam, "stepwise")
    c.reset()
    c.generate_rays()
    rays, pix = c.read_rays(0)
    assert np.array_equal(pix, np.arange(W * H, dtype=np.uint32))
    assert (rays["direction"][:, 3] == np.float32(20000.0)).all()
    assert (rays["origin"][:, 3] == 0.0).all()
    c.intersect(0)
    _, hpix = c.read_hits(0)
    assert np.array_equal(hpix, pix)
    c.shade_hits(0)
    rays1, pix1 = c.read_rays(1)
    assert len(rays1) > 0 and (rays1["direction"][:, 3] == np.float32(20000.0)).all()
    assert len(np.unique(pix1)) == len(pix1) and pix1.max() < W * H
    c.destroy()
