"""
GPU tests (-m gpu) of adaptive sampling at the sizes it runs at.  After every sample k_adaptive_update compacts the active pixels in
place with a decoupled look-back over 1024-entry tiles, 32 tiles per step; the next frame's primary rays come from that list, so a
wrong prefix drops or duplicates pixels.  test_gpu_adaptive.py renders at most 22 tiles, where the look-back always ends in its first
window; these tests run updates of 32 to 8 100 tiles.

Expected values come from tests/adaptive_model.py fed with the accumulations of a context with the feature off (or, for the small
images, with the oracle's), after every sample.  Every case checks, after each frame, n_ext[0] against the model's active count
before the update and active_pixels() against the count after it, and at the end, bit for bit, each pixel's count, its radiance
at that count, the resolved image and the sample count.  The feature-off accumulations themselves are held to the oracle: the
whole image for the small cases, a band of rows spread over the frame for the full-size ones.  Guards assert from the model's tile
report that each case reaches the look-back windows it is meant to.

Cost: about 30 s of wall time for the whole file on an H100 host, 4K and ShaderBalls included.  The GPU work is seconds; the rest
is the host's: a read-back after every full-size frame (33 MB at 1080p), the model's updates and the oracle's rows.
"""
import numpy as np
import pytest

from oracle.orcbind import Oracle
from raytracing_b200 import capi
from raytracing_b200.camera import default_camera
from tests.adaptive_model import AdaptiveModel
from tests.helpers import bits, scene, synthetic_sampler_tables
from tests.test_gpu_adaptive import EVERY, adaptive_ctx, assert_same, at_counts, resolve_at
from tests.test_gpu_parity import run_frame, schedule_ctx

pytestmark = pytest.mark.gpu

# The small cases: the update at n = min_samples (every pixel still active) has the stated number of tiles.
EDGE_ERROR, EDGE_MIN = 0.02, 2
# The full-size cases' (max_error, min_samples): chosen so that at least three consecutive updates run more than 96 tiles (four
# look-back windows), one of them with at least 10 % empty and 10 % partial tiles, and pixels are still active after the last sample
# (full_size_guard).  CornellBox's noise is spread evenly over the frame: below max_error 0.15 every tile keeps survivors, so its
# stops come late and together.  At these values (H100 runs): CornellBox 1080p, n = 12: 24 % of 2 025 tiles empty, 76 % partial,
# 51 833 pixels left after 16 samples; ShaderBalls 1080p, n = 2: 12 % empty, 88 % partial, 752 164 left after 16; CornellBox 4K,
# n = 4: 40 % of 8 100 tiles empty, 60 % partial, 64 737 left after 8.
FULL = {"CornellBox": (0.15, 12), "ShaderBalls": (0.02, 2), "CornellBox_4K": (0.2, 4)}
CB_ERROR, CB_MIN = FULL["CornellBox"]


def band_rows(h, first, step):
    rows = np.arange(first, h, step)
    assert len(rows) >= 17
    return rows


def check_end(c, m, n, rows=slice(None), where=()):
    """c's counts, radiance, resolve and sample count equal the model's (of c's rows) after n samples."""
    where = tuple(where)
    assert np.array_equal(c.pixel_samples()[rows], m.count), where
    assert np.array_equal(bits(c.read_radiance()[rows][..., :3]), bits(m.radiance)), where
    assert np.array_equal(bits(c.resolve()[rows]), bits(resolve_at(m.radiance, m.count))), where
    assert c.sample_count() == n, where
    assert c.active_pixels() == m.n_active, where


def check_update(c, u, where=()):
    """n_ext[0] of the frame that ran is the active count before the update, active_pixels() the count after it."""
    assert c.frame_stats()["n_ext"][0] == u.active_before, tuple(where) + (u,)
    assert c.active_pixels() == u.active_after, tuple(where) + (u,)


def full_size_guard(m):
    """The look-back runs past its fourth window in three consecutive updates, one update has >= 10 % empty and >= 10 % partial
    tiles (tiles publish very different aggregates), and the last update still leaves pixels active."""
    big = [u.tiles > 96 for u in m.updates]
    assert any(all(big[i:i + 3]) for i in range(len(big) - 2)), m.updates
    assert any(u.tiles > 96 and u.empty >= 0.1 * u.tiles and u.partial >= 0.1 * u.tiles for u in m.updates), m.updates
    assert m.n_active > 0, m.updates


def form_ctx(form, sc, cam, w, h, **kw):
    """An adaptive context for one call form: a schedule of test_gpu_parity.SCHEDULES, "stepwise", or "samples" (one
    rt_integrate_samples call under the default selection)."""
    return adaptive_ctx(None if form == "samples" else form, sc, cam, w, h, **kw)


# (w, h, rank, world, tiles of the first full update): 32 767 / 32 768 / 32 769 / 33 792 / 66 560 pixels, and rank 2 of a 3-way
# partition of 1000 x 100 (33 local rows, 33 000 pixels)
EDGES = {
    "217x151": (217, 151, 0, 1, 32),
    "256x128": (256, 128, 0, 1, 32),
    "331x99": (331, 99, 0, 1, 33),
    "264x128": (264, 128, 0, 1, 33),
    "1024x65": (1024, 65, 0, 1, 65),
    "1000x100_rank2of3": (1000, 100, 2, 3, 33),
}


@pytest.mark.parametrize("case,sampler", [(k, "random") for k in EDGES] + [("331x99", "blue_noise")])
def test_tile_boundaries_every_schedule(case, sampler):
    """CornellBox, 3 bounces, 12 samples, at sizes whose full update lands on the edges of the look-back's windows: every
    rt_integrate schedule, stepwise and rt_integrate_samples against the model of the oracle's accumulations of the whole image."""
    w, h, rank, world, want_tiles = EDGES[case]
    name, mb, n = "CornellBox", 3, 12
    sc, cam = scene(name), default_camera(w, h)
    tables = synthetic_sampler_tables() if sampler == "blue_noise" else None
    rows = np.arange(rank, h, world)
    forms = EVERY + ("samples",)
    kw = dict(tables=tables, max_error=EDGE_ERROR, min_samples=EDGE_MIN, rank=rank, world=world)
    ctxs = {f: form_ctx(f, sc, cam, w, h, **kw) for f in forms}
    off = schedule_ctx("frame", sc, cam, w, h, rank=rank, world=world)
    if tables is not None:
        off.upload_sampler_tables(*tables); off.set_option(capi.OPT_SAMPLER, 1)
    off.reset()
    m = AdaptiveModel((len(rows), w), EDGE_ERROR, EDGE_MIN)
    o = Oracle(sc)
    acc = np.zeros((h, w, 4), dtype="<f4")
    try:
        o.set_sampler_tables(tables)
        for s in range(n):
            acc, _, _ = o.render(cam, w, h, mb, sample_idx=s, radiance=acc, row_first=rank, row_step=world, want_hits=False)
            run_frame(off, "frame", mb)
            assert np.array_equal(bits(off.read_radiance()[rows][..., :3]), bits(acc[rows][..., :3])), ("off", s)
            u = m.update(acc[rows])
            for f in EVERY:
                run_frame(ctxs[f], f, mb)
                check_update(ctxs[f], u, (f, s))
        ctxs["samples"].integrate_samples(mb, n)
        assert ctxs["samples"].frame_stats()["n_ext"][0] == sum(u.active_before for u in m.updates)
        for f, c in ctxs.items():
            check_end(c, m, n, rows, (f,))
    finally:
        o.set_sampler_tables(None)
        for c in list(ctxs.values()) + [off]:
            c.destroy()
    first = m.updates[EDGE_MIN - 1]                 # the first update that can stop pixels: every local pixel still active
    assert first.tiles == want_tiles and 0 < first.active_after < first.active_before, first


def render_full_size(name, w, h, mb, n, forms, row_first, row_step, max_error, min_samples):
    """Renders n frames on a feature-off context (the per-phase graph at 1080p, the default selection at 4K) and on an adaptive
    context per form, checking each frame against the model; the oracle renders a band of rows through every sample, and each
    frame's feature-off band equals it.  -> (model, contexts by form, the band's rows, the oracle's band after each sample)."""
    sc, cam = scene(name), default_camera(w, h)
    brows = band_rows(h, row_first, row_step)
    ctxs = {f: form_ctx(f, sc, cam, w, h, max_error=max_error, min_samples=min_samples) for f in forms}
    off = schedule_ctx("phase_graph" if w * h < 4e6 else None, sc, cam, w, h); off.reset()
    m = AdaptiveModel((h, w), max_error, min_samples)
    o = Oracle(sc)
    acc = np.zeros((h, w, 4), dtype="<f4")
    band_accs = []
    for s in range(n):
        acc, _, _ = o.render(cam, w, h, mb, sample_idx=s, radiance=acc, row_first=row_first, row_step=row_step, want_hits=False)
        band_accs.append(acc[brows].copy())
        run_frame(off, "frame", mb)
        r = off.read_radiance()
        assert np.array_equal(bits(r[brows][..., :3]), bits(acc[brows][..., :3])), ("off band", s)
        u = m.update(r)
        for f in forms:
            if f != "samples":
                run_frame(ctxs[f], f, mb)
                check_update(ctxs[f], u, (name, f, s))
    off.destroy()
    if "samples" in ctxs:
        ctxs["samples"].integrate_samples(mb, n)
        assert ctxs["samples"].frame_stats()["n_ext"][0] == sum(u.active_before for u in m.updates)
    return m, ctxs, brows, np.stack(band_accs)


def check_full_size(m, ctxs, n, brows, band_accs, where=()):
    """The guards, the end checks of every context, and the band of every context against the oracle at the model's counts."""
    full_size_guard(m)
    want_band = at_counts(band_accs, m.count[brows])
    for f, c in ctxs.items():
        check_end(c, m, n, where=tuple(where) + (f,))
        assert np.array_equal(bits(c.read_radiance()[brows][..., :3]), bits(want_band[..., :3])), tuple(where) + (f, "band")


@pytest.mark.parametrize("name,row_first,row_step", [("CornellBox", 5, 61), ("ShaderBalls", 3, 59)])
def test_1080p_benchmarked_configurations(name, row_first, row_step):
    """1920x1080, 8 bounces, 16 samples: the per-phase graph (the 1080p default), RT_OPT_FRAME_KERNEL 1 (k_frame over the whole
    frame) and one rt_integrate_samples(8, 16) call, against the model; a band of rows against the oracle at the model's counts."""
    w, h, mb, n = 1920, 1080, 8, 16
    m, ctxs, brows, band_accs = render_full_size(name, w, h, mb, n, ("phase_graph", "frame", "samples"), row_first, row_step,
                                                 *FULL[name])
    try:
        check_full_size(m, ctxs, n, brows, band_accs, where=(name,))
    finally:
        for c in ctxs.values():
            c.destroy()


def test_4k():
    """CornellBox 3840x2160, 3 bounces, 8 samples, the default schedule: 8 100 tiles per full update."""
    w, h, mb, n, row_first, row_step = 3840, 2160, 3, 8, 11, 127
    m, ctxs, brows, band_accs = render_full_size("CornellBox", w, h, mb, n, (None,), row_first, row_step,
                                                 *FULL["CornellBox_4K"])
    try:
        assert m.updates[0].tiles == 8100
        check_full_size(m, ctxs, n, brows, band_accs, where=("4K",))
    finally:
        for c in ctxs.values():
            c.destroy()


def test_1080p_partition_rank_equals_single_rows():
    """Rank 1 of a 4-way rt_set_partition at 1080p (270 local rows, 507 tiles) holds the single context's rows: radiance, counts,
    resolve, and an active count equal to the rank's pixels that still advance on the single context; both equal the model."""
    name, w, h, mb, n, world = "CornellBox", 1920, 1080, 8, 16, 4
    rows = np.arange(1, h, world)
    sc, cam = scene(name), default_camera(w, h)
    off = schedule_ctx(None, sc, cam, w, h); off.reset()
    one = adaptive_ctx(None, sc, cam, w, h, max_error=CB_ERROR, min_samples=CB_MIN)
    part = adaptive_ctx(None, sc, cam, w, h, max_error=CB_ERROR, min_samples=CB_MIN, rank=1, world=world)
    m_one = AdaptiveModel((h, w), CB_ERROR, CB_MIN)
    m = AdaptiveModel((len(rows), w), CB_ERROR, CB_MIN)
    try:
        for s in range(n):
            for c in (off, one, part):
                run_frame(c, None, mb)
            r = off.read_radiance()
            check_update(one, m_one.update(r), ("single", s))
            check_update(part, m.update(r[rows]), ("rank 1", s))
        full_size_guard(m)
        check_end(one, m_one, n, where=("single",))
        check_end(part, m, n, rows, ("rank 1",))
        assert np.array_equal(bits(part.read_radiance()[rows][..., :3]), bits(one.read_radiance()[rows][..., :3]))
        assert np.array_equal(part.pixel_samples()[rows], one.pixel_samples()[rows])
        assert np.array_equal(bits(part.resolve()[rows]), bits(one.resolve()[rows]))
        left = part.active_pixels()
        run_frame(one, None, mb); run_frame(part, None, mb)          # the active pixels are the ones whose count advances
        assert left == int((one.pixel_samples()[rows] == n + 1).sum())
        assert np.array_equal(part.pixel_samples()[rows], one.pixel_samples()[rows])
    finally:
        for c in (off, one, part):
            c.destroy()


def test_1080p_multi_device_equals_one_device():
    """A multi-device context at 1080p (the node's GPUs, or one GPU listed three times: 675 tiles per device) equals one device in
    radiance, counts, resolve and active count, after rt_integrate frames and an rt_integrate_samples call."""
    name, w, h, mb = "CornellBox", 1920, 1080, 8
    sc, cam = scene(name), default_camera(w, h)
    n_dev = capi.device_count()
    devices = list(range(n_dev)) if n_dev >= 2 else [0, 0, 0]
    one = adaptive_ctx(None, sc, cam, w, h, max_error=CB_ERROR, min_samples=CB_MIN)
    multi = capi.Context(w, h, devices=devices)
    multi.upload_scene(sc); multi.set_camera(cam)
    multi.set_adaptive_sampling(CB_ERROR, CB_MIN); multi.reset()
    for c in (one, multi):
        for _ in range(8):
            run_frame(c, None, mb)
        c.integrate_samples(mb, 8)
    assert_same(multi, one, ("multi", devices))
    assert 0 < one.active_pixels() < w * h
    one.destroy(); multi.destroy()


def test_1080p_two_runs_agree():
    """Tiles are taken in CTA arrival order: two contexts built the same way (the per-phase graph, CornellBox 1080p, 8 bounces,
    16 samples) end with byte-identical radiance and counts."""
    name, w, h, mb, n = "CornellBox", 1920, 1080, 8, 16
    sc, cam = scene(name), default_camera(w, h)
    a, b = (form_ctx("phase_graph", sc, cam, w, h, max_error=CB_ERROR, min_samples=CB_MIN) for _ in range(2))
    for _ in range(n):
        run_frame(a, "phase_graph", mb); run_frame(b, "phase_graph", mb)
    assert a.read_radiance().tobytes() == b.read_radiance().tobytes()
    assert a.pixel_samples().tobytes() == b.pixel_samples().tobytes()
    assert a.active_pixels() == b.active_pixels() < w * h
    a.destroy(); b.destroy()
