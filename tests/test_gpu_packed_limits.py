"""
GPU tests (-m gpu) of the packed queue words at their limits, each on every schedule that reads or writes it:

- the light byte of a shadow record (sA.w = local pixel | light << 24, no sB for directional lights below index 255): scenes with
  254 .. 300 analytic lights and directional lights with edge origins, against the oracle;
- the 24-bit local pixel of that word: frames of exactly 2^24 local pixels (two-plane) and just past it (every ray three-plane),
  whole and as ranks of a partition, against the next partition up and against the oracle's rows;
- the 16-bit pixel coordinates of an extension ray (B.w = x | y << 16): frames 65535 pixels wide or high, and x >= 32768;
- the counter batch of rt_integrate_samples' N-frame one-kernel loop, whose 64-bit counter pairs are folded before the low word
  could carry into the high one.

"Every schedule" is the per-phase graph and direct launches, the one-kernel frame, the unmerged per-phase kernels under kernel
timing, the stepwise calls and the N-frame one-kernel loop (rt_integrate_samples with RT_OPT_FRAME_KERNEL 1).  A context of 2^24 local
pixels takes about 4 GB of device memory (3.98 GB at 4096 x 4096 after a frame, measured on an H100 80GB HBM3); one such context
exists at a time.  The file runs in about a minute there.
"""
import numpy as np
import pytest

from oracle.orcbind import Oracle
from raytracing_b200 import capi
from raytracing_b200.camera import default_camera
from tests.helpers import bits, scene, synthetic_sampler_tables
from tests.test_gpu_parity import check_stats, schedule_ctx
from tests.test_packed_limits_cpu import LIGHT_COUNTS, edge_origin_scene, light_scene, wall_scene

pytestmark = pytest.mark.gpu

STAT_KEYS = ("n_ext", "n_miss", "n_shadow", "n_cont", "n_unoccluded", "n_emissive_hits")
RUNS = ("frame", "phase_graph", "phase_direct", "timed", "stepwise", "samples_fk1")      # "samples_fk1": integrate_samples(mb, n), forced k_frame


def make(run, sc, cam, w, h, options=(), rank=0, world=1, tables=None):
    c = schedule_ctx("frame" if run == "samples_fk1" else run, sc, cam, w, h, options, rank, world)
    if tables is not None:
        c.upload_sampler_tables(*tables); c.set_option(capi.OPT_SAMPLER, 1)
    c.reset()
    return c


def render(c, run, mb, samples):
    """`samples` frames of `run` on c; -> the per-bounce statistics of each frame (one summed entry for "samples_fk1")."""
    if run == "samples_fk1":
        c.integrate_samples(mb, samples)
        return [c.frame_stats()]
    out = []
    for _ in range(samples):
        c.integrate_stepwise(mb) if run == "stepwise" else c.integrate(mb)
        out.append(c.frame_stats())
    return out


def summed(stats):
    return {k: np.sum([np.asarray(s[k], np.uint32) for s in stats], axis=0, dtype=np.uint32) for k in STAT_KEYS}


def check_run_stats(run, got, want, mb, where):
    """got: render()'s statistics; want: the reference's per-frame statistics ("samples_fk1" sums them)."""
    if run == "samples_fk1":
        got, want = [summed(got)], [summed(want)]
    check_stats(got[-1], want[-1], mb, where)


def same_rows(a, b, chunk=1024):
    """Bit equality of two radiance images (h, w, 4) in the rgb channels, a block of rows at a time."""
    for r in range(0, a.shape[0], chunk):
        if not np.array_equal(bits(a[r:r + chunk, :, :3]), bits(b[r:r + chunk, :, :3])):
            return False
    return True


def oracle(sc, cam, w, h, mb, samples, rank=0, world=1, tables=None):
    """Radiance of `samples` samples and the per-sample statistics of the rows rank::world."""
    o = Oracle(sc)
    acc = np.zeros((h, w, 4), "<f4"); stats = []
    try:
        o.set_sampler_tables(tables)
        for s in range(samples):
            acc, _, st = o.render(cam, w, h, mb, sample_idx=s, radiance=acc, row_first=rank, row_step=world, want_hits=False)
            stats.append(st)
    finally:
        o.set_sampler_tables(None)
    return acc, stats


def every_run_matches_oracle(sc, cam, w, h, mb, samples=2, rank=0, world=1, tables=None, runs=RUNS, where=()):
    oacc, ost = oracle(sc, cam, w, h, mb, samples, rank, world, tables)
    for run in runs:
        c = make(run, sc, cam, w, h, rank=rank, world=world, tables=tables)
        try:
            st = render(c, run, mb, samples)
            rad = c.read_radiance()
        finally:
            c.destroy()
        at = tuple(where) + (run, "rank %d/%d" % (rank, world))
        assert np.array_equal(bits(rad[rank::world, :, :3]), bits(oacc[rank::world, :, :3])), at
        check_run_stats(run, st, ost, mb, at)
    return oacc


# ------------------------------------------------------------------------------------ 1. the light byte
W1, H1, MB1 = 96, 64, 4
LIGHT_SCENES = {"lights_%d" % n: (lambda n=n: light_scene(n)) for n in LIGHT_COUNTS}
LIGHT_SCENES["edge_origins"] = edge_origin_scene


@pytest.mark.parametrize("name", sorted(LIGHT_SCENES))
def test_light_byte_every_schedule_matches_oracle(name):
    """Radiance bits and per-bounce counters (n_unoccluded above all) equal the oracle's on every schedule and on both ranks of a
    2-way partition: shadow rays toward lights 253 .. 256 and past them read their own light's direction and t_max."""
    sc = LIGHT_SCENES[name](); cam = default_camera(W1, H1)
    every_run_matches_oracle(sc, cam, W1, H1, MB1, where=(name,))
    for rank in (0, 1):
        every_run_matches_oracle(sc, cam, W1, H1, MB1, rank=rank, world=2, runs=("frame", "phase_graph"), where=(name,))


def test_light_byte_blue_noise_sampler():
    sc = light_scene(300); cam = default_camera(W1, H1)
    every_run_matches_oracle(sc, cam, W1, H1, MB1, tables=synthetic_sampler_tables(), where=("lights_300", "blue noise"))


@pytest.mark.parametrize("light", ("emitters", "environment", "both"))
def test_light_byte_beside_sampled_lights(light):
    """Emitter and environment samples keep three-plane records beside the two-plane and forced-three-plane records of 300
    analytic lights: every schedule equals the one-kernel frame."""
    sc = light_scene(300); cam = default_camera(W1, H1)
    opts = (((capi.OPT_EMITTER_SAMPLING, 1),) if light in ("emitters", "both") else ()) + \
           (((capi.OPT_ENV_SAMPLING, 1),) if light in ("environment", "both") else ())
    want = make("frame", sc, cam, W1, H1, opts)
    try:
        wst = render(want, "frame", MB1, 2)
        wrad = want.read_radiance()
    finally:
        want.destroy()
    assert int(np.asarray(wst[-1]["n_unoccluded"][: MB1 + 1]).sum()) > 0
    for run in ("phase_graph", "phase_direct", "timed", "stepwise"):
        c = make(run, sc, cam, W1, H1, opts)
        try:
            if run == "stepwise":
                c.integrate(MB1); c.reset()         # the stepwise steps take the frame's last bounce from the last rt_integrate call
            st = render(c, run, MB1, 2)
            assert np.array_equal(bits(c.read_radiance()[..., :3]), bits(wrad[..., :3])), (light, run)
            check_stats(st[-1], wst[-1], MB1, (light, run))
        finally:
            c.destroy()


# ------------------------------------------------------------------------------------ 2. 2^24 local pixels
MB2 = 3
# (width, height, rank, world): exactly 2^24 local pixels; one row past; 2^24 + 2048 on rank 0 and on rank 1 of two
BIG_FRAMES = [(4096, 4096, 0, 1), (4096, 4097, 0, 1), (2048, 16386, 0, 2), (2048, 16386, 1, 2)]


def band_rows(w, h, rank, world):
    """Global rows of row 0 of the rank, its last row and the rows of local pixels 2^24 - 1 and 2^24 (where it has them)."""
    n_rows = len(range(rank, h, world))
    local = {0, n_rows - 1} | {i // w for i in ((1 << 24) - 1, 1 << 24) if i < n_rows * w}
    return sorted(r * world + rank for r in local)


@pytest.mark.parametrize("w,h,rank,world", BIG_FRAMES, ids=lambda v: str(v))
def test_local_pixels_around_2_24(w, h, rank, world):
    """Every schedule renders the same bits and statistics; both ranks of the next partition up (two-plane) reproduce the rows;
    a band of rows (first, last, and those of local pixels 2^24 - 1 and 2^24) equals the oracle."""
    sc = scene("CornellBox"); cam = default_camera(w, h)
    n_local = len(range(rank, h, world)) * w
    assert (n_local == 1 << 24) if (w, h) == (4096, 4096) else (n_local > 1 << 24)
    ref = None
    for run in ("phase_graph",) + tuple(r for r in RUNS if r != "phase_graph"):
        c = make(run, sc, cam, w, h, rank=rank, world=world)
        try:
            assert c.local_pixel_count() == n_local
            st = render(c, run, MB2, 2)
            rad = c.read_radiance()
        finally:
            c.destroy()
        if ref is None:
            ref, ref_st = rad, st
            assert int(st[-1]["n_ext"][0]) == n_local
            continue
        assert same_rows(rad, ref), (w, h, rank, world, run)
        check_run_stats(run, st, ref_st, MB2, (w, h, rank, world, run))
        del rad
    # the next partition up: ranks rank and rank + world of 2 * world, each below 2^24 local pixels
    for sub in (rank, rank + world):
        c = make("phase_graph", sc, cam, w, h, rank=sub, world=2 * world)
        try:
            assert c.local_pixel_count() < 1 << 24
            render(c, "phase_graph", MB2, 2)
            rad = c.read_radiance()
        finally:
            c.destroy()
        assert same_rows(rad[sub::2 * world], ref[sub::2 * world]), (w, h, rank, world, "rank %d of %d" % (sub, 2 * world))
        del rad
    # a band of rows against the oracle
    o = Oracle(sc)
    acc = np.zeros((h, w, 4), "<f4")
    rows = band_rows(w, h, rank, world)
    for s in range(2):
        for r in rows:
            acc, _, _ = o.render(cam, w, h, MB2, sample_idx=s, radiance=acc, row_first=r, row_step=h, want_hits=False)
    for r in rows:
        assert np.array_equal(bits(ref[r, :, :3]), bits(acc[r, :, :3])), (w, h, rank, world, "row %d" % r)


def test_local_pixels_past_2_24_with_emitter_sampling():
    """4096 x 4097 with emitter sampling: sampled-light records (always three-plane) at this size; the per-phase frame equals the
    one-kernel frame and the rows of both ranks of a 2-way partition."""
    w, h = 4096, 4097
    sc = scene("CornellBox"); cam = default_camera(w, h)
    opts = ((capi.OPT_EMITTER_SAMPLING, 1),)
    ref = None
    for run in ("phase_graph", "frame"):
        c = make(run, sc, cam, w, h, opts)
        try:
            st = render(c, run, MB2, 2)
            rad = c.read_radiance()
        finally:
            c.destroy()
        if ref is None:
            ref, ref_st = rad, st
            continue
        assert same_rows(rad, ref), run
        check_stats(st[-1], ref_st[-1], MB2, (run,))
        del rad
    for sub in (0, 1):
        c = make("phase_graph", sc, cam, w, h, opts, rank=sub, world=2)
        try:
            render(c, "phase_graph", MB2, 2)
            rad = c.read_radiance()
        finally:
            c.destroy()
        assert same_rows(rad[sub::2], ref[sub::2]), ("rank %d of 2" % sub)
        del rad


# ------------------------------------------------------------------------------------ 3. 16-bit pixel coordinates
MB3 = 3
WIDE_FRAMES = [(65535, 2), (2, 65535), (32769, 3)]


@pytest.mark.parametrize("w,h", WIDE_FRAMES, ids=lambda v: str(v))
def test_pixel_coordinates_at_16_bits(w, h):
    """Every schedule equals the whole-frame oracle; at least a quarter of the primary rays hit."""
    sc = scene("CornellBox"); cam = default_camera(w, h)
    oacc = every_run_matches_oracle(sc, cam, w, h, MB3, where=(w, h))
    _, ost = oracle(sc, cam, w, h, MB3, 1)
    assert int(ost[0]["n_miss"][0]) * 4 <= 3 * w * h
    if (w, h) == (65535, 2):
        c = make("phase_graph", sc, cam, w, h)
        try:
            render(c, "phase_graph", MB3, 2)
            img = c.resolve()
        finally:
            c.destroy()
        z4, z1, z2 = np.zeros((h, w, 4), "<f4"), np.zeros((h, w), "<f4"), np.zeros((h, w, 2), "<f4")
        assert np.array_equal(bits(img), bits(Oracle(sc).resolve(0, oacc, z4, z1, z4, z2, 2)))


def test_pixel_coordinates_one_row_per_rank():
    """65535 x 3 over a 3-way partition: each rank's one row on every schedule equals the oracle's."""
    w, h = 65535, 3
    sc = scene("CornellBox"); cam = default_camera(w, h)
    for rank in range(3):
        every_run_matches_oracle(sc, cam, w, h, MB3, rank=rank, world=3, where=(w, h))


@pytest.mark.parametrize("w,h,rank,world", [(65535, 2, 0, 1), (2, 65535, 0, 1), (32769, 3, 0, 1), (65535, 3, 1, 3)],
                         ids=lambda v: str(v))
def test_pixel_coordinates_decoded_by_the_taps(w, h, rank, world):
    """rt_read_rays (k_unpack_rays, on the device) and rt_read_hits (on the host) decode B.w into the pixel index."""
    sc = scene("CornellBox"); cam = default_camera(w, h)
    c = make("stepwise", sc, cam, w, h, rank=rank, world=world)
    try:
        c.generate_rays(); c.intersect(0)
        want = (np.arange(rank, h, world)[:, None] * w + np.arange(w)[None, :]).ravel().astype(np.uint32)
        _, rpix = c.read_rays(0)
        _, hpix = c.read_hits(0)
    finally:
        c.destroy()
    assert np.array_equal(rpix, want), "rt_read_rays"
    assert np.array_equal(hpix, want), "rt_read_hits"


@pytest.mark.parametrize("w,h", WIDE_FRAMES, ids=lambda v: str(v))
def test_pixel_coordinates_adaptive_partial_active_list(w, h):
    """Adaptive sampling traces a partial list of pixels: the per-phase frames and the one-kernel frame equal the stepwise
    schedule, pixel counts included."""
    sc = scene("CornellBox"); cam = default_camera(w, h)

    def run(r):
        c = make(r, sc, cam, w, h)
        try:
            c.set_adaptive_sampling(0.05, 2); c.reset()
            st = render(c, r, MB3, 8)
            return c.read_radiance(), st[-1], c.pixel_samples()
        finally:
            c.destroy()
    wrad, wst, wcounts = run("stepwise")
    assert 0 < int(wst["n_ext"][0]) < w * h, int(wst["n_ext"][0])
    for r in ("phase_graph", "phase_direct", "frame"):
        rad, st, counts = run(r)
        assert np.array_equal(bits(rad), bits(wrad)), r
        check_stats(st, wst, MB3, (r,))
        assert np.array_equal(counts, wcounts), r


def test_frame_extents_accepted_and_refused():
    for w, h in ((65535, 1), (1, 65535)):
        capi.Context(w, h).destroy()
    for w, h in ((65536, 1), (1, 65536)):
        with pytest.raises(capi.RtError) as e:
            capi.Context(w, h)
        assert e.value.code == -1, (w, h)               # RT_ERR_INVALID_ARGUMENT


# ------------------------------------------------------------------------------------ 4. the counter batch of the N-frame loop
def test_counter_batch_of_the_n_frame_loop():
    """integrate_samples(1, 300) on the one-kernel frame with adaptive sampling that stops nothing: n k_frame launches whose
    packed counters are folded every 0xFFFFFFFF // 2^24 = 255 frames, so the call crosses one fold.  Every frame traces 2^24
    primary rays, all of which hit: the hit word of the {hit, miss} pair gains exactly 2^24 per frame, so a fold one frame late
    (256 x 2^24 = 2^32) would carry into n_miss.  All but a handful of hits per frame (a light sample or BSDF sample of zero) also
    spawn a shadow and a continuation ray.  The sums equal 300 per-phase frames', which wrap mod 2^32 like every uint32 counter."""
    w = h = 4096
    n, frames = 1 << 24, 300
    sc = wall_scene(); cam = default_camera(w, h)

    def ctx(run):
        c = make(run, sc, cam, w, h)
        c.set_adaptive_sampling(1e-6, 1000); c.reset()
        return c
    c = ctx("phase_graph")
    try:
        total = {k: np.zeros(capi.MAX_BOUNCES + 1, np.uint32) for k in STAT_KEYS}
        for f in range(frames):
            c.integrate(1)
            st = c.frame_stats()
            assert (int(st["n_ext"][0]), int(st["n_miss"][0])) == (n, 0), f
            assert min(int(st["n_shadow"][0]), int(st["n_cont"][0])) >= n - 256, f
            for k in STAT_KEYS:
                total[k] += st[k]
        want = c.read_radiance()
    finally:
        c.destroy()
    wrapped = (frames * n) % (1 << 32)
    assert int(total["n_ext"][0]) == wrapped
    assert int(total["n_shadow"][0]) + (1 << 32) >= frames * (n - 256)          # the sums wrapped once, as 300 x 2^24 does
    c = ctx("frame")
    try:
        c.integrate_samples(1, frames)
        st = c.frame_stats()
        rad = c.read_radiance()
    finally:
        c.destroy()
    assert (int(st["n_ext"][0]), int(st["n_miss"][0])) == (wrapped, 0), (int(st["n_ext"][0]), int(st["n_miss"][0]))
    for k in STAT_KEYS:
        assert np.array_equal(np.asarray(st[k][:2]), total[k][:2]), (k, np.asarray(st[k][:2]).tolist(), total[k][:2].tolist())
    assert same_rows(rad, want)
