"""
GPU tests (-m gpu) of what rt_integrate selects and of ground no other test renders: the automatic choice between the
one-kernel frame and the per-phase kernels and the CTA shape of the former at their thresholds, every CTA size option, paths
of up to RT_MAX_BOUNCES bounces, sample indices past the wrap of the blue-noise sampler, and the temporal denoiser fed by
rt_integrate.  Everything is compared with the CPU oracle bit for bit; the oracle itself is pinned to the reference's kernels
on the same ground in tests/test_oracle_vs_ref.py (long paths, late samples).
"""
import numpy as np
import pytest

from oracle.orcbind import Oracle
from raytracing_b200 import capi
from raytracing_b200.camera import default_camera
from tests.helpers import bits, scene, synthetic_sampler_tables
from tests.scenes_extra import closed_cornell
from tests.test_gpu_parity import BASIC, SCHEDULES, check_frame, check_stats, destroy, schedule_ctx, schedules_match_oracle

pytestmark = pytest.mark.gpu

STAT_KEYS = ("n_ext", "n_miss", "n_shadow", "n_cont", "n_unoccluded", "n_emissive_hits")


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def frame_launches(c, mb):
    """Renders one frame with rt_integrate; returns the number of kernels it launched."""
    before = c.launch_count()
    c.integrate(mb)
    return c.launch_count() - before


# staging of the BVH in the traversal kernels: ShaderBalls does not fit shared memory and is fetched through L1 (k_frame<0>),
# or stages the top of its tree (k_frame<2>); CornellBox is staged whole (k_frame<1>)
STAGING = {"l1": ("ShaderBalls", ()), "top": ("ShaderBalls", ((capi.OPT_TOP_SMEM, 100),)), "whole": ("CornellBox", ())}


@pytest.mark.parametrize("rows_per_sm_row", [512, 513, 896, 897], ids=lambda r: "%d_px_per_sm" % (8 * r))
def test_frame_kernel_selector_at_its_thresholds(rows_per_sm_row):
    """Images of width 8 x SMs and 512 / 513 / 896 / 897 rows: 4096, 4096 + one row, 7168 and 7168 + one row pixels per SM.
    RT_OPT_FRAME_KERNEL = 2 (default) runs the one-kernel frame (one launch) up to 7168 pixels per SM and the per-phase graph
    above (include/rt_b200.h); the automatic CTA shape of the one-kernel frame switches to 1024 threads above 4096 pixels per
    SM for scenes that are not staged whole.  Default, per-phase and one-kernel frames are bit-identical over the whole frame,
    and a band of rows equals the oracle."""
    sms = sm_count()
    w, h, mb = 8 * sms, rows_per_sm_row, 4
    one_kernel = w * h <= 7168 * sms
    sc = scene("ShaderBalls"); cam = default_camera(w, h)
    row_first, row_step = 3, 61
    orad, _, _ = Oracle(sc).render(cam, w, h, mb, row_first=row_first, row_step=row_step)
    rows = np.arange(row_first, h, row_step)
    for staging in ("l1", "top"):
        _, options = STAGING[staging]
        imgs, launches, stats = {}, {}, {}
        for fk in (2, 0, 1):
            c = schedule_ctx(None, sc, cam, w, h, options + ((capi.OPT_FRAME_KERNEL, fk),))
            c.reset()
            frame_launches(c, mb)                   # the per-phase schedule captures its graph on the first frame
            c.reset()
            launches[fk] = frame_launches(c, mb)
            imgs[fk] = c.read_radiance(); stats[fk] = c.frame_stats()
            c.destroy()
        assert launches[1] == 1 and launches[0] > 1, (staging, launches)
        assert launches[2] == launches[1 if one_kernel else 0], (staging, w, h, launches)
        for fk in (0, 1):
            assert np.array_equal(bits(imgs[fk]), bits(imgs[2])), (staging, w, h, fk)
            for k in STAT_KEYS:
                assert np.array_equal(stats[fk][k][: mb + 1], stats[2][k][: mb + 1]), (staging, w, h, fk, k)
        assert np.array_equal(bits(imgs[2][rows][..., :3]), bits(orad[rows][..., :3])), (staging, w, h)


@pytest.mark.parametrize("staging", list(STAGING))
def test_frame_threads_option_matches_oracle(staging):
    """RT_OPT_FRAME_THREADS 32 (one warp per CTA: the 32-CTA per SM occupancy cap), 96 (not a power of two), 512 and 1024 for
    each staging of the BVH, on the whole image and on a 3-way scanline partition, two progressive samples."""
    name, options = STAGING[staging]
    sc = scene(name)
    w, h, mb = 160, 91, 5
    cam = default_camera(w, h)
    o = Oracle(sc)
    oacc = np.zeros((h, w, 4), dtype="<f4")
    ost = []
    for sample in range(2):
        oacc, _, st = o.render(cam, w, h, mb, sample_idx=sample, radiance=oacc.copy())
        ost.append((oacc, st))
    for threads in (32, 96, 512, 1024):
        for world in (1, 3):
            ctxs = [schedule_ctx("frame", sc, cam, w, h, options + ((capi.OPT_FRAME_THREADS, threads),), rank=r, world=world)
                    for r in range(world)]
            for c in ctxs:
                c.reset()
            for sample, (want, st) in enumerate(ost):
                rad = np.zeros((h, w, 4), "<f4")
                total = {k: np.zeros(mb + 1, np.int64) for k in STAT_KEYS}
                for c in ctxs:
                    c.integrate(mb)
                    c.read_radiance(rad)
                    cst = c.frame_stats()
                    for k in STAT_KEYS:
                        total[k] += cst[k][: mb + 1]
                where = (name, staging, threads, world, "sample %d" % sample)
                check_stats(total, st, mb, where)
                assert np.array_equal(bits(rad[..., :3]), bits(want[..., :3])), where
            for c in ctxs:
                c.destroy()
    c = capi.Context(32, 32)
    for bad in (33, 1056):
        with pytest.raises(capi.RtError):
            c.set_option(capi.OPT_FRAME_THREADS, bad)
    c.destroy()


@pytest.mark.parametrize("mb,sampler", [(60, "blue_noise"), (60, "random"), (255, "random")])
def test_long_paths_match_oracle(mb, sampler):
    """Paths that never leave the closed box, up to RT_MAX_BOUNCES: the blue-noise dimension (bounce * 5 + type) & 255 wraps
    at bounce 51, and the throughput decays through the subnormal range, where the shadow-ray test dot(light_sample,
    light_sample) > 0 (hit_surface.cl:127) depends on subnormals being kept (no flush to zero)."""
    w, h = 64, 48
    sc = closed_cornell(); cam = default_camera(w, h)
    _, _, ost = Oracle(sc).render(cam, w, h, mb)
    # the case must stay what it is meant to be: long paths, and (at 255) a shadow-ray count that collapses while the paths go on
    assert ost["n_ext"][55] >= ost["n_ext"][0] // 2, ost["n_ext"][: mb + 1]
    if mb == 255:
        hit = ost["n_ext"] - ost["n_miss"]
        assert ost["n_ext"][255] >= ost["n_ext"][0] // 2 and ost["n_shadow"][10] > hit[10] // 4
        assert (ost["n_shadow"][200:256] < hit[200:256] // 10).all(), ost["n_shadow"][: mb + 1]
    tables = synthetic_sampler_tables() if sampler == "blue_noise" else None
    ctxs, _ = schedules_match_oracle(sc, cam, w, h, mb, BASIC, tables=tables, where=("closed_cornell", mb, sampler))
    with pytest.raises(capi.RtError):
        ctxs["frame"].integrate(256)
    destroy(ctxs)


@pytest.mark.parametrize("n", [255, 256, 257, 65537])
@pytest.mark.parametrize("sampler", ["random", "blue_noise"])
def test_late_sample_indices_match_oracle(n, sampler):
    """rt_advance_sample_count N times (no launch), then one frame: the frame of sample index N and its resolve with N + 1
    samples.  The blue-noise sampler wraps the index with & 255; kRandom hashes all 32 bits."""
    name, w, h, mb = "CornellBox", 136, 72, 3
    sc = scene(name); cam = default_camera(w, h)
    tables = synthetic_sampler_tables() if sampler == "blue_noise" else None
    o = Oracle(sc)
    try:
        o.set_sampler_tables(tables)
        orad, _, ost = o.render(cam, w, h, mb, sample_idx=n)
    finally:
        o.set_sampler_tables(None)
    z4, z1, z2 = np.zeros((h, w, 4), "<f4"), np.zeros((h, w), "<f4"), np.zeros((h, w, 2), "<f4")
    want = o.resolve(0, orad, z4, z1, z4, z2, n + 1)
    for schedule in ("frame", "phase_graph"):
        c = schedule_ctx(schedule, sc, cam, w, h)
        if tables is not None:
            c.upload_sampler_tables(*tables); c.set_option(capi.OPT_SAMPLER, 1)
        c.reset()
        for _ in range(n):
            c.advance_sample_count()
        c.integrate(mb)
        where = (name, schedule, sampler, "sample %d" % n)
        check_frame(c, ost, orad, mb, where)
        assert c.sample_count() == n + 1, where
        assert np.array_equal(bits(c.resolve()), bits(want)), where
        c.destroy()


@pytest.mark.parametrize("schedule", ["frame", "phase_graph", "phase_direct"])
def test_denoiser_fed_by_integrate_matches_oracle(schedule):
    """Integrator::Integrate with the denoiser on, driven by rt_integrate: per frame set_camera, reset, integrate, denoise,
    copy_history, resolve; three frames, the camera moves between the first two.  The AOVs (velocity from the previous
    SetCameraData camera, which the frame graph must refresh), the denoised radiance and the resolved image equal the oracle."""
    name, w, h, mb = "ShaderBalls", 192, 108, 3
    sc = scene(name)
    o = Oracle(sc)
    cams = [default_camera(w, h), default_camera(w, h, position=(0.05, -1.02, 1.01)), default_camera(w, h, position=(0.05, -1.02, 1.01))]
    c = capi.Context(w, h)
    c.upload_scene(sc)                          # no camera yet: the first frame's previous camera is the zero-initialised one
    for k, v in SCHEDULES[schedule] + ((capi.OPT_DENOISER, 1),):
        c.set_option(k, v)
    prev_cam = np.zeros((), dtype=cams[0].dtype)
    prev_rad = np.zeros((h, w, 4), "<f4"); prev_depth = np.zeros((h, w), "<f4")
    for f, cam in enumerate(cams):
        c.set_camera(cam); c.reset(); c.integrate(mb); c.denoise(); c.copy_history()
        img = c.resolve()
        where = (name, schedule, "frame %d" % f)
        rad, _, ost = o.render(cam, w, h, mb, sample_idx=f)
        check_stats(c.frame_stats(), ost, mb, where)
        al, de, no, ve = o.aovs(cam, prev_cam, w, h, sample_idx=f)
        gal, gde, gno, gve = c.read_aovs()
        assert np.array_equal(bits(gal[..., :3]), bits(al[..., :3])) and np.array_equal(bits(gde), bits(de)), where
        assert np.array_equal(bits(gno[..., :3]), bits(no[..., :3])), where
        assert np.array_equal(bits(gve), bits(ve)), where
        den = o.temporal_accumulation(rad, prev_rad, de, prev_depth, ve)
        assert np.array_equal(bits(c.read_radiance()[..., :3]), bits(den[..., :3])), where
        assert np.array_equal(bits(img), bits(o.resolve(0, den, al, de, no, ve, f + 1, denoiser=True))), where
        prev_rad, prev_depth, prev_cam = den, de, cam
    c.destroy()
