"""
CPU tests (-m "not gpu"): the oracle restatement against what the reference's own kernels (oracle/_ref, the reference's
OpenCL kernels compiled for the CPU by oracle/build_ref.py) produced on configurations other than the committed golden
images (different resolution / bounce count / sample index / options).  The reference's per-bounce counters and the
digests of its radiance bits and primary hits are stored in tests/golden/ref/ (tests/golden/make_ref_records.py writes
them from the same case lists).  Bar: bit-exact.
"""
import os

import numpy as np
import pytest

from oracle.orcbind import Oracle
from raytracing_b200.camera import default_camera
from tests.helpers import GOLDEN, assert_frames, bits, digest, frame_record, fuzz_configs, scene, synthetic_sampler_tables

BIT_EXACT_CASES = [
    ("CornellBox", 97, 61, 3, False),
    ("CornellBox", 64, 64, 5, True),
    ("ShaderBalls", 160, 90, 8, False),
    ("CornellBox_Dragon", 120, 68, 6, False),
]
AOV_CASES = ["CornellBox", "ShaderBalls"]
BLUE_NOISE_CASES = [
    ("CornellBox", 160, 136, 3, False),        # > 128 x 128: every tile pixel, incl. the ones whose ranking index runs past the table
    ("ShaderBalls", 144, 130, 8, False),
    ("CornellBox", 64, 64, 4, True),
]
LIGHTS_CASES = [("CornellBox", 150, 90, 5), ("ShaderBalls", 128, 72, 4)]
DEGENERATE_CASES = {"zero_bounces": ("CornellBox", 96, 64, 0, {}),
                    "all_miss": ("ShaderBalls", 80, 48, 4, {"position": (0.0, -30.0, 40.0), "pitch": 0.3}),
                    "inside_geometry": ("ShaderBalls", 80, 48, 4, {"position": (0.0, 0.0, 0.35), "pitch": 1.9})}
# the closed box (tests/scenes_extra.closed_cornell): paths that never leave it, throughput decaying through the subnormal range.
# 60 bounces passes the wrap of the blue-noise dimension (bounce * 5 + type) & 255 at bounce 51; 255 is RT_MAX_BOUNCES.
LONG_PATH_CASES = [(48, 32, 60, "blue_noise"), (48, 32, 255, "random")]
# late sample indices: 258 accumulated samples, records of the last four (the blue-noise sample index wraps at 256)
LATE_SAMPLE_CASES = [("CornellBox", 24, 16, 2, "random"), ("CornellBox", 24, 16, 2, "blue_noise")]
LATE_SAMPLE_COUNT, LATE_SAMPLE_KEEP = 258, (254, 255, 256, 257)
LIBM_CASES = [("CornellBox", 160, 90, 8, 0.02), ("ShaderBalls", 160, 90, 8, 0.02), ("CornellBox_Dragon", 160, 90, 16, 0.04)]
LIBM_SAMPLE = 1024          # pixels of each frame kept in tests/golden/ref/libm_sample.npz (seeded)


def libm_sample_index(w, h):
    return np.sort(np.random.default_rng(4321).choice(w * h, LIBM_SAMPLE, replace=False))


def aov_cameras(w, h):
    return [default_camera(w, h), default_camera(w, h, position=(0.05, -1.02, 1.01)), default_camera(w, h, position=(0.05, -1.02, 1.01))]


def lights_camera(w, h):
    return default_camera(w, h, position=(0.15, -1.3, 0.9), aperture=0.04, focus_distance=1.7)


def oracle_samples(sc, cam, w, h, mb, n, wf=False, with_hits=True, tables=None, keep=None):
    """Records of n progressively accumulated samples (sample_idx 0, 1, ...), or of the samples listed in `keep`; kBlueNoise
    with `tables`."""
    o = Oracle(sc)
    acc = np.zeros((h, w, 4), dtype="<f4")
    out = []
    try:
        o.set_sampler_tables(tables)
        for sample in range(n):
            acc, hits, st = o.render(cam, w, h, mb, sample_idx=sample, white_furnace=wf, radiance=acc)
            if keep is None or sample in keep:
                out.append(frame_record(st, mb, acc, hits if with_hits else None))
    finally:
        o.set_sampler_tables(None)
    return out, st


def sampler_tables(sampler):
    return synthetic_sampler_tables() if sampler == "blue_noise" else None


@pytest.mark.parametrize("name,w,h,mb,wf", BIT_EXACT_CASES)
def test_oracle_bit_exact_vs_reference_kernels(name, w, h, mb, wf):
    recs, _ = oracle_samples(scene(name), default_camera(w, h), w, h, mb, 2, wf)
    assert_frames("bit_exact/%s_%dx%d_b%d_wf%d" % (name, w, h, mb, wf), recs)


@pytest.mark.parametrize("name", AOV_CASES)
def test_aov_denoiser_resolve_restatements_vs_reference_kernels(name):
    """orc_aovs / orc_temporal_accumulation / orc_resolve against aov.cl, denoiser.cl, resolve_radiance.cl (3 frames, moving camera)."""
    sc = scene(name); w, h, mb = 128, 72, 3
    o = Oracle(sc)
    cams = aov_cameras(w, h)
    prev = np.zeros((), dtype=cams[0].dtype)
    prev_rad = np.zeros((h, w, 4), "<f4"); prev_depth = np.zeros((h, w), "<f4")
    recs = []
    for f, cam in enumerate(cams):
        rad, _, _ = o.render(cam, w, h, mb, sample_idx=f)
        al, de, no, ve = o.aovs(cam, prev, w, h, sample_idx=f)
        den = o.temporal_accumulation(rad, prev_rad, de, prev_depth, ve)
        recs.append({"albedo": digest(bits(al[..., :3])), "depth": digest(bits(de)), "normal": digest(bits(no[..., :3])),
                     "velocity": digest(bits(ve)), "radiance": digest(bits(den[..., :3])),
                     "resolved": digest(bits(o.resolve(0, den, al, de, no, ve, f + 1, denoiser=True)))})
        prev_rad, prev_depth, prev = den, de, cam
    assert_frames("aov/" + name, recs)


def test_textured_materials_bit_exact_vs_reference_kernels():
    """ApplyTextures / SampleTexture (material.h:251-264,319-369) on every texture slot, wrapped coordinates included."""
    from tests.scenes_extra import textured_cornell
    sc = textured_cornell()
    w, h, mb = 96, 64, 4
    cam = default_camera(w, h)
    rad, hits, st = Oracle(sc).render(cam, w, h, mb)
    assert_frames("textured", [frame_record(st, mb, rad, keys=("n_ext", "n_miss", "n_shadow", "n_cont", "n_unoccluded"))])
    # the textured image must differ from the untextured one (the textures are really used)
    plain, _, _ = Oracle(scene("CornellBox")).render(cam, w, h, mb)
    assert not np.array_equal(bits(plain), bits(rad))


@pytest.mark.parametrize("name,w,h,mb,wf", BLUE_NOISE_CASES)
def test_blue_noise_sampler_bit_exact_vs_reference_kernels(name, w, h, mb, wf):
    """SamplerType::kBlueNoise (sampling.h:40-61): the restatement against hit_surface.cl built with -DBLUE_NOISE_SAMPLER, both
    reading the seeded tables of tests/helpers.synthetic_sampler_tables, three progressive samples."""
    sc = scene(name)
    cam = default_camera(w, h)
    o = Oracle(sc)
    tables = synthetic_sampler_tables()
    try:
        o.set_sampler_tables(tables)
        acc = np.zeros((h, w, 4), dtype="<f4")
        recs = []
        for sample in range(3):
            acc, hits, st = o.render(cam, w, h, mb, sample_idx=sample, white_furnace=wf, radiance=acc)
            recs.append(frame_record(st, mb, acc))
        assert_frames("blue_noise/%s_%dx%d_b%d_wf%d" % (name, w, h, mb, wf), recs)
        # and the sampler did change the image
        o.set_sampler_tables(None)
        plain, _, _ = o.render(cam, w, h, mb, sample_idx=0, white_furnace=wf)
        first, _, _ = (o.set_sampler_tables(tables), o.render(cam, w, h, mb, sample_idx=0, white_furnace=wf))[1]
        assert not np.array_equal(bits(plain), bits(first))
    finally:
        o.set_sampler_tables(None)


@pytest.mark.parametrize("name,w,h,mb", LIGHTS_CASES)
def test_point_lights_and_thin_lens_bit_exact_vs_reference_kernels(name, w, h, mb):
    """Five analytic lights (point + directional, light.h:30-65) and a thin-lens camera (aperture > 0: the hexagonal
    aperture sampling of raygeneration.cl:40-49,108-124), moved off the default pose."""
    from tests.scenes_extra import many_lights_scene
    recs, st = oracle_samples(many_lights_scene(name), lights_camera(w, h), w, h, mb, 2)
    assert_frames("lights/%s_%dx%d_b%d" % (name, w, h, mb), recs)
    assert st["n_shadow"][:mb].min() > 0 and st["n_unoccluded"][:mb].min() > 0


@pytest.mark.parametrize("case", list(DEGENERATE_CASES))
def test_degenerate_frames_bit_exact_vs_reference_kernels(case):
    """max_bounces = 0 (one extension pass, one shadow pass); a camera that only sees the sky (every queue after bounce 0
    is empty); a camera placed inside a ShaderBall (rays start inside closed geometry: back faces are culled)."""
    name, w, h, mb, kw = DEGENERATE_CASES[case]
    recs, st = oracle_samples(scene(name), default_camera(w, h, **kw), w, h, mb, 2)
    assert_frames("degenerate/" + case, recs)
    if case == "all_miss":
        assert st["n_hit"][0] == 0 and st["n_ext"][1] == 0


@pytest.mark.parametrize("cfg", fuzz_configs(), ids=lambda c: f"{c[0]}_{c[1]}x{c[2]}_b{c[3]}")
def test_fuzzed_frames_bit_exact_vs_reference_kernels(cfg):
    """Seeded random scenes / sizes / bounce counts / camera poses and lenses, two progressive samples each."""
    name, w, h, mb, kw, wf = cfg
    recs, _ = oracle_samples(scene(name), default_camera(w, h, **kw), w, h, mb, 2, wf)
    assert_frames("fuzzed/%d" % fuzz_configs().index(cfg), recs)


@pytest.mark.parametrize("w,h,mb,sampler", LONG_PATH_CASES)
def test_long_paths_bit_exact_vs_reference_kernels(w, h, mb, sampler):
    """Paths of up to 256 segments inside the closed box (no Russian roulette in the reference): the blue-noise dimension
    wraps at bounce 51, the throughput underflows through the subnormals and the shadow-ray test dot(light_sample,
    light_sample) > 0 (hit_surface.cl:127) then turns on whether subnormals are kept.  Two progressive samples."""
    from tests.scenes_extra import closed_cornell
    recs, st = oracle_samples(closed_cornell(), default_camera(w, h), w, h, mb, 2, tables=sampler_tables(sampler))
    assert_frames("long_path/closed_cornell_%dx%d_b%d_%s" % (w, h, mb, sampler), recs)
    assert st["n_ext"][mb] == w * h                 # nothing escapes the box
    assert st["n_shadow"][mb] < st["n_shadow"][10] // 4


@pytest.mark.parametrize("name,w,h,mb,sampler", LATE_SAMPLE_CASES)
def test_late_sample_indices_bit_exact_vs_reference_kernels(name, w, h, mb, sampler):
    """Sample indices 254..257 of one accumulation (the blue-noise sampler wraps the index with & 255, kRandom hashes it)."""
    recs, _ = oracle_samples(scene(name), default_camera(w, h), w, h, mb, LATE_SAMPLE_COUNT, tables=sampler_tables(sampler),
                             keep=LATE_SAMPLE_KEEP)
    assert_frames("late_sample/%s_%dx%d_b%d_%s" % (name, w, h, mb, sampler), recs)


@pytest.mark.parametrize("name,w,h,mb,limit", LIBM_CASES)
def test_math_library_sensitivity_is_small(name, w, h, mb, limit):
    """The OpenCL driver's libm is unpinned (SURVEY 8c).  Swapping include/rt_math.h for glibc's libm inside the
    reference kernels must leave all but a small fraction of pixels within 1e-4 relative — on all three shipped scenes (the
    mirror / metal paths of the Dragon scene at 16 bounces are the most sensitive).  The libm build's frame is stored as a
    seeded sample of its pixels; the oracle stands in for the rt_math build (bit-identical to it, tests above).
    include/rt_math.h itself is pinned against double-precision libm in tests/test_rt_math.py."""
    b = np.load(os.path.join(GOLDEN, "ref", "libm_sample.npz"))[name].astype(np.float64)
    rad, _, _ = Oracle(scene(name)).render(default_camera(w, h), w, h, mb)
    a = rad[..., :3].reshape(-1, 3)[libm_sample_index(w, h)].astype(np.float64)
    rel = np.abs(a - b) / np.maximum(np.abs(a), 1e-6)
    frac_bad = (rel.max(axis=-1) > 1e-4).mean()
    assert frac_bad < limit, frac_bad
