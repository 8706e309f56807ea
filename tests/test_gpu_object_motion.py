"""
GPU tests (-m gpu) of object motion vectors (RT_OPT_OBJECT_MOTION, include/rt_b200.h): the AOVs after uploads and updates equal the
CPU model of tests/motion_model.cpp bit for bit on every schedule, with the previous positions being the array each update
replaced; radiance and per-bounce statistics equal those of the option off.  Also: the option on with no update changes no byte;
the host variant over several staging chunks and the device variant; rebuilds keep the previous positions and a re-upload resets
them; graph replay across updates; the temporal denoiser end to end; multi-device contexts, partitions and adaptive sampling;
argument errors and device memory; the C++ host path.
"""
import ctypes as C

import numpy as np
import pytest

from raytracing_b200 import capi
from raytracing_b200.camera import default_camera
from tests.helpers import bits, scene
from tests.motion_model import MotionModel, positions
from tests.refit_model import deform, refit
from tests.test_gpu_parity import SCHEDULES, check_stats, run_frame
from tests.test_gpu_refit import RUNS

pytestmark = pytest.mark.gpu

W, H, MB = 64, 48, 3
CAM_KEYS = ("n_ext", "n_miss", "n_shadow", "n_cont", "n_unoccluded", "n_emissive_hits")
MOTION = (capi.OPT_OBJECT_MOTION, 1)


def with_tris(sc, t):
    """The scene dict of triangles t (leaf order) with the uploaded tree refit over them (what the device traverses after an update)."""
    return {**sc, "triangles": t, "nodes": refit(sc["nodes"], t)}


def make(schedule, sc, cam, options=(), motion=True, prev_cam=None, w=W, h=H, **kw):
    """A context that runs `schedule` with the AOVs produced every frame; rt_set_camera is called twice (prev_cam, then cam), so that
    the previous camera is prev_cam (default: cam).  Object motion is switched on after the upload.  Not reset yet."""
    c = capi.Context(w, h, **kw)
    c.upload_scene(sc)
    c.set_camera(cam if prev_cam is None else prev_cam); c.set_camera(cam)
    for k, v in SCHEDULES.get(schedule, ()) + tuple(options) + ((capi.OPT_AOV_ALWAYS, 1),) + ((MOTION,) if motion else ()):
        c.set_option(k, v)
    return c


def assert_aovs(got, want, where):
    for g, x, name in zip(got, want, ("albedo", "depth", "normal", "velocity")):
        if name in ("albedo", "normal"):
            g, x = g[..., :3], x[..., :3]
        assert np.array_equal(bits(g), bits(x)), (name,) + tuple(where)


def frame(c, schedule, samples=1):
    c.reset()
    if samples > 1:
        c.integrate_samples(MB, samples)
    else:
        run_frame(c, schedule, MB)


def sequence(sc, cams):
    """upload A, update B, update C: (triangles, the previous positions Q after the step, the camera of the frame after it)."""
    a = sc["triangles"]
    b = deform(a, "rigid", seed=3, amount=0.08)
    cc = deform(b, "noise", seed=5)
    return [(a, a, cams[0]), (b, a, cams[1]), (cc, b, cams[1])]


def run_sequence(schedule, options=(), samples=1, name="ShaderBalls"):
    """The upload / update / update sequence with a frame after each step on a context with the option on and one with it off: the
    AOVs equal the model (Q = the array each update replaced; the camera moves with the first update), radiance and statistics equal
    the option off's."""
    sc = scene(name)
    cams = [default_camera(W, H), default_camera(W, H, position=(0.04, -1.03, 1.02))]
    on = make(schedule, sc, cams[0], options)
    off = make(schedule, sc, cams[0], options, motion=False)
    prev_cam = cams[0]                                           # the camera of the set_camera call before the last, throughout
    try:
        for step, (t, q, cam) in enumerate(sequence(sc, cams)):
            for c in (on, off):
                if step:
                    c.update_triangles(t)
                if step == 1:
                    c.set_camera(cam)
                frame(c, schedule, samples)
            where = (schedule, options, "step %d" % step)
            want = MotionModel(with_tris(sc, t)).mv_aovs(q, cam, prev_cam, W, H, sample_idx=samples - 1)
            assert_aovs(on.read_aovs(), want, where)
            assert np.array_equal(bits(on.read_radiance()[..., :3]), bits(off.read_radiance()[..., :3])), where
            check_stats(on.frame_stats(), off.frame_stats(), MB, where)
            if step:
                assert np.any(want[3] != MotionModel(with_tris(sc, t)).aovs(cam, prev_cam, W, H, sample_idx=samples - 1)[3]), where
    finally:
        on.destroy(); off.destroy()


@pytest.mark.parametrize("run", sorted(RUNS))
def test_every_run_matches_model(run):
    schedule, options = RUNS[run]
    run_sequence(schedule, options)


def test_forced_frame_kernel_samples_match_model():
    """rt_integrate_samples with RT_OPT_FRAME_KERNEL 1 (N one-kernel frames): the AOVs are those of the call's last sample."""
    run_sequence("frame", (), samples=3)


def test_sorted_shading_pass_matches_model():
    """A 4K frame takes the sorted shading pass (k_shade_queues<true, ...>): one update, the whole AOV planes against the model."""
    w, h = 3840, 2160
    sc = scene("CornellBox")
    cam = default_camera(w, h)
    t = deform(sc["triangles"], "rigid", seed=4, amount=0.08)
    c = make("phase_graph", sc, cam, w=w, h=h)
    off = make("phase_graph", sc, cam, motion=False, w=w, h=h)
    for x in (c, off):
        x.update_triangles(t); x.reset(); x.integrate(2)
    want = MotionModel(with_tris(sc, t)).mv_aovs(sc["triangles"], cam, cam, w, h)
    assert_aovs(c.read_aovs(), want, ("4K",))
    assert np.any(want[3] != 0)
    assert np.array_equal(bits(c.read_radiance()[..., :3]), bits(off.read_radiance()[..., :3]))
    c.destroy(); off.destroy()


def test_option_on_without_update_changes_nothing():
    """On with no update: every output (radiance, AOVs, the resolved views, statistics) is byte-identical to a context that never
    set it.  Switched on after an update, Q is the updated positions: camera-only velocity until the next update."""
    sc = scene("CornellBox_Dragon")
    cams = [default_camera(W, H), default_camera(W, H, position=(0.05, -1.02, 1.01))]
    on = make("frame", sc, cams[1], prev_cam=cams[0])
    off = make("frame", sc, cams[1], prev_cam=cams[0], motion=False)
    for view in (0, 4, 1):
        for c in (on, off):
            c.set_option(capi.OPT_AOV, view); c.reset(); c.integrate(MB)
        assert np.array_equal(on.resolve().view(np.uint8), off.resolve().view(np.uint8)), view
        for x, y in zip(on.read_aovs(), off.read_aovs()):
            assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), view
        assert np.array_equal(on.read_radiance().view(np.uint8), off.read_radiance().view(np.uint8))
        assert on.frame_stats().tobytes() == off.frame_stats().tobytes()
    on.destroy()

    b = deform(sc["triangles"], "rigid", seed=6, amount=0.08)
    cc = deform(b, "rigid", seed=7, amount=0.08)
    off.update_triangles(b)
    off.set_option(*MOTION)
    off.reset(); off.integrate(MB)
    m = MotionModel(with_tris(sc, b))
    assert_aovs(off.read_aovs(), m.mv_aovs(b, cams[1], cams[0], W, H), ("on after update",))
    assert_aovs(off.read_aovs(), m.aovs(cams[1], cams[0], W, H), ("camera-only",))
    off.update_triangles(cc)
    off.reset(); off.integrate(MB)
    want = MotionModel(with_tris(sc, cc)).mv_aovs(b, cams[1], cams[0], W, H)
    assert_aovs(off.read_aovs(), want, ("next update",))
    off.destroy()


def soup(n, seed=21):
    from raytracing_b200 import hostapi
    from raytracing_b200.layouts import TRIANGLE_DT
    rng = np.random.default_rng(seed)
    s = np.zeros(n, dtype=TRIANGLE_DT)
    centre = rng.uniform(-1.0, 1.0, (n, 3)).astype(np.float32) * np.float32([1.0, 1.0, 0.5]) + np.float32([0.0, 0.0, 0.5])
    for v in ("v1", "v2", "v3"):
        s[v]["position"][:, :3] = centre + rng.normal(0, 0.01, (n, 3)).astype(np.float32)
        s[v]["normal"][:, :3] = (0, 0, 1)
    tris, nodes, _ = hostapi.build_bvh(s)
    return {**scene("CornellBox"), "triangles": tris, "nodes": nodes, "emissive": np.zeros(0, "<u4")}


def test_host_chunks_and_device_variant():
    """A generated soup of 220 000 triangles (35 MB: two 32 MB staging chunks of the host variant) and the device variant from a
    torch tensor: the AOVs after each of two updates equal the model, and both variants give the same bytes."""
    import torch
    sc = soup(220_000)
    assert len(sc["triangles"]) * 160 > (32 << 20)
    cam = default_camera(W, H)
    b = deform(sc["triangles"], "noise", seed=9)
    cc = deform(b, "rigid", seed=10, amount=0.1)
    out = []
    for src in ("host", "device"):
        c = make(None, sc, cam)
        got = []
        for t, q in ((b, sc["triangles"]), (cc, b)):
            c.update_triangles(t if src == "host" else torch.from_numpy(t.view(np.uint8).reshape(len(t), 160).copy()).cuda())
            c.reset(); c.integrate(MB)
            aovs = c.read_aovs()
            if src == "host":
                assert_aovs(aovs, MotionModel(with_tris(sc, t)).mv_aovs(q, cam, cam, W, H), (src,))
            got.append(aovs)
        out.append(got)
        c.destroy()
    for x, y in zip(out[0], out[1]):
        for p, q in zip(x, y):
            assert np.array_equal(p.view(np.uint8), q.view(np.uint8))


@pytest.mark.parametrize("method", ["linear", "ploc"])
def test_rebuilds_keep_q_and_reupload_resets_it(method):
    """upload A, update B, rebuild, frame: Q is still A (the model on the rebuilt nodes); update C, rebuild again, frame: Q = B.
    Re-uploading A makes Q = A again: camera-only velocity."""
    sc = scene("ShaderBalls"); cam = default_camera(W, H)
    b = deform(sc["triangles"], "rigid", seed=12, amount=0.1)
    cc = deform(b, "noise", seed=13)
    c = make("frame", sc, cam)
    for t, q in ((b, sc["triangles"]), (cc, b)):
        c.update_triangles(t)
        c.rebuild_bvh(method)
        c.reset(); c.integrate(MB)
        nodes, _ = c.read_bvh()
        want = MotionModel({**sc, "triangles": t, "nodes": nodes}).mv_aovs(q, cam, cam, W, H)
        assert_aovs(c.read_aovs(), want, (method,))
        assert np.any(want[3] != 0)
    c.upload_scene(sc)
    c.reset(); c.integrate(MB)
    want = MotionModel(sc).aovs(cam, cam, W, H)
    assert_aovs(c.read_aovs(), want, ("re-upload",))
    assert np.all(want[3][np.isfinite(want[3])] == 0)
    c.destroy()


def test_graph_replay_across_updates_and_launch_count():
    """The per-phase frame graph captured before the updates is replayed after each (the updates move no buffer): AOVs equal the
    model.  An update launches as many kernels with the option on as with it off."""
    sc = scene("CornellBox_Dragon"); cam = default_camera(W, H)
    c = make("phase_graph", sc, cam)
    c.reset(); c.integrate(MB)
    q = sc["triangles"]
    for seed in (1, 2, 3):
        t = deform(q, "rigid", seed=seed, amount=0.05)
        c.update_triangles(t)
        c.reset(); c.integrate(MB)
        assert_aovs(c.read_aovs(), MotionModel(with_tris(sc, t)).mv_aovs(q, cam, cam, W, H), ("seed %d" % seed,))
        q = t
    counts = []
    for motion in (0, 1):
        c.set_option(capi.OPT_OBJECT_MOTION, motion)
        before = c.launch_count()
        c.update_triangles(sc["triangles"])
        counts.append(c.launch_count() - before)
    assert counts[0] == counts[1] == 2
    c.destroy()


@pytest.mark.parametrize("schedule", ["frame", "phase_graph", "phase_direct"])
def test_denoiser_fed_by_object_motion_matches_model(schedule):
    """Integrator::Integrate with the denoiser on: per frame an update and a camera move, then set_camera, reset, integrate,
    denoise, copy_history, resolve.  The AOVs equal the model, the denoised radiance and the resolved image equal
    orc_temporal_accumulation fed the model's velocity."""
    name, w, h, mb = "ShaderBalls", 192, 108, 3
    sc = scene(name)
    cams = [default_camera(w, h), default_camera(w, h, position=(0.05, -1.02, 1.01)), default_camera(w, h, position=(0.08, -1.04, 1.02))]
    tris = [sc["triangles"]]
    for seed in (31, 32):
        tris.append(deform(tris[-1], "rigid", seed=seed, amount=0.06))
    c = capi.Context(w, h)
    c.upload_scene(sc)
    for k, v in SCHEDULES[schedule] + ((capi.OPT_DENOISER, 1), MOTION):
        c.set_option(k, v)
    prev_cam = np.zeros((), dtype=cams[0].dtype)
    prev_rad = np.zeros((h, w, 4), "<f4"); prev_depth = np.zeros((h, w), "<f4")
    for f, cam in enumerate(cams):
        if f:
            c.update_triangles(tris[f])
        c.set_camera(cam); c.reset(); c.integrate(mb); c.denoise(); c.copy_history()
        img = c.resolve()
        where = (schedule, "frame %d" % f)
        m = MotionModel(with_tris(sc, tris[f]))
        rad, _, ost = m.render(cam, w, h, mb, sample_idx=f)
        check_stats(c.frame_stats(), ost, mb, where)
        al, de, no, ve = m.mv_aovs(tris[max(f - 1, 0)], cam, prev_cam, w, h, sample_idx=f)
        assert_aovs(c.read_aovs(), (al, de, no, ve), where)
        den = m.temporal_accumulation(rad, prev_rad, de, prev_depth, ve)
        assert np.array_equal(bits(c.read_radiance()[..., :3]), bits(den[..., :3])), where
        assert np.array_equal(bits(img), bits(m.resolve(0, den, al, de, no, ve, f + 1, denoiser=True))), where
        prev_rad, prev_depth, prev_cam = den, de, cam
    c.destroy()


def test_multi_device_partition_and_adaptive():
    """A context listing device 0 three times and the three ranks of a 3-way partition: velocity rows equal one device's.
    Adaptive sampling: after an update, pixels that stopped before it keep the velocity of their last traced sample."""
    sc = scene("CornellBox"); cam = default_camera(W, H)
    b = deform(sc["triangles"], "rigid", seed=14, amount=0.1)
    single = make("frame", sc, cam)
    multi = make("frame", sc, cam, devices=[0, 0, 0])
    ranks = [make("frame", sc, cam, rank=r, world=3) for r in range(3)]
    vel = np.zeros((H, W, 2), "<f4")
    for c in [single, multi] + ranks:
        c.update_triangles(b); c.reset(); c.integrate(MB)
    want = single.read_aovs()
    assert_aovs(want, MotionModel(with_tris(sc, b)).mv_aovs(sc["triangles"], cam, cam, W, H), ("single",))
    assert np.array_equal(bits(multi.read_aovs()[3]), bits(want[3]))
    for r, c in enumerate(ranks):
        vel[r::3] = c.read_aovs()[3][r::3]
    assert np.array_equal(bits(vel), bits(want[3]))
    for c in [single, multi] + ranks:
        c.destroy()

    c = make("frame", sc, cam)
    c.set_adaptive_sampling(0.03, 2)
    c.reset()
    for _ in range(8):
        c.integrate(MB)
    c.update_triangles(b)
    c.integrate(MB)
    counts = c.pixel_samples().reshape(H, W); n = c.sample_count()
    active = counts == n
    assert active.any() and not active.all()
    got = c.read_aovs()
    c.destroy()
    moved = MotionModel(with_tris(sc, b)).mv_aovs(sc["triangles"], cam, cam, W, H, sample_idx=n - 1)
    for k in np.unique(counts):
        sel = counts == k
        src = moved if k == n else MotionModel(sc).mv_aovs(sc["triangles"], cam, cam, W, H, sample_idx=int(k) - 1)
        for g, x in zip(got, src):
            assert np.array_equal(bits(g[sel]), bits(x[sel])), int(k)


def test_argument_errors_and_memory():
    """Values other than 0 and 1 are RT_ERR_INVALID_ARGUMENT and change nothing; turning the option off gives its device memory back
    (48 B per triangle: 10.6 MB on a 220 000-triangle soup; the card is shared, so this is a coarse guard)."""
    import torch
    L = capi.load_library()
    sc = soup(220_000, seed=5)
    cam = default_camera(W, H)
    c = make("frame", sc, cam, motion=False)
    for v in (2, 7, 0xFFFFFFFF):
        assert L.rt_set_option(c.h, capi.OPT_OBJECT_MOTION, C.c_uint32(v)) == -1
    c.reset(); c.integrate(MB)
    assert np.all(c.read_aovs()[3] == 0)

    def free():
        torch.cuda.synchronize()
        return torch.cuda.mem_get_info()[0]

    q_bytes = len(sc["triangles"]) * 48
    start = free()
    for _ in range(4):
        c.set_option(capi.OPT_OBJECT_MOTION, 1)
        assert start - free() >= q_bytes // 2
        c.set_option(capi.OPT_OBJECT_MOTION, 0)
    assert abs(start - free()) < q_bytes // 2, (start, free())
    c.destroy()


def test_host_render_object_motion_matches_the_c_abi(tmp_path):
    """Render::SetObjectMotion through hostapi with AOV view 4: the image after each of two updates equals the C ABI's."""
    from raytracing_b200 import hostapi
    from tests.test_host import PROC_OBJ, make_env
    w, h, mb = 96, 64, 3
    env_path, _ = make_env(tmp_path, w=64, h=32)
    s = hostapi.HostScene(PROC_OBJ)
    s.add_directional_light((-0.6, -1.5, 3.5), (15, 10, 5))
    r = hostapi.HostRender(s, w, h, env_path)
    r.set_max_bounces(mb)
    a = s.arrays(); a["nodes"] = r.nodes()
    t1 = deform(a["triangles"], "rigid", seed=5, amount=0.1)
    t2 = deform(t1, "noise", seed=6)
    cam = hostapi.default_camera(w, h)
    L = capi.load_library()
    c = capi.Context(w, h)
    c.upload_scene(a)
    try:
        r.set_object_motion(True)
        assert L.rt_set_option(C.c_void_p(r.context_handle()), capi.OPT_AOV, 4) == 0
        for k, v in ((capi.OPT_AOV, 4), MOTION):
            c.set_option(k, v)
        r.render_frame()
        c.set_camera(cam); c.reset(); c.integrate(mb)
        for t in (t1, t2):
            r.update_triangles(t); r.request_reset(); r.render_frame()
            c.update_triangles(t); c.set_camera(cam); c.reset(); c.integrate(mb)
            img = c.resolve()
            assert np.array_equal(bits(r.image()), bits(img))
            assert np.any(img[..., :2] != 0)
        r.set_object_motion(False)
    finally:
        r.close(); s.close(); c.destroy()
