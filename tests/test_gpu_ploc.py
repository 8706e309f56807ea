"""
GPU tests (-m gpu) of rt_rebuild_bvh_ploc: the device-built tree against the numpy model of tests/ploc_model.py bit for bit
(nodes), its records against rt_upload_scene's layout of the read-back nodes (build_layout) bit for bit, and every frame after a
rebuild against the oracle rendering the same triangles with the model's nodes, on every schedule of test_gpu_refit.RUNS; the
shared-memory staging and the octant records; an animation that alternates the two builds; the depth guard; ordering against
work in flight; emitter and environment sampling; multi-device contexts, the C++ host path, the errors and the launch counts.
"""
import ctypes as C

import numpy as np
import pytest

from oracle.orcbind import Oracle
from raytracing_b200 import capi
from raytracing_b200.camera import default_camera
from raytracing_b200.layouts import NODE_DT
from tests import lbvh_model, ploc_model
from tests.helpers import bits, scene
from tests.refit_model import deform, refit
from tests.test_bvh_layout import lib  # noqa: F401  (the build_layout fixture)
from tests.test_gpu_lbvh import check_tree
from tests.test_gpu_parity import check_frame, run_frame, schedule_ctx
from tests.test_gpu_refit import RUNS, TRAVERSAL_KEYS, capi_err
from tests.test_ploc_cpu import CASES, case, geometric_chain, soup_case

pytestmark = pytest.mark.gpu

W, H, MB = 64, 48, 4


def clustered(sc, t=None):
    """The scene dict with triangles t (default: sc's) and the PLOC model's tree over them."""
    t = sc["triangles"] if t is None else t
    return {**sc, "triangles": t, "nodes": ploc_model.build(t)[0]}


@pytest.mark.parametrize("which", CASES)
def test_ploc_tree_equals_the_model(lib, which):  # noqa: F811
    """Upload with the SAH tree, PLOC rebuild: 2n - 1 nodes equal to the model's, records equal to build_layout's."""
    sc = case(which)
    c = schedule_ctx(None, sc, default_camera(W, H), W, H)
    assert c.rebuild_bvh("ploc") == 2 * len(sc["triangles"]) - 1
    check_tree(lib, c, clustered(sc)["nodes"], sc["triangles"])
    c.destroy()


@pytest.mark.parametrize("name", ["CornellBox", "ShaderBalls", "CornellBox_Dragon"])
def test_frames_after_ploc_match_oracle_on_every_schedule(name):
    """A frame on the upload, a PLOC rebuild, then a frame: radiance bits and per-bounce counters equal the oracle on the model's
    tree, and so do the traversal counters of the counting kernels."""
    sc = scene(name); cam = default_camera(W, H)
    new_sc = clustered(sc)
    orad, _, ost = Oracle(new_sc).render(cam, W, H, MB)
    for run, (schedule, options) in RUNS.items():
        c = schedule_ctx(schedule, sc, cam, W, H, options)
        c.reset(); run_frame(c, schedule, MB)
        c.rebuild_bvh("ploc")
        c.reset(); run_frame(c, schedule, MB)
        check_frame(c, ost, orad, MB, (name, run))
        if schedule == "counted":
            st = c.frame_stats()
            for k in TRAVERSAL_KEYS:
                assert np.array_equal(st[k][: MB + 1], ost[k][: MB + 1]), (name, k)
        c.destroy()


def test_staging_and_octant_records_after_ploc():
    """CornellBox: both rebuilt trees have 63 nodes, so the staging mode after a PLOC rebuild is the one after rt_rebuild_bvh;
    RT_OPT_OCTANT_BVH on equals off after a PLOC rebuild."""
    from tests.test_gpu_octant_bvh import assert_on_equals_off
    sc = scene("CornellBox"); cam = default_camera(W, H)
    modes = []
    for method in ("linear", "ploc"):
        c = schedule_ctx(None, sc, cam, W, H)
        c.rebuild_bvh(method)
        modes.append(c.bvh_staging())
        c.destroy()
    assert modes[0] == modes[1]
    t = deform(sc["triangles"], "noise", seed=3, amount=0.3)

    def prepare(c):
        c.update_triangles(t)
        c.rebuild_bvh("ploc")
    assert_on_equals_off(sc, cam, W, H, MB, "ploc", runs=("frame", "phase_graph", "stepwise"), prepare=prepare)


@pytest.mark.parametrize("name", ["ShaderBalls", "CornellBox_Dragon"])
def test_animation_alternating_builds(lib, name):  # noqa: F811
    """upload, PLOC, frame, update, frame, LBVH rebuild, frame, PLOC, frame under RT_OPT_GRAPH 1: each tree is the model's (the
    update's the refit of the PLOC topology), every frame equals the oracle on it."""
    sc = scene(name); cam = default_camera(W, H)
    t1 = deform(sc["triangles"], "noise", seed=3, amount=0.3)
    t2 = deform(t1, "rigid", seed=4)
    c = schedule_ctx("phase_graph", sc, cam, W, H, ((capi.OPT_GRAPH, 1),))
    p0 = clustered(sc)
    upd = {**sc, "triangles": t1, "nodes": refit(p0["nodes"], t1)}
    lin = {**sc, "triangles": t2, "nodes": lbvh_model.build(t2)[0]}
    steps = [("ploc", p0), ("update", upd), ("update2", None), ("linear", lin), ("ploc", clustered(sc, t2))]
    for what, want in steps:
        if what == "update2":
            c.update_triangles(t2)
            continue
        if what == "update":
            c.update_triangles(want["triangles"])
        else:
            c.rebuild_bvh(what)
        check_tree(lib, c, want["nodes"], want["triangles"])
        orad, _, ost = Oracle(want).render(cam, W, H, MB)
        c.reset(); c.integrate(MB)
        check_frame(c, ost, orad, MB, (name, what))
    c.destroy()


def test_ploc_rebuilds_repeat_and_keep_the_captured_graph():
    """Two PLOC rebuilds give identical bytes; a frame replayed from the graph captured after the first equals the oracle on the
    tree of a later PLOC rebuild of moved triangles."""
    sc = scene("ShaderBalls"); cam = default_camera(W, H)
    t = deform(sc["triangles"], "noise", seed=8, amount=0.3)
    c = schedule_ctx("phase_graph", sc, cam, W, H, ((capi.OPT_GRAPH, 1),))
    c.rebuild_bvh("ploc")
    a = c.read_bvh()
    c.rebuild_bvh("ploc")
    b = c.read_bvh()
    assert np.array_equal(a[0].view(np.uint8), b[0].view(np.uint8)) and np.array_equal(bits(a[1]), bits(b[1]))
    c.reset(); c.integrate(MB)
    c.update_triangles(t)
    c.rebuild_bvh("ploc")
    new_sc = clustered(sc, t)
    assert np.array_equal(c.read_bvh()[0].view(np.uint8), new_sc["nodes"].view(np.uint8))
    orad, _, ost = Oracle(new_sc).render(cam, W, H, MB)
    c.reset(); c.integrate(MB)
    check_frame(c, ost, orad, MB, ("graph",))
    c.destroy()


@pytest.mark.parametrize("before", ["upload", "linear"])
def test_too_deep_a_tree_changes_nothing(before):
    """The 1.5^k chain: RT_ERR_UNSUPPORTED whose text names rt_rebuild_bvh; the tree read back is unchanged, and the frame after
    the call has the bits of the frame before it (the first call after an upload, and a call on a rebuilt tree)."""
    sc = soup_case("geometric_chain", geometric_chain)
    assert ploc_model.build(sc["triangles"], with_boxes=False)[1]["depth_error"]
    cam = default_camera(W, H)
    c = schedule_ctx("phase_graph", sc, cam, W, H, ((capi.OPT_GRAPH, 1),))
    if before == "linear":
        c.rebuild_bvh("linear")
    c.reset(); c.integrate(MB)
    want = c.read_radiance()
    nodes, rec = c.read_bvh()
    n = C.c_uint64(7)
    assert c.lib.rt_rebuild_bvh_ploc(c.h, C.byref(n)) == capi_err("UNSUPPORTED") and n.value == 7
    assert b"rt_rebuild_bvh " in c.lib.rt_last_error(c.h)
    nodes2, rec2 = c.read_bvh()
    assert np.array_equal(nodes.view(np.uint8), nodes2.view(np.uint8)) and np.array_equal(bits(rec), bits(rec2))
    c.reset(); c.integrate(MB)
    assert np.array_equal(bits(c.read_radiance()), bits(want))
    c.destroy()


@pytest.mark.parametrize("overlap", [0, 1, 2])
@pytest.mark.parametrize("how", ["phase_graph", "fused_steps"])
def test_ploc_is_ordered_after_work_in_flight(how, overlap):
    """reset; a frame on A; update(B); PLOC rebuild; a frame; no synchronisation in between: the oracle's frame on A at sample 0
    plus its frame on (B, the model's tree) at sample 1."""
    sc = scene("CornellBox"); cam = default_camera(W, H)
    t = deform(sc["triangles"], "rigid", seed=11)
    new_sc = clustered(sc, t)
    acc, _, _ = Oracle(sc).render(cam, W, H, MB, sample_idx=0)
    acc, _, ost = Oracle(new_sc).render(cam, W, H, MB, sample_idx=1, radiance=acc)
    c = schedule_ctx(None, sc, cam, W, H, ((capi.OPT_FRAME_KERNEL, 0), (capi.OPT_OVERLAP, overlap)))
    c.reset()
    if how == "fused_steps":
        c.generate_rays()
        for b in range(MB + 1):
            c.extend_shade(b); c.shadow_accumulate(b)
        c.update_triangles(t); c.rebuild_bvh("ploc")
        c.advance_sample_count()
    else:
        c.integrate(MB)
        c.update_triangles(t); c.rebuild_bvh("ploc")
    c.integrate(MB)
    check_frame(c, ost, acc, MB, (how, overlap))
    c.destroy()


def test_light_sampling_after_ploc():
    """Emitter and environment sampling on: the frame after a PLOC rebuild equals the light model on the model's tree."""
    from tests.light_model import LightModel
    sc = scene("CornellBox"); cam = default_camera(W, H)
    new_sc = clustered(sc)
    orad, _, ost = LightModel(new_sc).render(cam, W, H, MB, emitters=True, env=True)
    c = schedule_ctx(None, sc, cam, W, H)
    for k, v in ((capi.OPT_EMITTER_SAMPLING, 1), (capi.OPT_ENV_SAMPLING, 1)):
        c.set_option(k, v)
    c.reset(); c.integrate(MB)
    c.rebuild_bvh("ploc")
    c.reset(); c.integrate(MB)
    check_frame(c, ost, orad, MB, ("lights",))
    c.destroy()


def test_multi_device_host_path_errors_and_launch_counts(tmp_path):
    """Device 0 listed three times renders what one device renders after a PLOC rebuild; Render::RebuildBvh(BvhBuild::kPloc)
    through hostapi gives the C ABI's image; RT_ERR_NOT_READY before an upload; the launches count under RT_K_MISC."""
    sc = scene("ShaderBalls"); cam = default_camera(W, H)
    t = deform(sc["triangles"], "noise", seed=2, amount=0.3)
    one = schedule_ctx(None, sc, cam, W, H)
    one.update_triangles(t); assert one.rebuild_bvh("ploc") == 2 * len(t) - 1
    one.reset(); one.integrate(MB)
    want = one.read_radiance()
    one.destroy()
    m = capi.Context(W, H, devices=[0, 0, 0])
    m.upload_scene(sc); m.set_camera(cam)
    m.update_triangles(t); assert m.rebuild_bvh("ploc") == 2 * len(t) - 1
    m.reset(); m.integrate(MB)
    assert np.array_equal(bits(m.read_radiance()), bits(want))
    m.destroy()

    L = capi.load_library()
    fresh = capi.Context(W, H)
    n = C.c_uint64(7)
    assert L.rt_rebuild_bvh_ploc(fresh.h, C.byref(n)) == capi_err("NOT_READY") and n.value == 7
    with pytest.raises(ValueError):
        fresh.rebuild_bvh("sah")
    fresh.destroy()

    for name in ("CornellBox", "one"):
        s = scene("CornellBox")
        want_launches = 9 + 3 * ploc_model.build(s["triangles"], with_boxes=False)[1]["iterations"]
        if name == "one":
            s = {**s, "triangles": s["triangles"][:1], "emissive": np.zeros(0, "<u4")}
            leaf = np.zeros(1, dtype=NODE_DT); leaf["num_primitives_axis"] = 1 << 16
            s["nodes"] = refit(leaf, s["triangles"])
            want_launches = 2
        c = schedule_ctx(None, s, cam, W, H, ((capi.OPT_KERNEL_TIMING, 1),))
        c.kernel_times()
        before = c.launch_count()
        assert L.rt_rebuild_bvh_ploc(c.h, None) == 0
        assert c.launch_count() - before == want_launches       # bounds, keys, sort, init, 3 per iteration, number, flags, top, writes, refit
        assert c.kernel_times()["misc"][1] == want_launches
        c.destroy()

    from raytracing_b200 import hostapi
    from tests.test_host import PROC_OBJ, make_env
    w, h, mb = 96, 64, 4
    env_path, _ = make_env(tmp_path, w=64, h=32)
    s = hostapi.HostScene(PROC_OBJ)
    s.add_directional_light((-0.6, -1.5, 3.5), (15, 10, 5))
    r = hostapi.HostRender(s, w, h, env_path)
    r.set_max_bounces(mb)
    a = s.arrays(); a["nodes"] = r.nodes()
    t = deform(a["triangles"], "noise", seed=5, amount=0.3)
    cam = hostapi.default_camera(w, h)
    c = capi.Context(w, h)
    c.upload_scene(a); c.set_camera(cam)
    try:
        r.render_frame()
        r.update_triangles(t); assert r.rebuild_bvh("ploc") == 2 * len(t) - 1
        r.request_reset(); r.render_frame()
        c.update_triangles(t); c.rebuild_bvh("ploc"); c.reset(); c.integrate(mb)
        assert np.array_equal(bits(r.image()), bits(c.resolve()))
    finally:
        r.close(); s.close(); c.destroy()


@pytest.mark.slow
def test_synthetic_10m_ploc_matches_model_and_oracle():
    """Synthetic10M at full size: a PLOC rebuild after a rigid move of a third of the triangles gives rt_read_bvh nodes equal to
    the model byte for byte, and a band of rows equals the oracle on that tree."""
    from raytracing_b200 import scene_io, synthetic
    w, h, mb = 1920, 1080, 8
    sc = synthetic.bistro_scale_scene(scene_io.load_scene("ShaderBalls"), 183, w, h)
    cam = sc["camera_pose"]
    t = deform(sc["triangles"], "rigid", seed=2)
    new_sc = clustered(sc, t)
    c = capi.Context(w, h)
    c.upload_scene(sc); c.set_camera(cam)
    c.update_triangles(t)
    assert c.rebuild_bvh("ploc") == 2 * len(t) - 1
    nodes, _ = c.read_bvh()
    assert np.array_equal(nodes.view(np.uint8), new_sc["nodes"].view(np.uint8))
    c.reset(); c.integrate(mb)
    img = c.read_radiance(); c.destroy()
    orad, _, _ = Oracle(new_sc).render(cam, w, h, mb, row_first=7, row_step=70)
    rows = np.arange(7, h, 70)
    assert np.array_equal(bits(img[rows][..., :3]), bits(orad[rows][..., :3]))
