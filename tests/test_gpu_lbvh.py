"""
GPU tests (-m gpu) of rt_rebuild_bvh: the device-built tree against the numpy model of tests/lbvh_model.py bit for bit (nodes),
its records against rt_upload_scene's layout of the read-back nodes (build_layout) bit for bit, and every frame after a rebuild
against the oracle rendering the same triangles with the model's nodes, on every schedule of test_gpu_refit.RUNS; the
animation sequence (update, rebuild, update); repeatability and the captured frame graph; ordering against work in flight;
emitter and environment sampling; multi-device contexts, the C++ host path and the errors.
"""
import ctypes as C

import numpy as np
import pytest

from oracle.orcbind import Oracle
from raytracing_b200 import capi
from raytracing_b200.camera import default_camera
from raytracing_b200.layouts import NODE_DT
from tests import lbvh_model
from tests.helpers import bits, scene
from tests.refit_model import deform, refit
from tests.test_bvh_layout import build as layout_build
from tests.test_bvh_layout import lib  # noqa: F401  (the build_layout fixture)
from tests.test_gpu_parity import check_frame, run_frame, schedule_ctx
from tests.test_gpu_refit import RUNS, TRAVERSAL_KEYS, capi_err
from tests.test_lbvh_cpu import CASES, case

pytestmark = pytest.mark.gpu

W, H, MB = 64, 48, 4


def rebuilt(sc, t=None):
    """The scene dict with triangles t (default: sc's) and the model's tree over them."""
    t = sc["triangles"] if t is None else t
    return {**sc, "triangles": t, "nodes": lbvh_model.build(t)[0]}


def check_tree(L, c, want_nodes, tris):
    """rt_read_bvh: the nodes equal want_nodes byte for byte; the records equal build_layout of the read-back nodes bit for bit."""
    nodes, rec = c.read_bvh()
    assert np.array_equal(nodes.view(np.uint8), want_nodes.view(np.uint8))
    rc, err, wn, _, _, _, _ = layout_build(L, nodes, tris)
    assert rc == 0, err
    assert np.array_equal(bits(rec), bits(wn))
    return nodes, rec


@pytest.mark.parametrize("which", CASES)
def test_rebuilt_tree_equals_the_model(lib, which):  # noqa: F811
    """Upload with the SAH tree, rebuild: 2n - 1 nodes equal to the model's, records equal to build_layout's (breadth-first
    prefix, child references, axes, flags)."""
    sc = case(which)
    c = schedule_ctx(None, sc, default_camera(W, H), W, H)
    assert c.rebuild_bvh() == 2 * len(sc["triangles"]) - 1
    check_tree(lib, c, rebuilt(sc)["nodes"], sc["triangles"])
    c.destroy()


@pytest.mark.parametrize("name", ["CornellBox", "ShaderBalls", "CornellBox_Dragon"])
def test_frames_after_rebuild_match_oracle_on_every_schedule(name):
    """A frame on the upload (captures the graph, stages the tree), a rebuild, then a frame: radiance bits and per-bounce
    counters equal the oracle on the rebuilt tree, and so do the traversal counters of the counting kernels."""
    sc = scene(name); cam = default_camera(W, H)
    new_sc = rebuilt(sc)
    orad, _, ost = Oracle(new_sc).render(cam, W, H, MB)
    for run, (schedule, options) in RUNS.items():
        c = schedule_ctx(schedule, sc, cam, W, H, options)
        c.reset(); run_frame(c, schedule, MB)
        c.rebuild_bvh()
        c.reset(); run_frame(c, schedule, MB)
        check_frame(c, ost, orad, MB, (name, run))
        if schedule == "counted":
            st = c.frame_stats()
            for k in TRAVERSAL_KEYS:
                assert np.array_equal(st[k][: MB + 1], ost[k][: MB + 1]), (name, k)
        c.destroy()


@pytest.mark.parametrize("name", ["ShaderBalls", "CornellBox_Dragon"])
def test_animation_sequence(lib, name):  # noqa: F811
    """upload, frame, update, rebuild, frame, update, frame: after the first update the tree is the refit of the upload's, after
    the rebuild the model's, after the second update the refit of the model's topology; every frame equals the oracle."""
    sc = scene(name); cam = default_camera(W, H)
    t1 = deform(sc["triangles"], "noise", seed=3, amount=0.3)
    t2 = deform(t1, "rigid", seed=4)
    c = schedule_ctx("phase_graph", sc, cam, W, H)
    steps = [("frame", sc), ("update", t1, refit(sc["nodes"], t1)), ("rebuild",)]
    lb1 = rebuilt(sc, t1)
    steps += [("frame", lb1), ("update", t2, refit(lb1["nodes"], t2)), ("frame", {**sc, "triangles": t2, "nodes": refit(lb1["nodes"], t2)})]
    tris = sc["triangles"]
    for st in steps:
        if st[0] == "frame":
            orad, _, ost = Oracle(st[1]).render(cam, W, H, MB)
            c.reset(); c.integrate(MB)
            check_frame(c, ost, orad, MB, (name, len(steps)))
        elif st[0] == "update":
            tris = st[1]
            c.update_triangles(tris)
            check_tree(lib, c, st[2], tris)
        else:
            c.rebuild_bvh()
            check_tree(lib, c, lb1["nodes"], tris)
    c.destroy()


def test_rebuilds_repeat_and_keep_the_captured_graph():
    """Two rebuilds give identical bytes.  Under RT_OPT_GRAPH 1, a frame replayed from the graph captured after the first rebuild
    (no re-capture: the second rebuild reuses every buffer) equals the oracle on the second rebuild's tree."""
    sc = scene("ShaderBalls"); cam = default_camera(W, H)
    t = deform(sc["triangles"], "noise", seed=8, amount=0.3)
    c = schedule_ctx("phase_graph", sc, cam, W, H, ((capi.OPT_GRAPH, 1),))
    c.rebuild_bvh()
    a = c.read_bvh()
    c.rebuild_bvh()
    b = c.read_bvh()
    assert np.array_equal(a[0].view(np.uint8), b[0].view(np.uint8)) and np.array_equal(bits(a[1]), bits(b[1]))
    c.reset(); c.integrate(MB)                                   # captures the graph on the rebuilt buffers
    c.update_triangles(t)
    c.rebuild_bvh()
    new_sc = rebuilt(sc, t)
    assert np.array_equal(c.read_bvh()[0].view(np.uint8), new_sc["nodes"].view(np.uint8))
    orad, _, ost = Oracle(new_sc).render(cam, W, H, MB)
    c.reset(); c.integrate(MB)
    check_frame(c, ost, orad, MB, ("graph",))
    c.destroy()


@pytest.mark.parametrize("overlap", [0, 1, 2])
@pytest.mark.parametrize("how", ["phase_graph", "fused_steps"])
def test_rebuild_is_ordered_after_work_in_flight(how, overlap):
    """reset; a frame on A; update(B); rebuild; a frame; no synchronisation in between.  The radiance is the oracle's frame on A at
    sample 0 plus its frame on (B, the model's tree) at sample 1.  fused_steps leaves the last shadow pass of the frame on A
    deferred (RT_OPT_OVERLAP 2) or on the second stream (1) when the update and the rebuild arrive."""
    sc = scene("CornellBox"); cam = default_camera(W, H)
    t = deform(sc["triangles"], "rigid", seed=11)
    new_sc = rebuilt(sc, t)
    acc, _, _ = Oracle(sc).render(cam, W, H, MB, sample_idx=0)
    acc, _, ost = Oracle(new_sc).render(cam, W, H, MB, sample_idx=1, radiance=acc)
    c = schedule_ctx(None, sc, cam, W, H, ((capi.OPT_FRAME_KERNEL, 0), (capi.OPT_OVERLAP, overlap)))
    c.reset()
    if how == "fused_steps":
        c.generate_rays()
        for b in range(MB + 1):
            c.extend_shade(b); c.shadow_accumulate(b)
        c.update_triangles(t); c.rebuild_bvh()
        c.advance_sample_count()
    else:
        c.integrate(MB)
        c.update_triangles(t); c.rebuild_bvh()
    c.integrate(MB)
    check_frame(c, ost, acc, MB, (how, overlap))
    c.destroy()


@pytest.mark.parametrize("order", ["on_then_rebuild", "rebuild_then_on"])
def test_light_sampling_after_rebuild(order):
    """Emitter and environment sampling on: the frame after a rebuild equals the light model on the rebuilt tree, whose tables
    are built from the same triangles (the rebuild leaves them unchanged)."""
    from tests.light_model import LightModel
    sc = scene("CornellBox"); cam = default_camera(W, H)
    new_sc = rebuilt(sc)
    orad, _, ost = LightModel(new_sc).render(cam, W, H, MB, emitters=True, env=True)
    c = schedule_ctx(None, sc, cam, W, H)
    opts = ((capi.OPT_EMITTER_SAMPLING, 1), (capi.OPT_ENV_SAMPLING, 1))
    if order == "on_then_rebuild":
        for k, v in opts:
            c.set_option(k, v)
        c.reset(); c.integrate(MB)
        c.rebuild_bvh()
    else:
        c.rebuild_bvh()
        for k, v in opts:
            c.set_option(k, v)
    c.reset(); c.integrate(MB)
    check_frame(c, ost, orad, MB, (order,))
    c.destroy()


def test_multi_device_host_path_errors_and_launch_counts(tmp_path):
    """Device 0 listed three times renders what one device renders after a rebuild; Render::RebuildBvh through hostapi gives the
    C ABI's image; RT_ERR_NOT_READY before an upload; the launches count under RT_K_MISC."""
    sc = scene("ShaderBalls"); cam = default_camera(W, H)
    t = deform(sc["triangles"], "noise", seed=2, amount=0.3)
    one = schedule_ctx(None, sc, cam, W, H)
    one.update_triangles(t); assert one.rebuild_bvh() == 2 * len(t) - 1
    one.reset(); one.integrate(MB)
    want = one.read_radiance()
    one.destroy()
    m = capi.Context(W, H, devices=[0, 0, 0])
    m.upload_scene(sc); m.set_camera(cam)
    m.update_triangles(t); assert m.rebuild_bvh() == 2 * len(t) - 1
    m.reset(); m.integrate(MB)
    assert np.array_equal(bits(m.read_radiance()), bits(want))
    m.destroy()

    L = capi.load_library()
    fresh = capi.Context(W, H)
    n = C.c_uint64(7)
    assert L.rt_rebuild_bvh(fresh.h, C.byref(n)) == capi_err("NOT_READY") and n.value == 7
    fresh.destroy()

    for name, want_launches in (("CornellBox", 8), ("one", 2)):
        s = scene("CornellBox")
        if name == "one":
            s = {**s, "triangles": s["triangles"][:1], "emissive": np.zeros(0, "<u4")}
            leaf = np.zeros(1, dtype=NODE_DT); leaf["num_primitives_axis"] = 1 << 16
            s["nodes"] = refit(leaf, s["triangles"])
        c = schedule_ctx(None, s, cam, W, H, ((capi.OPT_KERNEL_TIMING, 1),))
        c.kernel_times()
        before = c.launch_count()
        assert L.rt_rebuild_bvh(c.h, None) == 0
        assert c.launch_count() - before == want_launches        # bounds, keys, sort, Karras, numbering, top, writes, refit
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
        r.update_triangles(t); assert r.rebuild_bvh() == 2 * len(t) - 1
        r.request_reset(); r.render_frame()
        c.update_triangles(t); c.rebuild_bvh(); c.reset(); c.integrate(mb)
        assert np.array_equal(bits(r.image()), bits(c.resolve()))
    finally:
        r.close(); s.close(); c.destroy()


@pytest.mark.slow
def test_synthetic_10m_rebuild_matches_model_and_oracle():
    """Synthetic10M at full size: a rebuild after a rigid move of a third of the triangles gives rt_read_bvh nodes equal to the
    model byte for byte, and a band of rows equals the oracle on the rebuilt tree."""
    from raytracing_b200 import scene_io, synthetic
    w, h, mb = 1920, 1080, 8
    sc = synthetic.bistro_scale_scene(scene_io.load_scene("ShaderBalls"), 183, w, h)
    cam = sc["camera_pose"]
    t = deform(sc["triangles"], "rigid", seed=2)
    new_sc = rebuilt(sc, t)
    c = capi.Context(w, h)
    c.upload_scene(sc); c.set_camera(cam)
    c.update_triangles(t)
    assert c.rebuild_bvh() == 2 * len(t) - 1
    nodes, _ = c.read_bvh()
    assert np.array_equal(nodes.view(np.uint8), new_sc["nodes"].view(np.uint8))
    c.reset(); c.integrate(mb)
    img = c.read_radiance(); c.destroy()
    orad, _, _ = Oracle(new_sc).render(cam, w, h, mb, row_first=7, row_step=70)
    rows = np.arange(7, h, 70)
    assert np.array_equal(bits(img[rows][..., :3]), bits(orad[rows][..., :3]))
