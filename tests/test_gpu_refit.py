"""
GPU tests (-m gpu) of geometry updates (rt_update_triangles, rt_update_triangles_device, rt_read_bvh): the refit boxes against
the numpy model of tests/refit_model.py bit for bit, and every frame after an update against the oracle rendering the updated
arrays with the model's nodes, on every schedule; the same state as a fresh upload; ordering against work in flight; the emitter
table after an update; the device variant, its errors and multi-device contexts; the C++ host path.
"""
import ctypes as C

import numpy as np
import pytest

from oracle.orcbind import Oracle
from raytracing_b200 import capi
from raytracing_b200.camera import default_camera
from tests.helpers import bits, scene
from tests.refit_model import deform, records_match_nodes, refit
from tests.test_gpu_parity import SCHEDULES, check_frame, check_stats, run_frame, schedule_ctx

pytestmark = pytest.mark.gpu

W, H, MB = 64, 48, 4
SCENES = ["CornellBox", "ShaderBalls", "CornellBox_Dragon"]
KINDS = ["noise", "rigid", "scale"]
# every way a frame can run: (schedule of test_gpu_parity.SCHEDULES or "stepwise", extra options)
RUNS = {
    "frame": ("frame", ()),
    "phase_graph": ("phase_graph", ()),
    "phase_direct": ("phase_direct", ()),
    "phase_no_pdl": ("phase_graph", ((capi.OPT_PDL, 0),)),
    "stepwise": ("stepwise", ()),
    "literal": ("frame", ((capi.OPT_TRAVERSAL, 0),)),
    "counted": ("counted", ()),
    "no_smem": ("frame", ((capi.OPT_SMEM_BVH, 0),)),
    "top_smem": ("phase_graph", ((capi.OPT_TOP_SMEM, 100),)),      # on scenes that do not fit shared memory
}
TRAVERSAL_KEYS = ("nodes_ext", "tris_ext", "nodes_shadow", "tris_shadow")


def moved(sc, kind, seed=7):
    """(updated scene dict for the oracle / a fresh upload, the new triangles)."""
    t = deform(sc["triangles"], kind, seed=seed)
    return {**sc, "triangles": t, "nodes": refit(sc["nodes"], t)}, t


def assert_nodes_equal(got, want, exact):
    for f in ("offset", "num_primitives_axis", "padding"):
        assert np.array_equal(got[f], want[f]), f
    for f in ("bounds_min", "bounds_max"):
        assert np.array_equal(got[f][:, 3].view("<u4"), want[f][:, 3].view("<u4")), f
        if exact:
            assert np.array_equal(bits(got[f][:, :3]), bits(want[f][:, :3])), f
        else:
            assert (got[f][:, :3] == want[f][:, :3]).all(), f


def records_equal(a, b):
    return (a[:, :12] == b[:, :12]).all() and np.array_equal(a[:, 12:].view("<u4"), b[:, 12:].view("<u4"))


def primary_hits(c):
    c.generate_rays(); c.intersect(0)
    hits, pix = c.read_hits(0)
    prim = np.full(W * H, 0xFFFFFFFE, np.uint32); prim[pix] = hits["primitive_id"]
    return prim


@pytest.mark.parametrize("name", SCENES)
def test_identity_update_keeps_bvh_and_frames(name):
    """An update with the uploaded array: nodes and records value-equal to the upload's, frames bit-identical (radiance,
    per-bounce counters, primary hits)."""
    sc = scene(name); cam = default_camera(W, H)
    c = schedule_ctx(None, sc, cam, W, H)
    n0, r0 = c.read_bvh()
    assert_nodes_equal(n0, sc["nodes"], exact=True)
    frames = []
    for update in (False, True):
        if update:
            c.update_triangles(sc["triangles"])
            n1, r1 = c.read_bvh()
            assert_nodes_equal(n1, n0, exact=False)
            assert records_equal(r1, r0)
        c.reset(); c.integrate(MB)
        frames.append((c.read_radiance(), c.frame_stats(), primary_hits(c)))
    (ra, sa, ha), (rb, sb, hb) = frames
    assert np.array_equal(bits(ra), bits(rb)) and np.array_equal(ha, hb)
    check_stats(sb, sa, MB)
    c.destroy()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("name", ["CornellBox", "ShaderBalls"])
def test_deformed_frames_match_oracle_on_every_schedule(name, kind):
    """A frame on the upload (captures the graph, stages the tree), an update, then a frame: rt_read_bvh equals the numpy model
    bit for bit and every record holds its children's boxes; the frame equals the oracle on the updated arrays."""
    sc = scene(name); cam = default_camera(W, H)
    new_sc, t = moved(sc, kind)
    orad, _, ost = Oracle(new_sc).render(cam, W, H, MB)
    for run, (schedule, options) in RUNS.items():
        if run == "top_smem" and name == "CornellBox":
            continue                                             # staged whole
        c = schedule_ctx(schedule, sc, cam, W, H, options)
        c.reset(); run_frame(c, schedule, MB)
        c.update_triangles(t)
        nodes, rec = c.read_bvh()
        assert_nodes_equal(nodes, new_sc["nodes"], exact=True)
        assert records_match_nodes(nodes, rec) == rec.shape[0]
        c.reset(); run_frame(c, schedule, MB)
        check_frame(c, ost, orad, MB, (name, kind, run))
        c.destroy()


def test_update_equals_fresh_upload():
    """upload(A) + update(B) against upload(B with the model's nodes): radiance, AOVs and the spatial-denoised resolve are
    bit-identical; A -> B -> A gives back A's frame and traversal counters."""
    sc = scene("ShaderBalls"); cam = default_camera(W, H)
    new_sc, t = moved(sc, "rigid")
    a = schedule_ctx(None, sc, cam, W, H); a.update_triangles(t)
    b = schedule_ctx(None, new_sc, cam, W, H)
    out = []
    for c in (a, b):
        c.set_spatial_denoiser(2, 0.5, 0.2, 0.1)
        c.reset(); c.integrate(MB); c.integrate(MB)
        out.append((c.read_radiance(), c.read_aovs(), c.resolve()))
    for x, y in zip(out[0][1], out[1][1]):
        assert np.array_equal(bits(x), bits(y))
    assert np.array_equal(bits(out[0][0]), bits(out[1][0])) and np.array_equal(bits(out[0][2]), bits(out[1][2]))
    b.destroy(); a.destroy()

    c = schedule_ctx(None, sc, cam, W, H, ((capi.OPT_COUNT_TRAVERSAL, 1),))
    res = []
    for step in ("A", "B", "A"):
        if step == "B":
            c.update_triangles(t)
            continue
        if res:
            c.update_triangles(sc["triangles"])
        c.reset(); c.integrate(MB)
        res.append((c.read_radiance(), c.frame_stats()))
    assert np.array_equal(bits(res[0][0]), bits(res[1][0]))
    for k in TRAVERSAL_KEYS:
        assert np.array_equal(res[0][1][k][: MB + 1], res[1][1][k][: MB + 1]), k
    check_stats(res[1][1], res[0][1], MB)
    c.destroy()


@pytest.mark.parametrize("overlap", [2, 1])
@pytest.mark.parametrize("how", ["frame_kernel", "phase_graph", "fused_steps"])
def test_update_is_ordered_after_work_in_flight(how, overlap):
    """reset; a frame on A; update(B); a frame; no synchronisation in between.  The radiance is the oracle's frame on A at sample 0
    plus its frame on B at sample 1.  fused_steps leaves the last shadow pass of the frame on A deferred (RT_OPT_OVERLAP 2) or
    on the second stream (1) when the update arrives; the per-phase graph chains its kernels with PDL, whose traversal kernels
    stage the tree before waiting."""
    sc = scene("CornellBox"); cam = default_camera(W, H)
    new_sc, t = moved(sc, "rigid", seed=11)
    acc, _, _ = Oracle(sc).render(cam, W, H, MB, sample_idx=0)
    acc, _, ost = Oracle(new_sc).render(cam, W, H, MB, sample_idx=1, radiance=acc)
    fk = 1 if how == "frame_kernel" else 0
    c = schedule_ctx(None, sc, cam, W, H, ((capi.OPT_FRAME_KERNEL, fk), (capi.OPT_OVERLAP, overlap)))
    c.reset()
    if how == "fused_steps":
        c.generate_rays()
        for b in range(MB + 1):
            c.extend_shade(b); c.shadow_accumulate(b)
        c.update_triangles(t)
        c.advance_sample_count()
    else:
        c.integrate(MB)
        c.update_triangles(t)
    c.integrate(MB)
    check_frame(c, ost, acc, MB, (how, overlap))
    c.destroy()


def light_moved(sc, seed=3):
    """CornellBox with its light moved down and stretched (the emissive triangles only)."""
    t = sc["triangles"].copy()
    em = np.asarray(sc["emissive"], dtype=np.int64)
    pos = np.stack([t[v]["position"][em, :3] for v in ("v1", "v2", "v3")], axis=1)
    c = pos.reshape(-1, 3).mean(0)
    pos = (c + (pos - c) * np.array([1.6, 1.3, 1.0])).astype(np.float32)
    pos[..., 2] -= np.float32(0.05)
    for i, v in enumerate(("v1", "v2", "v3")):
        t[v]["position"][em, :3] = pos[:, i]
    return {**sc, "triangles": t, "nodes": refit(sc["nodes"], t)}, t


@pytest.mark.parametrize("order", ["on_then_update", "update_then_on"])
def test_emitter_table_follows_the_update(order):
    """Emitter and environment sampling on: after an update that moves and stretches the light, the frame equals the light model
    on the updated arrays (the emitter areas come from the new positions), whether the options were on before the update or
    turned on after it."""
    from tests.light_model import LightModel
    sc = scene("CornellBox"); cam = default_camera(W, H)
    assert len(sc["emissive"]) > 0
    new_sc, t = light_moved(sc)
    orad, _, ost = LightModel(new_sc).render(cam, W, H, MB, emitters=True, env=True)
    c = schedule_ctx(None, sc, cam, W, H)
    opts = ((capi.OPT_EMITTER_SAMPLING, 1), (capi.OPT_ENV_SAMPLING, 1))
    if order == "on_then_update":
        for k, v in opts:
            c.set_option(k, v)
        c.reset(); c.integrate(MB)
        c.update_triangles(t)
    else:
        c.update_triangles(t)
        for k, v in opts:
            c.set_option(k, v)
    c.reset(); c.integrate(MB)
    check_frame(c, ost, orad, MB, (order,))
    c.destroy()


def test_device_variant_and_errors():
    """A CUDA torch tensor (uint8 (n, 160) and float32 (n, 40)) gives the host variant's nodes, records and frames.  Errors: a
    wrong count, a host pointer, the device variant on a multi-device context, an update before an upload.  A host-variant
    update of a multi-device context renders what one device renders."""
    import torch
    sc = scene("ShaderBalls"); cam = default_camera(W, H)
    _, t = moved(sc, "noise")
    L = capi.load_library()
    want = None
    for src in ("host", "u8", "f32"):
        c = schedule_ctx(None, sc, cam, W, H)
        if src == "host":
            c.update_triangles(t)
        else:
            d = torch.from_numpy(t.view(np.uint8).reshape(len(t), 160).copy()).cuda()
            c.update_triangles(d if src == "u8" else d.view(torch.float32))
        c.reset(); c.integrate(MB)
        got = c.read_bvh() + (c.read_radiance(),)
        if want is None:
            want = got
        else:
            assert np.array_equal(got[0].view(np.uint8), want[0].view(np.uint8)) and np.array_equal(bits(got[1]), bits(want[1]))
            assert np.array_equal(bits(got[2]), bits(want[2])), src
        if src == "u8":
            assert L.rt_update_triangles_device(c.h, C.c_void_p(d.data_ptr()), len(t) - 1) == capi_err("INVALID")
            assert L.rt_update_triangles(c.h, t.ctypes.data, len(t) + 1) == capi_err("INVALID")
            assert L.rt_update_triangles_device(c.h, C.c_void_p(t.ctypes.data), len(t)) == capi_err("INVALID")
            assert L.rt_update_triangles(c.h, None, len(t)) == capi_err("INVALID")
        c.destroy()

    fresh = capi.Context(W, H)
    d = torch.zeros((len(t), 160), dtype=torch.uint8, device="cuda")
    assert L.rt_update_triangles(fresh.h, t.ctypes.data, len(t)) == capi_err("NOT_READY")
    assert L.rt_update_triangles_device(fresh.h, C.c_void_p(d.data_ptr()), len(t)) == capi_err("NOT_READY")
    n = C.c_uint64()
    assert L.rt_read_bvh(fresh.h, None, None, C.byref(n)) == capi_err("NOT_READY")
    fresh.destroy()

    m = capi.Context(W, H, devices=[0, 0])
    m.upload_scene(sc); m.set_camera(cam)
    assert L.rt_update_triangles_device(m.h, C.c_void_p(d.data_ptr()), len(t)) == capi_err("UNSUPPORTED")
    m.update_triangles(t)
    m.reset(); m.integrate(MB)
    assert np.array_equal(bits(m.read_radiance()), bits(want[2]))
    m.destroy()


def test_dropped_tensor_is_not_reused_before_the_update_reads_it():
    """Fresh geometry tensors, each dropped right after update_triangles while a frame is still queued on the render stream, and
    torch allocations of the same size filled with 0xFF at once: the update reads the geometry it was given (Context.update_triangles
    records the tensor on the render stream, so the allocator keeps its block until the update has run)."""
    import torch
    sc = scene("ShaderBalls"); cam = default_camera(W, H)
    c = schedule_ctx(None, sc, cam, W, H)
    c.reset()
    for seed in (1, 2, 3):
        new_sc, t = moved(sc, "noise", seed=seed)
        c.integrate(MB)                                          # keeps the render stream busy
        d = torch.from_numpy(t.view(np.uint8).reshape(len(t), 160).copy()).cuda()
        c.update_triangles(d)
        del d
        junk = torch.full((len(t), 160), 255, dtype=torch.uint8, device="cuda")
        nodes, _ = c.read_bvh()
        assert_nodes_equal(nodes, new_sc["nodes"], exact=True)
        del junk
    c.destroy()


def capi_err(name):
    return {"INVALID": -1, "NOT_READY": -4, "UNSUPPORTED": -5}[name]


def test_update_launches_count_as_misc():
    sc = scene("CornellBox"); cam = default_camera(W, H)
    _, t = moved(sc, "scale")
    c = schedule_ctx(None, sc, cam, W, H, ((capi.OPT_KERNEL_TIMING, 1),))
    c.kernel_times()
    before = c.launch_count()
    c.update_triangles(t)
    assert c.launch_count() - before == 2                        # records + refit
    assert c.kernel_times()["misc"][1] == 2
    c.destroy()


def test_host_render_update_triangles_matches_the_c_abi(tmp_path):
    """Render::UpdateTriangles through hostapi: the image after an update and a reset equals the C ABI's."""
    from raytracing_b200 import hostapi
    from tests.test_host import PROC_OBJ, make_env
    w, h, mb = 96, 64, 4
    env_path, _ = make_env(tmp_path, w=64, h=32)
    s = hostapi.HostScene(PROC_OBJ)
    s.add_directional_light((-0.6, -1.5, 3.5), (15, 10, 5))
    r = hostapi.HostRender(s, w, h, env_path)
    r.set_max_bounces(mb)
    a = s.arrays(); a["nodes"] = r.nodes()
    t = deform(a["triangles"], "noise", seed=5)
    cam = hostapi.default_camera(w, h)
    c = capi.Context(w, h)
    c.upload_scene(a); c.set_camera(cam)
    try:
        r.render_frame()
        r.update_triangles(t); r.request_reset(); r.render_frame()
        c.update_triangles(t); c.reset(); c.integrate(mb)
        assert np.array_equal(bits(r.image()), bits(c.resolve()))
    finally:
        r.close(); s.close(); c.destroy()


def test_host_variant_streams_several_chunks():
    """A generated soup of 450 000 triangles (72 MB) passes through the host variant's 32 MB staging halves in three chunks, the
    third reusing the first half: nodes bit-equal to the numpy model, every record holding its children's boxes, the device
    variant's nodes and records, and a frame equal to the oracle on the updated arrays."""
    import torch
    from raytracing_b200 import hostapi
    from raytracing_b200.layouts import TRIANGLE_DT
    n = 450_000
    rng = np.random.default_rng(21)
    soup = np.zeros(n, dtype=TRIANGLE_DT)
    centre = rng.uniform(-1.0, 1.0, (n, 3)).astype(np.float32) * np.float32([1.0, 1.0, 0.5]) + np.float32([0.0, 0.0, 0.5])
    for v in ("v1", "v2", "v3"):
        soup[v]["position"][:, :3] = centre + rng.normal(0, 0.01, (n, 3)).astype(np.float32)
        soup[v]["normal"][:, :3] = (0, 0, 1)
    tris, nodes, _ = hostapi.build_bvh(soup)
    sc = {**scene("CornellBox"), "triangles": tris, "nodes": nodes, "emissive": np.zeros(0, "<u4")}
    cam = default_camera(W, H)
    new_sc, t = moved(sc, "noise", seed=9)
    assert t.nbytes > 2 * (32 << 20)
    c = schedule_ctx(None, sc, cam, W, H)
    c.reset(); c.integrate(MB)
    c.update_triangles(t)
    got_nodes, got_rec = c.read_bvh()
    assert_nodes_equal(got_nodes, new_sc["nodes"], exact=True)
    assert records_match_nodes(got_nodes, got_rec) == got_rec.shape[0]
    c.reset(); c.integrate(MB)
    orad, _, ost = Oracle(new_sc).render(cam, W, H, MB)
    check_frame(c, ost, orad, MB, ("soup", n))
    c.destroy()
    d = schedule_ctx(None, sc, cam, W, H)
    d.update_triangles(torch.from_numpy(t.view(np.uint8).reshape(n, 160).copy()).cuda())
    dev_nodes, dev_rec = d.read_bvh()
    assert np.array_equal(dev_nodes.view(np.uint8), got_nodes.view(np.uint8)) and np.array_equal(bits(dev_rec), bits(got_rec))
    d.destroy()


@pytest.mark.slow
def test_synthetic_10m_refit_matches_model_and_oracle():
    """Synthetic10M at full size (183 copies of ShaderBalls + ground): a refit after a rigid move of a third of the triangles
    gives rt_read_bvh nodes bit-equal to the numpy model, and a band of rows equals the oracle on the updated arrays."""
    from raytracing_b200 import scene_io, synthetic
    w, h, mb = 1920, 1080, 8
    sc = synthetic.bistro_scale_scene(scene_io.load_scene("ShaderBalls"), 183, w, h)
    cam = sc["camera_pose"]
    new_sc, t = moved(sc, "rigid", seed=2)
    c = capi.Context(w, h)
    c.upload_scene(sc); c.set_camera(cam)
    c.update_triangles(t)
    nodes, _ = c.read_bvh()
    assert_nodes_equal(nodes, new_sc["nodes"], exact=True)
    c.reset(); c.integrate(mb)
    img = c.read_radiance(); c.destroy()
    orad, _, _ = Oracle(new_sc).render(cam, w, h, mb, row_first=7, row_step=70)
    rows = np.arange(7, h, 70)
    assert np.array_equal(bits(img[rows][..., :3]), bits(orad[rows][..., :3]))


def test_headless_render_animate(tmp_path):
    """examples/headless_render --animate 3 writes the image HostRender renders after the same two moves of one mesh (the
    triangles of the first triangle's material, +1 % of the z extent per frame, accumulation restarted each frame)."""
    import os
    import subprocess
    from tests.helpers import REPO
    from tests.test_gpu_env_sampling import host_render_setup
    from tests.test_host import PROC_OBJ
    exe = str(tmp_path / "headless_render")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-I" + os.path.join(REPO, "include"), "-I" + os.path.join(REPO, "raytracing_b200", "host"),
                    os.path.join(REPO, "examples", "headless_render.cpp"), "-L" + os.path.join(REPO, "raytracing_b200"), "-l:librt_host.so",
                    "-l:librt_b200.so", "-Wl,-rpath," + os.path.join(REPO, "raytracing_b200"), "-o", exe], check=True)
    w, h, n = 64, 40, 4
    s, r, env_path = host_render_setup(tmp_path, w, h)
    out = str(tmp_path / "out.pfm")
    p = subprocess.run([exe, PROC_OBJ, env_path, str(w), str(h), str(n), out, "--animate", "3"], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    with open(out, "rb") as f:
        assert f.readline() == b"PF\n" and f.readline() == b"%d %d\n" % (w, h) and f.readline() == b"-1.0\n"
        img = np.frombuffer(f.read(), "<f4").reshape(h, w, 3)[::-1]
    t = s.arrays()["triangles"]
    z = np.concatenate([t[v]["position"][:, 2] for v in ("v1", "v2", "v3")])
    step = np.float32(0.01) * (z.max() - z.min())
    mesh = t["mtlIndex"] == t["mtlIndex"][0]
    assert 0 < mesh.sum() < len(t)
    r.set_max_bounces(8); r.set_samples_per_frame(n)
    r.render_frame()
    still = r.image()[..., :3]
    for _ in range(2):
        for v in ("v1", "v2", "v3"):
            t[v]["position"][mesh, 2] += step
        r.update_triangles(t); r.request_reset(); r.render_frame()
    want = r.image()[..., :3]
    r.close(); s.close()
    assert np.array_equal(bits(img), bits(want))
    assert not np.array_equal(bits(img), bits(still))
    assert subprocess.run([exe, PROC_OBJ, env_path, str(w), str(h), str(n), out, "--animate", "0"], capture_output=True).returncode == 2
