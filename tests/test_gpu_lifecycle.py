"""
GPU tests (-m gpu) of the device resources a context owns.  One context walks through every resource group's creation,
replacement and release (AOV buffers, spatial-denoiser planes, adaptive-sampling state, the pipelined read-back, the update
staging and refit map, the rebuilt tree, the light tables, the partition's buffers, the scene); after every step its frame
equals, bit for bit, that of a fresh context configured directly into the same state.  And contexts created with every group on
and destroyed again give their device memory back.
"""
import numpy as np
import pytest

from raytracing_b200 import capi
from raytracing_b200.camera import default_camera
from tests.helpers import bits, scene
from tests.refit_model import deform, refit
from tests.test_gpu_parity import SCHEDULES, check_stats

pytestmark = pytest.mark.gpu

W, H, MB = 64, 48, 4
SD = (2, 0.5, 0.2, 0.1)
LIGHTS = ((capi.OPT_EMITTER_SAMPLING, 1), (capi.OPT_ENV_SAMPLING, 1))


def soup_scene(n_soup=230_000, seed=5):
    """CornellBox plus a cloud of small triangles, enough (> 32 MB) for a host update to stream through several staging chunks.
    The emitters are found again by material after the host build reorders the triangles."""
    from raytracing_b200 import hostapi
    from raytracing_b200.layouts import TRIANGLE_DT
    sc = scene("CornellBox")
    light_mtl = set(sc["triangles"]["mtlIndex"][np.asarray(sc["emissive"], np.int64)].tolist())
    plain_mtl = next(int(m) for m in sc["triangles"]["mtlIndex"] if int(m) not in light_mtl)
    rng = np.random.default_rng(seed)
    soup = np.zeros(n_soup, dtype=TRIANGLE_DT)
    centre = rng.uniform(-0.4, 0.4, (n_soup, 3)).astype(np.float32) + np.float32([0.0, 0.0, 0.4])
    for v in ("v1", "v2", "v3"):
        soup[v]["position"][:, :3] = centre + rng.normal(0, 0.003, (n_soup, 3)).astype(np.float32)
        soup[v]["normal"][:, :3] = (0, 0, 1)
    soup["mtlIndex"] = plain_mtl
    tris, nodes, _ = hostapi.build_bvh(np.concatenate([sc["triangles"], soup]))
    emissive = np.flatnonzero(np.isin(tris["mtlIndex"], list(light_mtl))).astype("<u4")
    return {**sc, "triangles": tris, "nodes": nodes, "emissive": emissive}


def configure(c, st):
    """Puts a context that has its scene and camera into the walk's state `st` (options, filters, sampling, tree)."""
    if st["rebuilt"]:
        c.rebuild_bvh()
    for k, v in SCHEDULES[st["schedule"]] + ((capi.OPT_AOV, st["aov"]),) + (LIGHTS if st["lights"] else ()):
        c.set_option(k, v)
    c.set_spatial_denoiser(*(SD if st["sd"] else (0,)))
    c.set_adaptive_sampling(*((0.05, 2) if st["adaptive"] else (0.0,)))


def fresh(st, cam):
    c = capi.Context(W, H, rank=st["rank"], world=st["world"])
    c.upload_scene(st["scene"]); c.set_camera(cam)
    configure(c, st)
    return c


def frame(c):
    """Two frames from a reset: radiance, statistics and the resolved image."""
    c.reset(); c.integrate(MB); c.integrate(MB)
    return c.read_radiance(), c.frame_stats(), c.resolve()


def assert_same(got, want, where):
    check_stats(got[1], want[1], MB, where)
    assert np.array_equal(bits(got[0]), bits(want[0])), where
    assert np.array_equal(bits(got[2]), bits(want[2])), where


@pytest.mark.parametrize("schedule", ["frame", "phase_graph"])
def test_every_group_through_create_replace_release(schedule):
    import torch
    sc = soup_scene(); cam = default_camera(W, H)
    t_host = deform(sc["triangles"], "noise", seed=11)
    t_dev = deform(sc["triangles"], "rigid", seed=12)
    assert t_host.nbytes > 32 << 20
    st = {"schedule": schedule, "scene": sc, "rebuilt": False, "aov": 0, "sd": False, "adaptive": False, "lights": False,
          "rank": 0, "world": 1}
    c = fresh(st, cam)

    def set_(**kw):
        st.update(kw)
        configure_walked(kw)

    def configure_walked(kw):
        if "aov" in kw:
            c.set_option(capi.OPT_AOV, kw["aov"])
        if "sd" in kw:
            c.set_spatial_denoiser(*(SD if kw["sd"] else (0,)))
        if "adaptive" in kw:
            c.set_adaptive_sampling(*((0.05, 2) if kw["adaptive"] else (0.0,)))
        if "lights" in kw:
            for k, v in LIGHTS:
                c.set_option(k, v if kw["lights"] else 0)

    def check(where):
        f = fresh(st, cam)
        assert_same(frame(c), frame(f), (schedule, where))
        f.destroy()

    check("start")
    set_(aov=1); check("aov view on")
    set_(aov=0, sd=True); check("spatial denoiser on")
    set_(sd=False); check("spatial denoiser off")
    set_(adaptive=True); check("adaptive on")
    check("adaptive reset")
    set_(adaptive=False); check("adaptive off")

    c.reset(); c.integrate(MB)
    out = np.zeros((H, W, 4), "<f4")
    for _ in range(3):                                      # both resolve buffers, the first one again
        c.resolve_async(out); c.resolve_wait()
    f = fresh(st, cam); f.reset(); f.integrate(MB)
    assert np.array_equal(bits(out), bits(f.resolve())), (schedule, "resolve_async")
    f.destroy()

    c.update_triangles(t_host)
    st["scene"] = {**sc, "triangles": t_host, "nodes": refit(sc["nodes"], t_host)}; check("host update")
    c.update_triangles(t_host)
    check("host update again")
    c.update_triangles(torch.from_numpy(t_dev.view(np.uint8).reshape(len(t_dev), 160).copy()).cuda())
    st["scene"] = {**sc, "triangles": t_dev, "nodes": refit(sc["nodes"], t_dev)}; check("device update")
    c.rebuild_bvh(); st["rebuilt"] = True; check("first rebuild")
    c.rebuild_bvh(); check("second rebuild")

    set_(lights=True); check("light sampling on")
    set_(lights=False); check("light sampling off")

    c._ck(c.lib.rt_set_partition(c.h, 1, 2))
    st["rank"], st["world"] = 1, 2; check("re-partition")

    c.upload_scene(sc)
    st["scene"], st["rebuilt"] = sc, False; check("scene re-upload")
    c.destroy()


def test_contexts_give_their_memory_back():
    """At 1920x1080: the free device memory after 8 cycles of create, every group on, render, destroy is within one cycle's
    footprint of where it started (a group lost per cycle would show as several footprints).  The card is shared, so this is
    a coarse guard, not an exact count."""
    import torch
    w, h = 1920, 1080
    sc = scene("CornellBox"); cam = default_camera(w, h)
    t = deform(sc["triangles"], "noise", seed=3)
    out = np.zeros((h, w, 4), "<f4")

    def free():
        torch.cuda.synchronize()
        return torch.cuda.mem_get_info()[0]

    def cycle(destroy=True):
        c = capi.Context(w, h)
        c.upload_scene(sc); c.set_camera(cam)
        for k, v in ((capi.OPT_AOV_ALWAYS, 1), (capi.OPT_OVERLAP, 1), (capi.OPT_KERNEL_TIMING, 1)) + LIGHTS:
            c.set_option(k, v)
        c.set_spatial_denoiser(*SD)
        c.set_adaptive_sampling(0.05, 2)
        c.update_triangles(t); c.rebuild_bvh()
        c.reset(); c.integrate_samples(MB, 2)
        c.read_rays(1)
        c.resolve_async(out); c.resolve_async(out); c.resolve_wait()
        c.kernel_times()
        if destroy:
            c.destroy()
        return c

    start = free()
    c = cycle(destroy=False)
    footprint = start - free()
    c.destroy()
    assert footprint > 0
    for _ in range(8):
        cycle()
    assert start - free() <= footprint, (start, free(), footprint)
