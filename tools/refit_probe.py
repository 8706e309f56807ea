"""
Geometry updates on one GPU (rt_update_triangles, include/rt_b200.h): what an update costs against a rebuild, and how a refit
tree ages as the deformation grows.

  python tools/refit_probe.py [--scenes CornellBox_Dragon,Synthetic10M] [--width 1920 --height 1080 --bounces 8] [--out FILE]

Per scene: the first update (builds the refit map), then the median of 5 updates through the host variant (numpy array) and the
device variant (CUDA torch tensor), each as wall time from the call to the end of rt_sync and as the device time of its two
kernels (CUDA events of RT_OPT_KERNEL_TIMING, class RT_K_MISC); an update while emitter and environment sampling are on (the
call blocks while the light tables are rebuilt: wall time); the host rebuild (hostapi.build_bvh) plus rt_upload_scene of the
same geometry; and, for per-vertex noise of growing amplitude, the median device time of a frame (rt_integrate between CUDA
events on the render stream, 3 runs) after a refit against a context that rebuilt and uploaded the deformed scene.  Prints one JSON line per measurement, headed by
the GPU's name and power limit read in the same run.

  python tools/refit_probe.py --motion [--scenes ...]

Object motion vectors (RT_OPT_OBJECT_MOTION) off against on, alternated twice on one context: the median host and device update
as above, and the median device time of a frame with AOV view 4 (the velocity AOV computed every frame) after an update.

  python tools/refit_probe.py --rebuild [--scenes ...] [--rigid 0.05,0.2] [--amplitudes 0.01,0.02,0.05,0.2,1.0]

The device rebuilds instead (rt_rebuild_bvh "linear" and rt_rebuild_bvh_ploc "ploc", --methods), each in a context of its own:
the first call (allocates and re-captures) and the median of 5 later calls as wall time to the end of rt_sync, their device time
(RT_K_MISC events) and, from torch.profiler, the device time of each kernel and the PLOC iteration count; the frame time of the
undeformed scene with the uploaded SAH tree and with the rebuilt tree; and, for rigid moves and per-vertex noise of growing
amplitude, the frame time after a refit of the uploaded tree against the frame time after each device rebuild.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from raytracing_b200 import capi, hostapi, scene_io, synthetic  # noqa: E402
from raytracing_b200.camera import default_camera  # noqa: E402
from tests.refit_model import deform  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def load(name, w, h):
    if name == "Synthetic10M":
        sc = synthetic.bistro_scale_scene(scene_io.load_scene("ShaderBalls"), 183, w, h)
        return sc, sc["camera_pose"]
    return scene_io.load_scene(name), default_camera(w, h)


def timed(fn, sync):
    t0 = time.perf_counter(); fn(); sync(); return (time.perf_counter() - t0) * 1e3


def frame_ms(c, mb, runs=3):
    """Median device time of rt_integrate: CUDA events recorded on the render stream around it."""
    import torch
    stream = torch.cuda.ExternalStream(c.stream_handle())
    c.reset(); c.integrate(mb); c.sync()
    out = []
    for _ in range(runs):
        c.reset()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream); c.integrate(mb); b.record(stream)
        c.sync(); b.synchronize()
        out.append(a.elapsed_time(b))
    return float(np.median(out))


def update_ms(c, src, runs=5):
    """(median wall ms of the update to the end of rt_sync, median device ms of its kernels)."""
    wall, dev = [], []
    c.set_option(capi.OPT_KERNEL_TIMING, 1)
    for _ in range(runs):
        c.kernel_times()
        wall.append(timed(lambda: c.update_triangles(src), c.sync))
        dev.append(c.kernel_times()["misc"][0])
    c.set_option(capi.OPT_KERNEL_TIMING, 0)
    return float(np.median(wall)), float(np.median(dev))


def rebuild_ms(c, method, runs=5):
    """(median wall ms of the rebuild to the end of rt_sync, median device ms of its launches)."""
    wall, dev = [], []
    c.set_option(capi.OPT_KERNEL_TIMING, 1)
    for _ in range(runs):
        c.kernel_times()
        wall.append(timed(lambda: c.rebuild_bvh(method), c.sync))
        dev.append(c.kernel_times()["misc"][0])
    c.set_option(capi.OPT_KERNEL_TIMING, 0)
    return float(np.median(wall)), float(np.median(dev))


def kernel_ms(c, method, runs=3):
    """(device ms per kernel name of one rebuild, launches per kernel name of one rebuild) from torch.profiler, mean over `runs`
    rebuilds; the PLOC iterations are the launches of k_ploc_nearest."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(runs):
            c.rebuild_bvh(method)
        c.sync()
    out, count = {}, {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" and e.device_time_total > 0:
            out[e.key[:60]] = round(e.device_time_total / 1e3 / runs, 4)
            count[e.key[:60]] = e.count // runs
    return out, count


def rebuild_arm(a, name, sc, cam, emit):
    n = len(sc["triangles"])
    ctx = {}
    for method in a.methods.split(","):
        c = ctx[method] = capi.Context(a.width, a.height)
        c.upload_scene(sc); c.set_camera(cam)
        sah_ms = frame_ms(c, a.bounces)
        first = timed(lambda: c.rebuild_bvh(method), c.sync)
        wall, dev = rebuild_ms(c, method)
        kernels, launches = kernel_ms(c, method)
        emit({"scene": name, "method": method, "triangles": n, "nodes_sah": len(sc["nodes"]), "first_rebuild_ms": first,
              "rebuild_ms": wall, "rebuild_device_ms": dev, "iterations": next((v for k, v in launches.items() if k.startswith("k_ploc_nearest")), None),
              "kernels_ms": kernels, "frame_ms_sah": sah_ms, "frame_ms_rebuilt": frame_ms(c, a.bounces)})
    refit = capi.Context(a.width, a.height)
    refit.upload_scene(sc); refit.set_camera(cam)
    moves = [("rigid", float(x)) for x in a.rigid.split(",") if x] + [("noise", float(x)) for x in a.amplitudes.split(",") if x]
    for kind, amp in moves:
        tt = deform(sc["triangles"], kind, seed=3, amount=amp)
        refit.update_triangles(tt)
        row = {"scene": name, "deformation": kind, "amplitude": amp, "frame_ms_refit": frame_ms(refit, a.bounces)}
        for method, c in ctx.items():
            c.update_triangles(tt); c.rebuild_bvh(method)
            row["frame_ms_" + method] = frame_ms(c, a.bounces)
        emit(row)
    refit.destroy()
    for c in ctx.values():
        c.destroy()


def motion_arm(a, name, sc, cam, emit):
    """RT_OPT_OBJECT_MOTION off against on, alternated twice on one context: the host and device update (update_ms) and the frame
    time with AOV view 4 (the velocity AOV produced every frame) after an update."""
    import torch
    n = len(sc["triangles"])
    t = deform(sc["triangles"], "rigid", seed=1, amount=0.02)
    d = torch.from_numpy(t.view(np.uint8).reshape(n, 160).copy()).cuda()
    torch.cuda.synchronize()
    c = capi.Context(a.width, a.height)
    c.upload_scene(sc); c.set_camera(cam); c.set_camera(cam)
    c.set_option(capi.OPT_AOV, 4)
    c.update_triangles(t); c.sync()                          # builds the refit map
    for rep in range(2):
        for motion in (0, 1):
            c.set_option(capi.OPT_OBJECT_MOTION, motion)
            host, host_k = update_ms(c, t)
            dev, dev_k = update_ms(c, d)
            emit({"scene": name, "triangles": n, "object_motion": motion, "rep": rep, "update_host_ms": host,
                  "update_host_kernels_ms": host_k, "update_device_ms": dev, "update_device_kernels_ms": dev_k,
                  "frame_ms_aov4": frame_ms(c, a.bounces), "prev_positions_bytes": n * 48 if motion else 0})
    c.destroy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", default="CornellBox_Dragon,Synthetic10M")
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--bounces", type=int, default=8)
    ap.add_argument("--amplitudes", default="0.01,0.05,0.2,1.0")
    ap.add_argument("--out", default=None)
    ap.add_argument("--rebuild", action="store_true", help="measure rt_rebuild_bvh instead of rt_update_triangles")
    ap.add_argument("--motion", action="store_true", help="measure updates and AOV frames with RT_OPT_OBJECT_MOTION off and on")
    ap.add_argument("--rigid", default="0.05,0.2", help="--rebuild: amplitudes of the rigid moves (empty: none)")
    ap.add_argument("--methods", default="linear,ploc", help="--rebuild: the device builds to measure (rt_rebuild_bvh, rt_rebuild_bvh_ploc)")
    a = ap.parse_args()
    import torch

    def emit(r):
        print(json.dumps(r), flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(json.dumps(r) + "\n")

    emit({"gpu": gpu_info()})

    for name in a.scenes.split(","):
        sc, cam = load(name, a.width, a.height)
        if a.rebuild:
            rebuild_arm(a, name, sc, cam, emit)
            continue
        if a.motion:
            motion_arm(a, name, sc, cam, emit)
            continue
        n = len(sc["triangles"])
        t = deform(sc["triangles"], "noise", seed=1, amount=0.01)
        c = capi.Context(a.width, a.height)
        c.upload_scene(sc); c.set_camera(cam)
        first = timed(lambda: c.update_triangles(t), c.sync)
        host, host_k = update_ms(c, t)
        d = torch.from_numpy(t.view(np.uint8).reshape(n, 160).copy()).cuda()
        torch.cuda.synchronize()
        dev, dev_k = update_ms(c, d)
        lit = capi.Context(a.width, a.height)
        lit.upload_scene(sc); lit.set_camera(cam)
        lit.set_option(capi.OPT_EMITTER_SAMPLING, 1); lit.set_option(capi.OPT_ENV_SAMPLING, 1)
        lit.update_triangles(t); lit.sync()
        lights = float(np.median([timed(lambda: lit.update_triangles(t), lit.sync) for _ in range(5)]))
        lit.destroy()
        t0 = time.perf_counter()
        rt, rn, _ = hostapi.build_bvh(t)
        build = (time.perf_counter() - t0) * 1e3
        fresh = capi.Context(a.width, a.height)
        upload = timed(lambda: fresh.upload_scene({**sc, "triangles": rt, "nodes": rn}), fresh.sync)
        fresh.destroy()
        emit({"scene": name, "triangles": n, "nodes": len(sc["nodes"]), "first_update_ms": first,
              "update_host_ms": host, "update_host_kernels_ms": host_k, "update_device_ms": dev, "update_device_kernels_ms": dev_k,
              "update_with_light_sampling_ms": lights, "emitters": int(len(sc["emissive"])),
              "rebuild_ms": build, "upload_ms": upload, "record_bytes_per_update": n * (160 + 48 + 48 + 112)})
        c.update_triangles(sc["triangles"])
        base = frame_ms(c, a.bounces)
        for amp in [float(x) for x in a.amplitudes.split(",")]:
            tt = deform(sc["triangles"], "noise", seed=3, amount=amp)
            c.update_triangles(tt)
            refit_ms = frame_ms(c, a.bounces)
            rt, rn, _ = hostapi.build_bvh(tt)
            f = capi.Context(a.width, a.height)
            f.upload_scene({**sc, "triangles": rt, "nodes": rn}); f.set_camera(cam)
            rebuilt_ms = frame_ms(f, a.bounces)
            f.destroy()
            emit({"scene": name, "noise_amplitude": amp, "frame_ms_undeformed": base, "frame_ms_refit": refit_ms,
                  "frame_ms_rebuilt": rebuilt_ms})
        c.destroy()


if __name__ == "__main__":
    main()
