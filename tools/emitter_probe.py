"""Emitter sampling (RT_OPT_EMITTER_SAMPLING) at 1920x1080 x 8 bounces on one GPU, CornellBox and ShaderBalls.

cost     ms per frame with the option on against off, arms alternating, median of --reps repetitions of 16 frames each: the whole
         frame on the per-phase graph (RT_OPT_FRAME_KERNEL 0) and rank 0 of a 4-way partition on k_frame (RT_OPT_FRAME_KERNEL 1).
benefit  RMSE of the displayed (Reinhard) image against a converged image (option off, samples 256 .. 256 + REF_SPP - 1, disjoint
         from the arms' samples 0 .. 255), with the option on and off at 1, 4, 16 and 64 spp; for each row the option-off spp that
         reaches the option-on RMSE (interpolated in log-log between measured counts 1 .. 256), and the option-off RMSE at equal time
         (the option-on spp times the cost ratio of the per-phase graph).

    python tools/emitter_probe.py [--out DIR] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from raytracing_b200 import capi, scene_io  # noqa: E402
from raytracing_b200.camera import default_camera  # noqa: E402

W, H, MB = 1920, 1080, 8
REF_SPP = 2048
SPPS = (1, 4, 16, 64)
MAX_OFF_SPP = 256
SCENES = ("CornellBox", "ShaderBalls")


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name(0)


def context(sc, world=1, fk=0, emitters=0):
    c = capi.Context(W, H, device=0, rank=0, world=world)
    c.upload_scene(sc); c.set_camera(default_camera(W, H))
    c.set_option(capi.OPT_FRAME_KERNEL, fk)
    c.set_option(capi.OPT_EMITTER_SAMPLING, emitters)
    return c


def frames_ms(c, n):
    """ms per frame of n rt_integrate calls, timed with CUDA events on the render stream."""
    stream = torch.cuda.ExternalStream(c.stream_handle())
    c.sync()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(n):
        c.integrate(MB)
    e1.record(stream); c.sync(); e1.synchronize()
    return e0.elapsed_time(e1) / n


def cost(sc, reps):
    out = {}
    for label, world, fk in (("graph_whole_frame", 1, 0), ("kframe_rank0_of_4", 4, 1)):
        ctxs = {on: context(sc, world, fk, on) for on in (0, 1)}
        for c in ctxs.values():
            c.reset(); frames_ms(c, 4)                 # warm-up: graph capture, first launches
        ms = {0: [], 1: []}
        for _ in range(reps):
            for on in (0, 1):
                ms[on].append(frames_ms(ctxs[on], 16))
        for c in ctxs.values():
            c.destroy()
        off, on = float(np.median(ms[0])), float(np.median(ms[1]))
        out[label] = {"ms_off": off, "ms_on": on, "ratio": on / off, "runs_off": ms[0], "runs_on": ms[1]}
    return out


def display(radiance, spp):
    x = radiance[..., :3].astype(np.float64) / spp
    return x / (1.0 + x)


def rmse(a, b):
    return float(np.sqrt(np.mean((a - b) ** 2)))


def benefit(sc, ratio):
    c = context(sc)
    c.reset()
    c.integrate_samples(MB, 256)
    skip = c.read_radiance().astype(np.float64)
    c.integrate_samples(MB, REF_SPP)
    ref = display(c.read_radiance().astype(np.float64) - skip, REF_SPP)
    c.destroy()
    curves = {}
    for on in (0, 1):
        c = context(sc, emitters=on)
        c.reset()
        counts = range(1, (MAX_OFF_SPP if on == 0 else max(SPPS)) + 1)
        curves[on] = {}
        for n in counts:
            c.integrate(MB)
            if on == 0 or n in SPPS:
                curves[on][n] = rmse(display(c.read_radiance(), n), ref)
        c.destroy()
    off_n = np.array(sorted(curves[0])); off_e = np.array([curves[0][n] for n in off_n])

    def off_spp_for(e):
        """option-off spp with the same RMSE: log-log interpolation on the measured curve (it decreases)"""
        if e >= off_e[0]:
            return 1.0
        if e < off_e[-1]:
            return float("inf")
        return float(np.exp(np.interp(-np.log(e), -np.log(off_e), np.log(off_n))))

    rows = []
    for n in SPPS:
        e_on = curves[1][n]
        eq = max(1, int(round(n / ratio)))
        rows.append({"spp": n, "rmse_off": curves[0][n], "rmse_on": e_on, "off_spp_same_rmse": off_spp_for(e_on),
                     "equal_time_off_spp": eq, "rmse_off_equal_time": curves[0].get(eq)})
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    result = {"gpu": card(), "workload": "%dx%d x %d bounces" % (W, H, MB), "scenes": {}}
    print(result["gpu"])
    for name in SCENES:
        sc = scene_io.load_scene(name)
        cst = cost(sc, args.reps)
        for k, v in cst.items():
            print("%-12s %-18s off %.3f ms  on %.3f ms  (x%.3f)" % (name, k, v["ms_off"], v["ms_on"], v["ratio"]))
        rows = benefit(sc, cst["graph_whole_frame"]["ratio"])
        for r in rows:
            print("%-12s %3d spp  RMSE off %.5f  on %.5f  off spp for the same RMSE %.1f  equal time: off at %d spp %.5f"
                  % (name, r["spp"], r["rmse_off"], r["rmse_on"], r["off_spp_same_rmse"], r["equal_time_off_spp"], r["rmse_off_equal_time"]))
        result["scenes"][name] = {"cost": cst, "rmse": rows}
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "emitter_probe.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
