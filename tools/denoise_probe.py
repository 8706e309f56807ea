"""The spatial denoiser (rt_set_spatial_denoiser) at 1920x1080 x 8 bounces on one GPU.

cost     ms per device-only resolve (rt_resolve with no host image) with the filter off and at 1..5 iterations, arms alternating, median
         over repetitions of 20 resolves each; the per-pass split is the difference of consecutive iteration counts (pass 0 includes the
         guide pack), with the achieved bytes/s of the assumed traffic (48 B/pixel per pass: colour and guide read, colour written;
         36 B/pixel for the pack) against the H100's 3.35 TB/s.
guides   frame time with AOV production forced on (RT_OPT_AOV_ALWAYS, what the filter turns on) against off, for the whole frame on the
         per-phase graph and for rank 0 of a 4-way partition on k_frame; radiance checked byte-identical first; 16 samples per call.
quality  CornellBox and ShaderBalls: RMSE of the displayed image against a 1024-spp reference rendered in the same run, unfiltered and
         filtered for several sigma settings at 1, 4, 16 and 64 spp, over all pixels and over edge pixels (the reference's depth changes
         by more than 10 % or its normal by more than 25 degrees inside a 3x3 window); and the spp an unfiltered image needs to match.

    python tools/denoise_probe.py [--out DIR] [--reps 5]
"""
import argparse
import ctypes as C
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
REF_SPP = 1024
SPPS = (1, 4, 16, 64)
SIGMAS = {"c0.3_n0.25_z0.15": (0.3, 0.25, 0.15), "c0.1_n0.25_z0.15": (0.1, 0.25, 0.15), "c1.0_n0.25_z0.15": (1.0, 0.25, 0.15),
          "c0.3_n0.25_z0": (0.3, 0.25, 0.0), "c0.3_n0_z0.15": (0.3, 0.0, 0.15), "c0_n0.25_z0.15": (0.0, 0.25, 0.15)}
HBM_TBPS = 3.35


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name(0)


def context(sc, world=1, fk=0, options=()):
    c = capi.Context(W, H, device=0, rank=0, world=world)
    c.upload_scene(sc); c.set_camera(default_camera(W, H))
    c.set_option(capi.OPT_FRAME_KERNEL, fk)
    for k, v in options:
        c.set_option(k, v)
    return c


class Timer:
    def __init__(self, c):
        self.c, self.stream = c, torch.cuda.ExternalStream(c.stream_handle())

    def __enter__(self):
        self.c.sync()
        self.e0, self.e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        self.e0.record(self.stream)
        return self

    def __exit__(self, *exc):
        self.e1.record(self.stream); self.c.sync(); self.e1.synchronize()
        self.ms = self.e0.elapsed_time(self.e1)


def device_resolve(c):
    c._ck(c.lib.rt_resolve(c.h, C.c_void_p(None)))


def cost(reps):
    sc = scene_io.load_scene("CornellBox")
    c = context(sc)
    c.set_spatial_denoiser(5, *SIGMAS["c0.3_n0.25_z0.15"])
    c.reset(); c.integrate_samples(MB, 8)
    arms = list(range(6))                     # iterations, 0 = off
    ms = {i: [] for i in arms}
    for rep in range(reps + 1):               # the first round warms up
        for i in arms:
            c.set_spatial_denoiser(i, *SIGMAS["c0.3_n0.25_z0.15"])
            device_resolve(c)                 # allocates the scratch planes outside the timed resolves
            with Timer(c) as t:
                for _ in range(20):
                    device_resolve(c)
            if rep:
                ms[i].append(t.ms / 20)
    c.destroy()
    med = {i: float(np.median(v)) for i, v in ms.items()}
    n = W * H
    passes = []
    for i in range(1, 6):
        d = med[i] - med[i - 1]
        nbytes = n * (48 + (36 if i == 1 else 0))
        passes.append({"pass": i - 1, "step": 1 << (i - 1), "ms": round(d, 4), "bytes_per_s_TB": round(nbytes / (d * 1e-3) / 1e12, 3),
                       "of_hbm_pct": round(100.0 * nbytes / (d * 1e-3) / (HBM_TBPS * 1e12), 1)})
    return {"what": "cost", "ms_per_resolve": {str(i): round(med[i], 4) for i in arms},
            "spread": {str(i): [round(min(v), 4), round(max(v), 4)] for i, v in ms.items()},
            "filter_ms_5_iterations": round(med[5] - med[0], 4), "passes": passes}


def guides(reps, n=16):
    out = []
    sc = scene_io.load_scene("CornellBox")
    for cfg, (world, fk) in {"whole_phase_graph": (1, 0), "rank0of4_k_frame": (4, 2)}.items():
        c = context(sc, world, fk)
        res = {}
        for v in (0, 1):
            c.set_option(capi.OPT_AOV_ALWAYS, v); c.reset(); c.integrate_samples(MB, n)
            res[v] = c.read_radiance().tobytes()
        if res[0] != res[1]:
            raise SystemExit("AOV production changed the radiance")
        ms = {0: [], 1: []}
        for rep in range(reps + 1):
            for v in (0, 1):
                c.set_option(capi.OPT_AOV_ALWAYS, v); c.reset(); c.integrate(MB); c.reset()   # re-capture outside the timed call
                with Timer(c) as t:
                    c.integrate_samples(MB, n)
                if rep:
                    ms[v].append(t.ms / n)
        c.destroy()
        off, on = float(np.median(ms[0])), float(np.median(ms[1]))
        out.append({"what": "guides", "config": cfg, "ms_per_frame_aov_off": round(off, 4), "ms_per_frame_aov_on": round(on, 4),
                    "cost_pct": round(100.0 * (on / off - 1.0), 2),
                    "spread": {k: [round(min(v), 4), round(max(v), 4)] for k, v in (("off", ms[0]), ("on", ms[1]))}})
    return out


def rmse(a, b, mask=None):
    d = a[..., :3].astype(np.float64) - b[..., :3].astype(np.float64)
    ok = np.isfinite(d).all(axis=-1)
    if mask is not None:
        ok &= mask
    return float(np.sqrt(np.mean(d[ok] ** 2)))


def edge_mask(depth, normal):
    """pixels where the depth changes by more than 10 % or the normal by more than 25 degrees inside the 3x3 window"""
    h, w = depth.shape
    m = np.zeros((h, w), bool)
    zp = np.pad(depth, 1, mode="edge"); npd = np.pad(normal[..., :3], ((1, 1), (1, 1), (0, 0)), mode="edge")
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            zq = zp[1 + dy: 1 + dy + h, 1 + dx: 1 + dx + w]; nq = npd[1 + dy: 1 + dy + h, 1 + dx: 1 + dx + w]
            m |= np.abs(zq - depth) > 0.1 * depth
            m |= (nq * normal[..., :3]).sum(-1) < np.cos(np.radians(25.0))
    return m


def quality(name):
    sc = scene_io.load_scene(name)
    c = context(sc, options=((capi.OPT_AOV_ALWAYS, 1),))
    c.reset()
    for _ in range(REF_SPP // 256):
        c.integrate_samples(MB, 256)
    ref = c.resolve()
    _, rdepth, rnormal, _ = c.read_aovs()
    edges = edge_mask(rdepth, rnormal)
    ladder = {}                                   # unfiltered RMSE at 1, 2, 4, ... 256 spp
    c.reset()
    done = 0
    for spp in (1, 2, 4, 8, 16, 32, 64, 128, 256):
        c.integrate_samples(MB, spp - done) if spp - done > 1 else c.integrate(MB)
        done = spp
        ladder[spp] = rmse(c.resolve(), ref)
    rows = []
    for spp in SPPS:
        c.reset()
        c.integrate_samples(MB, spp) if spp > 1 else c.integrate(MB)
        c.set_spatial_denoiser(0)
        raw = c.resolve()
        row = {"what": "quality", "scene": name, "spp": spp, "unfiltered": {"rmse": round(rmse(raw, ref), 6), "edge_rmse": round(rmse(raw, ref, edges), 6)}}
        for key, sig in SIGMAS.items():
            c.set_spatial_denoiser(5, *sig)
            img = c.resolve()
            e = rmse(img, ref)
            match = next((s for s in sorted(ladder) if ladder[s] <= e), None)
            row[key] = {"rmse": round(e, 6), "edge_rmse": round(rmse(img, ref, edges), 6),
                        "unfiltered_spp_to_match": match if match is not None else ">256"}
        c.set_spatial_denoiser(0)
        rows.append(row)
    c.destroy()
    return rows, {"edge_pct": round(100.0 * float(edges.mean()), 2), "unfiltered_ladder": {str(k): round(v, 6) for k, v in ladder.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--parts", default="cost,guides,quality")
    a = ap.parse_args()
    info = {"card": card(), "width": W, "height": H, "max_bounces": MB, "results": []}
    print("card:", info["card"], flush=True)
    parts = a.parts.split(",")
    if "cost" in parts:
        row = cost(a.reps); print(json.dumps(row), flush=True); info["results"].append(row)
    if "guides" in parts:
        for row in guides(a.reps):
            print(json.dumps(row), flush=True); info["results"].append(row)
    if "quality" in parts:
        for name in ("CornellBox", "ShaderBalls"):
            rows, extra = quality(name)
            print(json.dumps({"scene": name, **extra}), flush=True); info["results"].append({"scene": name, **extra})
            for row in rows:
                print(json.dumps(row), flush=True); info["results"].append(row)
    info["card_after"] = card()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "denoise_probe.json"), "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
