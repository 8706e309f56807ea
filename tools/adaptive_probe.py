"""Adaptive sampling (rt_set_adaptive_sampling) at 1920x1080 x 8 bounces, on the whole frame (per-phase graph) and on rank 0 of a 4-way
scanline partition (k_frame, the default selection there), one GPU.

overhead  the feature on with nothing stopping (min_samples above N) against the feature off, N = 64 samples per rt_integrate_samples
          call: first checked byte-identical (radiance and summed statistics), then timed with CUDA events, the arms alternating.
benefit   for each max_error, progressive rendering in calls of 16 samples until no pixel is active or 256 samples are spent (what
          examples/headless_render does): mean samples per pixel, time, rays traced, and the RMSE of the resolved image against a
          2048-sample reference rendered in the same call; then uniform sampling for the same time (the sample count that the
          feature-off time per sample fits into it) and its RMSE; for min_samples 4 and 16.
per_ray   one frame at a time for the largest max_error (min_samples 4): the time per traced ray (extension + shadow rays) as the active fraction
          falls, and the time of a frame with no active pixel.

    python tools/adaptive_probe.py [--out DIR] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from raytracing_b200 import capi, scene_io  # noqa: E402
from raytracing_b200.camera import default_camera  # noqa: E402

W, H, MB = 1920, 1080, 8
STAT_KEYS = ("n_ext", "n_miss", "n_shadow", "n_cont", "n_unoccluded", "n_emissive_hits")
# name: (world, RT_OPT_FRAME_KERNEL).  Rank 0 of 4 takes the default selection, which is k_frame there (518 400 pixels <= 132 SMs x 7168).
CONFIGS = {"whole": (1, 0), "rank0of4": (4, 2)}
CHUNK, CAP, REF_SPP = 16, 256, 2048


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name(0)


def context(sc, world, fk):
    c = capi.Context(W, H, device=0, rank=0, world=world)
    c.upload_scene(sc); c.set_camera(default_camera(W, H))
    c.set_option(capi.OPT_FRAME_KERNEL, fk)
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


def rays(st):
    return int(st["n_ext"].astype(np.int64).sum() + st["n_shadow"].astype(np.int64).sum())


def rows_of(img, world):
    return img[0::world]


def rmse(a, b):
    """over the pixels finite in both images (a few ShaderBalls pixels accumulate a NaN sample)"""
    d = a[..., :3].astype(np.float64) - b[..., :3].astype(np.float64)
    ok = np.isfinite(d).all(axis=-1)
    return float(np.sqrt(np.mean(d[ok] ** 2)))


def configure(c, max_error, min_samples):
    """The setting, a reset, one untimed frame and a reset again: a changed setting changes the frame's launch arguments, and the
    per-phase frame graph is re-captured in that untimed frame instead of inside a timed call."""
    c.set_adaptive_sampling(max_error, min_samples)
    c.reset(); c.integrate(MB); c.reset()


def overhead(c, n, reps):
    c.set_adaptive_sampling(0, 0)
    out = {}
    for arm in ("off", "on_nothing_stops"):
        configure(c, 0, 0) if arm == "off" else configure(c, 0.01, 1 << 30)
        c.integrate_samples(MB, n)
        st = c.frame_stats()
        out[arm] = (c.read_radiance().tobytes(), {k: st[k].tobytes() for k in STAT_KEYS})
    if out["off"] != out["on_nothing_stops"]:
        raise SystemExit("feature on with nothing stopping is not byte-identical to the feature off")
    ms = {"off": [], "on_nothing_stops": []}
    for rep in range(reps + 1):                          # the first round warms up
        for arm in ms:
            configure(c, 0, 0) if arm == "off" else configure(c, 0.01, 1 << 30)
            with Timer(c) as t:
                c.integrate_samples(MB, n)
            if rep:
                ms[arm].append(t.ms / n)
    c.set_adaptive_sampling(0, 0); c.reset()
    return {arm: round(float(np.median(v)), 4) for arm, v in ms.items()}, {arm: [round(min(v), 4), round(max(v), 4)] for arm, v in ms.items()}


def progressive(c, max_error, min_samples):
    """Calls of CHUNK samples until nothing is active or CAP samples are spent -> (ms, wall ms, samples, rays, per-pixel counts)."""
    configure(c, max_error, min_samples)
    total_rays, spent = 0, 0
    c.sync()
    t0 = time.perf_counter()
    with Timer(c) as t:
        while spent < CAP:
            c.integrate_samples(MB, CHUNK); spent += CHUNK
            total_rays += rays(c.frame_stats())
            if c.active_pixels() == 0:
                break
    wall = (time.perf_counter() - t0) * 1e3
    spp = c.pixel_samples()
    return t.ms, wall, spent, total_rays, spp


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--scenes", default="CornellBox,ShaderBalls")
    ap.add_argument("--errors", default="0.02,0.01,0.005,0.0025")
    ap.add_argument("--min-samples", default="4,16")
    ap.add_argument("--configs", default=",".join(CONFIGS))
    a = ap.parse_args()
    info = {"card": card(), "width": W, "height": H, "max_bounces": MB, "results": []}
    print("card:", info["card"], flush=True)
    for name in a.scenes.split(","):
        sc = scene_io.load_scene(name)
        ref = None
        for cfg in a.configs.split(","):
            world, fk = CONFIGS[cfg]
            c = context(sc, world, fk)
            n_local = c.local_pixel_count()
            if ref is None:                              # the 2048-sample reference of the whole frame (the rank's rows are a subset)
                full = context(sc, 1, 0); full.reset()
                for _ in range(REF_SPP // 256):
                    full.integrate_samples(MB, 256)
                ref = full.resolve(); full.destroy()
            ref_rows = rows_of(ref, world)
            med, spread = overhead(c, 64, a.reps)
            row = {"scene": name, "config": cfg, "what": "overhead", "n": 64, "ms_per_sample": med, "spread": spread,
                   "overhead_pct": round(100.0 * (med["on_nothing_stops"] / med["off"] - 1.0), 2)}
            print(json.dumps(row), flush=True); info["results"].append(row)
            ms_uniform = med["off"]
            # uniform rays per sample, for the rays-per-ms comparison
            c.reset(); c.integrate(MB); uniform_rays = rays(c.frame_stats())
            errors = [float(x) for x in a.errors.split(",") if x]          # --errors "": the overhead only
            if not errors:
                c.destroy()
                continue
            c.set_adaptive_sampling(0, 0); c.reset(); c.integrate_samples(MB, CAP)
            cap_img = rows_of(c.resolve(), world)
            for me, mins in [(e, m) for m in map(int, a.min_samples.split(",")) for e in errors]:
                ms, wall, spent, n_rays, spp = progressive(c, me, mins)
                img = rows_of(c.resolve(), world)
                mean_spp = float(spp[0::world].astype(np.float64).mean())
                n_eq = max(1, int(round(ms / ms_uniform)))
                c.set_adaptive_sampling(0, 0); c.reset(); c.integrate_samples(MB, n_eq) if n_eq > 1 else c.integrate(MB)
                uni = rows_of(c.resolve(), world)
                row = {"scene": name, "config": cfg, "what": "benefit", "max_error": me, "min_samples": mins, "samples_spent": spent,
                       "mean_spp": round(mean_spp, 2), "ms": round(ms, 2), "wall_ms": round(wall, 2), "rays": n_rays,
                       "ns_per_ray": round(ms * 1e6 / max(n_rays, 1), 3), "uniform_ns_per_ray": round(ms_uniform * 1e6 / uniform_rays, 3),
                       "rmse": round(rmse(img, ref_rows), 6), "uniform_equal_time_spp": n_eq, "uniform_equal_time_rmse": round(rmse(uni, ref_rows), 6),
                       "uniform_256_rmse": round(rmse(cap_img, ref_rows), 6), "uniform_256_ms": round(ms_uniform * CAP, 2),
                       "stopped_pct": round(100.0 * float((spp[0::world] < spent).mean()), 2),
                       "nonfinite_px": int((~np.isfinite(ref_rows[..., :3]).all(axis=-1)).sum())}
                print(json.dumps(row), flush=True); info["results"].append(row)
            # time per traced ray as the active fraction falls, one frame at a time
            me = errors[0]
            configure(c, me, 4)
            trace = []
            for f in range(CAP):
                act = c.active_pixels()
                with Timer(c) as t:
                    c.integrate(MB)
                st = c.frame_stats()
                trace.append((f, act / n_local, t.ms, rays(st)))
                if act == 0:
                    break
            pts = []
            for target in (1.0, 0.75, 0.5, 0.25, 0.1, 0.05, 0.02, 0.0):
                best = min(trace, key=lambda r: abs(r[1] - target))
                pts.append({"active": round(best[1], 4), "frame": best[0], "ms": round(best[2], 3), "rays": best[3],
                            "ns_per_ray": round(best[2] * 1e6 / best[3], 3) if best[3] else None})
            row = {"scene": name, "config": cfg, "what": "per_ray", "max_error": me, "points": pts}
            print(json.dumps(row), flush=True); info["results"].append(row)
            c.destroy()
    info["card_after"] = card()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "adaptive_probe.json"), "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
