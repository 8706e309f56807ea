"""Sampled lights at 1920x1080 x 8 bounces on one GPU: emitter sampling (RT_OPT_EMITTER_SAMPLING), environment sampling
(RT_OPT_ENV_SAMPLING) and the light-kind weights (rt_set_light_selection), on CornellBox, ShaderBalls, procedural and ShaderBalls
under a synthetic sun sky (the shipped sky plus a 3x2-texel sun of luma 1e4 at about 45 degrees elevation) that lights it alone
(its directional light dark).

Settings: off, emitters, env, both (default weights), and both with weights chosen per scene (WEIGHTS below).
cost      ms per frame of rt_integrate (the default schedule: the per-phase graph at 1080p), settings alternating, median of --reps
          repetitions of 8 frames each.
variance  mean over pixels and channels of the per-pixel variance of one sample, from samples 0 .. VAR_SPP - 1 (pixels whose
          radiance is NaN, which the renderer produces on a few ShaderBalls pixels with every setting, are left out here and below).
rmse      RMSE of the displayed (Reinhard) image at equal time against a converged image (option off, REF_SPP samples starting at
          sample index REF_FIRST, disjoint from the settings' samples): every setting gets the time of BUDGET_SPP samples of the
          setting off, i.e. round(BUDGET_SPP * ms_off / ms_setting) samples.

    python tools/light_probe.py [--out DIR] [--reps 3]
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
from tests.test_emitter_sampling_cpu import procedural_scene  # noqa: E402

W, H, MB = 1920, 1080, 8
REF_SPP, REF_FIRST = 1024, 4096
VAR_SPP = 16
BUDGET_SPP = 32
SETTINGS = {"off": (0, 0, None), "emitters": (1, 0, None), "env": (0, 1, None), "both": (1, 1, None), "chosen": (1, 1, "scene")}
# hand-chosen from what lights each scene: (analytic, emitters, environment)
WEIGHTS = {"CornellBox": (1.0, 3.0, 0.5), "ShaderBalls": (2.0, 0.5, 1.0), "procedural": (4.0, 1.0, 1.0), "ShaderBalls_sun": (1.0, 0.25, 2.0)}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name(0)


def sun_sky(env, w, h, seed=5):
    rng = np.random.default_rng(seed)
    img = np.array(env, dtype="<f4").reshape(h, w, 4)
    j, i = h // 4 + int(rng.integers(-5, 6)), int(rng.integers(0, w - 3))
    img[j:j + 2, i:i + 3, :3] = np.float32(1e4)
    return img.reshape(-1)


def load(name):
    if name == "procedural":
        return procedural_scene()
    sc = dict(scene_io.load_scene(name.replace("_sun", "")))
    if name.endswith("_sun"):
        sc["env"] = sun_sky(sc["env"], int(sc["env_width"]), int(sc["env_height"]))
        sc["lights"] = sc["lights"].copy(); sc["lights"]["radiance"] = 0          # the sun is in the sky: no directional light
    return sc


def context(sc, name, setting):
    em, env, wts = SETTINGS[setting]
    c = capi.Context(W, H, device=0)
    c.upload_scene(sc); c.set_camera(default_camera(W, H))
    c.set_option(capi.OPT_EMITTER_SAMPLING, em); c.set_option(capi.OPT_ENV_SAMPLING, env)
    if wts:
        c.set_light_selection(*WEIGHTS[name])
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


def display(radiance, spp):
    x = radiance[..., :3].astype(np.float64) / spp
    return x / (1.0 + x)


def probe_scene(name, reps):
    sc = load(name)
    ctxs = {s: context(sc, name, s) for s in SETTINGS}
    for c in ctxs.values():
        c.reset(); frames_ms(c, 2)                     # warm-up: graph capture, first launches
    runs = {s: [] for s in SETTINGS}
    for _ in range(reps):
        for s, c in ctxs.items():
            runs[s].append(frames_ms(c, 8))
    ms = {s: float(np.median(r)) for s, r in runs.items()}
    c = ctxs["off"]
    c.reset()
    for _ in range(REF_FIRST):
        c.advance_sample_count()
    c.integrate_samples(MB, REF_SPP)
    ref = display(c.read_radiance(), REF_SPP)
    out = {}
    for s, c in ctxs.items():
        c.reset()
        prev = np.zeros((H, W, 3), np.float64)
        s1 = np.zeros((H, W, 3), np.float64); s2 = np.zeros((H, W, 3), np.float64)
        for _ in range(VAR_SPP):
            c.integrate(MB)
            cur = c.read_radiance()[..., :3].astype(np.float64)
            x = cur - prev; prev = cur
            s1 += x; s2 += x * x
        mean = s1 / VAR_SPP
        var = float(np.nanmean(s2 / VAR_SPP - mean * mean) * VAR_SPP / (VAR_SPP - 1))
        n = max(1, int(round(BUDGET_SPP * ms["off"] / ms[s])))
        c.reset(); c.integrate_samples(MB, n)
        err = float(np.sqrt(np.nanmean((display(c.read_radiance(), n) - ref) ** 2)))
        out[s] = {"ms": ms[s], "runs_ms": runs[s], "variance": var, "equal_time_spp": n, "rmse_equal_time": err}
        print("%-16s %-9s %7.3f ms/frame  variance %.4g  equal time: %3d spp, RMSE %.5f" % (name, s, ms[s], var, n, err))
    for c in ctxs.values():
        c.destroy()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--scenes", default=",".join(WEIGHTS))
    args = ap.parse_args()
    result = {"gpu": card(), "workload": "%dx%d x %d bounces" % (W, H, MB), "weights": WEIGHTS, "scenes": {}}
    print(result["gpu"])
    for name in args.scenes.split(","):
        result["scenes"][name] = probe_scene(name, args.reps)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "light_probe.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
