"""N samples per pixel: N calls of rt_integrate against one rt_integrate_samples(..., N), as rank 0 of 1-, 2-, 4- and 8-way scanline
partitions at 1920x1080 x 8 bounces (one GPU renders rank 0's rows, as tools/partition_probe.py does).

For every scene, partition and N the two arms are first checked to give byte-identical radiance and summed per-bounce statistics,
then timed with CUDA events around the whole call (ms per sample), the arms alternating, the set repeated.  "frames" and
"samples" run the default schedule selection (the per-phase graph on the whole frame and on a 2-way partition, k_frame below);
"frames_fk1" (N x k_frame) forces the one-kernel frame and must give the same radiance.

    python tools/spp_probe.py [--out DIR] [--reps 3] [--rounds 2]
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
STAT_KEYS = ("n_ext", "n_miss", "n_shadow", "n_cont", "n_unoccluded", "n_emissive_hits")


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name(0)


def context(sc, world, fk):
    c = capi.Context(W, H, device=0, rank=0, world=world)
    c.upload_scene(sc); c.set_camera(default_camera(W, H))
    if fk is not None:
        c.set_option(capi.OPT_FRAME_KERNEL, fk)
    return c


def run(c, arm, n):
    """One reset and the arm's N samples; returns the summed statistics."""
    c.reset()
    if arm.startswith("samples"):
        c.integrate_samples(MB, n)
        st = c.frame_stats()
        return {k: st[k].copy() for k in STAT_KEYS}
    total = {k: np.zeros(capi.MAX_BOUNCES + 1, np.uint32) for k in STAT_KEYS}
    for _ in range(n):
        c.integrate(MB)
        st = c.frame_stats()
        for k in STAT_KEYS:
            total[k] += st[k]
    return total


def timed(c, arm, n):
    c.reset(); c.sync()
    stream = torch.cuda.ExternalStream(c.stream_handle())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    if arm.startswith("samples"):
        c.integrate_samples(MB, n)
    else:
        for _ in range(n):
            c.integrate(MB)
    e1.record(stream)
    c.sync(); e1.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--scenes", default="CornellBox,ShaderBalls")
    ap.add_argument("--worlds", default="1,2,4,8")
    ap.add_argument("--ns", default="1,8,64")
    a = ap.parse_args()
    info = {"card": card(), "width": W, "height": H, "max_bounces": MB, "results": []}
    print("card:", info["card"], flush=True)
    for name in a.scenes.split(","):
        sc = scene_io.load_scene(name)
        for world in map(int, a.worlds.split(",")):
            arms = {"frames": None, "samples": None, "frames_fk1": 1}
            ctxs = {arm: context(sc, world, fk) for arm, fk in arms.items()}
            for n in map(int, a.ns.split(",")):
                # correctness first: the arms give the same bytes
                outs = {}
                for arm, c in ctxs.items():
                    st = run(c, arm, n)
                    outs[arm] = (c.read_radiance().tobytes(), st)
                f, s = outs["frames"], outs["samples"]
                if f[0] != s[0] or not all(np.array_equal(f[1][k], s[1][k]) for k in STAT_KEYS):
                    raise SystemExit(f"{name} world {world} N {n}: samples differs from frames")
                if outs["frames"][0] != outs["frames_fk1"][0]:
                    raise SystemExit(f"{name} world {world} N {n}: the schedules differ")
                for arm, c in ctxs.items():            # warm-up
                    timed(c, arm, n)
                ms = {arm: [] for arm in ctxs}
                for _ in range(a.rounds):
                    for _ in range(a.reps):
                        for arm, c in ctxs.items():    # alternating
                            ms[arm].append(timed(c, arm, n))
                row = {"scene": name, "world": world, "n": n, "identical": True,
                       "ms_per_sample": {arm: round(float(np.median(v)), 4) for arm, v in ms.items()},
                       "spread": {arm: [round(float(min(v)), 4), round(float(max(v)), 4)] for arm, v in ms.items()}}
                info["results"].append(row)
                print(json.dumps(row), flush=True)
            for c in ctxs.values():
                c.destroy()
    info["card_after"] = card()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "spp_probe.json"), "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
