"""Same-card A/B of the 4-wide octant tables (RT_OPT_OCTANT_BVH): 1920x1080 x 8 bounces, CornellBox (staged whole in shared
memory: the scene the tables exist for) and ShaderBalls (traversed through L1/L2: the control that must not move).
Arms: "parent" = a library built from the parent commit (a path, or a variant name of tools/build_variant.py; skipped when the
file does not exist), "off" = the in-tree library with the option 0, "on" = the in-tree library with the option 1.  Schedules:
"phase" = the per-phase kernels on the whole frame (what bench.py's headline runs), "frame" = the one-kernel frame (k_frame) on
rank 0 of a 4-way partition (it keeps the canonical records: a control that must not move either).  First asserts that every arm leaves the same radiance bits and frame statistics as the first one,
then alternates the arms: median over the repetitions of the best of 3 windows of 20 frames (CUDA events, ms per frame), and
for the per-phase schedule the per-kernel split of OPT_KERNEL_TIMING (individual launches, shadow pass on its own).
usage: octant_probe.py [--reps R] [--parent LIB] [--json FILE]"""
import argparse, json, os, statistics, subprocess, sys
HERE = os.path.dirname(os.path.abspath(__file__)); REPO = os.path.dirname(HERE)
CHILD = r'''
import hashlib, json, os, sys, torch
sys.path.insert(0, %r)
from raytracing_b200 import capi, scene_io
from raytracing_b200.camera import default_camera
octant, check = sys.argv[1], sys.argv[2] == "1"
w, h, mb = 1920, 1080, 8
out = {}
for name in ("CornellBox", "ShaderBalls"):
    sc = scene_io.load_scene(name)
    for sched in ("phase", "frame"):
        ctx = capi.Context(w, h, device=0, rank=0, world=4 if sched == "frame" else 1)
        ctx.set_option(capi.OPT_FRAME_KERNEL, 1 if sched == "frame" else 0)
        if octant != "-":
            ctx.set_option(capi.OPT_OCTANT_BVH, int(octant))
        ctx.upload_scene(sc); ctx.set_camera(sc["camera_pose"] if "camera_pose" in sc else default_camera(w, h))
        r = {}
        if check:
            ctx.reset(); ctx.integrate(mb); ctx.sync()
            r["radiance"] = hashlib.sha256(ctx.read_radiance().tobytes()).hexdigest()
            r["stats"] = hashlib.sha256(ctx.frame_stats().tobytes()).hexdigest()
        stream = torch.cuda.ExternalStream(ctx.stream_handle())
        best = 1e9
        for rep in range(3):
            for _ in range(3):
                ctx.reset(); ctx.integrate(mb)
            ctx.sync()
            n = 20
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(n):
                ctx.reset(); ctx.integrate(mb)
            e1.record(stream); ctx.sync(); torch.cuda.synchronize()
            best = min(best, e0.elapsed_time(e1) / n)
        r["ms"] = best
        if sched == "phase":
            ctx.set_option(capi.OPT_KERNEL_TIMING, 1); ctx.set_option(capi.OPT_OVERLAP, 0)
            for _ in range(2):
                ctx.reset(); ctx.integrate(mb)
            ctx.sync(); ctx.kernel_times()
            for _ in range(10):
                ctx.reset(); ctx.integrate(mb)
            ctx.sync()
            r["kernels"] = {k: v[0] / 10 for k, v in ctx.kernel_times().items() if v[1]}
        ctx.destroy()
        out[name + " " + sched] = r
print(json.dumps(out))
''' % REPO


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--parent", default="parent")
    ap.add_argument("--json", default=None, help="also write the raw runs to this file")
    args = ap.parse_args()
    cur = os.path.join(REPO, "raytracing_b200", "librt_b200.so")
    parent = args.parent if os.path.sep in args.parent else os.path.join(REPO, "raytracing_b200", "variants", f"librt_b200_{args.parent}.so")
    arms = [("off", cur, "0"), ("on", cur, "1")]
    if os.path.exists(parent):
        arms.insert(0, ("parent", parent, "-"))
    else:
        print(f"no parent library at {parent}: arms off / on only")
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
        gpu = q.stdout.strip() or q.stderr.strip()
    except OSError as e:
        gpu = repr(e)
    print(f"GPU: {gpu}  (name, power limit, max SM clock, SM clock at idle)")
    runs = {a[0]: [] for a in arms}
    for rep in range(args.reps):
        for name, lib, octant in arms:
            r = subprocess.run([sys.executable, "-c", CHILD, octant, "1" if rep == 0 else "0"], capture_output=True, text=True,
                               env=dict(os.environ, RT_B200_LIB=lib))
            if r.returncode:
                sys.exit(f"{name}: {r.stderr.strip()[-2000:]}")
            runs[name].append(json.loads(r.stdout.strip().splitlines()[-1]))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(runs, f)
    first = arms[0][0]
    same = True
    for name, _, _ in arms[1:]:
        for case, r in runs[name][0].items():
            for k in ("radiance", "stats"):
                ok = r[k] == runs[first][0][case][k]
                same &= ok
                print(f"{case:18s} {name} vs {first}: {k} {'byte-identical' if ok else 'DIFFERENT'}")
    for case in runs[first][0]:
        print(f"{case}, 1920x1080 x 8: median of {args.reps} repetitions of the best of 3 windows (ms per frame; per kernel ms per frame)")
        for name, _, _ in arms:
            ms = [r[case]["ms"] for r in runs[name]]
            ks = runs[name][0][case].get("kernels", {})
            ks = {k: statistics.median(r[case]["kernels"][k] for r in runs[name]) for k in ks}
            split = "  ".join(f"{k} {v:.3f}" for k, v in sorted(ks.items(), key=lambda kv: -kv[1]) if v >= 0.001)
            print(f"  {name:7s} {statistics.median(ms):.3f}  (runs {' '.join(f'{m:.3f}' for m in ms)})  {split}")
    sys.exit(0 if same else 1)


if __name__ == "__main__":
    main()
