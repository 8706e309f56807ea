"""Where the time of the unsorted shading pass (k_shade_queues<false>) goes: 1920x1080 x 8 bounces, per-phase schedule, CornellBox
and ShaderBalls.  Arms (libraries; build the variants first with tools/build_variant.py):
  parent  the parent commit's library (a path, or a variant name; skipped when the file does not exist)
  built   the in-tree library
  mem     variant "shade_mem"  -DRT_SHADE_PROBE=1: memory floor (the same entry, ray, shading-record, material and blue-noise reads
          and the same kind of queue stores, with the shading arithmetic replaced by a few adds; every hit spawns both rays)
  math    variant "shade_math" -DRT_SHADE_PROBE=2: math floor (each warp shades its first hit group's entries and rays again for
          every hit group it takes, so those reads hit L1/L2; the stores stay)
First asserts that parent and built leave the same radiance bits and frame statistics, then alternates the arms: median over the
repetitions of the best of 3 windows of 20 frames (CUDA events, ms per frame) and the per-kernel split of OPT_KERNEL_TIMING
(individual launches, shadow pass on its own).  The floors change which rays are spawned, so the shading pass handles a different
number of queue entries: the table also gives the shade_queues time per shaded entry (hit and miss entries of bounces 0..7, in
picoseconds of the whole GPU).  The split is per frame: the library times kernel classes, not single bounces.
usage: shade_probe.py [--reps R] [--parent LIB] [--json FILE]"""
import argparse, json, os, statistics, subprocess, sys
HERE = os.path.dirname(os.path.abspath(__file__)); REPO = os.path.dirname(HERE)
CHILD = r'''
import hashlib, json, sys, torch
sys.path.insert(0, %r)
from raytracing_b200 import capi, scene_io
from raytracing_b200.camera import default_camera
check = sys.argv[1] == "1"
w, h, mb = 1920, 1080, 8
out = {}
for name in ("CornellBox", "ShaderBalls"):
    sc = scene_io.load_scene(name)
    ctx = capi.Context(w, h, device=0)
    ctx.set_option(capi.OPT_FRAME_KERNEL, 0)
    ctx.upload_scene(sc); ctx.set_camera(sc["camera_pose"] if "camera_pose" in sc else default_camera(w, h))
    r = {}
    ctx.reset(); ctx.integrate(mb); ctx.sync()
    st = ctx.frame_stats()
    r["entries"] = int(st["n_ext"][:mb].sum())
    if check:
        r["radiance"] = hashlib.sha256(ctx.read_radiance().tobytes()).hexdigest()
        r["stats"] = hashlib.sha256(st.tobytes()).hexdigest()
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
    ctx.set_option(capi.OPT_KERNEL_TIMING, 1); ctx.set_option(capi.OPT_OVERLAP, 0)
    for _ in range(2):
        ctx.reset(); ctx.integrate(mb)
    ctx.sync(); ctx.kernel_times()
    for _ in range(10):
        ctx.reset(); ctx.integrate(mb)
    ctx.sync()
    r["kernels"] = {k: v[0] / 10 for k, v in ctx.kernel_times().items() if v[1]}
    ctx.destroy()
    out[name] = r
print(json.dumps(out))
''' % REPO


def variant(name):
    return name if os.path.sep in name else os.path.join(REPO, "raytracing_b200", "variants", f"librt_b200_{name}.so")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--parent", default="parent")
    ap.add_argument("--json", default=None, help="also write the raw runs to this file")
    args = ap.parse_args()
    arms = [("parent", variant(args.parent)), ("built", os.path.join(REPO, "raytracing_b200", "librt_b200.so")),
            ("mem", variant("shade_mem")), ("math", variant("shade_math"))]
    for name, lib in list(arms):
        if not os.path.exists(lib):
            print(f"no library at {lib}: arm {name} skipped")
            arms.remove((name, lib))
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
        gpu = q.stdout.strip() or q.stderr.strip()
    except OSError as e:
        gpu = repr(e)
    print(f"GPU: {gpu}  (name, power limit, max SM clock, SM clock at idle)")
    runs = {a[0]: [] for a in arms}
    for rep in range(args.reps):
        for name, lib in arms:
            r = subprocess.run([sys.executable, "-c", CHILD, "1" if rep == 0 else "0"], capture_output=True, text=True,
                               env=dict(os.environ, RT_B200_LIB=lib))
            if r.returncode:
                sys.exit(f"{name}: {r.stderr.strip()[-2000:]}")
            runs[name].append(json.loads(r.stdout.strip().splitlines()[-1]))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(runs, f)
    same = True
    exact = [a[0] for a in arms if a[0] in ("parent", "built")]
    for name in exact[1:]:
        for case, r in runs[name][0].items():
            for k in ("radiance", "stats"):
                ok = r[k] == runs[exact[0]][0][case][k]
                same &= ok
                print(f"{case:12s} {name} vs {exact[0]}: {k} {'byte-identical' if ok else 'DIFFERENT'}")
    first = arms[0][0]
    for case in runs[first][0]:
        print(f"{case}, 1920x1080 x 8, per-phase: median of {args.reps} repetitions (ms per frame; shade_queues ms per frame and ps per "
              f"shaded entry; per kernel ms per frame)")
        for name, _ in arms:
            ms = [r[case]["ms"] for r in runs[name]]
            ks = {k: statistics.median(r[case]["kernels"][k] for r in runs[name]) for k in runs[name][0][case]["kernels"]}
            sq, ent = ks.get("shade_queues", float("nan")), runs[name][0][case]["entries"]
            split = "  ".join(f"{k} {v:.3f}" for k, v in sorted(ks.items(), key=lambda kv: -kv[1]) if v >= 0.001)
            print(f"  {name:7s} {statistics.median(ms):.3f}  (runs {' '.join(f'{m:.3f}' for m in ms)})  shade_queues {sq:.3f} ms, "
                  f"{ent} entries, {sq * 1e9 / ent:.1f} ps/entry  |  {split}")
    sys.exit(0 if same else 1)


if __name__ == "__main__":
    main()
