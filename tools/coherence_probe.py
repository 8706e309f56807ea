"""Same-box A/B of the sorted continuation-ray writes of k_shade_queues: the per-phase schedule (whole 1080p x 8 frame on one GPU)
of two or more libraries, CornellBox and ShaderBalls.  First checks that every library leaves the same radiance bits and frame
statistics as the first one, then alternates the libraries: median ms per frame over the repetitions (CUDA events, 20 frames
per repetition, best of 3 windows) and the per-kernel split of OPT_KERNEL_TIMING (individual launches, shadow pass on its own).
usage: coherence_probe.py [--reps R] [lib ...]   (lib = path or variant name of tools/build_variant.py; "cur" = the in-tree
library; default: variant "parent" against "cur").  At 1080p the in-tree library runs the unsorted pass; a variant built with
`tools/build_variant.py sorted -DRT_SORT_MIN_PIXELS_PER_SM=0` runs the sorted one at every size."""
import argparse, json, os, statistics, subprocess, sys
HERE = os.path.dirname(os.path.abspath(__file__)); REPO = os.path.dirname(HERE)
CHILD = r'''
import hashlib, json, os, sys, torch
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


def lib_path(spec):
    if os.path.sep in spec:
        return spec
    if spec == "cur":
        return os.path.join(REPO, "raytracing_b200", "librt_b200.so")
    return os.path.join(REPO, "raytracing_b200", "variants", f"librt_b200_{spec}.so")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("libs", nargs="*", default=["parent", "cur"])
    args = ap.parse_args()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                           capture_output=True, text=True)
        gpu = q.stdout.strip() or q.stderr.strip()
    except OSError as e:
        gpu = repr(e)
    print(f"GPU: {gpu}  (name, power limit, max SM clock, SM clock at idle)")
    runs = {spec: [] for spec in args.libs}
    for rep in range(args.reps):
        for spec in args.libs:
            env = dict(os.environ, RT_B200_LIB=lib_path(spec))
            r = subprocess.run([sys.executable, "-c", CHILD, "1" if rep == 0 else "0"], capture_output=True, text=True, env=env)
            if r.returncode:
                sys.exit(f"{spec}: {r.stderr.strip()[-2000:]}")
            runs[spec].append(json.loads(r.stdout.strip().splitlines()[-1]))
    first = args.libs[0]
    same = True
    for spec in args.libs[1:]:
        for scene, r in runs[spec][0].items():
            r0 = runs[first][0][scene]
            for k in ("radiance", "stats"):
                ok = r[k] == r0[k]
                same &= ok
                print(f"{scene:12s} {spec} vs {first}: {k} {'byte-identical' if ok else 'DIFFERENT'}")
    for scene in runs[first][0]:
        print(f"{scene}, 1920x1080 x 8, per-phase schedule: median of {args.reps} (ms per frame; per kernel ms per frame)")
        for spec in args.libs:
            ms = [r[scene]["ms"] for r in runs[spec]]
            ks = {k: statistics.median(r[scene]["kernels"][k] for r in runs[spec]) for k in runs[spec][0][scene]["kernels"]}
            split = "  ".join(f"{k} {v:.3f}" for k, v in sorted(ks.items(), key=lambda kv: -kv[1]) if v >= 0.001)
            print(f"  {spec:10s} {statistics.median(ms):.3f}  (runs {' '.join(f'{m:.3f}' for m in ms)})  {split}")
    sys.exit(0 if same else 1)


if __name__ == "__main__":
    main()
