"""
Instanced against flattened Synthetic10M (C5): replicate()'s 183 rotated ShaderBalls copies and the ground quad, once as 10 M
flattened triangles under the host SAH tree (bench.py's secondary workload) and once as two meshes and 184 instances
(synthetic.instanced_field, rt_upload_instanced_scene / rt_set_instances).

  python tools/instance_probe.py [--width 1920 --height 1080 --bounces 8 --frames 20 --warmup 5] [--out FILE]

Per arm: ms per frame (rt_reset + rt_integrate) from CUDA events on the render stream after --warmup frames, the device memory the
scene holds (free memory before the context's upload minus after it, cudaMemGetInfo), and for the instanced arm the cost of one
rt_set_instances with the 184 instances (host clock around 50 calls, each followed by rt_sync, warm buffer).  Prints one JSON line
per arm, headed by the GPU's name and power limit read in the same run.  Frames of the two arms are not equal: the instanced matrices
round differently from the flattened vertices (tests/test_instancing_cpu.py bounds the difference).

  python tools/instance_probe.py --mesh-update [--width ... --frames ... --warmup ... --calls 20] [--out FILE]

Mesh updates in the instanced field (rt_update_mesh_triangles*) instead: the time of one update of the ShaderBalls mesh (54 790
triangles, under 183 instances) by the host variant (a TRIANGLE_DT array) and by the device variant (a CUDA uint8 tensor), host
clock around --calls calls, each returning after its blocking root-box read-back and followed by rt_sync; the time of a 32-byte
device-to-host copy with its synchronise, the read-back's floor; and ms per frame after a deforming update (refit tree) against a
fresh context that uploaded the same triangles and refit nodes (tests/refit_model.py) with the same instance list.

  python tools/instance_probe.py --materials [--width ... --frames ... --warmup ... --repeats 5] [--out FILE]

Per-instance materials in the instanced field (rt_set_instance_materials) instead, three arms on one context, alternated --repeats
times: no assignment; every instance with its own row (a seeded permutation of the scene's materials); every instance with the
identity row.  ms per frame of each repeat from CUDA events; the identity arm's radiance is checked to equal the first arm's bits.
With RT_B200_LIB naming a library built from a commit before rt_set_instance_materials, only the first arm runs (the parent's
frame time on the same scene).
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from raytracing_b200 import capi, scene_io, synthetic  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed_frames(c, bounces, frames, warmup):
    import torch
    for _ in range(warmup):
        c.reset(); c.integrate(bounces)
    c.sync()
    stream = torch.cuda.ExternalStream(c.stream_handle())
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    for _ in range(frames):
        c.reset(); c.integrate(bounces)
    b.record(stream)
    b.synchronize()
    return a.elapsed_time(b) / frames


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--bounces", type=int, default=8)
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--copies", type=int, default=183)
    ap.add_argument("--out", default=None)
    ap.add_argument("--mesh-update", action="store_true")
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--materials", action="store_true")
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    import torch
    torch.cuda.init()
    base = scene_io.load_scene("ShaderBalls")
    lines = [{"gpu": gpu_info()}]
    if args.mesh_update:
        lines += mesh_update(args, base)
        emit(lines, args.out)
        return
    if args.materials:
        lines += instance_materials(args, base)
        emit(lines, args.out)
        return

    def free():
        torch.cuda.synchronize()
        return torch.cuda.mem_get_info()[0]

    fld = synthetic.instanced_field(base, copies=args.copies, width=args.width, height=args.height)
    cam = fld["camera_pose"]
    c = capi.Context(args.width, args.height)
    c.set_camera(cam)
    f0 = free()
    c.upload_instanced_scene(fld["meshes"], fld["shared"])
    c.set_instances(fld["mesh_ids"], fld["transforms"])
    c.sync()
    mem = f0 - free()
    ms = timed_frames(c, args.bounces, args.frames, args.warmup)
    t = time.perf_counter()
    for _ in range(50):
        c.set_instances(fld["mesh_ids"], fld["transforms"]); c.sync()
    set_ms = (time.perf_counter() - t) * 1e3 / 50
    c.destroy()
    lines.append({"arm": "instanced", "instances": len(fld["mesh_ids"]), "mesh_triangles": [len(m["triangles"]) for m in fld["meshes"]],
                  "ms_per_frame": ms, "scene_device_bytes": int(mem), "set_instances_ms": set_ms,
                  "frame": f"{args.width}x{args.height}x{args.bounces}"})

    flat = synthetic.bistro_scale_scene(base, copies=args.copies, width=args.width, height=args.height)
    c = capi.Context(args.width, args.height)
    c.set_camera(cam)
    f0 = free()
    c.upload_scene(flat)
    c.sync()
    mem = f0 - free()
    ms = timed_frames(c, args.bounces, args.frames, args.warmup)
    c.destroy()
    lines.append({"arm": "flattened", "triangles": len(flat["triangles"]), "ms_per_frame": ms, "scene_device_bytes": int(mem),
                  "frame": f"{args.width}x{args.height}x{args.bounces}"})
    emit(lines, args.out)


def emit(lines, out):
    text = "\n".join(json.dumps(x) for x in lines)
    print(text)
    if out:
        with open(out, "w") as f:
            f.write(text + "\n")


def mesh_update(args, base):
    import torch
    from tests.refit_model import deform, refit
    fld = synthetic.instanced_field(base, copies=args.copies, width=args.width, height=args.height)
    meshes, ids, mats, cam = fld["meshes"], fld["mesh_ids"], fld["transforms"], fld["camera_pose"]
    t0 = meshes[0]["triangles"]
    shapes = [deform(t0, "noise", seed=s, amount=0.02) for s in range(2)]
    c = capi.Context(args.width, args.height)
    c.set_camera(cam)
    c.upload_instanced_scene(meshes, fld["shared"])
    c.set_instances(ids, mats)
    out = []
    for variant in ("host", "device"):
        src = shapes if variant == "host" else [torch.from_numpy(x.view(np.uint8).reshape(len(x), 160).copy()).cuda() for x in shapes]
        for k in range(3):
            c.update_mesh_triangles(0, src[k % 2])
        c.sync()
        t = time.perf_counter()
        for k in range(args.calls):
            c.update_mesh_triangles(0, src[k % 2]); c.sync()
        out.append({"update": variant, "mesh_triangles": len(t0), "instances": len(ids),
                    "ms_per_update": (time.perf_counter() - t) * 1e3 / args.calls})
    x = torch.zeros(8, device="cuda")
    y = torch.empty(8, pin_memory=False)
    for _ in range(10):
        y.copy_(x); torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(200):
        y.copy_(x); torch.cuda.synchronize()
    out.append({"readback_32B_ms": (time.perf_counter() - t) * 1e3 / 200})
    c.update_mesh_triangles(0, shapes[1])
    upd = timed_frames(c, args.bounces, args.frames, args.warmup)
    c.destroy()
    cur = list(meshes)
    cur[0] = {"triangles": shapes[1], "nodes": refit(meshes[0]["nodes"], shapes[1])}
    f = capi.Context(args.width, args.height)
    f.set_camera(cam)
    f.upload_instanced_scene(cur, fld["shared"])
    f.set_instances(ids, mats)
    fresh = timed_frames(f, args.bounces, args.frames, args.warmup)
    f.destroy()
    c = capi.Context(args.width, args.height)                # the updated arm again, after the fresh one: alternation shows drift
    c.set_camera(cam)
    c.upload_instanced_scene(meshes, fld["shared"])
    c.set_instances(ids, mats)
    c.update_mesh_triangles(0, shapes[1])
    upd2 = timed_frames(c, args.bounces, args.frames, args.warmup)
    c.destroy()
    out.append({"frame": f"{args.width}x{args.height}x{args.bounces}", "ms_per_frame_after_update": [upd, upd2],
                "ms_per_frame_fresh_upload": fresh})
    return out


def instance_materials(args, base):
    fld = synthetic.instanced_field(base, copies=args.copies, width=args.width, height=args.height)
    ids, n_mat = fld["mesh_ids"], len(base["materials"])
    rng = np.random.default_rng(7)
    own = np.stack([rng.permutation(n_mat) for _ in ids]).astype(np.uint32)
    arms = {"none": ([], []), "own_rows": (own, list(range(len(ids)))),
            "identity_rows": (np.arange(n_mat, dtype=np.uint32)[None], [0] * len(ids))}
    c = capi.Context(args.width, args.height)
    c.set_camera(fld["camera_pose"])
    c.upload_instanced_scene(fld["meshes"], fld["shared"])
    c.set_instances(ids, fld["transforms"])
    if not hasattr(capi.load_library(), "rt_set_instance_materials"):
        arms = {"none": arms["none"]}
    ms = {k: [] for k in arms}
    image = {}
    for _ in range(args.repeats):
        for arm, (rows, of) in arms.items():
            if len(arms) > 1:
                c.set_instance_materials(rows, of)
            ms[arm].append(timed_frames(c, args.bounces, args.frames, args.warmup))
            image.setdefault(arm, c.read_radiance()[..., :3].view(np.uint32).copy())
    c.destroy()
    out = [{"arm": arm, "instances": len(ids), "materials": n_mat, "ms_per_frame": v, "median": float(np.median(v)),
            "spread": float(max(v) - min(v)), "frame": f"{args.width}x{args.height}x{args.bounces}"} for arm, v in ms.items()]
    if len(arms) > 1:
        out.append({"identity_rows_equal_none": bool(np.array_equal(image["identity_rows"], image["none"])),
                    "own_rows_differ": bool(not np.array_equal(image["own_rows"], image["none"]))})
    out.append({"library": capi.LIB_PATH, "none_radiance_sha1": hashlib.sha1(image["none"].tobytes()).hexdigest()})
    return out


if __name__ == "__main__":
    main()
