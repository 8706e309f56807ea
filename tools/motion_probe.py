"""
What object motion vectors (RT_OPT_OBJECT_MOTION, include/rt_b200.h) buy the temporal denoiser.

  python tools/motion_probe.py [--width 960 --height 540 --bounces 5 --frames 32 --step 0.02 --ref-spp 1024] [--out FILE]

CornellBox_Dragon with the dragon (the largest material group) translating along +x over the floor by --step per frame, the
camera fixed.  Each frame: rt_update_triangles (from the second frame on), rt_set_camera, rt_reset, one sample (rt_integrate),
rt_denoise, rt_copy_history, rt_resolve, as Integrator::Integrate runs the denoiser; once with the option off (camera-only motion
vectors, the reference's) and once with it on.  The displayed last frame is compared with a --ref-spp render of the last frame's
geometry (rt_integrate_samples, denoiser off): RMSE of the resolved RGB over the pixels whose primary ray hits the dragon in the
reference and over the whole image, both over the pixels where both images are finite (the count of the others is reported).  Prints one JSON line per arm, headed by the GPU's name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from raytracing_b200 import capi, scene_io  # noqa: E402
from raytracing_b200.camera import default_camera  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def moved(tris, mesh, dx):
    t = tris.copy()
    for v in ("v1", "v2", "v3"):
        t[v]["position"][mesh, 0] += np.float32(dx)
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--width", type=int, default=960)
    ap.add_argument("--height", type=int, default=540)
    ap.add_argument("--bounces", type=int, default=5)
    ap.add_argument("--frames", type=int, default=32)
    ap.add_argument("--step", type=float, default=0.02)
    ap.add_argument("--ref-spp", type=int, default=1024)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    w, h, mb = a.width, a.height, a.bounces

    def emit(r):
        print(json.dumps(r), flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(json.dumps(r) + "\n")

    emit({"gpu": gpu_info()})
    sc = scene_io.load_scene("CornellBox_Dragon")
    cam = default_camera(w, h)
    ids, counts = np.unique(sc["triangles"]["mtlIndex"], return_counts=True)
    mesh = sc["triangles"]["mtlIndex"] == ids[counts.argmax()]
    frames = [moved(sc["triangles"], mesh, a.step * f) for f in range(a.frames)]

    ref = capi.Context(w, h)
    ref.upload_scene(sc); ref.set_camera(cam)
    ref.update_triangles(frames[-1])
    ref.generate_rays(); ref.intersect(0)
    hits, pix = ref.read_hits(0)
    on_mesh = np.zeros(w * h, bool)
    prim = hits["primitive_id"]
    hit = prim < len(mesh)
    on_mesh[pix[hit]] = mesh[prim[hit]]
    on_mesh = on_mesh.reshape(h, w)
    ref.reset(); ref.integrate_samples(mb, a.ref_spp)
    want = ref.resolve()[..., :3].astype(np.float64)
    ref.destroy()

    for motion in (0, 1):
        c = capi.Context(w, h)
        c.upload_scene(sc)
        c.set_option(capi.OPT_DENOISER, 1); c.set_option(capi.OPT_OBJECT_MOTION, motion)
        for f, t in enumerate(frames):
            if f:
                c.update_triangles(t)
            c.set_camera(cam); c.reset(); c.integrate(mb); c.denoise(); c.copy_history()
            img = c.resolve()
        c.destroy()
        err = ((img[..., :3].astype(np.float64) - want) ** 2).mean(axis=-1)
        ok = np.isfinite(err)
        emit({"object_motion": motion, "width": w, "height": h, "bounces": mb, "frames": a.frames, "step": a.step,
              "ref_spp": a.ref_spp, "mesh_pixels": int((on_mesh & ok).sum()), "non_finite_pixels": int((~ok).sum()),
              "rmse_mesh": float(np.sqrt(err[on_mesh & ok].mean())), "rmse_image": float(np.sqrt(err[ok].mean()))})


if __name__ == "__main__":
    main()
