"""
Ray queue bytes per frame, pass by pass, for three layouts:
  - "raygen": before the pixel moved from plane A to plane B (every primary ray written whole by k_raygen, every shaded entry
    reading planes A, B and C, every shadow ray three planes);
  - "3-plane": primary rays generated in the bounce-0 traversal, which stores plane B only; the shading pass reads B, and C after
    bounce 0, and A only for the depth AOV at bounce 0 or the emitter MIS term after it; shadow rays still three planes;
  - "now": as "3-plane", but a shadow ray toward a directional light stores planes sA and sC only, and the shadow pass reads sA
    (and sC for an unoccluded ray), taking direction and t_max from the light's record.  Every light of the shipped scenes is
    directional, so the model counts every shadow ray as two-plane.
A byte model from the per-bounce counters, not a measurement: queue planes are 16 B
float4s, hit-queue entries 16 B, miss-queue entries 4 B; BVH, material and radiance traffic is left out (the same in both).

    python tools/stream_bytes.py                          # the oracle's counters on the CPU (CornellBox, ShaderBalls)
    python tools/stream_bytes.py --device --scenes CornellBox ShaderBalls CornellBox_Dragon Synthetic10M
                                                          # one frame's counters from the device (rt_read_frame_stats)
"""
import argparse
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

PLANE, HITQ, MISSQ = 16, 16, 4


def counters(name, device):
    """-> (max_bounces, dict of per-bounce arrays n_ext, n_miss, n_shadow, n_cont, n_unoccluded) for the bench workload `name`."""
    import bench
    sname, w, h, mb = bench.WORKLOADS[name]
    sc, cam = bench.load_workload_scene(name, w, h)
    if device:
        from raytracing_b200 import capi
        c = capi.Context(w, h)
        c.upload_scene(sc); c.set_camera(cam); c.reset(); c.integrate(mb)
        st = c.frame_stats()
        c.destroy()
    else:
        from oracle.orcbind import Oracle
        _, _, st = Oracle(sc).render(cam, w, h, mb, want_hits=False)
    return mb, {k: np.asarray(st[k][: mb + 1], dtype=np.int64) for k in ("n_ext", "n_miss", "n_shadow", "n_cont", "n_unoccluded")}


def passes(mb, s, fused, aov=False, emit=False, two_plane=False):
    """Bytes per pass of one frame: (pass name, bytes read, bytes written)."""
    shadow_planes = 2 if two_plane else 3
    out = []
    n0 = int(s["n_ext"][0])
    if not fused:
        out.append(("raygen", 0, 3 * PLANE * n0))
    for b in range(mb + 1):
        n, miss = int(s["n_ext"][b]), int(s["n_miss"][b])
        hit = n - miss
        if fused and b == 0:          # generated in registers; B stored for the shading pass (A as well with AOVs)
            out.append(("trace %d" % b, 0, (2 if aov else 1) * PLANE * n + HITQ * hit + MISSQ * miss))
        else:
            out.append(("trace %d" % b, 2 * PLANE * n, HITQ * hit + MISSQ * miss))
        if fused:
            hit_planes = (1 + (1 if aov else 0)) if b == 0 else (2 + (1 if emit else 0))
            miss_planes = 1 if b == 0 else 2
        else:
            hit_planes = miss_planes = 3
        written = shadow_planes * PLANE * int(s["n_shadow"][b]) + 3 * PLANE * int(s["n_cont"][b])
        out.append(("shade %d" % b, (HITQ + hit_planes * PLANE) * hit + (MISSQ + miss_planes * PLANE) * miss, written))
        sh = int(s["n_shadow"][b])
        out.append(("shadow %d" % b, (shadow_planes - 1) * PLANE * sh + PLANE * int(s["n_unoccluded"][b]), 0))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--scenes", nargs="+", default=["CornellBox", "ShaderBalls"])
    ap.add_argument("--device", action="store_true", help="counters of one rt_integrate frame on cuda:0 instead of the oracle's")
    ap.add_argument("--per-pass", action="store_true", help="print every pass, not only the totals by kind")
    args = ap.parse_args()
    for name in args.scenes:
        mb, s = counters(name, args.device)
        arms = (("raygen", passes(mb, s, False)), ("3-plane", passes(mb, s, True)), ("now", passes(mb, s, True, two_plane=True)))
        print("%s (max_bounces %d, %s counters): extension rays per bounce %s, shadow rays %d (%d unoccluded)"
              % (name, mb, "device" if args.device else "oracle", s["n_ext"].tolist(), int(s["n_shadow"].sum()), int(s["n_unoccluded"].sum())))
        print("  %-10s" % "pass" + "".join("%14s" % (a + " MB") for a, _ in arms))
        kinds, order = {}, []
        for rows in zip(*[[x for x in ps if x[0] != "raygen"] for _, ps in arms]):
            p = rows[0][0]
            k = p.split()[0] if not p.endswith(" 0") else p
            if k not in kinds: kinds[k] = [0] * len(arms); order.append(k)
            for j, (_, r, w) in enumerate(rows):
                kinds[k][j] += r + w
            if args.per_pass:
                print("  %-10s" % p + "".join("%14.1f" % ((r + w) / 1e6) for _, r, w in rows))
        rg = sum(r + w for p, r, w in arms[0][1] if p == "raygen")
        print("  %-10s" % "raygen" + "%14.1f" % (rg / 1e6) + "%14.1f" % 0.0 * (len(arms) - 1))
        for k in order:
            print("  %-10s" % k + "".join("%14.1f" % (v / 1e6) for v in kinds[k]))
        tot = [sum(r + w for _, r, w in ps) for _, ps in arms]
        print("  %-10s" % "frame" + "".join("%14.1f" % (t / 1e6) for t in tot)
              + "   (now saves %.1f MB = %.1f %% of the 3-plane layout's queue bytes)" % ((tot[1] - tot[2]) / 1e6, 100.0 * (tot[1] - tot[2]) / tot[1]))

if __name__ == "__main__":
    main()
