"""
Extension-ray queue bytes per frame, pass by pass: the layout before the pixel moved from plane A to plane B (every primary ray
written whole by k_raygen, every shaded entry reading planes A, B and C) against the current one (primary rays generated in the
bounce-0 traversal, which stores plane B only; the shading pass reads B, and C after bounce 0, and A only for the depth AOV at
bounce 0 or the emitter MIS term after it).  A byte model from the per-bounce counters, not a measurement: queue planes are 16 B
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


def passes(mb, s, fused, aov=False, emit=False):
    """Bytes per pass of one frame: (pass name, bytes read, bytes written)."""
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
        written = 3 * PLANE * (int(s["n_shadow"][b]) + int(s["n_cont"][b]))
        out.append(("shade %d" % b, (HITQ + hit_planes * PLANE) * hit + (MISSQ + miss_planes * PLANE) * miss, written))
        sh = int(s["n_shadow"][b])
        out.append(("shadow %d" % b, 2 * PLANE * sh + PLANE * int(s["n_unoccluded"][b]), 0))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--scenes", nargs="+", default=["CornellBox", "ShaderBalls"])
    ap.add_argument("--device", action="store_true", help="counters of one rt_integrate frame on cuda:0 instead of the oracle's")
    ap.add_argument("--per-pass", action="store_true", help="print every pass, not only the totals by kind")
    args = ap.parse_args()
    for name in args.scenes:
        mb, s = counters(name, args.device)
        old, new = passes(mb, s, False), passes(mb, s, True)
        print("%s (max_bounces %d, %s counters): extension rays per bounce %s" % (name, mb, "device" if args.device else "oracle",
                                                                               s["n_ext"].tolist()))
        print("  %-10s %14s %14s %14s" % ("pass", "before MB", "now MB", "saved MB"))
        kinds = {}
        for (p, r0, w0), (_, r1, w1) in zip([x for x in old if x[0] != "raygen"], new):
            k = p.split()[0] if not p.endswith(" 0") else p
            a = kinds.setdefault(k, [0, 0])
            a[0] += r0 + w0; a[1] += r1 + w1
            if args.per_pass:
                print("  %-10s %14.1f %14.1f %14.1f" % (p, (r0 + w0) / 1e6, (r1 + w1) / 1e6, (r0 + w0 - r1 - w1) / 1e6))
        rg = sum(r + w for p, r, w in old if p == "raygen")
        print("  %-10s %14.1f %14.1f %14.1f" % ("raygen", rg / 1e6, 0.0, rg / 1e6))
        for k, (a, b) in kinds.items():
            print("  %-10s %14.1f %14.1f %14.1f" % (k, a / 1e6, b / 1e6, (a - b) / 1e6))
        to = sum(r + w for _, r, w in old); tn = sum(r + w for _, r, w in new)
        print("  %-10s %14.1f %14.1f %14.1f  (%.1f %% of the queue bytes)" % ("frame", to / 1e6, tn / 1e6, (to - tn) / 1e6,
                                                                               100.0 * (to - tn) / to))


if __name__ == "__main__":
    main()
