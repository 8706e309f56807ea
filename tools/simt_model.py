"""Issue-slot model of the traversal kernels' warp schedules (analysis only, CPU; see tools/simt_model.cpp).
usage: python tools/simt_model.py [scene] [width height max_bounces]
       python tools/simt_model.py shadow [scene] [width height max_bounces]   the SMEM 3 any-hit loop near to far, far to near and with postponed leaves"""
import ctypes as C, os, subprocess, sys, tempfile
import numpy as np
HERE = os.path.dirname(os.path.abspath(__file__)); REPO = os.path.dirname(HERE)
sys.path.insert(0, REPO)
from oracle.orcbind import Oracle
from raytracing_b200 import scene_io
from raytracing_b200.camera import default_camera
from raytracing_b200.layouts import RAY_DT

lib_path = os.path.join(tempfile.gettempdir(), "libsimt_model.so")
subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-fopenmp", "-ffp-contract=off", "-I" + os.path.join(REPO, "include"),
                "-shared", "-o", lib_path, os.path.join(HERE, "simt_model.cpp")], check=True)
M = C.CDLL(lib_path)
M.simt_model.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_uint32, C.c_void_p, C.c_void_p]
M.simt_any_model.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int, C.c_int, C.c_void_p, C.c_void_p]


def shadow_rays(sc, rays, hits, seed=0):
    """The shadow rays the shading pass makes at these hits (oracle.cpp, direct lighting), as (n, 7) float32 rows of origin,
    direction, t_max: origin = position + shading normal * RT_EPS, towards the light (a directional light: origin *
    RT_MAX_RENDER_DIST), t_max = that distance.  The light is chosen by a uniform draw (the scenes here have one); a ray is kept
    when the light is above the shading normal."""
    hit = hits["primitive_id"] != 0xFFFFFFFF
    t = sc["triangles"][hits["primitive_id"][hit]]
    u = hits["bc"][hit, 0:1].astype(np.float32); v = hits["bc"][hit, 1:2].astype(np.float32)
    def interp(f):
        return t["v1"][f][:, :3] * (1.0 - u - v) + t["v2"][f][:, :3] * u + t["v3"][f][:, :3] * v
    pos = interp("position"); nrm = interp("normal"); nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    lights = sc["lights"]; pick = np.random.default_rng(seed).integers(0, len(lights), len(pos))
    lo = lights["origin"][pick, :3]
    point = (lights["type"][pick] == 0)[:, None]
    out = np.where(point, lo - pos, lo * np.float32(20000.0)).astype(np.float32)
    dist = np.linalg.norm(out, axis=1); d = out / dist[:, None]
    keep = (d * nrm).sum(1) > 0.0
    r = np.zeros((int(keep.sum()), 7), np.float32)
    r[:, 0:3] = (pos + nrm * np.float32(1e-3))[keep]; r[:, 3:6] = d[keep]; r[:, 6] = dist[keep]
    return np.ascontiguousarray(r)


def shadow_main(argv):
    from tests.test_wide_octant_cpu import layout, tables
    so = os.path.join(tempfile.gettempdir(), "libsimt_wide_octant.so")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-I" + os.path.join(REPO, "include"),
                    "-I" + os.path.join(REPO, "raytracing_b200", "csrc"), "-o", so, os.path.join(REPO, "tests", "wide_octant_host.cpp"),
                    os.path.join(REPO, "tests", "bvh_layout_host.cpp")], check=True)
    L = C.CDLL(so)
    L.wide_tables.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32)]
    L.bvh_layout_build.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int),
                                   C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.c_char_p, C.c_int]
    name = argv[0] if argv else "CornellBox"
    w, h, mb = (int(argv[1]), int(argv[2]), int(argv[3])) if len(argv) > 3 else (1920, 1080, 8)
    sc = scene_io.load_scene(name); orc = Oracle(sc); cam = default_camera(w, h)
    recs, wt, root, nodes = layout(L, sc)
    ok, _, tab, _ = tables(L, recs)
    assert ok == 1
    root_box = np.concatenate([nodes["bounds_min"][0, :3], nodes["bounds_max"][0, :3]]).astype("<f4")
    # issue slots: wide step (2..4 ordered slab tests + push/pop), triangle stages as for the binary loop, fetch + setup +
    # accumulate, and the postponing overhead per interior step (the postpone test and the warp vote)
    wide_steps = (70.0, 100.0, 130.0)
    variants = [("near to far", 0, 0), ("postponed, all lanes", 1, 0), ("postponed, >= 24 lanes", 1, 24),
                ("postponed, >= 16 lanes", 1, 16), ("postponed, >= 8 lanes", 1, 8), ("postponed, no vote", 1, -1), ("far child first", 2, 0)]
    total = {v[0]: np.zeros(len(wide_steps)) for v in variants}
    print(f"{name} {w}x{h}, bounces 0..{mb}: shadow rays of each bounce on the SMEM 3 any-hit loop")
    print(f"   {'bounce':>6s} {'rays':>8s} {'unocc':>6s} {'variant':24s} {'lanes':>6s} " + " ".join(f"{'x@' + str(int(s)):>7s}" for s in wide_steps))
    for bounce in range(0, mb + 1):
        rays = np.zeros(w * h, dtype=RAY_DT); work = np.zeros((w * h, 2), np.uint32); cnt = C.c_uint32(0)
        orc.lib.orc_set_dump(bounce, rays.ctypes.data_as(C.c_void_p), work.ctypes.data_as(C.c_void_p), C.byref(cnt))
        orc.render(cam, w, h, mb, want_hits=False)
        orc.lib.orc_set_dump(-1, None, None, None)
        if cnt.value == 0:
            continue
        ext = np.ascontiguousarray(rays[:cnt.value])
        hits, _ = orc.trace(ext)
        sr = shadow_rays(sc, ext, hits)
        if len(sr) == 0:
            continue
        res = {}
        for label, var, trig in variants:
            row = []
            for ws in wide_steps:
                costs = np.array([ws, 24.0, 48.0, 66.0, 78.0, 90.0, 6.0]); out = np.zeros(3)
                assert M.simt_any_model(tab.ctypes.data, len(recs), wt.ctypes.data, root, root_box.ctypes.data, sr.ctypes.data, len(sr),
                                        var, trig, costs.ctypes.data, out.ctypes.data) == 0
                row.append(out.copy())
            res[label] = row
        unocc = res["near to far"][0][2]
        for label, var, trig in variants:
            assert res[label][0][2] == unocc                # the same rays reach the end unoccluded
            lanes = res[label][1][1] / res[label][1][0]
            sp = [res["near to far"][k][0] / res[label][k][0] for k in range(len(wide_steps))]
            total[label] += [res[label][k][0] for k in range(len(wide_steps))]
            print(f"   {bounce:6d} {len(sr):8d} {unocc / len(sr):6.2f} {label:24s} {lanes:6.1f} " + " ".join(f"{s:6.3f}x" for s in sp))
    print("   all bounces:")
    for label, _, _ in variants:
        print(f"   {'':6s} {'':8s} {'':6s} {label:24s} {'':6s} " + " ".join(f"{total['near to far'][k] / total[label][k]:6.3f}x" for k in range(len(wide_steps))))


if len(sys.argv) > 1 and sys.argv[1] == "shadow":
    shadow_main(sys.argv[2:])
    sys.exit(0)

name = sys.argv[1] if len(sys.argv) > 1 else "CornellBox"
w, h, mb = (int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4])) if len(sys.argv) > 4 else (960, 540, 3)
sc = scene_io.load_scene(name); o = Oracle(sc); cam = default_camera(w, h)
nodes = np.ascontiguousarray(sc["nodes"]); tris = np.ascontiguousarray(sc["triangles"])
# issue slots: interior record step, triangle test by exit stage (det / u / v / full), ray fetch + setup + result write
costs = np.array([75.0, 24.0, 48.0, 66.0, 78.0, 90.0])

def run(rays, any_hit, schedule, K, per):
    out = np.zeros(4)
    rc = M.simt_model(nodes.ctypes.data, len(nodes), tris.ctypes.data, len(tris), rays.ctypes.data, len(rays), any_hit, schedule, K, per,
                      costs.ctypes.data, out.ctypes.data)
    assert rc == 0
    return out

for bounce in range(0, mb + 1):
    rays = np.zeros(w * h, dtype=RAY_DT); work = np.zeros((w * h, 2), np.uint32); cnt = C.c_uint32(0)
    o.lib.orc_set_dump(bounce, rays.ctypes.data_as(C.c_void_p), work.ctypes.data_as(C.c_void_p), C.byref(cnt))
    o.render(cam, w, h, mb, want_hits=False)
    o.lib.orc_set_dump(-1, None, None, None)
    n = cnt.value
    if n == 0:
        continue
    r = np.ascontiguousarray(rays[:n])
    base = run(r, 0, 0, 1, 32)
    print(f"{name} bounce {bounce}: {n} rays, {base[2] / n:.1f} record steps + {base[3] / n:.1f} triangle tests per ray")
    print(f"   {'schedule':34s} {'slots/ray':>10s} {'lanes':>6s} {'speed-up':>8s}")
    rows = [("1 ray / lane, batch of 32 (round 1)", 0, 1, 32)]
    for K in (2, 4, 8, 16):
        rows.append((f"{K} rays / lane, static", 1, K, 32 * K))
    rows.append(("ideal dynamic refill", 2, 1, 32 * 256))
    for label, sch, K, per in rows:
        out = run(r, 0, sch, K, per)
        print(f"   {label:34s} {out[0] / n:10.1f} {out[1] / out[0]:6.1f} {base[0] / out[0]:8.2f}x")

# ---- effect of re-ordering the bounce's ray queue on the round-1 schedule (phase coherence, not only length variance)
def octant(d): return (d[:, 0] < 0).astype(np.int64) | ((d[:, 1] < 0).astype(np.int64) << 1) | ((d[:, 2] < 0).astype(np.int64) << 2)
def morton_cells(org, bits):
    mn, mx = org.min(0), org.max(0)
    cell = np.clip(((org - mn) / np.maximum(mx - mn, 1e-9) * (1 << bits)).astype(np.int64), 0, (1 << bits) - 1)
    m = np.zeros(len(org), np.int64)
    for b in range(bits):
        for a in range(3):
            m |= ((cell[:, a] >> b) & 1) << (3 * b + a)
    return m
def dir_cells(d, bits):
    # octahedral-ish: quantised direction
    q = np.clip(((d * 0.5 + 0.5) * (1 << bits)).astype(np.int64), 0, (1 << bits) - 1)
    m = np.zeros(len(d), np.int64)
    for b in range(bits):
        for a in range(3):
            m |= ((q[:, a] >> b) & 1) << (3 * b + a)
    return m

print("\nre-ordering (schedule: 1 ray / lane, batch of 32)")
for bounce in (1, 2):
    rays = np.zeros(w * h, dtype=RAY_DT); work = np.zeros((w * h, 2), np.uint32); cnt = C.c_uint32(0)
    o.lib.orc_set_dump(bounce, rays.ctypes.data_as(C.c_void_p), work.ctypes.data_as(C.c_void_p), C.byref(cnt))
    o.render(cam, w, h, mb, want_hits=False)
    o.lib.orc_set_dump(-1, None, None, None)
    n = cnt.value
    r = np.ascontiguousarray(rays[:n])
    org = r["origin"][:, :3].astype(np.float64); d = r["direction"][:, :3].astype(np.float64)
    base = run(r, 0, 0, 1, 32)
    oc = octant(d)
    orders = {"queue order": np.arange(n),
              "octant (8 sub-queues, stable)": np.argsort(oc, kind="stable"),
              "octant + origin cell 4b": np.argsort(oc * (1 << 12) + morton_cells(org, 4), kind="stable"),
              "origin cell 4b + octant": np.argsort(morton_cells(org, 4) * 8 + oc, kind="stable"),
              "origin cell 3b + dir cell 3b": np.argsort(morton_cells(org, 3) * 512 + dir_cells(d, 3), kind="stable"),
              "dir cell 3b + origin cell 3b": np.argsort(dir_cells(d, 3) * 512 + morton_cells(org, 3), kind="stable"),
              "dir cell 4b + origin cell 4b": np.argsort(dir_cells(d, 4) * 4096 + morton_cells(org, 4), kind="stable"),
              "random": np.random.default_rng(1).permutation(n)}
    print(f"{name} bounce {bounce}")
    for label, order in orders.items():
        rr = np.ascontiguousarray(r[order])
        out = run(rr, 0, 0, 1, 32)
        print(f"   {label:34s} {out[0] / n:10.1f} {out[1] / out[0]:6.1f} {base[0] / out[0]:8.2f}x")
