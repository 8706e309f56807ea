"""Issue-slot model (tools/simt_model.cpp): what a CTA-local sort of the one-kernel frame's private ray queue would give.
Rays of bounce b are dealt to CTAs the way k_frame deals pixels (groups of 32 consecutive entries, round-robin over n_cta CTAs);
each CTA's queue is then traced in its own order, or sorted by a small key first."""
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
name = sys.argv[1] if len(sys.argv) > 1 else "CornellBox"
w, h, mb = 960, 540, 4
n_cta = int(sys.argv[2]) if len(sys.argv) > 2 else 132
sc = scene_io.load_scene(name); o = Oracle(sc); cam = default_camera(w, h)
nodes = np.ascontiguousarray(sc["nodes"]); tris = np.ascontiguousarray(sc["triangles"])
costs = np.array([75.0, 24.0, 48.0, 66.0, 78.0, 90.0])
root_min = np.array(nodes[0]["bounds_min"][:3], dtype=np.float64); root_max = np.array(nodes[0]["bounds_max"][:3], dtype=np.float64)
def run(rays):
    out = np.zeros(4)
    assert M.simt_model(nodes.ctypes.data, len(nodes), tris.ctypes.data, len(tris), rays.ctypes.data, len(rays), 0, 0, 1, 32, costs.ctypes.data, out.ctypes.data) == 0
    return out
def interleave(q, bits):
    m = np.zeros(len(q), np.int64)
    for b in range(bits):
        for a in range(3):
            m |= ((q[:, a] >> b) & 1) << (3 * b + a)
    return m
def ocell(org, bits):
    q = np.clip(((org - root_min) / np.maximum(root_max - root_min, 1e-9) * (1 << bits)), 0, (1 << bits) - 1).astype(np.int64)
    return interleave(q, bits)
def dcell(d, bits):
    q = np.clip(((d * 0.5 + 0.5) * (1 << bits)), 0, (1 << bits) - 1).astype(np.int64)
    return interleave(q, bits)
def octant(d): return (d[:, 0] < 0).astype(np.int64) | ((d[:, 1] < 0).astype(np.int64) << 1) | ((d[:, 2] < 0).astype(np.int64) << 2)
for bounce in (1, 2, 3):
    rays = np.zeros(w * h, dtype=RAY_DT); work = np.zeros((w * h, 2), np.uint32); cnt = C.c_uint32(0)
    o.lib.orc_set_dump(bounce, rays.ctypes.data_as(C.c_void_p), work.ctypes.data_as(C.c_void_p), C.byref(cnt))
    o.render(cam, w, h, mb, want_hits=False)
    o.lib.orc_set_dump(-1, None, None, None)
    n = cnt.value
    r = np.ascontiguousarray(rays[:n])
    grp = np.arange(n) // 32
    cta = grp % n_cta
    order_cta = np.argsort(cta, kind="stable")             # each CTA's queue, in its own (pixel) order
    r_cta = np.ascontiguousarray(r[order_cta]); cta_sorted = cta[order_cta]
    org = r_cta["origin"][:, :3].astype(np.float64); d = r_cta["direction"][:, :3].astype(np.float64)
    base_global = run(r)
    base = run(r_cta)
    line = f"{name} bounce {bounce}: {n} rays, {n // n_cta} per CTA; global queue order {base_global[0] / n:.1f} slots/ray ({base_global[1] / base_global[0]:.1f} lanes); CTA-private order {base[0] / n:.1f} ({base[1] / base[0]:.1f} lanes)"
    print(line)
    keys = {"octant": octant(d), "dir2": dcell(d, 2), "dir3": dcell(d, 3), "org1+dir2": ocell(org, 1) * 64 + dcell(d, 2),
            "org2+dir2": ocell(org, 2) * 64 + dcell(d, 2), "org2+dir3": ocell(org, 2) * 512 + dcell(d, 3), "dir3+org2": dcell(d, 3) * 64 + ocell(org, 2),
            "org3+dir3": ocell(org, 3) * 512 + dcell(d, 3)}
    res = []
    for label, key in keys.items():
        order = np.lexsort((key, cta_sorted))              # sort by key within each CTA
        out = run(np.ascontiguousarray(r_cta[order]))
        res.append(f"{label} {base[0] / out[0]:.2f}x ({out[1] / out[0]:.1f} lanes)")
    print("   sorted within the CTA: " + "  ".join(res))
