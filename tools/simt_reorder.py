"""Issue-slot model (tools/simt_model.cpp): effect of CTA-local re-ordering of the ray queue (blocks of B rays sorted by a small key).
usage: simt_reorder.py [scene [width height max_bounces [bounces [blocks]]]]   (bounces and blocks comma-separated; block 0 = the whole queue)"""
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
w, h, mb = (int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4])) if len(sys.argv) > 4 else (960, 540, 3)
bounces = [int(b) for b in sys.argv[5].split(",")] if len(sys.argv) > 5 else [1, 2]
blocks = [int(b) for b in sys.argv[6].split(",")] if len(sys.argv) > 6 else [1024, 2048, 4096, 16384, 0]     # 0 = the whole queue
sc = scene_io.load_scene(name); o = Oracle(sc); cam = default_camera(w, h)
nodes = np.ascontiguousarray(sc["nodes"]); tris = np.ascontiguousarray(sc["triangles"])
costs = np.array([75.0, 24.0, 48.0, 66.0, 78.0, 90.0])
root_min = np.array(nodes[0]["bounds_min"][:3], dtype=np.float64); root_max = np.array(nodes[0]["bounds_max"][:3], dtype=np.float64)
def run(rays, any_hit=0, schedule=0, K=1, per=32):
    out = np.zeros(4)
    assert M.simt_model(nodes.ctypes.data, len(nodes), tris.ctypes.data, len(tris), rays.ctypes.data, len(rays), any_hit, schedule, K, per, costs.ctypes.data, out.ctypes.data) == 0
    return out
def octant(d): return (d[:, 0] < 0).astype(np.int64) | ((d[:, 1] < 0).astype(np.int64) << 1) | ((d[:, 2] < 0).astype(np.int64) << 2)
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
def blocked(key, B):
    n = len(key); order = np.arange(n)
    for s in range(0, n, B):
        e = min(n, s + B); order[s:e] = s + np.argsort(key[s:e], kind="stable")
    return order
for bounce in bounces:
    rays = np.zeros(w * h, dtype=RAY_DT); work = np.zeros((w * h, 2), np.uint32); cnt = C.c_uint32(0)
    o.lib.orc_set_dump(bounce, rays.ctypes.data_as(C.c_void_p), work.ctypes.data_as(C.c_void_p), C.byref(cnt))
    o.render(cam, w, h, mb, want_hits=False)
    o.lib.orc_set_dump(-1, None, None, None)
    n = cnt.value
    r = np.ascontiguousarray(rays[:n])
    org = r["origin"][:, :3].astype(np.float64); d = r["direction"][:, :3].astype(np.float64)
    base = run(r)
    print(f"{name} bounce {bounce}: {n} rays, queue order {base[0] / n:.1f} slots/ray, {base[1] / base[0]:.1f} lanes")
    keys = {"octant": octant(d), "dir2": dcell(d, 2), "dir3": dcell(d, 3),
            "oct+org1": octant(d) * 8 + ocell(org, 1), "oct+org2": octant(d) * 64 + ocell(org, 2),
            "org2+oct": ocell(org, 2) * 8 + octant(d), "org2+dir2": ocell(org, 2) * 64 + dcell(d, 2), "dir2+org2": dcell(d, 2) * 64 + ocell(org, 2),
            "org3+dir3": ocell(org, 3) * 512 + dcell(d, 3), "dir3+org3": dcell(d, 3) * 512 + ocell(org, 3), "org2+dir3": ocell(org, 2) * 512 + dcell(d, 3)}
    for B in [b or n for b in blocks]:
        line = f"   block {B if B != n else 'all':>6}: "
        for label, key in keys.items():
            out = run(np.ascontiguousarray(r[blocked(key, B)]))
            line += f"{label} {base[0] / out[0]:.2f}x  "
        print(line)
