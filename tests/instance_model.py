"""
The CPU model of instanced scenes (tests/instance_model.cpp: the oracle's frame with the two-level traversal and instanced shading
of include/rt_b200.h), built with g++ -ffp-contract=off into a temporary shared library on first use.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle.orcbind import STATS_DT, Oracle
from oracle.refbind import CAMERA_DT
from raytracing_b200.capi import INSTANCE_DT
from raytracing_b200.layouts import HIT_DT, NODE_DT, RAY_DT, TRIANGLE_DT

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="instance_model_")
        so = os.path.join(d, "libinstance_model.so")
        subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", "-fno-fast-math",
                        "-Wno-unknown-pragmas", "-I" + os.path.join(REPO, "include"), "-I" + os.path.join(REPO, "oracle"),
                        "-I" + os.path.join(REPO, "raytracing_b200", "csrc"), "-o", so, os.path.join(HERE, "instance_model.cpp")], check=True)
        L = C.CDLL(so)
        os.remove(so); os.rmdir(d)
        L.im_render.restype = C.c_int
        L.im_render.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32,
                                C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.im_trace.restype = C.c_int
        L.im_trace.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_int, C.c_void_p,
                               C.c_void_p]
        L.im_trace_mesh.restype = None
        L.im_trace_mesh.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_float, C.c_void_p]
        _lib = L
    return _lib


def instances(mesh_ids, transforms):
    rec = np.zeros(len(mesh_ids), dtype=INSTANCE_DT)
    rec["object_to_world"] = np.ascontiguousarray(transforms, dtype="<f4").reshape(-1, 12)
    rec["mesh"] = np.asarray(mesh_ids, dtype="<u4")
    return rec


class InstanceModel(Oracle):
    """The instanced scene of meshes (dicts with "triangles", "nodes") and shared (materials, lights, environment), as
    Context.upload_instanced_scene takes them."""

    def __init__(self, meshes, shared):
        tris = np.concatenate([np.ascontiguousarray(m["triangles"], dtype=TRIANGLE_DT) for m in meshes])
        nodes = np.concatenate([np.ascontiguousarray(m["nodes"], dtype=NODE_DT) for m in meshes])
        super().__init__(dict(shared, triangles=tris, nodes=nodes, emissive=np.zeros(0, "<u4")))
        self.desc = np.zeros((len(meshes), 4), dtype="<u8")
        t0 = n0 = 0
        for k, m in enumerate(meshes):
            self.desc[k] = (t0, len(m["triangles"]), n0, len(m["nodes"]))
            t0 += len(m["triangles"]); n0 += len(m["nodes"])

    def render_instanced(self, mesh_ids, transforms, cam, width, height, max_bounces, sample_idx=0, prev=None, radiance=None):
        """-> (radiance (h, w, 4) accumulated into `radiance`, primary hits (h*w,) HIT_DT, stats, velocity (h, w, 2) with the camera
        as its own previous camera and `prev` (n, 3, 4) as the previous transforms)."""
        inst = instances(mesh_ids, transforms)
        if radiance is None:
            radiance = np.zeros((height, width, 4), dtype="<f4")
        hits = np.zeros(width * height, dtype=HIT_DT)
        stats = np.zeros((), dtype=STATS_DT)
        vel = np.zeros((height, width, 2), dtype="<f4")
        pv = None if prev is None else np.ascontiguousarray(prev, dtype="<f4").reshape(-1, 12)
        c = np.ascontiguousarray(cam, dtype=CAMERA_DT)
        rc = lib().im_render(C.addressof(self.scene), self.desc.ctypes.data, len(self.desc), inst.ctypes.data if len(inst) else None, len(inst),
                             pv.ctypes.data if pv is not None else None, c.ctypes.data, width, height, max_bounces, sample_idx,
                             radiance.ctypes.data, hits.ctypes.data, stats.ctypes.data, vel.ctypes.data)
        if rc != 0:
            raise ValueError("instance list rejected")
        return radiance, hits, stats, vel

    def trace_instanced(self, mesh_ids, transforms, rays, any_hit=False):
        """The two-level traversal of a batch of rays (RAY_DT; origin.w = t_min, direction.w = t_max) -> closest hits (HIT_DT, virtual
        ids), or for any_hit a uint32 per ray: 0 if occluded, 0xFFFFFFFF if not."""
        inst = instances(mesh_ids, transforms)
        rays = np.ascontiguousarray(rays, dtype=RAY_DT)
        hits = np.zeros(len(rays), dtype=HIT_DT)
        flags = np.zeros(len(rays), dtype="<u4")
        rc = lib().im_trace(C.addressof(self.scene), self.desc.ctypes.data, len(self.desc), inst.ctypes.data if len(inst) else None,
                            len(inst), rays.ctypes.data, len(rays), int(any_hit), hits.ctypes.data, flags.ctypes.data)
        if rc != 0:
            raise ValueError("instance list rejected")
        return flags if any_hit else hits

    def trace_mesh(self, mesh, rays, cull=1.0):
        """Mesh `mesh`'s own tree alone on object-space rays, culling on det * cull -> closest hits (HIT_DT, mesh triangle ids)."""
        rays = np.ascontiguousarray(rays, dtype=RAY_DT)
        hits = np.zeros(len(rays), dtype=HIT_DT)
        lib().im_trace_mesh(C.addressof(self.scene), self.desc.ctypes.data, mesh, rays.ctypes.data, len(rays), cull, hits.ctypes.data)
        return hits
