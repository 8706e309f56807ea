"""
The velocity model of deforming meshes in instanced scenes (tests/mesh_motion_model.cpp: the previous mesh positions Q of
RT_OPT_OBJECT_MOTION placed by the previous transforms, evaluated on the primary hits of tests/instance_model.cpp's frame), built
with g++ -ffp-contract=off into a temporary shared library on first use.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle.refbind import CAMERA_DT
from tests.instance_model import InstanceModel, instances

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="mesh_motion_model_")
        so = os.path.join(d, "libmesh_motion_model.so")
        subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", "-fno-fast-math",
                        "-Wno-unknown-pragmas", "-I" + os.path.join(REPO, "include"), "-I" + os.path.join(REPO, "oracle"),
                        "-I" + os.path.join(REPO, "raytracing_b200", "csrc"), "-I" + HERE, "-o", so,
                        os.path.join(HERE, "mesh_motion_model.cpp")], check=True)
        L = C.CDLL(so)
        os.remove(so); os.rmdir(d)
        L.mm_velocity.restype = C.c_int
        L.mm_velocity.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


class MeshMotionModel(InstanceModel):
    """InstanceModel whose velocity also follows the previous mesh positions."""

    def velocity(self, mesh_ids, transforms, cam, width, height, hits, prev=None, prev_positions=None):
        """-> velocity (h, w, 2) of the primary hits `hits` (h*w,) HIT_DT, with the camera as its own previous camera, `prev`
        (n, 3, 4) the previous transforms and `prev_positions` (one (3, 3) per triangle of the concatenated meshes: q1, q2, q3) the
        previous mesh positions; None for either = the current ones."""
        inst = instances(mesh_ids, transforms)
        pv = None if prev is None else np.ascontiguousarray(prev, dtype="<f4").reshape(-1, 12)
        pq = None if prev_positions is None else np.ascontiguousarray(prev_positions, dtype="<f4").reshape(-1, 9)
        if pq is not None and len(pq) != int(self.desc[:, 1].sum()):
            raise ValueError("prev_positions: one (3, 3) per triangle")
        h = np.ascontiguousarray(hits)
        vel = np.zeros((height, width, 2), dtype="<f4")
        c = np.ascontiguousarray(cam, dtype=CAMERA_DT)
        rc = lib().mm_velocity(C.addressof(self.scene), self.desc.ctypes.data, len(self.desc), inst.ctypes.data if len(inst) else None,
                               len(inst), pv.ctypes.data if pv is not None else None, pq.ctypes.data if pq is not None else None,
                               c.ctypes.data, width, height, h.ctypes.data, vel.ctypes.data)
        if rc != 0:
            raise ValueError("instance list rejected")
        return vel

    def render_instanced(self, mesh_ids, transforms, cam, width, height, max_bounces, sample_idx=0, prev=None, radiance=None,
                         prev_positions=None):
        """InstanceModel.render_instanced, with the velocity of the previous mesh positions when prev_positions is given."""
        rad, hits, st, vel = super().render_instanced(mesh_ids, transforms, cam, width, height, max_bounces, sample_idx, prev, radiance)
        if prev_positions is not None:
            vel = self.velocity(mesh_ids, transforms, cam, width, height, hits, prev, prev_positions)
        return rad, hits, st, vel
