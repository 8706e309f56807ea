"""
The CPU model of object motion vectors (tests/motion_model.cpp: the oracle's GenerateAOV with the rule stated at
RT_OPT_OBJECT_MOTION in include/rt_b200.h), built with g++ -ffp-contract=off into a temporary shared library on first use.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle.orcbind import Oracle
from oracle.refbind import CAMERA_DT

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="motion_model_")
        so = os.path.join(d, "libmotion_model.so")
        subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", "-fno-fast-math",
                        "-Wno-unknown-pragmas", "-I" + os.path.join(REPO, "include"), "-I" + os.path.join(REPO, "oracle"),
                        "-o", so, os.path.join(HERE, "motion_model.cpp")], check=True)
        L = C.CDLL(so)
        os.remove(so); os.rmdir(d)
        L.mv_aovs.argtypes = [C.c_void_p] * 4 + [C.c_uint32] * 3 + [C.c_void_p] * 4
        _lib = L
    return _lib


def positions(triangles):
    """The previous-position array of a triangle array: 3 float4 per triangle (tris_ref's layout, .w words included)."""
    return np.ascontiguousarray(np.stack([triangles[v]["position"] for v in ("v1", "v2", "v3")], axis=1), dtype="<f4")


class MotionModel(Oracle):
    """The oracle plus object motion: mv_aovs(prev_positions, cam, prev_cam, ...) follows the RT_OPT_OBJECT_MOTION rule."""

    def mv_aovs(self, prev_positions, cam, prev_cam, width, height, sample_idx=0):
        """-> albedo[h,w,4], depth[h,w], normal[h,w,4], velocity[h,w,2]; prev_positions: (n, 3, 4) float32 or a triangle array."""
        q = np.asarray(prev_positions)
        if q.dtype.names:
            q = positions(q)
        q = np.ascontiguousarray(q, dtype="<f4")
        assert q.shape == (int(self.scene.n_triangles), 3, 4)
        c = np.ascontiguousarray(cam, dtype=CAMERA_DT); pc = np.ascontiguousarray(prev_cam, dtype=CAMERA_DT)
        al = np.zeros((height, width, 4), "<f4"); de = np.zeros((height, width), "<f4")
        no = np.zeros((height, width, 4), "<f4"); ve = np.zeros((height, width, 2), "<f4")
        lib().mv_aovs(C.addressof(self.scene), q.ctypes.data, c.ctypes.data, pc.ctypes.data, width, height, sample_idx,
                      al.ctypes.data, de.ctypes.data, no.ctypes.data, ve.ctypes.data)
        return al, de, no, ve
