"""
The CPU model of emitter sampling (tests/emitter_model.cpp: the oracle's frame with the rule stated at RT_OPT_EMITTER_SAMPLING in
include/rt_b200.h), built with g++ -ffp-contract=off into a temporary shared library on first use.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle.orcbind import STATS_DT, Oracle
from oracle.refbind import CAMERA_DT

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="emitter_model_")
        so = os.path.join(d, "libemitter_model.so")
        subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", "-fno-fast-math",
                        "-Wno-unknown-pragmas", "-I" + os.path.join(REPO, "include"), "-I" + os.path.join(REPO, "oracle"),
                        "-I" + os.path.join(REPO, "raytracing_b200", "csrc"), "-o", so, os.path.join(HERE, "emitter_model.cpp")], check=True)
        L = C.CDLL(so)
        os.remove(so); os.rmdir(d)
        L.em_table.restype = C.c_int
        L.em_table.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.em_render.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int,
                                C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


class EmitterModel(Oracle):
    """The oracle plus emitter sampling: render(..., emitters=True) follows the RT_OPT_EMITTER_SAMPLING rule."""

    def __init__(self, scene, emissive=None):
        super().__init__(scene)
        em = scene["emissive"] if emissive is None else emissive
        self.emissive = np.ascontiguousarray(em, dtype="<u4")

    def set_sampler_tables(self, tables):
        super().set_sampler_tables(tables)
        L = lib()
        L.orc_set_sampler_tables.argtypes = [C.c_void_p] * 3
        if tables is None:
            L.orc_set_sampler_tables(None, None, None)
        else:
            L.orc_set_sampler_tables(*[t.ctypes.data for t in self._bn])

    def table(self, white_furnace=False):
        """-> (list, cdf, pdfA, p_e) as rt_upload_scene builds them, or None for an invalid emitter list."""
        n, nt = self.emissive.size, int(self.scene.n_triangles)
        lst = np.zeros(max(n, 1), "<u4"); cdf = np.zeros(max(n, 1), "<f4"); pdfa = np.zeros(nt, "<f4")
        n_out = C.c_uint32(0); pe = C.c_float(0.0)
        ok = lib().em_table(C.addressof(self.scene), self.emissive.ctypes.data, n, int(white_furnace), lst.ctypes.data, cdf.ctypes.data,
                            pdfa.ctypes.data, C.byref(n_out), C.byref(pe))
        if not ok:
            return None
        return lst[: n_out.value], cdf[: n_out.value], pdfa, pe.value

    def render(self, cam, width, height, max_bounces, sample_idx=0, white_furnace=False, row_first=0, row_step=1,
               radiance=None, want_hits=True, emitters=False):
        if not emitters:
            return super().render(cam, width, height, max_bounces, sample_idx, white_furnace, row_first, row_step, radiance, want_hits)
        if radiance is None:
            radiance = np.zeros((height, width, 4), dtype="<f4")
        stats = np.zeros((), dtype=STATS_DT)
        c = np.ascontiguousarray(cam, dtype=CAMERA_DT)
        lib().em_render(C.addressof(self.scene), self.emissive.ctypes.data, self.emissive.size, c.ctypes.data, width, height, max_bounces,
                        sample_idx, int(white_furnace), row_first, row_step, radiance.ctypes.data, stats.ctypes.data)
        return radiance, None, stats
