"""
oracle/orcbind.py — TEST INFRASTRUCTURE.  ctypes binding of oracle/liboracle.so (the
CPU restatement of the reference hot path, oracle/oracle.cpp).  Only tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from .refbind import (CAMERA_DT, HIT_DT, LIGHT_DT, MATERIAL_DT, NODE_DT, RAY_DT, SCENE_INFO_DT, TEXTURE_DT, TRIANGLE_DT)

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "liboracle.so")
MAX_BOUNCES = 256        # entries of the per-bounce counters: bounces 0..255, as the CUDA path (RT_MAX_BOUNCES)


class OrcScene(C.Structure):
    _fields_ = [("triangles", C.c_void_p), ("n_triangles", C.c_uint32),
                ("nodes", C.c_void_p), ("n_nodes", C.c_uint32),
                ("materials", C.c_void_p), ("n_materials", C.c_uint32),
                ("lights", C.c_void_p), ("n_lights", C.c_uint32),
                ("textures", C.c_void_p), ("n_textures", C.c_uint32),
                ("texels", C.c_void_p), ("n_texels", C.c_uint32),
                ("env", C.c_void_p), ("env_width", C.c_uint32), ("env_height", C.c_uint32),
                ("info", C.c_uint32 * 4)]


STATS_DT = np.dtype([(k, "<u4", MAX_BOUNCES) for k in ("n_ext", "n_miss", "n_hit", "n_shadow", "n_cont", "n_unoccluded", "n_emissive_hits")] +
                    [(k, "<u8", MAX_BOUNCES) for k in ("nodes_ext", "tris_ext", "nodes_shadow", "tris_shadow")])


def build():
    subprocess.run(["make", "-C", HERE, "-s"], check=True)


class Oracle:
    def __init__(self, scene: dict, lib: str = None):
        """lib: another build of oracle.cpp (tools/fma_sensitivity.py loads the contracted-traversal model liboracle_fma.so)."""
        if lib is None and not os.path.exists(LIB):
            build()
        L = self.lib = C.CDLL(lib or LIB)
        L.orc_wang_hash.restype = C.c_uint32
        L.orc_wang_hash.argtypes = [C.c_uint32]
        L.orc_set_sampler_tables.argtypes = [C.c_void_p] * 3
        L.orc_sample_random.restype = C.c_float
        L.orc_sample_random.argtypes = [C.c_uint32] * 5
        L.orc_generate_rays.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]
        L.orc_trace.argtypes = [C.POINTER(OrcScene), C.c_void_p, C.c_uint32, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_sample_sky.argtypes = [C.POINTER(OrcScene), C.c_void_p, C.c_uint32, C.c_void_p]
        L.orc_render.argtypes = [C.POINTER(OrcScene), C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int,
                                 C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_aovs.argtypes = [C.POINTER(OrcScene), C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32] + [C.c_void_p] * 4
        L.orc_temporal_accumulation.argtypes = [C.c_uint32, C.c_uint32] + [C.c_void_p] * 5
        L.orc_resolve.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32] + [C.c_void_p] * 5 + [C.c_uint32, C.c_int, C.c_void_p]
        a = self._a = {
            "triangles": np.ascontiguousarray(scene["triangles"], dtype=TRIANGLE_DT),
            "nodes": np.ascontiguousarray(scene["nodes"], dtype=NODE_DT),
            "materials": np.ascontiguousarray(scene["materials"], dtype=MATERIAL_DT),
            "lights": np.ascontiguousarray(scene["lights"], dtype=LIGHT_DT),
            "textures": np.ascontiguousarray(scene["textures"], dtype=TEXTURE_DT),
            "texels": np.ascontiguousarray(scene["texels"], dtype="<u4"),
            "env": np.ascontiguousarray(scene["env"], dtype="<f4"),
            "scene_info": np.ascontiguousarray(scene["scene_info"], dtype=SCENE_INFO_DT),
        }
        s = self.scene = OrcScene()
        for k in ("triangles", "nodes", "materials", "lights", "textures", "texels"):
            setattr(s, k, a[k].ctypes.data)
            setattr(s, "n_" + k, a[k].shape[0])
        s.env = a["env"].ctypes.data
        s.env_width, s.env_height = int(scene["env_width"]), int(scene["env_height"])
        info = a["scene_info"].view("<u4").ravel()
        for i in range(4):
            s.info[i] = int(info[i])

    def wang_hash(self, x): return self.lib.orc_wang_hash(x)
    def set_sampler_tables(self, tables):
        """kBlueNoise with (sobol, scrambling, ranking) int32 arrays, kRandom with None.  Process-wide, like the option it mirrors."""
        if tables is None:
            self._bn = None
            self.lib.orc_set_sampler_tables(None, None, None)
            return
        self._bn = [np.ascontiguousarray(t, dtype=np.int32) for t in tables]
        assert [t.size for t in self._bn] == [65536, 131072, 131072]
        self.lib.orc_set_sampler_tables(*[t.ctypes.data for t in self._bn])

    def sample_random(self, px, py, sample, bounce, typ): return self.lib.orc_sample_random(px, py, sample, bounce, typ)

    def generate_rays(self, cam, width, height, sample_idx=0, first=0, count=None):
        count = width * height - first if count is None else count
        rays = np.zeros(count, dtype=RAY_DT)
        c = np.ascontiguousarray(cam, dtype=CAMERA_DT)
        self.lib.orc_generate_rays(c.ctypes.data, width, height, sample_idx, first, count, rays.ctypes.data)
        return rays

    def trace(self, rays, any_hit=False):
        rays = np.ascontiguousarray(rays, dtype=RAY_DT)
        n = rays.shape[0]
        counters = np.zeros(2, dtype="<u8")
        if any_hit:
            flags = np.zeros(n, dtype="<u4")
            self.lib.orc_trace(C.byref(self.scene), rays.ctypes.data, n, 1, None, flags.ctypes.data, counters.ctypes.data)
            return flags, counters
        hits = np.zeros(n, dtype=HIT_DT)
        self.lib.orc_trace(C.byref(self.scene), rays.ctypes.data, n, 0, hits.ctypes.data, None, counters.ctypes.data)
        return hits, counters

    def sample_sky(self, dirs):
        d = np.ascontiguousarray(dirs, dtype="<f4").reshape(-1, 3)
        out = np.zeros_like(d)
        self.lib.orc_sample_sky(C.byref(self.scene), d.ctypes.data, d.shape[0], out.ctypes.data)
        return out

    def aovs(self, cam, prev_cam, width, height, sample_idx=0):
        """-> albedo[h,w,4], depth[h,w], normal[h,w,4], velocity[h,w,2] as GenerateAOV leaves them."""
        c = np.ascontiguousarray(cam, dtype=CAMERA_DT); pc = np.ascontiguousarray(prev_cam, dtype=CAMERA_DT)
        al = np.zeros((height, width, 4), "<f4"); de = np.zeros((height, width), "<f4")
        no = np.zeros((height, width, 4), "<f4"); ve = np.zeros((height, width, 2), "<f4")
        self.lib.orc_aovs(C.byref(self.scene), c.ctypes.data, pc.ctypes.data, width, height, sample_idx,
                          al.ctypes.data, de.ctypes.data, no.ctypes.data, ve.ctypes.data)
        return al, de, no, ve

    def temporal_accumulation(self, radiance, prev_radiance, depth, prev_depth, velocity):
        h, w = depth.shape
        r = np.ascontiguousarray(radiance, "<f4").copy()
        pr = np.ascontiguousarray(prev_radiance, "<f4"); d = np.ascontiguousarray(depth, "<f4")
        pd = np.ascontiguousarray(prev_depth, "<f4"); v = np.ascontiguousarray(velocity, "<f4")
        self.lib.orc_temporal_accumulation(w, h, r.ctypes.data, pr.ctypes.data, d.ctypes.data, pd.ctypes.data, v.ctypes.data)
        return r

    def resolve(self, aov, radiance, albedo, depth, normal, velocity, sample_count, denoiser=False):
        h, w = depth.shape
        out = np.zeros((h, w, 4), "<f4")
        arrs = [np.ascontiguousarray(x, "<f4") for x in (radiance, albedo, depth, normal, velocity)]
        self.lib.orc_resolve(w, h, aov, *[x.ctypes.data for x in arrs], sample_count, int(denoiser), out.ctypes.data)
        return out

    def render(self, cam, width, height, max_bounces, sample_idx=0, white_furnace=False, row_first=0, row_step=1,
               radiance=None, want_hits=True):
        """One sample per pixel; returns (radiance[h,w,4] accumulated, primary_hits[h*w] or None, stats)."""
        if radiance is None:
            radiance = np.zeros((height, width, 4), dtype="<f4")
        hits = np.zeros(width * height, dtype=HIT_DT) if want_hits else None
        if hits is not None:
            hits["primitive_id"] = 0xFFFFFFFE   # "pixel not traced by this partition"
        stats = np.zeros((), dtype=STATS_DT)
        c = np.ascontiguousarray(cam, dtype=CAMERA_DT)
        self.lib.orc_render(C.byref(self.scene), c.ctypes.data, width, height, max_bounces, sample_idx, int(white_furnace),
                            row_first, row_step, radiance.ctypes.data, hits.ctypes.data if hits is not None else None,
                            stats.ctypes.data)
        return radiance, hits, stats
