"""
The CPU model of the sampled lights (tests/light_model.cpp: the oracle's frame with the rules stated at RT_OPT_EMITTER_SAMPLING,
RT_OPT_ENV_SAMPLING and rt_set_light_selection in include/rt_b200.h), built with g++ -ffp-contract=off into a temporary shared
library on first use.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle.orcbind import STATS_DT
from oracle.refbind import CAMERA_DT
from tests.emitter_model import EmitterModel

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="light_model_")
        so = os.path.join(d, "liblight_model.so")
        subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", "-fno-fast-math",
                        "-Wno-unknown-pragmas", "-I" + HERE, "-I" + os.path.join(REPO, "include"), "-I" + os.path.join(REPO, "oracle"),
                        "-I" + os.path.join(REPO, "raytracing_b200", "csrc"), "-o", so, os.path.join(HERE, "light_model.cpp")], check=True)
        L = C.CDLL(so)
        os.remove(so); os.rmdir(d)
        L.lm_env_table.restype = C.c_int
        L.lm_env_table.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_float, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        L.lm_env_pdf.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p]
        L.lm_env_sample.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p]
        L.lm_select.argtypes = [C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_void_p]
        L.lm_sinf.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
        L.lm_render.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int,
                                C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_set_sampler_tables.argtypes = [C.c_void_p] * 3
        _lib = L
    return _lib


def env_table(env, w, h, p_v=1.0, white_furnace=False):
    """-> (marg, cond, pdf) of an RGBA32F image as rt_envmap.h builds it (pdf scaled by p_v), or None when inactive."""
    env = np.ascontiguousarray(env, dtype="<f4")
    marg = np.zeros(h, "<f4"); cond = np.zeros(w * h, "<f4"); pdf = np.zeros(w * h, "<f4")
    ok = lib().lm_env_table(env.ctypes.data, w, h, p_v, int(white_furnace), marg.ctypes.data, cond.ctypes.data, pdf.ctypes.data)
    return (marg, cond.reshape(h, w), pdf.reshape(h, w)) if ok else None


def env_pdf(pdf, dirs):
    """p_v(dir) for (n, 3) directions."""
    h, w = pdf.shape
    pdf = np.ascontiguousarray(pdf, dtype="<f4"); d = np.ascontiguousarray(dirs, dtype="<f4")
    out = np.zeros(len(d), "<f4")
    lib().lm_env_pdf(pdf.ctypes.data, w, h, d.ctypes.data, len(d), out.ctypes.data)
    return out


def env_sample(marg, cond, r):
    """Directions of (n, 4) draws."""
    h, w = cond.shape
    r = np.ascontiguousarray(r, dtype="<f4")
    out = np.zeros((len(r), 3), "<f4")
    lib().lm_env_sample(np.ascontiguousarray(marg, "<f4").ctypes.data, np.ascontiguousarray(cond, "<f4").ctypes.data, w, h,
                        r.ctypes.data, len(r), out.ctypes.data)
    return out


def rt_sinf(x):
    x = np.ascontiguousarray(x, dtype="<f4")
    out = np.zeros_like(x)
    lib().lm_sinf(x.ctypes.data, x.size, out.ctypes.data)
    return out


def select(analytic, emitters, env, weights=(1.0, 1.0, 1.0)):
    """-> (P_e, P_v, P_e + P_v, no_analytic) of the light-kind rule."""
    out = np.zeros(4, "<f4")
    lib().lm_select(int(analytic), int(emitters), int(env), *[float(x) for x in weights], out.ctypes.data)
    return tuple(float(x) for x in out)


class LightModel(EmitterModel):
    """The oracle plus the sampled lights: render(..., emitters=, env=, weights=) follows the rules of include/rt_b200.h;
    with both options False it is the oracle's own render unless model=True."""

    def set_sampler_tables(self, tables):
        super().set_sampler_tables(tables)
        if tables is None:
            lib().orc_set_sampler_tables(None, None, None)
        else:
            lib().orc_set_sampler_tables(*[t.ctypes.data for t in self._bn])

    def render(self, cam, width, height, max_bounces, sample_idx=0, white_furnace=False, row_first=0, row_step=1,
               radiance=None, want_hits=True, emitters=False, env=False, weights=(1.0, 1.0, 1.0), model=False):
        if not (emitters or env or model):
            return super().render(cam, width, height, max_bounces, sample_idx, white_furnace, row_first, row_step, radiance, want_hits)
        if radiance is None:
            radiance = np.zeros((height, width, 4), dtype="<f4")
        stats = np.zeros((), dtype=STATS_DT)
        c = np.ascontiguousarray(cam, dtype=CAMERA_DT)
        wts = np.ascontiguousarray(weights, dtype="<f4")
        lib().lm_render(C.addressof(self.scene), self.emissive.ctypes.data, self.emissive.size, c.ctypes.data, width, height, max_bounces,
                        sample_idx, int(white_furnace), row_first, row_step, int(emitters), int(env), wts.ctypes.data,
                        radiance.ctypes.data, stats.ctypes.data)
        return radiance, None, stats
