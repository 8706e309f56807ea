"""
The BSDF sampler and the BSDF of the sampled lights in batches (tests/bsdf_harness.cpp: the oracle's SampleBxdf, the model's
BxdfEvalSampled and EvaluateMaterial), built with g++ -ffp-contract=off into a temporary shared library on first use.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="bsdf_harness_")
        so = os.path.join(d, "libbsdf_harness.so")
        subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", "-fno-fast-math",
                        "-Wno-unknown-pragmas", "-I" + HERE, "-I" + os.path.join(REPO, "include"), "-I" + os.path.join(REPO, "oracle"),
                        "-I" + os.path.join(REPO, "raytracing_b200", "csrc"), "-o", so, os.path.join(HERE, "bsdf_harness.cpp")], check=True)
        L = C.CDLL(so)
        os.remove(so); os.rmdir(d)
        for f in (L.bh_sample, L.bh_eval, L.bh_evaluate_material):
            f.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
        _lib = L
    return _lib


def _f4(x):
    return np.ascontiguousarray(x, dtype="<f4")


def sample(mat, normal, incoming, s):
    """SampleBxdf for (n, 3) draws (s1, s.x, s.y): -> outgoing (n, 3), pdf (n,), bxdf (n, 3), offset (n,)."""
    mat, normal, incoming, s = _f4(mat), _f4(normal), _f4(incoming), _f4(s)
    out = np.zeros((len(s), 8), "<f4")
    lib().bh_sample(mat.ctypes.data, normal.ctypes.data, incoming.ctypes.data, s.ctypes.data, len(s), out.ctypes.data)
    return out[:, :3], out[:, 3], out[:, 4:7], out[:, 7]


def eval_sampled(mat, normal, incoming, o):
    """BxdfEvalSampled for (n, 3) directions: -> g (n, 3), p_b (n,), spec_pdf (n,), alpha (n,)."""
    mat, normal, incoming, o = _f4(mat), _f4(normal), _f4(incoming), _f4(o)
    out = np.zeros((len(o), 6), "<f4")
    lib().bh_eval(mat.ctypes.data, normal.ctypes.data, incoming.ctypes.data, o.ctypes.data, len(o), out.ctypes.data)
    return out[:, :3], out[:, 3], out[:, 4], out[:, 5]


def evaluate_material(mat, normal, incoming, o):
    """EvaluateMaterial for (n, 3) directions: -> (n, 3)."""
    mat, normal, incoming, o = _f4(mat), _f4(normal), _f4(incoming), _f4(o)
    out = np.zeros((len(o), 3), "<f4")
    lib().bh_evaluate_material(mat.ctypes.data, normal.ctypes.data, incoming.ctypes.data, o.ctypes.data, len(o), out.ctypes.data)
    return out
