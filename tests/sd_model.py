"""
The scalar model of the spatial denoiser (tests/spatial_denoise_model.c, the rule stated with rt_set_spatial_denoiser in
include/rt_b200.h) and the host rt_expf, built with gcc -ffp-contract=off into a temporary shared library on first use.
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
        d = tempfile.mkdtemp(prefix="sd_model_")
        so = os.path.join(d, "libsd_model.so")
        subprocess.run(["/usr/bin/gcc", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-I" + os.path.join(REPO, "include"),
                        "-o", so, os.path.join(HERE, "spatial_denoise_model.c"), "-lm"], check=True)
        L = C.CDLL(so)
        os.remove(so); os.rmdir(d)
        L.sdm_expf.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
        L.sdm_filter.argtypes = [C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_float, C.c_float, C.c_float, C.c_void_p]
        _lib = L
    return _lib


def expf(x):
    """include/rt_math.h rt_expf evaluated on the host."""
    x = np.ascontiguousarray(x, dtype="<f4")
    out = np.zeros_like(x)
    lib().sdm_expf(x.ctypes.data, out.ctypes.data, x.size)
    return out


def filter_image(ldr, normal, depth, iterations, sigma_color, sigma_normal, sigma_depth):
    """ldr (h, w, 4) resolved colour, normal (h, w, 4), depth (h, w) -> the filtered (h, w, 4) image, alpha 1."""
    h, w = depth.shape
    a = [np.ascontiguousarray(x, dtype="<f4") for x in (ldr, normal, depth)]
    assert a[0].shape == (h, w, 4) and a[1].shape == (h, w, 4)
    out = np.zeros((h, w, 4), "<f4")
    lib().sdm_filter(w, h, a[0].ctypes.data, a[1].ctypes.data, a[2].ctypes.data, int(iterations), float(sigma_color), float(sigma_normal),
                     float(sigma_depth), out.ctypes.data)
    return out
