"""
include/rt_math.h pinned INDEPENDENTLY of the renderers.  The reference kernels compiled for the CPU (oracle/_ref), the
oracle and the CUDA kernels all use this one header, so a wrong rt_atan2f would be bit-identical on every side and invisible to
the parity tests.  Here every function is checked (a) on the CPU against glibc's double-precision libm rounded to float
(correctly rounded up to double rounding) on >= 1 M seeded arguments per function plus edge cases, with the ulp bound stated,
and (b) on the GPU: the device evaluation of the same header must equal the host evaluation bit for bit.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
N = 1 << 20
FN = {"sin": 0, "cos": 1, "tan": 2, "atan2": 3, "acos": 4, "pow": 5, "fmin": 6, "fmax": 7, "rsqrt": 8, "div": 9}


@pytest.fixture(scope="module")
def host():
    so = os.path.join(tempfile.gettempdir(), f"librt_math_host_{os.getpid()}.so")
    subprocess.run(["/usr/bin/gcc", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-I" + os.path.join(REPO, "include"),
                    "-o", so, os.path.join(HERE, "rt_math_host.c"), "-lm"], check=True)
    L = C.CDLL(so)
    L.rtm_eval.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]

    def ev(fn, a, b=None):
        a = np.ascontiguousarray(a, dtype="<f4"); b = np.ascontiguousarray(np.zeros_like(a) if b is None else b, dtype="<f4")
        out = np.zeros_like(a)
        L.rtm_eval(FN[fn], a.ctypes.data, b.ctypes.data, out.ctypes.data, a.size)
        return out
    yield ev
    os.remove(so)


def ulp_diff(got, want):
    """|got - want| in units of the last place of float32 `want` (same-sign finite values; NaN == NaN counts as 0)."""
    g = np.asarray(got, dtype="<f4"); w = np.asarray(want, dtype="<f4")
    both_nan = np.isnan(g) & np.isnan(w)
    gi = g.view("<i4").astype(np.int64); wi = w.view("<i4").astype(np.int64)
    gi = np.where(gi < 0, -(gi & 0x7FFFFFFF), gi); wi = np.where(wi < 0, -(wi & 0x7FFFFFFF), wi)
    d = np.abs(gi - wi)
    d[both_nan] = 0
    d[np.isnan(g) ^ np.isnan(w)] = 1 << 40
    return d


def arguments(fn, rng):
    """(a, b) float32 arguments covering the ranges the path uses, plus edge cases."""
    if fn in ("sin", "cos", "tan"):
        a = np.concatenate([rng.uniform(-7.0, 7.0, N // 2), rng.uniform(-1000.0, 1000.0, N // 2 - 16),
                            [0.0, -0.0, np.pi, -np.pi, np.pi / 2, 2 * np.pi, 1e-30, -1e-30, 6.2831855, 0.6544, 1.5707964, 3.1415927, 99999.0, -99999.0, 1e-5, 0.5]])
        return a.astype("<f4"), np.zeros(N, "<f4")
    if fn == "atan2":
        a = rng.normal(0, 1, N).astype("<f4"); b = rng.normal(0, 1, N).astype("<f4")
        edge = np.array([[0.0, 1.0], [-0.0, 1.0], [0.0, -1.0], [-0.0, -1.0], [1.0, 0.0], [-1.0, 0.0], [1.0, -0.0], [0.0, 0.0], [1e-30, 1e30], [1e30, 1e-30],
                         [1.0, 1.0], [-1.0, 1.0], [1.0, -1.0], [-1.0, -1.0], [0.125, 1.0], [0.375, 1.0]], dtype="<f4")
        a[: len(edge)] = edge[:, 0]; b[: len(edge)] = edge[:, 1]
        a[len(edge): 2 * len(edge)] *= 1e-20                     # tiny / huge ratios
        return a, b
    if fn == "acos":
        a = np.concatenate([rng.uniform(-1.0, 1.0, N - 8), [1.0, -1.0, 0.0, -0.0, 0.99999994, -0.99999994, 1e-20, 0.5]]).astype("<f4")
        return a, np.zeros(N, "<f4")
    if fn == "pow":
        half = N // 2
        a = np.concatenate([rng.uniform(-1.0, 1.0, half), rng.uniform(0.0, 1.0, N - half)]).astype("<f4")     # Schlick (1 - cos)^5, texture gamma
        b = np.concatenate([np.full(half, 5.0), np.full(N - half, 2.2)]).astype("<f4")
        a[:6] = [0.0, 1.0, -1.0, 0.5, 1e-10, 0.99999994]
        return a, b
    if fn in ("fmin", "fmax"):
        a = rng.normal(0, 10, N).astype("<f4"); b = rng.normal(0, 10, N).astype("<f4")
        a[:8] = [0.0, -0.0, np.nan, 1.0, np.nan, np.inf, -np.inf, 3.0]; b[:8] = [-0.0, 0.0, 1.0, np.nan, np.nan, 1.0, 1.0, 3.0]
        return a, b
    if fn == "rsqrt":
        return np.concatenate([rng.uniform(1e-6, 1e6, N - 4), [1.0, 4.0, 1e-30, 1e30]]).astype("<f4"), np.zeros(N, "<f4")
    a = rng.normal(0, 100, N).astype("<f4"); b = rng.normal(0, 100, N).astype("<f4")
    b[b == 0] = 1.0
    return a, b


REFERENCE = {
    "sin": lambda a, b: np.sin(a.astype(np.float64)), "cos": lambda a, b: np.cos(a.astype(np.float64)), "tan": lambda a, b: np.tan(a.astype(np.float64)),
    "atan2": lambda a, b: np.arctan2(a.astype(np.float64), b.astype(np.float64)), "acos": lambda a, b: np.arccos(a.astype(np.float64)),
    "pow": lambda a, b: np.power(a.astype(np.float64), b.astype(np.float64)),
    "rsqrt": None, "div": None, "fmin": None, "fmax": None,
}
# stated bounds: the double-precision evaluation is accurate to well under 1e-9 float ulps, so the float result is the correctly
# rounded one except where the exact value lies within that distance of a rounding boundary (double rounding): <= 1 ulp always,
# and identical to round(libm double) on all but a vanishing fraction of arguments
MAX_ULP = {"sin": 1, "cos": 1, "tan": 1, "atan2": 1, "acos": 1, "pow": 1}
MAX_MISMATCH_FRACTION = 2e-6


@pytest.mark.parametrize("fn", ["sin", "cos", "tan", "atan2", "acos", "pow"])
def test_rt_math_against_double_libm(host, fn):
    rng = np.random.default_rng(1234 + FN[fn])
    a, b = arguments(fn, rng)
    got = host(fn, a, b)
    with np.errstate(all="ignore"):
        want = REFERENCE[fn](a, b).astype("<f4")
    if fn == "pow":                                   # rt_powf(x < 0, 2.2) is NaN by construction; only the exponent 5 takes negative bases
        keep = ~((a < 0) & (b != 5.0))
        got, want = got[keep], want[keep]
    d = ulp_diff(got, want)
    assert d.max() <= MAX_ULP[fn], (fn, int(d.max()), a[np.argmax(d)], b[np.argmax(d)] if fn in ("atan2", "pow") else None)
    assert (d != 0).mean() <= MAX_MISMATCH_FRACTION, (fn, float((d != 0).mean()))


def test_rt_math_exact_building_blocks(host):
    """fmin/fmax follow IEEE minNum/maxNum (NaN operand ignored, -0 < +0) — what PTX min.f32/max.f32 do; 1/sqrt and division are
    the correctly rounded IEEE operations (checked against double arithmetic rounded once: exact for these two operations)."""
    rng = np.random.default_rng(99)
    a, b = arguments("fmin", rng)
    with np.errstate(all="ignore"):
        for fn, ref in (("fmin", np.fmin), ("fmax", np.fmax)):
            got = host(fn, a, b); want = ref(a, b)
            ok = (got.view("<u4") == want.view("<u4")) | (np.isnan(got) & np.isnan(want))
            zero_pair = (a == 0) & (b == 0)                                     # numpy leaves the sign of min(+0, -0) unspecified
            assert ok[~zero_pair].all(), fn
        assert host("fmin", [0.0, -0.0], [-0.0, 0.0]).view("<u4").tolist() == [0x80000000, 0x80000000]
        assert host("fmax", [0.0, -0.0], [-0.0, 0.0]).view("<u4").tolist() == [0, 0]
        a, b = arguments("div", rng)
        assert np.array_equal(host("div", a, b).view("<u4"), (a.astype(np.float64) / b.astype(np.float64)).astype("<f4").view("<u4"))
        a, _ = arguments("rsqrt", rng)
        s = np.sqrt(a.astype(np.float64)).astype("<f4")                          # IEEE sqrtf, then IEEE 1/x: two correctly rounded steps
        assert np.array_equal(host("rsqrt", a).view("<u4"), (np.float32(1.0) / s).view("<u4"))


@pytest.mark.gpu
@pytest.mark.parametrize("fn", sorted(FN))
def test_device_rt_math_equals_host_rt_math(host, fn):
    """sm_90a (-fmad=false) and x86-64 (-ffp-contract=off) evaluate include/rt_math.h to the same bits."""
    from raytracing_b200 import capi
    rng = np.random.default_rng(4321 + FN[fn])
    a, b = arguments(fn, rng)
    dev = capi.math_eval(fn, a, b)
    hst = host(fn, a, b)
    same = (dev.view("<u4") == hst.view("<u4")) | (np.isnan(dev) & np.isnan(hst))
    assert same.all(), (fn, int((~same).sum()), a[~same][:4], b[~same][:4], dev[~same][:4], hst[~same][:4])
