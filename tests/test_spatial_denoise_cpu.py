"""
CPU tests (-m "not gpu") of the spatial denoiser's building blocks: the accuracy of include/rt_math.h rt_expf over the range the
edge-stopping weights use, its edge cases, and properties of the scalar model of the filter (tests/spatial_denoise_model.c) that the
GPU tests compare the kernels with bit for bit.
"""
import numpy as np
import pytest

from tests import sd_model

N = 1 << 20
# measured: the largest error is 1.21 ulp of the exact value (float Horner evaluation after an exact reduction); a tenth of the
# results are not the correctly rounded float
MAX_ULP = 1.25


def expf_arguments(seed):
    rng = np.random.default_rng(seed)
    a = np.concatenate([rng.uniform(-87.3, 0.0, N // 2), rng.uniform(-12.0, 0.0, N // 4), rng.uniform(-87.3, 88.7, N // 4)]).astype("<f4")
    edge = np.array([0.0, -0.0, 1e-30, -1e-30, 1.0, -1.0, -0.34657359, 0.34657359, -87.33654, -87.3366, 88.72283, 88.7229,
                     -104.0, 200.0, np.inf, -np.inf, np.nan], "<f4")
    return np.concatenate([edge, a])


def test_rt_expf_accuracy_against_double_exp():
    x = expf_arguments(7)
    x = x[np.isfinite(x) & (x >= np.float32(-87.33654)) & (x <= np.float32(88.72283))]
    got = sd_model.expf(x).astype(np.float64)
    want = np.exp(x.astype(np.float64))
    ulp = np.spacing(want.astype(np.float32)).astype(np.float64)
    err = np.abs(got - want) / ulp
    assert err.max() <= MAX_ULP, (float(err.max()), x[np.argmax(err)])
    assert np.all(got > 0)


def test_rt_expf_edge_cases():
    x = np.array([0.0, -0.0, -87.3366, -104.0, -np.inf, 88.7229, 200.0, np.inf, np.nan, 88.72283], "<f4")
    got = sd_model.expf(x)
    assert got[:2].tolist() == [1.0, 1.0]
    assert got[2:5].tolist() == [0.0, 0.0, 0.0]                       # below ln(FLT_MIN): 0, no subnormals
    assert np.isposinf(got[5:8]).all() and np.isnan(got[8])
    assert np.isfinite(got[9]) and got[9] > np.float32(3.4e38)
    # monotone over the weights' range
    y = np.sort(expf_arguments(11)[np.isfinite(expf_arguments(11))])
    y = y[(y <= 0.0) & (y >= -87.3)]
    assert np.all(np.diff(sd_model.expf(y)) >= 0)


def _guides(h, w, seed=0):
    rng = np.random.default_rng(seed)
    n = rng.normal(size=(h, w, 4)).astype("<f4")
    n[..., :3] /= np.linalg.norm(n[..., :3], axis=-1, keepdims=True)
    n[..., 3] = 0
    return n, rng.uniform(1.0, 10.0, (h, w)).astype("<f4")


def test_model_keeps_a_constant_image_and_leaves_no_nan():
    h, w = 23, 31
    n, z = _guides(h, w)
    ldr = np.full((h, w, 4), 0.25, "<f4")
    out = sd_model.filter_image(ldr, n, z, 5, 0.5, 0.3, 0.2)
    assert np.allclose(out[..., :3], 0.25, rtol=1e-6, atol=0) and (out[..., 3] == 1).all()
    ldr[5, 7, 0] = np.nan; ldr[11, 2, 1] = np.inf; ldr[0, 0, 2] = -np.inf
    out = sd_model.filter_image(ldr, n, z, 5, 0.5, 0.3, 0.2)
    assert np.isfinite(out).all()                                     # non-finite taps get weight 0; those pixels are filled in


def test_model_isolated_pixel_keeps_its_value():
    """A 1x1 image has only its own tap; a pixel whose every tap is non-finite keeps its input."""
    ldr = np.array([[[0.5, 0.25, 0.125, 1.0]]], "<f4")
    n = np.zeros((1, 1, 4), "<f4"); z = np.ones((1, 1), "<f4")
    assert np.array_equal(sd_model.filter_image(ldr, n, z, 5, 1.0, 1.0, 1.0), ldr)
    ldr = np.full((3, 3, 4), np.nan, "<f4"); ldr[..., 3] = 1
    out = sd_model.filter_image(ldr, np.zeros((3, 3, 4), "<f4"), np.ones((3, 3), "<f4"), 2, 1.0, 1.0, 1.0)
    assert np.isnan(out[..., :3]).all()


def test_model_depth_edge_stops_the_blur():
    """Two flat halves at different depths: with the depth guide the halves do not mix; without it they do."""
    h, w = 16, 16
    ldr = np.zeros((h, w, 4), "<f4"); ldr[:, w // 2:, :3] = 0.8; ldr[..., 3] = 1
    n = np.zeros((h, w, 4), "<f4"); n[..., 2] = 1
    z = np.ones((h, w), "<f4"); z[:, w // 2:] = 5.0
    kept = sd_model.filter_image(ldr, n, z, 3, 0.0, 0.0, 0.01)
    assert np.array_equal(kept, ldr)
    mixed = sd_model.filter_image(ldr, n, z, 3, 0.0, 0.0, 0.0)
    assert 0.0 < mixed[0, w // 2 - 1, 0] < 0.8
