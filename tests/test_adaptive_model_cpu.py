"""
CPU tests of tests/adaptive_model.py, the streaming model of adaptive sampling's stop rule that the GPU tests hold
k_adaptive_update to: it equals the batch model of test_gpu_adaptive.py on oracle accumulations, it gives hand-derived answers on
streams whose statistics have a closed form, its float64 decisions equal the decisions of exact rational arithmetic on the same
float32 luma values, and its tile report counts what the compaction's tiles hold.
"""
import warnings
from fractions import Fraction

import numpy as np
import pytest

from raytracing_b200.camera import default_camera
from tests.adaptive_model import TILE, AdaptiveModel, luma, rule
from tests.helpers import scene
from tests.test_gpu_adaptive import at_counts, model, oracle_accs

W, H, MB, N = 64, 48, 3, 12
SETTINGS = ((0.01, 4), (0.05, 2))


@pytest.fixture(scope="module")
def accs():
    """The oracle's accumulations of CornellBox 64x48, 3 bounces, after samples 1..12: (12, 48, 64, 4)."""
    return oracle_accs(scene("CornellBox"), default_camera(W, H), W, H, MB, N)


def run(accs, max_error, min_samples):
    m = AdaptiveModel(accs.shape[1:3], max_error, min_samples)
    return m, [m.update(a) for a in accs]


@pytest.mark.parametrize("max_error,min_samples", SETTINGS)
def test_streaming_equals_batch_model(accs, max_error, min_samples):
    """Counts, the active count before every update, the active count after the last and the radiance at each pixel's count equal
    the batch model's, exactly."""
    count, n_active, left = model(accs, max_error, min_samples)
    m, ups = run(accs, max_error, min_samples)
    assert (count < N).any() and (count == N).any()                       # pixels stop and pixels survive
    assert np.array_equal(m.count, count)
    assert [u.active_before for u in ups] == n_active
    assert m.n_active == left == ups[-1].active_after
    assert np.array_equal(m.radiance.view(np.uint32), at_counts(accs, count)[..., :3].view(np.uint32))
    for a, b in zip(ups, ups[1:]):
        assert b.active_before == a.active_after


def test_constant_radiance_stops_at_min_samples():
    """A sample radiance that never changes: zero radiance and a luma stream of exact multiples have e == 0 and stop exactly at
    min_samples; a constant grey (whose float32 luma rounds) has e far below 1e-6 and stops there too."""
    for min_samples in (2, 3, 7):
        m = AdaptiveModel((1, 3), 1e-6, min_samples)
        for n in range(1, 10):
            acc = np.zeros((1, 3, 3), np.float32)
            acc[0, 1] = np.float32(0.5) * n                          # grey 0.5 per sample: exact sums, luma rounds
            Y = luma(acc)
            Y[0, 2] = np.float32(0.25) * n                            # luma 0.25 per sample, exact
            if m.active.all():                                      # the state is the full stream's
                _, _, e = rule(Y, m.y_prev, m.q, m.n + 1)
                assert e[0, 0] == 0.0 and e[0, 2] == 0.0 and e[0, 1] < 1e-6
            m.update_luma(Y, acc)
        assert np.array_equal(m.count, np.full((1, 3), min_samples, np.uint32)), min_samples
        assert m.n_active == 0


def alternating_e2(a, b, n):
    """Exact e^2 after n samples whose per-sample luma alternates a, b, a, ...: n = 2k gives m = (a + b) / 2, v = ((a - b) / 2)^2;
    n = 2k + 1 gives m = ((k + 1) a + k b) / n, v = k (k + 1) (a - b)^2 / n^2."""
    a, b = Fraction(a), Fraction(b)
    k = n // 2
    if n % 2 == 0:
        m, v = (a + b) / 2, ((a - b) / 2) ** 2
    else:
        m, v = ((k + 1) * a + k * b) / n, k * (k + 1) * (a - b) ** 2 / n ** 2
    return v / n / (1 + m) ** 4


@pytest.mark.parametrize("a,b,max_error,min_samples", [(0.5, 0.25, 0.02, 2), (1.0, 0.0, 0.05, 2), (0.125, 2.0, 0.03, 5)])
def test_alternating_luma_stops_where_the_closed_form_says(a, b, max_error, min_samples):
    """Per-sample luma a, b, a, b, ... (exact float32 sums): the model's e equals the closed form at every n to 1e-15 relative,
    and the pixel stops at the first n >= min_samples whose exact e is <= max_error."""
    me = Fraction(float(np.float32(max_error)))
    want = next(n for n in range(1, 400) if n >= min_samples and alternating_e2(a, b, n) <= me * me)
    assert want > min_samples + 2                                   # guard: the stop comes from e, not from min_samples
    m = AdaptiveModel((1, 1), max_error, min_samples)
    Y = np.float32(0)
    for n in range(1, want + 3):
        Y = np.float32(Y + np.float32(a if n % 2 else b))
        assert Fraction(float(Y)) == sum(Fraction(a if i % 2 else b) for i in range(1, n + 1))      # exact luma sums
        _, _, e = rule(np.full((1, 1), Y), m.y_prev, m.q, n)
        if m.active.all():
            want_e2 = float(alternating_e2(a, b, n))
            assert abs(e[0, 0] ** 2 - want_e2) <= 4e-15 * want_e2, n
        m.update_luma(np.full((1, 1), Y))
    assert m.count[0, 0] == want and m.n_active == 0


def test_nan_and_inf_never_stop():
    """A pixel whose radiance becomes NaN, +inf or -inf (from the first sample or later) never stops, even with max_error 1e30;
    the finite pixels beside them stop at min_samples."""
    m = AdaptiveModel((1, 6), 1e30, 4)
    acc = np.zeros((1, 6, 3), np.float32)
    for n in range(1, 11):
        acc = acc + np.float32(0.3)
        if n == 1:
            acc[0, 0] = np.nan; acc[0, 1] = np.inf
        if n == 2:
            acc[0, 2, 1] = -np.inf
        if n == 5:
            acc[0, 3, 2] = np.nan                                   # after min_samples: the pixel stopped before this
        m.update(acc)
    assert list(m.count[0]) == [10, 10, 10, 4, 4, 4]
    assert list(m.active[0]) == [True, True, True, False, False, False]


def test_negative_variance_is_clamped_and_stops():
    """Q / n - m^2 of a zero-variance state can round below 0 in double: the clamp makes v = 0, so e = 0 and the pixel stops."""
    Y, y_prev, n = np.float32(1.0), np.float32(2.0 / 3.0), 3
    y = float(Y) - float(y_prev)
    q = 3.0 * (float(Y) / 3.0) ** 2 - y * y                           # Q = n m^2 in exact arithmetic
    for _ in range(256):                                            # the largest such state whose raw v rounds below 0
        _, raw, _ = rule(Y, y_prev, q, n)
        if raw < 0.0:
            break
        q = np.nextafter(q, -np.inf)
    assert q >= 0.0 and raw < 0.0                                   # guard: the state is a sum of squares and does round below 0
    _, raw, e = rule(Y, y_prev, q, n)
    assert e == 0.0
    m = AdaptiveModel((1, 1), 1e-9, 2)
    m.n, m.y_prev[:], m.q[:] = n - 1, y_prev, q
    m.update_luma(np.full((1, 1), Y))
    assert m.count[0, 0] == n and m.n_active == 0


@pytest.mark.parametrize("min_samples", [0, 1])
def test_min_samples_below_two_stops_at_the_first_sample(accs, min_samples):
    """After one sample Q = Y^2 and m = Y, so v = 0 and e = 0: with min_samples 0 or 1 every finite pixel stops at n = 1."""
    m = AdaptiveModel(accs.shape[1:3], 1e-12, min_samples)
    u = m.update(accs[0])
    assert u.active_before == W * H and u.active_after == 0
    assert (m.count == 1).all()


def test_huge_max_error_stops_everything_at_min_samples(accs):
    for min_samples in (2, 5):
        m, ups = run(accs, 1e30, min_samples)
        assert (m.count == min_samples).all()
        assert [u.active_before for u in ups] == [W * H] * min_samples + [0] * (N - min_samples)


def test_tile_report():
    """The report follows the active list: tile t is entries [1024 t, 1024 t + 1024) of the ascending list of active pixels."""
    n_pix = 3 * TILE - 72
    m = AdaptiveModel((1, n_pix), 1e-3, 2)
    u = m.update_luma(np.ones((1, n_pix), np.float32))             # n = 1 < min_samples: nothing stops
    assert (u.tiles, list(u.survivors), u.empty, u.full, u.partial) == (3, [TILE, TILE, n_pix - 2 * TILE], 0, 3, 0)
    Y = np.full((1, n_pix), 2.0, np.float32)                        # increments 1, 1: e = 0, stops
    Y[0, :TILE] = 5.0                                               # increments 1, 4: e = 0.087, survives: tile 0 whole ..
    Y[0, 2 * TILE::2] = 5.0                                         # .. and every other entry of tile 2
    u = m.update_luma(Y)
    half = (n_pix - 2 * TILE) // 2
    assert (u.tiles, list(u.survivors), u.empty, u.full, u.partial) == (3, [TILE, 0, half], 1, 1, 1)
    assert u.active_after == m.n_active == TILE + half
    Y = np.full((1, n_pix), 15.0, np.float32)                       # increments 1, 4, 10: e = 0.06, survives
    Y[0, 2 * TILE:] = 1e6                                           # e ~ 1e-6: list entries 1024 .. (pixels 2048 ..) stop
    u = m.update_luma(Y)
    assert (u.tiles, list(u.survivors), u.empty, u.full, u.partial) == (2, [TILE, 0], 1, 1, 0)
    assert list(np.flatnonzero(m.active[0])) == list(range(TILE))


@pytest.mark.parametrize("max_error,min_samples", SETTINGS + ((0.0203, 3),))
def test_float64_decisions_equal_exact_arithmetic(accs, max_error, min_samples):
    """Q, m, v and e^2 in exact rational arithmetic from the same float32 luma values: the float64 rule takes the same stop decision
    for every pixel and sample wherever e is not within 1e-12 relative of max_error.  Decisions that close are reported as
    warnings, never skipped silently."""
    me = Fraction(float(np.float32(max_error)))
    Ys = luma(accs)
    h, w = Ys.shape[1:]
    y_prev, q = np.zeros((h, w), np.float32), np.zeros((h, w))
    near, checked = [], 0
    exact_q = [[Fraction(0)] * w for _ in range(h)]
    exact_prev = [[Fraction(0)] * w for _ in range(h)]
    for n in range(1, N + 1):
        q, _, e = rule(Ys[n - 1], y_prev, q, n)
        y_prev = Ys[n - 1]
        stop64 = (n >= min_samples) & (e <= float(me))
        for i in range(h):
            for j in range(w):
                Yf = Fraction(float(Ys[n - 1, i, j]))
                y = Yf - exact_prev[i][j]
                exact_q[i][j] += y * y
                exact_prev[i][j] = Yf
                m = Yf / n
                v = max(exact_q[i][j] / n - m * m, Fraction(0))
                assert 1 + m > 0
                e2 = v / n / (1 + m) ** 4
                ratio = e2 / (me * me)
                if abs(ratio - 1) <= Fraction(2, 10 ** 12) + Fraction(1, 10 ** 24):
                    near.append((n, i, j, float(ratio)))
                    continue
                checked += 1
                assert bool(stop64[i, j]) == (n >= min_samples and e2 <= me * me), (n, i, j, float(e2), float(me * me))
    assert checked >= N * h * w - len(near)
    if near:
        warnings.warn("max_error %r: %d decisions with e within 1e-12 relative of max_error (n, row, col, e^2/max_error^2): %r"
                      % (max_error, len(near), near[:20]))
