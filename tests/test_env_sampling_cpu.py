"""
Environment sampling (RT_OPT_ENV_SAMPLING) and the light-kind weights (rt_set_light_selection) on the CPU: the environment table
(raytracing_b200/csrc/rt_envmap.h) against a numpy restatement, its density and sampling walk, the model's inactive cases against
the emitter model and the oracle, and the estimator's expectation against the option off.
"""
import numpy as np
import pytest

from raytracing_b200.camera import default_camera
from tests.helpers import bits, scene
from tests.light_model import LightModel, env_pdf, env_sample, env_table, rt_sinf, select
from tests.test_emitter_sampling_cpu import get_scene

SKEW = (0.5, 2.0, 3.0)


def sun_sky(env, w, h, seed=5):
    """The shipped sky plus a seeded few-texel sun of luma ~1e4 at about 45 degrees elevation."""
    rng = np.random.default_rng(seed)
    img = np.array(env, dtype="<f4").reshape(h, w, 4)
    j, i = h // 4 + int(rng.integers(-5, 6)), int(rng.integers(0, w - 3))
    img[j:j + 2, i:i + 3, :3] = np.float32(1e4)
    return img.reshape(-1)


def sun_scene(name):
    """The scene under the sun sky and lit by it alone: its analytic lights are dark, as when the environment image carries the sun."""
    sc = dict(get_scene(name))
    sc["env"] = sun_sky(sc["env"], int(sc["env_width"]), int(sc["env_height"]))
    sc["lights"] = sc["lights"].copy(); sc["lights"]["radiance"] = 0
    return sc


def numpy_table(env, w, h, p_v):
    """The rule of rt_envmap.h restated in numpy float32 (rt_sinf from the model: it is rt_math.h's)."""
    f = np.float32
    img = np.asarray(env, "<f4").reshape(h, w, 4)
    luma = (img[..., 0] * f(0.299) + img[..., 1] * f(0.587)) + img[..., 2] * f(0.114)
    luma = np.where(np.isfinite(luma) & (luma >= 0), luma, f(0)).astype(f)
    s = rt_sinf(f(np.pi) * ((np.arange(h, dtype=f) + f(0.5)) / f(h)))
    W = (luma * s[:, None]).astype(f)
    cond = np.cumsum(W, axis=1, dtype=f)            # running float32 sums in order
    row = cond[:, -1].copy()
    marg = np.cumsum(row, dtype=f)
    total = marg[-1]
    if not (np.isfinite(total) and total > 0):
        return None
    marg = (marg / total).astype(f); marg[-1] = 1
    cond = np.where(row[:, None] > 0, cond / np.where(row > 0, row, f(1))[:, None], f(1)).astype(f); cond[:, -1] = 1
    pdf = (f(p_v) * (((f(w) * f(h)) * W) / total)).astype(f)
    return marg, cond, pdf


def shipped():
    sc = scene("CornellBox")
    return sc["env"], int(sc["env_width"]), int(sc["env_height"])


@pytest.mark.parametrize("sky", ["shipped", "sun"])
@pytest.mark.parametrize("p_v", [1.0, 0.5, 0.2])
def test_table_matches_numpy_restatement(sky, p_v):
    env, w, h = shipped()
    if sky == "sun":
        env = sun_sky(env, w, h)
    got, want = env_table(env, w, h, p_v), numpy_table(env, w, h, p_v)
    for g, e in zip(got, want):
        assert np.array_equal(bits(g), bits(e))
    marg, cond, pdf = got
    assert np.all(np.diff(marg) >= 0) and np.all(np.diff(cond, axis=1) >= 0)
    # p_uv integrates to 1 over the texture square
    assert abs(pdf.astype(np.float64).sum() / (w * h) - p_v) < 1e-4 * p_v


def test_table_inactive_cases():
    env, w, h = shipped()
    assert env_table(env, w, h, white_furnace=True) is None
    assert env_table(np.zeros_like(env), w, h) is None
    neg = -np.abs(np.asarray(env, "<f4"))
    assert env_table(neg, w, h) is None
    img = np.array(env, "<f4").reshape(h, w, 4)
    img[7, 11, 0] = np.nan; img[20, 3, 1] = np.inf
    t = env_table(img.reshape(-1), w, h)
    assert t is not None and t[2][7, 11] == 0 and t[2][20, 3] == 0
    assert env_table(np.full(4, 0.2, "<f4"), 1, 1) is not None          # the procedural scene's 1x1 sky


def test_light_selection_rule():
    # env off, default weights: the emitter rule (P_e = 0.5, or 1 with the analytic lights dark)
    assert select(True, True, False) == (0.5, 0.0, 0.5, 0.0)
    assert select(False, True, False) == (1.0, 0.0, 1.0, 1.0)
    assert select(True, False, True) == (0.0, 0.5, 0.5, 0.0)
    assert select(False, False, True) == (0.0, 1.0, 1.0, 1.0)
    assert select(False, False, False) == (0.0, 0.0, 0.0, 0.0)
    f = np.float32
    pe, pv, pev, na = select(True, True, True, SKEW)
    s = (f(SKEW[0]) + f(SKEW[1])) + f(SKEW[2])
    assert (pe, pv, pev, na) == (float(f(SKEW[1]) / s), float(f(SKEW[2]) / s), float(f(f(SKEW[1]) / s) + f(f(SKEW[2]) / s)), 0.0)


@pytest.mark.parametrize("sky", ["shipped", "sun"])
def test_density_integrates_to_p_v(sky):
    env, w, h = shipped()
    if sky == "sun":
        env = sun_sky(env, w, h)
    p_v = 0.25
    _, _, pdf = env_table(env, w, h, p_v)
    # 2 x 2 directions per texel at the midpoints of its quarters: sum of p_v(dir) * d(omega), d(omega) = 2 pi^2 sin(theta) du dv
    k = 2
    u = (np.arange(w * k) + 0.5) / (w * k)
    v = (np.arange(h * k) + 0.5) / (h * k)
    uu, vv = np.meshgrid(u, v)
    phi, theta = uu * 2 * np.pi - np.pi, vv * np.pi
    d = np.stack([np.sin(theta) * np.sin(phi), np.sin(theta) * np.cos(phi), np.cos(theta)], -1).reshape(-1, 3)
    p = env_pdf(pdf, d).astype(np.float64)
    integral = (p * 2 * np.pi ** 2 * np.sin(theta).reshape(-1)).sum() / (w * k * h * k)
    assert abs(integral - p_v) < 1e-3 * p_v, integral


@pytest.mark.parametrize("sky", ["shipped", "sun"])
def test_samples_land_in_their_cell(sky):
    env, w, h = shipped()
    if sky == "sun":
        env = sun_sky(env, w, h)
    marg, cond, pdf = env_table(env, w, h)
    rng = np.random.default_rng(3)
    r = rng.random((200000, 4), dtype=np.float32)
    d = env_sample(marg, cond, r).astype(np.float64)
    j = np.searchsorted(marg, np.minimum(r[:, 0], np.float32(0.99999994)), side="right")
    i = np.array([np.searchsorted(cond[jj], x, side="right") for jj, x in zip(j, np.minimum(r[:, 1], np.float32(0.99999994)))])
    assert np.all(pdf[j, i] > 0)                       # only cells with weight are drawn
    cu = (np.arctan2(d[:, 0], d[:, 1]) + np.pi) / (2 * np.pi) * w
    cv = np.arccos(np.clip(d[:, 2], -1, 1)) / np.pi * h
    # away from cell borders (where the float rounding of the walk and the mapping may move it a texel) every direction lies in
    # the drawn cell
    inner = (np.abs(cu - np.round(cu)) > 1e-3) & (np.abs(cv - np.round(cv)) > 1e-3)
    assert inner.mean() > 0.99
    assert np.array_equal(np.floor(cu[inner]).astype(int) % w, i[inner])
    assert np.array_equal(np.floor(cv[inner]).astype(int), j[inner])
    # the density of the directions drawn: p_v(dir) equals the drawn cell's density in sin(theta)-weighted solid angle
    p = env_pdf(pdf, d)
    st = np.sqrt(np.maximum(1 - d[:, 2] ** 2, 0))
    assert np.allclose(p[inner] * 2 * np.pi ** 2 * st[inner], pdf[j, i][inner], rtol=1e-4)


@pytest.mark.parametrize("name", ["CornellBox", "ShaderBalls", "procedural"])
def test_model_inactive_cases_equal_emitter_model_and_oracle(name):
    sc = get_scene(name)
    m = LightModel(sc)
    w, h = 24, 16
    cam = default_camera(w, h)
    for s in range(2):
        # both options off: the oracle
        a, _, sa = m.render(cam, w, h, 3, s)
        b, _, sb = m.render(cam, w, h, 3, s, model=True)
        assert np.array_equal(bits(a), bits(b)) and sa.tobytes() == sb.tobytes()
        # environment off, default weights: the emitter model
        a, _, sa = m.render(cam, w, h, 3, s, emitters=True, model=True)
        b, _, sb = EmitterModel_render(sc, cam, w, h, 3, s)
        assert np.array_equal(bits(a), bits(b)) and sa.tobytes() == sb.tobytes()
        # white furnace: the environment table is inactive
        a, _, sa = m.render(cam, w, h, 3, s, white_furnace=True)
        b, _, sb = m.render(cam, w, h, 3, s, white_furnace=True, env=True, weights=SKEW)
        assert np.array_equal(bits(a), bits(b)) and sa.tobytes() == sb.tobytes()


def EmitterModel_render(sc, cam, w, h, mb, s):
    from tests.emitter_model import EmitterModel
    return EmitterModel(sc).render(cam, w, h, mb, s, emitters=True)


def batch_means(m, cam, w, h, mb, n, batches, first=0, **kw):
    """Per-batch mean images of samples first .. first + n - 1, and the mean per-pixel variance of one sample (over the pixels
    whose radiance is finite: a few ShaderBalls paths produce NaN with every setting)."""
    out = np.zeros((batches, h, w, 3), np.float64)
    per = n // batches
    sq = np.zeros((h, w, 3), np.float64)
    for b in range(batches):
        acc = np.zeros((h, w, 3), np.float64)
        for s in range(first + b * per, first + (b + 1) * per):
            r = m.render(cam, w, h, mb, s, **kw)[0][..., :3].astype(np.float64)
            acc += r
            sq += r * r
        out[b] = acc / per
    mean = out.mean(0)
    return out, np.nanmean(sq / n - mean * mean)


def z_scores(on, off, w, h, batches):
    tile = lambda x: x.reshape(x.shape[0], h // 8, 8, w // 8, 8, 3).mean((2, 4))
    ton, toff = tile(on), tile(off)
    se = lambda t: t.std(0, ddof=1) / np.sqrt(batches)
    # tiles without noise (the sky seen directly) differ only by the rounding of the float accumulations: tiles whose standard
    # error is below 3e-4 of their value are left out
    var = se(ton) ** 2 + se(toff) ** 2
    z = (ton.mean(0) - toff.mean(0)) / np.sqrt(var)
    return z[np.isfinite(z) & (np.sqrt(var) > 3e-4 * np.abs(toff.mean(0)))]


@pytest.mark.parametrize("weights", ["default", "skewed"])
@pytest.mark.parametrize("name", ["ShaderBalls", "procedural", "ShaderBalls_sun"])
def test_same_expectation_as_the_option_off(name, weights):
    """Per 8x8 tile and channel, z = (m_on - m_off) / sqrt(se_on^2 + se_off^2), environment and emitter sampling on against both off.
    Under the sun sky the option-off arm is dominated by rare BSDF hits of the sun, whose batch means are far from normal at this
    sample count; there the reference arm is environment sampling alone at the default weights (a different mixture of strategies,
    so a bias that depends on the weights or on emitter sampling still shows)."""
    sun = name == "ShaderBalls_sun"
    sc = sun_scene("ShaderBalls") if sun else get_scene(name)
    m = LightModel(sc)
    w = h = 32
    cam = default_camera(w, h)
    n, batches = 1200, 20
    wts = SKEW if weights == "skewed" else (1.0, 1.0, 1.0)
    on, var_on = batch_means(m, cam, w, h, 3, n, batches, env=True, emitters=True, weights=wts)
    off, var_off = batch_means(m, cam, w, h, 3, n, batches, first=n, env=sun)
    z = z_scores(on, off, w, h, batches)
    assert z.size > 0
    print("%s %s: %d tiles x channels, max |z| %.2f, mean z^2 %.2f; mean per-pixel variance on %.4g, off %.4g"
          % (name, weights, z.size, np.abs(z).max(), np.mean(z * z), var_on, var_off))
    assert np.all(np.abs(z) < 5)
    assert 0.5 <= np.mean(z * z) <= 2.0


@pytest.mark.parametrize("sky", ["shipped", "sun"])
def test_noise_at_equal_samples(sky):
    """Per-pixel variance at equal samples, environment sampling alone on against off, on ShaderBalls.  Under the sun sky it must
    fall; the shipped sky's numbers are printed whatever they are."""
    sc = sun_scene("ShaderBalls") if sky == "sun" else get_scene("ShaderBalls")
    m = LightModel(sc)
    w = h = 32
    cam = default_camera(w, h)
    n, batches = 400, 4
    _, var_on = batch_means(m, cam, w, h, 3, n, batches, env=True)
    _, var_off = batch_means(m, cam, w, h, 3, n, batches)
    print("ShaderBalls, %s sky: mean per-pixel variance env on %.4g, off %.4g" % (sky, var_on, var_off))
    if sky == "sun":
        assert var_on < 0.5 * var_off
