"""
The BSDF sampler against the density and the integrand the sampled lights weigh it with (include/rt_b200.h,
RT_OPT_EMITTER_SAMPLING / RT_OPT_ENV_SAMPLING; rt_device.cuh sample_bxdf and bxdf_eval_sampled, held bit for bit to the CPU copies
this file calls).  MIS weights sum to 1 whatever p_b is, so a wrong p_b only adds noise to the frame-level expectation tests, and
a wrong g biases every light sample: here, per material and shading point,

- the directions sample_bxdf draws have the density p_b (chi-square on an equal-area grid, expected counts from p_b integrated
  by adaptive Gauss-Legendre quadrature in float64),
- the fraction with pdf > 0 is the integral of p_b (the support),
- the mean of bxdf / pdf is the integral of g,
- p_b and g equal an independent float64 restatement (tests/analytic_light.py),

with negative controls showing that the chi-square and the integrand test reject the usual mistakes.
"""
import numpy as np
import pytest
from scipy.stats import chi2

from tests import bsdf_harness as bh
from tests.analytic_light import Bsdf, directions, frame, integrate_cells, unpack, unpack_packed
from tests.helpers import scene

N_SAMPLES = 1 << 20
NC, NP = 40, 64                # cos theta x phi bins about the shading normal (equal area; an edge at the horizon)
ANGLES = (0.0, 0.5, 1.0, 1.3, 1.55)
TILTED = (0.3, -0.5, 0.8)
NORMALS = {"z": (0.0, 0.0, 1.0), "tilted": TILTED, "x_small": (0.0008, 0.6, 0.8)}     # |n.x| <= 0.001: tangent_frame's other axis


def unit64(v):
    v = np.asarray(v, np.float64)
    return v / np.linalg.norm(v)


def unit32(v):
    return unit64(v).astype(np.float32)


def grid_materials():
    """Packed-byte grid: roughness 26..255 x metalness 0 / 128 / 255 x ior 25 / 38 / 51, seeded coloured albedos."""
    rng = np.random.default_rng(11)
    out = []
    for r in (26, 64, 128, 255):
        for mt in (0, 128, 255):
            for ior in (25, 38, 51):
                d = tuple(int(x) for x in rng.integers(20, 256, 3))
                s = tuple(int(x) for x in rng.integers(20, 256, 3))
                out.append(("grid_r%d_m%d_i%d" % (r, mt, ior), unpack(d, s, r, mt, ior)))
    return out


def scene_materials():
    """Every distinct material of CornellBox, ShaderBalls and the procedural scene that reflects light (lamps with black albedos
    have no lobe weights, pass-through sheets are the edge-case tests')."""
    from tests.test_emitter_sampling_cpu import procedural_scene
    seen, out = set(), []
    for name, sc in (("CornellBox", scene("CornellBox")), ("ShaderBalls", scene("ShaderBalls")), ("procedural", procedural_scene())):
        for k, pm in enumerate(sc["materials"]):
            m = unpack_packed(pm)
            if m.tobytes() in seen or m[9] < 0.5 or (m[0:3].max() == 0 and m[4:7].max() == 0):
                continue
            seen.add(m.tobytes())
            out.append(("%s_%d" % (name, k), m))
    return out


MATERIALS = grid_materials() + scene_materials()
# one shading point per material, cycling through the incoming angles and the normals so that every pair occurs
CASES = [(name, m, ANGLES[k % len(ANGLES)], list(NORMALS)[(k // len(ANGLES)) % len(NORMALS)]) for k, (name, m) in enumerate(MATERIALS)]
# The sampling tests meet the most grazing angle at 1.45 rad: at 1.55 the specular lobe reaches o = -i, where p_b's 1 / (4 h.o) is
# singular, and the quadrature would need far more nodes than this suite's budget to hold the sphere total to 1e-6 there.  The
# pointwise test takes 1.55 itself.
SAMPLING_CASES = [(name, m, 1.45 if a == 1.55 else a, n) for name, m, a, n in CASES]
P_REJECT = 1e-6 / len(CASES)


def shading_point(angle, normal, azimuth=0.7):
    """(n, i) as float32: the normal and an incoming direction at `angle` from it."""
    n = unit32(NORMALS[normal])
    t, b = frame(n.astype(np.float64))
    i = unit32(np.sin(angle) * (np.cos(azimuth) * t + np.sin(azimuth) * b) + np.cos(angle) * n.astype(np.float64))
    return n, i


def draws(seed, n=N_SAMPLES):
    return np.random.default_rng(seed).random((n, 3), dtype=np.float32)


class Case:
    """One material at one shading point: samples, their histogram and the quadrature of the densities and integrands."""

    def __init__(self, mat, angle, normal, seed=0, n=N_SAMPLES):
        self.mat = mat
        self.n32, self.i32 = shading_point(angle, normal)
        self.nd, idd = unit64(self.n32), unit64(self.i32)
        self.t, self.b = frame(self.nd)
        self.ref = Bsdf(mat, self.nd, idd)
        s = draws(seed, n)
        o, pdf, f, _ = bh.sample(mat, self.n32, self.i32, s)
        self.N = n
        self.o, self.pdf, self.f = o.astype(np.float64), pdf, f.astype(np.float64)
        # the kernels' rule for a delta sample (the mirror lobe of alpha <= 1e-4): outside p_b and g, weighted by BSDF sampling alone
        _, _, spec_pdf, alpha = bh.eval_sampled(mat, self.n32, self.i32, self.n32[None, :])
        self.delta = (s[:, 0] <= spec_pdf[0]) & (alpha[0] <= np.float32(1e-4))
        self.pos = (pdf > 0) & ~self.delta
        self.ce = np.linspace(-1.0, 1.0, NC + 1)
        self.pe = np.linspace(-np.pi, np.pi, NP + 1)

    def counts(self):
        o = self.o[self.pos]
        c = np.clip(o @ self.nd, -1.0, 1.0)
        phi = np.arctan2(o @ self.b, o @ self.t)
        ic = np.clip(np.searchsorted(self.ce, c, side="right") - 1, 0, NC - 1)
        ip = np.clip(np.searchsorted(self.pe, phi, side="right") - 1, 0, NP - 1)
        return np.bincount(ic * NP + ip, minlength=NC * NP).astype(np.float64)

    def integrals(self):
        """Per bin: [product p_b, product g rgb, reference p_b, reference g rgb, p_b without the Jacobian, p_b with the cos^2
        diffuse density, g without Fresnel rgb], integrated in float64."""
        if hasattr(self, "_int"):
            return self._int

        def f(c, p):
            d = directions(c, p, self.nd, self.t, self.b)
            g, pb, _, _ = bh.eval_sampled(self.mat, self.n32, self.i32, d.astype(np.float32))
            rp, rg = self.ref.terms(d)
            nj, _ = self.ref.terms(d, jacobian=False)
            c2, _ = self.ref.terms(d, diffuse_cos2=True)
            _, nf = self.ref.terms(d, fresnel=False)
            return np.concatenate([pb[:, None], g, rp[:, None], rg, nj[:, None], c2[:, None], nf], 1).astype(np.float64)
        c0, p0 = np.meshgrid(self.ce[:-1], self.pe[:-1], indexing="ij")
        c1, p1 = np.meshgrid(self.ce[1:], self.pe[1:], indexing="ij")
        self._int = integrate_cells(f, c0.ravel(), c1.ravel(), p0.ravel(), p1.ravel(), tol=3e-7, check=np.arange(4, 13), max_depth=12,
                                    must_split=self.near_lobe)
        return self._int

    def near_lobe(self, r):
        """Rectangles (theta0, theta1, phi0, phi1) wider than half the specular lobe (~2 alpha about the mirror direction) that
        come within a few lobe widths of it."""
        if not self.ref.rough:
            return np.zeros(len(r), bool)
        width = 2 * self.ref.alpha
        i = self.ref.i
        mirror = 2 * (i @ self.nd) * self.nd - i
        tc, pc = (r[:, 0] + r[:, 1]) / 2, (r[:, 2] + r[:, 3]) / 2
        centre = directions(np.cos(tc), pc, self.nd, self.t, self.b)
        dist = np.arccos(np.clip(centre @ mirror, -1, 1))
        size = np.maximum(r[:, 1] - r[:, 0], (r[:, 3] - r[:, 2]) * np.sin(np.minimum(r[:, 1], np.pi / 2)))
        return (size > width / 2) & (dist < size + 4 * width)
        return self._int


def chi2_test(case, density_col):
    """chi-square statistic, degrees of freedom and p-value of the bin counts of the samples with pdf > 0 against their number
    times the share of each bin in the integral of a density (the shape of the density; the mass test checks its total), the
    bins expecting fewer than 5 pooled."""
    obs = case.counts()
    I = case.integrals()[:, density_col]
    if I.sum() == 0:                                          # no non-delta lobe: no sample may land anywhere
        return float(obs.sum() * 1e300), 0, float(obs.sum() == 0)
    e = obs.sum() * I / I.sum()
    small = e < 5
    o_b = np.concatenate([obs[~small], [obs[small].sum()]])
    e_b = np.concatenate([e[~small], [e[small].sum()]])
    if e_b[-1] < 5:                                           # fold a pooled remainder that is still small into the smallest bin
        k = np.argmin(e_b[:-1])
        o_b[k] += o_b[-1]; e_b[k] += e_b[-1]
        o_b, e_b = o_b[:-1], e_b[:-1]
    stat = float(np.sum((o_b - e_b) ** 2 / e_b))
    dof = len(e_b) - 1
    return stat, dof, float(chi2.sf(stat, dof))


@pytest.mark.parametrize("name,mat,angle,normal", SAMPLING_CASES, ids=[c[0] for c in SAMPLING_CASES])
def test_sampler_density_support_and_integrand(name, mat, angle, normal):
    case = Case(mat, angle, normal)
    I = case.integrals()
    ref = case.ref
    # quadrature self-check: the reference density's sphere total against the analytic mass (to 1e-5: near o = -i, which rough
    # and grazing lobes reach, p_b's 1 / (4 h.o) is singular and the (theta, phi) rule converges slowly)
    mass = ref.mass()
    assert abs(I[:, 4].sum() - mass) < 1e-5, (I[:, 4].sum(), mass)
    # chi-square: the sampler's directions have the density p_b
    stat, dof, p = chi2_test(case, 0)
    # mass: the fraction of samples with pdf > 0 is the integral of p_b (binomial, 5 sigma)
    frac = case.pos.mean()
    sig = np.sqrt(max(mass * (1 - mass), 1.0 / case.N) / case.N)
    # integrand: the mean of bxdf / pdf (0 where pdf <= 0) is the integral of the float64 g, per channel (5 sigma; the standard
    # error is floored at 1e-6 of the integral for the Lambert-like materials, whose estimate has no variance but float rounding)
    est = np.where(case.pos[:, None], case.f / np.where(case.pos, case.pdf, 1.0)[:, None], 0.0)
    mean, se = est.mean(0), est.std(0) / np.sqrt(case.N)
    want = I[:, 5:8].sum(0)
    z = (mean - want) / np.maximum(se, 1e-6 * np.abs(want) + 1e-12)
    print("%s angle %.2f normal %s: chi2 %.0f / %d dof (p %.3g), mass %.6f vs %.6f (%.1f sigma), integrand z %s"
          % (name, angle, normal, stat, dof, p, frac, mass, (frac - mass) / sig, np.round(z, 2)))
    assert p > P_REJECT, (stat, dof, p)
    assert abs(frac - mass) < 5 * sig
    assert np.all(np.abs(z) < 5), z
    # the product's density integrates to the same mass.  Its float rounding is far below the statistics but for the sharpest
    # lobes, where D's denominator n.h^2 (alpha^2 - 1) + 1 loses ~1e-3 to the rounding of n.h (the MIS weights still sum to 1)
    assert abs(I[:, 0].sum() - mass) < 2e-3 * max(mass, 1e-3)


@pytest.mark.parametrize("name,mat,angle,normal", CASES, ids=[c[0] for c in CASES])
def test_pointwise_against_float64_restatement(name, mat, angle, normal):
    """The model's float p_b and g (bxdf_eval_sampled's CPU copy) equal the float64 restatement to 1e-4 relative wherever the value
    is above 1e-3 of its maximum, beyond what the float rounding of n.h allows where the GGX lobe is sharp."""
    n32, i32 = shading_point(angle, normal)
    nd = unit64(n32)
    t, b = frame(nd)
    rng = np.random.default_rng(5)
    # directions spread over the sphere plus a cluster about the mirror direction, where sharp lobes live
    d = rng.normal(size=(200000, 3))
    mirror = 2 * (i32.astype(np.float64) @ nd) * nd - i32
    m2 = mirror + rng.normal(size=(200000, 3)) * (mat[3] ** 2) * rng.uniform(0.1, 4, (200000, 1))
    d = np.concatenate([d, m2])
    d32 = (d / np.linalg.norm(d, axis=1)[:, None]).astype(np.float32)
    g, pb, spec_pdf, alpha = bh.eval_sampled(mat, n32, i32, d32)
    ref = Bsdf(mat, nd, unit64(i32))
    rp, rg = ref.terms(d32.astype(np.float64))
    assert abs(spec_pdf[0] - ref.spec_pdf) < 1e-5 and abs(alpha[0] - ref.alpha) < 1e-6 * max(ref.alpha, 1e-3)
    # conditioning of the float evaluation: D depends on n.h through 1 - (n.h)^2, which float rounding of n.h moves by ~2^-24
    hv = i32.astype(np.float64) + d32.astype(np.float64)
    nh = (hv / np.linalg.norm(hv, axis=1)[:, None]) @ nd
    a2 = ref.alpha ** 2
    den = nh * nh * (a2 - 1) + 1
    cond = np.where(ref.rough, 4 * np.abs(nh * nh * (a2 - 1)) / np.maximum(den, 1e-30), 0.0)
    # and h = normalize(i + o) loses the digits of i + o as o nears -i, where the specular density's 1 / (4 h.o) grows
    cond += np.where(ref.rough, 1.0 / np.maximum(1.0 + d32.astype(np.float64) @ unit64(i32), 1e-30), 0.0)
    # and g's cos_o = n.o, and the diffuse density with it, keep only the digits of n.o above its rounding near the horizon
    cond += 1.0 / np.maximum(np.abs(d32.astype(np.float64) @ nd), 1e-30)
    allow = 1e-4 + 8 * 2.0 ** -24 * cond
    # o = -i itself (where h = normalize(i + o) is undefined and 1 / (4 h.o) infinite) is left out
    away = np.arccos(np.clip(-(d32.astype(np.float64) @ unit64(i32)), -1, 1)) > 1e-3
    for got, want in ((pb.astype(np.float64), rp), *[(g[:, k].astype(np.float64), rg[:, k]) for k in range(3)]):
        big = (want > 1e-3 * want.max()) & away
        assert np.all(np.isfinite(got[big]))
        rel = np.abs(got[big] - want[big]) / want[big]
        assert np.all(rel <= allow[big]), (rel.max(), (rel / allow[big]).max())


def test_pass_through_materials_have_no_density():
    mat = unpack((200, 100, 50), (30, 30, 30), 128, 0, 38, transparency=64)
    n32, i32 = shading_point(0.5, "z")
    d = np.random.default_rng(1).normal(size=(1000, 3)).astype(np.float32)
    d /= np.linalg.norm(d, axis=1)[:, None]
    g, pb, _, _ = bh.eval_sampled(mat, n32, i32, d)
    assert np.all(g == 0) and np.all(pb == 0)
    o, pdf, f, off = bh.sample(mat, n32, i32, draws(2, 1000))
    assert np.all(pdf == 1) and np.all(off == -1) and np.array_equal(o, np.broadcast_to(-i32, o.shape))


@pytest.mark.parametrize("rbyte", [0, 2])
def test_delta_specular_is_outside_p_b_and_g(rbyte):
    """alpha <= 1e-4: no specular term in p_b or g.  The sampler's specular samples are the mirror direction (the delta lobe),
    drawn with probability spec_pdf, and the rest follow p_b, whose mass is diffuse_pdf."""
    mat = unpack((180, 120, 60), (200, 200, 200), rbyte, 128, 38)
    case = Case(mat, 0.8, "tilted", seed=3, n=1 << 19)
    assert not case.ref.rough
    mirror = 2 * (case.i32 @ case.n32) * case.n32 - case.i32
    assert np.all(np.linalg.norm(case.o[case.delta] - mirror, axis=1) < 1e-6)
    sig = np.sqrt(case.ref.spec_pdf * (1 - case.ref.spec_pdf) / case.N)
    assert abs(case.delta.mean() - case.ref.spec_pdf) < 5 * sig
    g, pb, _, _ = bh.eval_sampled(mat, case.n32, case.i32, mirror[None, :].astype(np.float32))
    rp, rg = case.ref.terms(mirror[None, :].astype(np.float64))
    assert np.allclose(pb, rp, rtol=1e-5) and np.allclose(g, rg, rtol=1e-5)
    assert abs(case.ref.mass() - case.ref.diffuse_pdf) < 1e-12
    assert abs(case.integrals()[:, 4].sum() - case.ref.diffuse_pdf) < 1e-6
    stat, dof, p = chi2_test(case, 0)
    assert p > P_REJECT, (stat, dof, p)


NEGATIVE = {"rough_metal": (unpack((200, 150, 100), (230, 180, 120), 128, 255, 38), 0.5, "tilted"),
            "diffuse": (unpack((200, 150, 100), (40, 40, 40), 255, 0, 38), 1.0, "z")}


@pytest.mark.parametrize("control", ["no_jacobian", "cos2_diffuse", "no_fresnel"])
def test_negative_controls_are_rejected(control):
    """The tests above have the power to see the usual mistakes: the chi-square rejects the reference's specular density without
    the 1/(4 h.o) Jacobian and a diffuse density of cos^2 theta 3 / (2 pi); the integrand test rejects g without Fresnel."""
    mat, angle, normal = NEGATIVE["diffuse" if control == "cos2_diffuse" else "rough_metal"]
    case = Case(mat, angle, normal)
    I = case.integrals()
    # the same samples pass against the reference's own density
    assert chi2_test(case, 4)[2] > P_REJECT
    if control == "no_fresnel":
        est = np.where(case.pos[:, None], case.f / np.where(case.pos, case.pdf, 1.0)[:, None], 0.0)
        se = est.std(0) / np.sqrt(case.N)
        z_ok = (est.mean(0) - I[:, 5:8].sum(0)) / se
        z_bad = (est.mean(0) - I[:, 10:13].sum(0)) / se
        print("%s: z against g %s, against g without Fresnel %s" % (control, np.round(z_ok, 2), np.round(z_bad, 1)))
        assert np.all(np.abs(z_ok) < 5) and np.all(np.abs(z_bad) > 5)
    else:
        stat, dof, p = chi2_test(case, 8 if control == "no_jacobian" else 9)
        print("%s: chi2 %.0f / %d dof, p %.3g" % (control, stat, dof, p))
        assert p < P_REJECT


@pytest.mark.parametrize("rbyte", [2, 3, 4])
def test_near_the_delta_threshold_everything_is_finite(rbyte):
    """Roughness bytes 2 (alpha 6.2e-5, a delta), 3 (alpha 1.4e-4: alpha^2 is below half an ulp of 1, so alpha^2 - 1 rounds to -1)
    and 4: p_b and g are never NaN, and finite wherever D's denominator n.h^2 (alpha^2 - 1) + 1 is not 0 (n.h rounding to 1 in
    float: the sampler's own pdf is infinite on those directions too, so the light strategies give them MIS weight 0)."""
    mat = unpack((180, 120, 60), (200, 200, 200), rbyte, 255, 38)
    for normal in NORMALS:
        n32, i32 = shading_point(0.6, normal)
        mirror = 2 * (unit64(i32) @ unit64(n32)) * unit64(n32) - unit64(i32)
        rng = np.random.default_rng(9)
        d = np.concatenate([rng.normal(size=(20000, 3)), mirror + rng.normal(size=(20000, 3)) * 1e-4, mirror[None, :]])
        d = (d / np.linalg.norm(d, axis=1)[:, None]).astype(np.float32)
        g, pb, _, _ = bh.eval_sampled(mat, n32, i32, d)
        assert not np.any(np.isnan(g)) and not np.any(np.isnan(pb)), (rbyte, normal)
        far = np.arccos(np.clip(d.astype(np.float64) @ mirror, -1, 1)) > 1e-3
        assert np.all(np.isfinite(g[far])) and np.all(np.isfinite(pb[far])), (rbyte, normal)
        assert np.array_equal(np.isinf(pb), np.isinf(g).any(1) | (np.isinf(pb) & (d.astype(np.float64) @ unit64(n32) <= 0)))
