"""
Independent float64 references for the sampled lights (include/rt_b200.h: RT_OPT_EMITTER_SAMPLING, RT_OPT_ENV_SAMPLING,
rt_set_light_selection).  Everything here is restated in numpy from the formulas stated in include/rt_b200.h and
raytracing_b200/csrc/rt_device.cuh; nothing calls the model or the library, so a formula written wrongly into both of them does
not pass by agreeing with itself.

- the BSDF: GGX D, the height-correlated Smith V, Schlick Fresnel at n.i times the specular albedo, the lobe weights, the density
  p_b of sample_bxdf's non-delta lobes and the integrand g it estimates (bxdf_eval_sampled), and evaluate_material, the BRDF the
  analytic-light samples weigh (Fresnel at h.o, dots clamped at RT_EPS);
- an adaptive Gauss-Legendre quadrature on (cos theta, phi) rectangles of the sphere, and the mass of p_b as a 1-D integral;
- known-answer scenes (a floor under lamps, a sky and a point light) and their per-pixel expectations.
"""
import numpy as np

RT_EPS = np.float32(1e-3)
LUMA = np.array([0.299, 0.587, 0.114])


# ------------------------------------------------------------------------------------------------------------------- materials
def unpack(diffuse=(0, 0, 0), specular=(0, 0, 0), roughness=255, metalness=0, ior=38, transparency=255):
    """The Material fields of packed bytes as the upload unpacks them (float32 byte / 255, ior byte / 25.5): diffuse rgb, roughness,
    specular rgb, metalness, ior, transparency."""
    f = np.float32
    d = [f(x) / f(255) for x in diffuse]
    s = [f(x) / f(255) for x in specular]
    return np.array(d + [f(roughness) / f(255)] + s + [f(metalness) / f(255), f(ior) / f(25.5), f(transparency) / f(255)], "<f4")


def unpack_packed(pm):
    """unpack() of a PackedMaterial record (untextured)."""
    rgb = lambda w: [(int(w) >> s) & 0xFF for s in (0, 8, 16)]
    rm, it = int(pm["roughness_metalness"]), int(pm["ior_emission_idx_transparency"])
    return unpack(rgb(pm["diffuse_albedo"]), rgb(pm["specular_albedo"]), rm & 0xFF, (rm >> 16) & 0xFF, it & 0xFF, (it >> 16) & 0xFF)


class Bsdf:
    """The BSDF of one material at one shading point (normal n, incoming direction i), in float64."""

    def __init__(self, mat, n, i):
        m = np.asarray(mat, np.float64)
        self.diffuse, self.roughness, self.specular = m[0:3], m[3], m[4:7]
        self.metalness, self.ior, self.transparency = m[7], m[8], m[9]
        self.n, self.i = np.asarray(n, np.float64), np.asarray(i, np.float64)       # i: (3,) or a batch (m, 3)
        self.alpha = self.roughness * self.roughness
        self.n_dot_i = self.i @ self.n
        f0d = ((self.ior - 1.0) / (self.ior + 1.0)) ** 2
        self.f0 = f0d + (self.specular - f0d) * self.metalness
        self.diffuse_albedo = (1.0 - self.metalness) * self.diffuse
        self.specular_albedo = self.specular + (1.0 - self.specular) * self.metalness
        # Schlick Fresnel at n.i times the specular albedo, and the lobe weights of sample_bxdf
        self.fresnel = (self.f0 + (1.0 - self.f0) * ((1.0 - self.n_dot_i) ** 5)[..., None]) * self.specular_albedo
        ws = (self.specular_albedo * self.fresnel) @ LUMA
        wd = (self.diffuse_albedo * (1.0 - self.fresnel)) @ LUMA
        self.spec_pdf, self.diffuse_pdf = ws / (ws + wd), wd / (ws + wd)
        self.rough = self.alpha > 1e-4              # alpha <= 1e-4: the specular lobe is a delta (mirror), outside p_b and g
        self.pass_through = self.transparency < 0.5

    def terms(self, o, fresnel=True, jacobian=True, diffuse_cos2=False):
        """p_b(o) and g(o) (rgb) for unit directions o (q, 3), or (m, q, 3) with a batch of m incoming directions.  The keywords
        build the wrong densities and integrands the negative controls feed the tests: no 1/(4 h.o) Jacobian, a cos^2 diffuse
        density, no Fresnel factor on g's specular term."""
        o = np.asarray(o, np.float64)
        if self.pass_through:
            return np.zeros(o.shape[:-1]), np.zeros(o.shape)
        ex = lambda a: np.asarray(a)[..., None]                  # per incoming direction -> broadcast over the q directions
        cos_o = o @ self.n
        c = np.maximum(cos_o, 0.0)
        pd = c * c * 1.5 / np.pi if diffuse_cos2 else c / np.pi
        p = ex(self.diffuse_pdf) * pd
        g = ((1.0 - self.fresnel) * self.diffuse_albedo / np.pi)[..., None, :] * c[..., None]
        if self.rough:
            hv = self.i[..., None, :] + o
            hl = np.linalg.norm(hv, axis=-1)
            h = hv / np.where(hl > 0, hl, 1.0)[..., None]
            n_dot_h, h_dot_o = h @ self.n, np.sum(h * o, axis=-1)
            ok = (n_dot_h > 0) & (h_dot_o > 0)
            d = ggx_d(self.alpha, n_dot_h)
            jac = 1.0 / (4.0 * np.where(ok, h_dot_o, 1.0)) if jacobian else 1.0
            p = p + np.where(ok, ex(self.spec_pdf) * d * n_dot_h * jac, 0.0)
            v = v_smith_ggx_correlated(ex(self.n_dot_i), np.where(c > 0, cos_o, 1.0), self.alpha)
            spec = np.where(ok & (c > 0), d * v * c, 0.0)
            g = g + (self.fresnel[..., None, :] if fresnel else 1.0) * spec[..., None]
        return p, g

    def mass(self):
        """The integral of p_b over the sphere: diffuse_pdf + spec_pdf * P(i.h > 0) for half vectors h drawn with density
        D(h) n.h, as a 1-D integral over the sampler's variable s (tan^2 theta_h = alpha^2 s / (1 - s), phi_h uniform)."""
        if self.pass_through:
            return 0.0
        if not self.rough:
            return self.diffuse_pdf
        from scipy.integrate import quad
        ti = np.arccos(np.clip(self.n_dot_i, -1, 1))
        a2 = self.alpha ** 2

        def frac(s):       # the fraction of phi_h with i.h = sin ti sin th cos phi + cos ti cos th > 0
            th = np.arctan(np.sqrt(a2 * s / (1.0 - s))) if s < 1.0 else np.pi / 2
            a, b = np.sin(ti) * np.sin(th), np.cos(ti) * np.cos(th)
            return 1.0 if b >= a else np.arccos(-b / a) / np.pi
        brk = []
        if ti > 1e-9:
            t2 = 1.0 / np.tan(ti) ** 2          # b = a at tan th = cot ti
            brk = [t2 / (a2 + t2)]
        p_h = quad(frac, 0.0, 1.0, points=brk or None, epsabs=1e-13, epsrel=1e-13, limit=400)[0]
        return self.diffuse_pdf + self.spec_pdf * p_h


def ggx_d(alpha, n_dot_h):
    a2 = alpha * alpha
    d = n_dot_h * n_dot_h * (a2 - 1.0) + 1.0
    return a2 / np.pi / (d * d)


def v_smith_ggx_correlated(n_dot_i, n_dot_o, alpha):
    a2 = alpha * alpha
    lv = n_dot_o * np.sqrt(n_dot_i * n_dot_i * (1.0 - a2) + a2)
    ll = n_dot_i * np.sqrt(n_dot_o * n_dot_o * (1.0 - a2) + a2)
    return 0.5 / (lv + ll)


def evaluate_material(mat, n, i, o):
    """evaluate_material (rt_device.cuh, material.h:132-169): Fresnel at h.o without the specular albedo, dots clamped at RT_EPS;
    (m, 3) directions o and one or (m, 3) incoming directions i -> (m, 3)."""
    m = np.asarray(mat, np.float64)
    o = np.asarray(o, np.float64).reshape(-1, 3)
    n, i = np.asarray(n, np.float64), np.broadcast_to(np.asarray(i, np.float64), o.shape)       # one incoming direction per o
    if m[9] < 0.5:
        return np.zeros((len(o), 3))
    eps = float(RT_EPS)
    h = i + o
    h = h / np.linalg.norm(h, axis=1)[:, None]
    n_dot_i = np.maximum(i @ n, eps)
    n_dot_o = np.maximum(o @ n, eps)
    n_dot_h = np.maximum(h @ n, eps)
    h_dot_o = np.maximum(np.sum(h * o, axis=1), eps)
    alpha = m[3] * m[3]
    f0d = ((m[8] - 1.0) / (m[8] + 1.0)) ** 2
    f0 = f0d + (m[4:7] - f0d) * m[7]
    fres = f0[None, :] + (1.0 - f0[None, :]) * ((1.0 - h_dot_o) ** 5)[:, None]
    spec = ggx_d(alpha, n_dot_h) * v_smith_ggx_correlated(n_dot_i, n_dot_o, alpha)
    return fres * spec[:, None] + (1.0 - fres) * ((1.0 - m[7]) * m[0:3] / np.pi)[None, :]


# ------------------------------------------------------------------------------------------------------------------ quadrature
def frame(n):
    """An orthonormal frame (t, b) about the unit vector n (any frame: the (cos theta, phi) grid is equal-area in each)."""
    n = np.asarray(n, np.float64)
    a = np.array([1.0, 0.0, 0.0]) if abs(n[0]) < 0.9 else np.array([0.0, 1.0, 0.0])
    t = np.cross(a, n); t /= np.linalg.norm(t)
    return t, np.cross(n, t)


def directions(c, phi, n, t, b):
    s = np.sqrt(np.maximum(1.0 - c * c, 0.0))
    return (s * np.cos(phi))[..., None] * t + (s * np.sin(phi))[..., None] * b + c[..., None] * n


def integrate_cells(f, c0, c1, p0, p1, tol, check=None, k=6, max_depth=14, must_split=None):
    """Integrals of f (callable: (m,) cos theta, (m,) phi -> (m, q)) over the rectangles [c0, c1] x [p0, p1] of (cos theta, phi),
    by Gauss-Legendre with k x k nodes in (theta, phi) (d omega = sin theta d theta d phi: smooth at the poles, where cos theta is
    not a smooth coordinate), splitting a rectangle in four until the rule on it and on its quarters agree within
    tol * (its solid angle / 4 pi) in the components `check` (all by default; leave out float-valued components, whose rounding
    noise never settles).  must_split(rects) -> bool array forces the split of rectangles (theta0, theta1, phi0, phi1) that may
    hold a feature narrower than the rule's nodes (a sharp lobe the rule on the rectangle and on its quarters could both miss)."""
    x, w = np.polynomial.legendre.leggauss(k)
    x, w = (x + 1.0) / 2.0, w / 2.0
    ww = (w[:, None] * w[None, :]).reshape(-1)

    def rule(r):
        parts = []
        for s in range(0, len(r), 16384):
            q = r[s:s + 16384]
            dt, dp = q[:, 1] - q[:, 0], q[:, 3] - q[:, 2]
            tt = (q[:, 0:1, None] + dt[:, None, None] * x[None, :, None]) * np.ones((1, 1, k))
            pp = (q[:, 2:3, None] + dp[:, None, None] * x[None, None, :]) * np.ones((1, k, 1))
            tt, pp = tt.reshape(-1), pp.reshape(-1)
            v = (f(np.cos(tt), pp) * np.sin(tt)[:, None]).reshape(len(q), k * k, -1)
            parts.append(np.einsum("j,ijq->iq", ww, v) * (dt * dp)[:, None])
        return np.concatenate(parts)

    def quarters(r):
        cm, pm = (r[:, 0] + r[:, 1]) / 2, (r[:, 2] + r[:, 3]) / 2
        q = [np.stack(v, 1) for v in ((r[:, 0], cm, r[:, 2], pm), (cm, r[:, 1], r[:, 2], pm), (r[:, 0], cm, pm, r[:, 3]), (cm, r[:, 1], pm, r[:, 3]))]
        return np.stack(q, 1).reshape(-1, 4)

    rects = np.stack([np.arccos(np.clip(np.asarray(v, np.float64), -1, 1)) for v in (c1, c0)]
                     + [np.asarray(v, np.float64) for v in (p0, p1)], 1)
    ids = np.arange(len(rects))
    whole = rule(rects)
    out = np.zeros_like(whole)
    for depth in range(max_depth):
        if len(rects) == 0:
            break
        ch = quarters(rects)
        sub = rule(ch)
        sums = sub.reshape(len(rects), 4, -1).sum(1)
        area = (np.cos(rects[:, 0]) - np.cos(rects[:, 1])) * (rects[:, 3] - rects[:, 2])
        err = np.abs(sums - whole) if check is None else np.abs(sums - whole)[:, check]
        done = np.all(err <= tol * area[:, None] / (4 * np.pi), axis=1)
        if must_split is not None:
            done &= ~must_split(rects)
        done |= depth == max_depth - 1
        np.add.at(out, ids[done], sums[done])
        keep = np.repeat(~done, 4)
        rects, whole, ids = ch[keep], sub[keep], np.repeat(ids, 4)[keep]
    return out


# ------------------------------------------------------------------------------------------------------------ known-answer scenes
# A large floor at z = 0 (normal +z) under two lamps that face down: a rectangle at z = 1 and a tilted triangle higher up and far
# enough to the side that, from every floor point the camera sees, neither lamp hides the other.  Lamp materials reflect nothing
# (black albedos, roughness 0: evaluate_material and g are 0, and sample_bxdf's pdf is NaN), so a path that reaches a lamp ends
# there.  The camera looks down from above the lamps, whose back faces the traversal culls: every primary ray hits the floor, and
# the floor sees only lamps, sky and the point light.
RECT = ((-1.6, -0.3), (-0.8, 0.3), 1.0)             # x range, y range, height
TILTED_TRI = ((1.0, -0.4, 1.2), (1.6, -0.2, 1.4), (1.2, 0.4, 1.35))
POINT = (0.3, 0.8, 0.7)                             # below both lamps: they cannot shadow it
CAMERA = dict(position=(0.0, 0.0, 3.0), yaw=1.5707964, pitch=2.95)
FLOORS = {"lambert": dict(diffuse=(170, 120, 60), specular=(0, 0, 0), roughness=255, metalness=0, ior=38),
          "ggx": dict(diffuse=(90, 90, 90), specular=(230, 180, 120), roughness=128, metalness=255, ior=38)}
LAMP_RGB = {"rect": (4.0, 3.0, 2.0), "tri": (1.0, 2.5, 6.0)}
LAMP_TEXELS = ((255, 255, 255), (255, 128, 40), (60, 200, 255), (140, 140, 140))   # 2x2, row-major from the top row of the image


def rgbe(rgb):
    """Packed RGBE emission (UnpackRGBE: mantissa bytes * 2^(e - 136)) of an exactly representable colour."""
    e = 136
    while max(rgb) * 2.0 ** (136 - e) >= 256:
        e += 1
    while max(rgb) * 2.0 ** (136 - e) < 128:
        e -= 1
    m = [int(round(c * 2.0 ** (136 - e))) for c in rgb]
    assert all(abs(mm * 2.0 ** (e - 136) - c) < 1e-12 for mm, c in zip(m, rgb))
    return m[0] | (m[1] << 8) | (m[2] << 16) | (e << 24)


def packed(diffuse=(0, 0, 0), specular=(0, 0, 0), roughness=255, metalness=0, ior=38, emission=None, emission_tex=0xFF):
    rgb = lambda c: int(c[0]) | (int(c[1]) << 8) | (int(c[2]) << 16) | (0xFF << 24)
    return (rgb(diffuse), rgb(specular), rgbe(emission) if emission else 0, (roughness & 0xFF) | (0xFF << 8) | (metalness << 16) | (0xFF << 24),
            (ior & 0xFF) | (emission_tex << 8) | (255 << 16) | (0xFF << 24))


def lamp_triangles():
    """(positions (3, 3), uvs (3, 2), lamp name) of the lamp triangles, wound so that the geometric normal points down."""
    (x0, x1), (y0, y1), z = RECT[0], RECT[1], RECT[2]
    c = {(0, 0): (x0, y0), (1, 0): (x1, y0), (1, 1): (x1, y1), (0, 1): (x0, y1)}
    rect = []
    for tri in (((0, 0), (0, 1), (1, 1)), ((0, 0), (1, 1), (1, 0))):
        rect.append((np.array([c[k] + (z,) for k in tri]), np.array(tri, np.float64), "rect"))
    p = np.array(TILTED_TRI, np.float64)
    if np.cross(p[1] - p[0], p[2] - p[0])[2] > 0:
        p = p[[0, 2, 1]]
    return rect + [(p, np.zeros((3, 2)), "tri")]


def known_answer_scene(floor="lambert", sky=None, point=0.0, textured=False):
    """The scene dict: floor material `floor`, sky an RGBA32F image (h, w, 4) or None for black, the point light's radiance
    (0: dark, as rt_upload_scene needs one light), the rectangle lamp with a 2x2 emission texture aligned with its uv."""
    from raytracing_b200 import hostapi
    from raytracing_b200.layouts import TEXTURE_DT
    from tests.helpers import scene as fixture
    base = fixture("CornellBox")
    tdt, mdt = base["triangles"].dtype, base["materials"].dtype
    mats = np.zeros(3, mdt)
    for k, m in enumerate([packed(**FLOORS[floor]), packed(emission=LAMP_RGB["rect"], roughness=0, emission_tex=0 if textured else 0xFF),
                           packed(emission=LAMP_RGB["tri"], roughness=0)]):
        mats[k] = m
    L = 20.0
    tris = []
    for q in (((-L, -L), (L, -L), (L, L)), ((-L, -L), (L, L), (-L, L))):
        tris.append((np.array([v + (0.0,) for v in q]), np.zeros((3, 2)), 0, (0.0, 0.0, 1.0)))
    for p, uv, name in lamp_triangles():
        tris.append((p, uv, 1 if name == "rect" else 2, tuple(np.cross(p[1] - p[0], p[2] - p[0]) / np.linalg.norm(np.cross(p[1] - p[0], p[2] - p[0])))))
    arr = np.zeros(len(tris), tdt)
    for k, (p, uv, mtl, nrm) in enumerate(tris):
        for j, v in enumerate(("v1", "v2", "v3")):
            arr[v]["position"][k, :3] = p[j]
            arr[v]["texcoord"][k, :2] = uv[j]
            arr[v]["normal"][k, :3] = nrm
        arr["mtlIndex"][k] = mtl
    ordered, nodes, _ = hostapi.build_bvh(arr)
    sc = {"triangles": ordered, "nodes": nodes, "materials": mats}
    sc["emissive"] = np.flatnonzero(ordered["mtlIndex"] > 0).astype("<u4")
    lights = np.zeros(1, base["lights"].dtype)
    lights[0]["origin"][:3] = POINT; lights[0]["radiance"][:3] = point; lights[0]["type"] = 0
    sc["lights"] = lights
    if textured:
        sc["textures"] = np.array([(0, 2, 2, 0)], dtype=TEXTURE_DT)
        sc["texels"] = np.array([r | (g << 8) | (b << 16) | (255 << 24) for r, g, b in LAMP_TEXELS], "<u4")
    else:
        sc["textures"], sc["texels"] = np.zeros(0, TEXTURE_DT), np.zeros(0, "<u4")
    info = np.array(base["scene_info"], copy=True)
    info["analytic_light_count"] = 1; info["emissive_count"] = len(sc["emissive"])
    sc["scene_info"] = info
    img = np.zeros((1, 1, 4), "<f4") if sky is None else np.asarray(sky, "<f4")
    sc["env"], sc["env_height"], sc["env_width"] = img.reshape(-1), img.shape[0], img.shape[1]
    return sc


def gradient_sky(w, h, sun=True, i_sun=5):
    """A sky with a vertical gradient (bright near the zenith, row 0) and a two-texel sun above the horizon.  The sun is a few
    times the sky, not orders of magnitude: the lamps hide it from some floor points, and the kinks of the bilinear lookup at its
    texel centres are what the lamp-area quadrature of the hidden sky must resolve."""
    v = (np.arange(h) + 0.5) / h
    img = np.zeros((h, w, 4), "<f4")
    img[..., 0], img[..., 1], img[..., 2] = (0.9 - 0.6 * v)[:, None], (1.0 - 0.6 * v)[:, None], (1.3 - 0.7 * v)[:, None]
    if sun and h >= 4 and w >= 4:
        j = max(h // 5, 1)
        img[j, i_sun:i_sun + 2, :3] = np.array([4.0, 3.6, 3.0], "<f4")
    return img


# --------------------------------------------------------------------------------------------------------------- references
def gl01(k):
    x, w = np.polynomial.legendre.leggauss(k)
    return (x + 1.0) / 2.0, w / 2.0


def primary(cam, w, h, k=4):
    """Floor points x (h, w, k*k, 3) and view directions d of generate_primary_ray (pinhole) at a k x k Gauss-Legendre grid of
    the sub-pixel jitter; the mean over the last axis with weights wt (k*k,) is the pixel's expectation."""
    x, wx = gl01(k)
    jx, jy = np.meshgrid(x, x, indexing="ij")
    wt = np.outer(wx, wx).reshape(-1)
    front, up, pos = [np.asarray(cam[f][:3], np.float64) for f in ("front", "up", "position")]
    right = np.cross(front, up)
    tanh = np.tan(0.5 * float(cam["fov"]))
    px = (np.arange(w)[None, :, None] + jx.reshape(-1)[None, None, :]) / w
    py = (np.arange(h)[:, None, None] + jy.reshape(-1)[None, None, :]) / h
    X = (px * 2 - 1) * tanh * float(cam["aspect_ratio"])
    Y = (py * 2 - 1) * tanh
    d = X[..., None] * right + Y[..., None] * up + front
    d = d / np.linalg.norm(d, axis=-1, keepdims=True)
    d = np.broadcast_to(d, (h, w, len(wt), 3))
    t = -pos[2] / d[..., 2]
    return pos + t[..., None] * d, d, wt


def polygon_form_factor(o, verts):
    """Lambert's closed form: (1 / 2 pi) sum_k beta_k (z . gamma_k) for points o (..., 3) with normal +z and a planar polygon; 0
    where the polygon turns its back (its normal points away from o)."""
    r = verts[None, :, :] - o.reshape(-1, 1, 3)
    r = r / np.linalg.norm(r, axis=-1, keepdims=True)
    tot = np.zeros(len(r))
    for k in range(len(verts)):
        a, b = r[:, k], r[:, (k + 1) % len(verts)]
        cr = np.cross(a, b)
        beta = np.arctan2(np.linalg.norm(cr, axis=-1), np.sum(a * b, -1))
        tot += beta * cr[:, 2] / np.linalg.norm(cr, axis=-1)
    nrm = np.cross(verts[1] - verts[0], verts[2] - verts[0])
    front = (o.reshape(-1, 3) - verts[0]) @ nrm > 0
    return (np.abs(tot) / (2 * np.pi) * front).reshape(o.shape[:-1])


def sky_radiance(img, u, v):
    """sample_sky restated in double at texture coordinates (u, v): bilinear, texel centres at +0.5, REPEAT on both axes."""
    h, w = img.shape[:2]
    U, V = (u - np.floor(u)) * w, (v - np.floor(v)) * h
    fu, fv = np.floor(U - 0.5), np.floor(V - 0.5)
    a, b = (U - 0.5 - fu)[..., None], (V - 0.5 - fv)[..., None]
    i0, j0 = fu.astype(int) % w, fv.astype(int) % h
    i1, j1 = (i0 + 1) % w, (j0 + 1) % h
    t = np.asarray(img, np.float64)[..., :3]
    return t[j0, i0] * (1 - a) * (1 - b) + t[j0, i1] * a * (1 - b) + t[j1, i0] * (1 - a) * b + t[j1, i1] * a * b


def sky_dir_radiance(img, d):
    u = (np.arctan2(d[..., 0], d[..., 1]) + np.pi) / (2 * np.pi)
    v = np.arccos(np.clip(d[..., 2], -1, 1)) / np.pi
    return sky_radiance(img, u, v)


def sky_irradiance(img, k=8):
    """The integral over the upper hemisphere of L_sky cos theta d omega: Gauss-Legendre on the cells between texel centres (where
    the bilinear lookup is smooth), d omega = 2 pi^2 sin theta du dv, theta = pi v, up to the horizon v = 1/2."""
    h, w = img.shape[:2]
    ue = np.unique(np.concatenate([[0.0, 1.0], (np.arange(w) + 0.5) / w]))
    ve = np.unique(np.concatenate([[0.0, 0.5], (np.arange(h) + 0.5) / h]))
    ve = ve[ve <= 0.5]
    x, wx = gl01(k)
    uu = (ue[:-1, None] + np.diff(ue)[:, None] * x[None, :]).reshape(-1)
    wu = (np.diff(ue)[:, None] * wx[None, :]).reshape(-1)
    vv = (ve[:-1, None] + np.diff(ve)[:, None] * x[None, :]).reshape(-1)
    wv = (np.diff(ve)[:, None] * wx[None, :]).reshape(-1)
    U, Vv = np.meshgrid(uu, vv, indexing="ij")
    W = np.outer(wu, wv)
    th = np.pi * Vv
    f = sky_radiance(img, U, Vv) * (2 * np.pi ** 2 * np.sin(th) * np.cos(th))[..., None]
    return np.einsum("ij,ijc->c", W, f)


def triangle_nodes(p, k):
    """Gauss-Legendre nodes (m, 3), weights (m,) (area measure) and barycentrics (m, 3) on triangle p (Duffy map of the square)."""
    x, wx = gl01(k)
    s, t = np.meshgrid(x, x, indexing="ij")
    s, t = s.reshape(-1), t.reshape(-1)
    b1, b2 = s * (1 - t), s * t
    area2 = np.linalg.norm(np.cross(p[1] - p[0], p[2] - p[0]))
    wts = np.outer(wx, wx).reshape(-1) * s * area2
    bc = np.stack([1 - b1 - b2, b1, b2], 1)
    return bc @ p, wts, bc


def lamp_emission(name, uv=None, textured=False):
    """L_e at lamp points: the material's constant emission times, on the textured rectangle, pow(texel / 255, 2.2) of the 2x2
    texture under uv (sample_texture: v flipped, nearest texel)."""
    le = np.array(LAMP_RGB[name], np.float64)
    if not (textured and name == "rect"):
        return np.broadcast_to(le, (1 if uv is None else len(uv), 3))
    tx = np.clip(np.floor(uv[:, 0] * 2), 0, 1).astype(int)
    ty = np.clip(np.floor((1 - uv[:, 1]) * 2), 0, 1).astype(int)
    tex = (np.array(LAMP_TEXELS, np.float64) / 255.0) ** 2.2
    return le * tex[ty * 2 + tx]


def rect_quarters():
    """The rectangle lamp's four constant sub-rectangles of the 2x2 texture: (vertices (4, 3), texel index)."""
    (x0, x1), (y0, y1), z = RECT[0], RECT[1], RECT[2]
    xm, ym = (x0 + x1) / 2, (y0 + y1) / 2
    out = []
    for tx, (a, b) in enumerate(((x0, xm), (xm, x1))):
        for ty, (c, d) in enumerate(((ym, y1), (y0, ym))):          # ty 0: uv.y in [1/2, 1] (top row of the image)
            out.append((np.array([(a, c, z), (a, d, z), (b, d, z), (b, c, z)]), ty * 2 + tx))
    return out


def expected_image(sc_kind, cam, w, h, k=4, lamp_k=12):
    """Per-pixel float64 expectation (h, w, 3) of the known-answer scene described by sc_kind = dict(floor=, sky=, point=,
    textured=) for every max_bounces >= 1."""
    floor, img, point, textured = sc_kind.get("floor", "lambert"), sc_kind.get("sky"), sc_kind.get("point", 0.0), sc_kind.get("textured", False)
    X, D, wt = primary(cam, w, h, k)
    eps = float(RT_EPS)
    O = X + np.array([0.0, 0.0, eps])
    mat = unpack(**FLOORS[floor])
    flat_o, flat_x, flat_d = O.reshape(-1, 3), X.reshape(-1, 3), D.reshape(-1, 3)
    m = len(flat_o)
    rad = np.zeros((m, 3))
    if floor == "lambert":
        rho = mat[0:3].astype(np.float64)
        for p, uv, name in lamp_triangles():
            if name == "rect" and textured:
                continue
            rad += rho / np.pi * np.pi * polygon_form_factor(flat_o, p)[:, None] * lamp_emission(name)[0]
        if textured:
            tex = (np.array(LAMP_TEXELS, np.float64) / 255.0) ** 2.2
            for verts, ti in rect_quarters():
                rad += rho * polygon_form_factor(flat_o, verts)[:, None] * (np.array(LAMP_RGB["rect"]) * tex[ti])
        if img is not None:
            hidden = np.zeros((m, 3))
            for p, uv, name in lamp_triangles():
                y, wy, _ = triangle_nodes(p, lamp_k)
                nl = np.cross(p[1] - p[0], p[2] - p[0]); nl /= np.linalg.norm(nl)
                for s in range(0, m, 4096):
                    r = y[None, :, :] - flat_o[s:s + 4096, None, :]
                    d2 = np.sum(r * r, -1)
                    om = r / np.sqrt(d2)[..., None]
                    cos_x, cos_y = om[..., 2], -(om @ nl)
                    hidden[s:s + 4096] += np.einsum("ij,ijc->ic", wy[None, :] * np.maximum(cos_x, 0) * np.maximum(cos_y, 0) / d2,
                                                    sky_dir_radiance(img, om))
            rad += rho / np.pi * (sky_irradiance(img)[None, :] - hidden)
    else:
        assert img is None and not textured
        for p, uv, name in lamp_triangles():
            y, wy, _ = triangle_nodes(p, lamp_k)
            nl = np.cross(p[1] - p[0], p[2] - p[0]); nl /= np.linalg.norm(nl)
            le = lamp_emission(name)[0]
            for s in range(0, m, 2048):
                r = y[None, :, :] - flat_o[s:s + 2048, None, :]
                d2 = np.sum(r * r, -1)
                om = r / np.sqrt(d2)[..., None]
                cos_y = np.maximum(-(om @ nl), 0)
                _, g = Bsdf(mat, (0.0, 0.0, 1.0), -flat_d[s:s + 2048]).terms(om)
                rad[s:s + 2048] += np.einsum("ijc,ij->ic", g, wy[None, :] * cos_y / d2) * le
    if point:
        r = np.array(POINT) - flat_x
        d2 = np.sum(r * r, -1)
        om = r / np.sqrt(d2)[:, None]
        rad += evaluate_material(mat, (0.0, 0.0, 1.0), -flat_d, om) * (point * np.maximum(om[:, 2], 0.0) / d2)[:, None]
    return np.einsum("k,ijkc->ijc", wt, rad.reshape(h, w, len(wt), 3))
