"""
A closest-hit and occlusion reference that knows nothing about the BVH: every ray against every triangle.

- closest() / any_hit(): the triangle test of trace_bvh.cl (rt_traverse.cuh trace_literal / trace_fast, oracle.cpp RayTriangle)
  restated in numpy float32, the same operations in the same order and no contraction: e1 = p2 - p1, e2 = p3 - p1,
  pvec = cross(d, e2), det = dot(e1, pvec), reject det < 1e-8, inv_det = 1 / det, u, v and t, inclusive bounds.  For each ray it
  gives the minimum accepted t and the tie set: every triangle accepted at exactly that t.
- classify(): a float64 evaluation of the same intersections that tags each ray with one class.  It never decides a verdict; it
  says which rule applies: `clean` (the nearest hit is more than 2^-20 from the next one and from its triangle's edges),
  `near_tie`, `near_edge`, or `near_box_face` (the hit lies within 2^-20 of a face of a box on its root-to-leaf path, where the
  float32 slab test may round a grazing interval to empty).
- verdict(): the rules a traversal's hits must meet (check them on the device's hits or the oracle's):
  a reported hit is accepted by the restatement with the same bits of (u, v, t); its t is the minimum t (so its triangle is in the
  tie set, and is the closest triangle where the tie set has one member); a miss or a farther hit is allowed only on a
  near_box_face ray, and those rays are counted.

dot(a, b) = (a.x * b.x + a.y * b.y) + a.z * b.z and cross as rt_device.cuh states them.  Every triangle is tested against every
ray; for scenes of more than 256 triangles a float64 bounding-sphere bound (padded by 2^-16 of the scene's scale, far beyond float32 rounding) first drops the pairs that cannot
meet, which changes no result (test_trace_reference_cpu.py checks that on a shipped scene).
"""
import hashlib

import numpy as np

from raytracing_b200.layouts import INVALID_ID

F = np.float32
EPS = 2.0 ** -20
CLASSES = ("clean", "near_tie", "near_edge", "near_box_face")


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def tri_points(tris):
    """-> p1, p2, p3 float32 (n, 3) of TRIANGLE_DT records."""
    return [np.ascontiguousarray(tris[v]["position"][:, :3], dtype=F) for v in ("v1", "v2", "v3")]


def ray_arrays(rays, t_min=None, t_max=None):
    """-> o, d float32 (n, 3), t_min, t_max float32 (n,): the ray's own origin.w / direction.w unless given."""
    o = np.ascontiguousarray(rays["origin"][:, :3], dtype=F)
    d = np.ascontiguousarray(rays["direction"][:, :3], dtype=F)
    lo = rays["origin"][:, 3] if t_min is None else np.broadcast_to(F(t_min) if np.isscalar(t_min) else t_min, len(rays))
    hi = rays["direction"][:, 3] if t_max is None else np.broadcast_to(F(t_max) if np.isscalar(t_max) else t_max, len(rays))
    return o, d, np.asarray(lo, F), np.asarray(hi, F)


def triangle_test(o, d, p1, p2, p3, t_min, t_max, sign=None):
    """The float32 test on matching rows (broadcast) -> accepted, u, v, t (u, v, t as computed; meaningful where accepted).
    sign (an instance's sign(det M), broadcast): the back-face test reads det * sign; u, v and t still divide by det."""
    with np.errstate(all="ignore"):
        e1, e2 = p2 - p1, p3 - p1
        pvec = _cross(d, e2)
        det = _dot(e1, pvec)
        ok = ~((det if sign is None else det * F(sign)) < F(1e-8))
        inv_det = F(1.0) / det
        tvec = o - p1
        u = _dot(tvec, pvec) * inv_det
        ok &= ~((u < F(0.0)) | (u > F(1.0)))
        qvec = _cross(tvec, e1)
        v = _dot(d, qvec) * inv_det
        ok &= ~((v < F(0.0)) | (u + v > F(1.0)))
        t = _dot(e2, qvec) * inv_det
        ok &= ~((t < t_min) | (t > t_max))
    return ok, u, v, t


def _near_spheres(c, rad, o, d, t_max):
    """(sphere, ray) pairs of rows whose ray line passes within the sphere (c, rad) at a t in [-rad, t_max + rad]; float64, d unit."""
    cd = ((c - o) * d).sum(-1)                                  # t of the point of the line nearest to c
    dist2 = np.maximum(((c - o) ** 2).sum(-1) - cd * cd, 0.0)
    return (dist2 <= rad * rad) & (cd >= -rad) & (cd <= t_max + rad)


def candidate_pairs(p, o, d, t_max, prefilter, chunk=1 << 21, block=64):
    """(ray, triangle) index pairs to test: all of them, or those whose line passes within the triangle's bounding sphere (float64,
    radius padded by 2^-16 of itself and of the scene's scale) at a t below the ray's t_max plus the radius.  The spheres are
    first tested in blocks of `block` consecutive triangles, each block under one sphere that holds its triangles' spheres: any
    grouping gives the same pairs, and consecutive triangles (leaf order) make the blocks small."""
    n_r, n_t = len(o), len(p[0])
    if not prefilter:
        step = max(1, chunk // max(n_t, 1))
        for a in range(0, n_r, step):
            r = np.arange(a, min(a + step, n_r))
            yield np.repeat(r, n_t), np.tile(np.arange(n_t), len(r))
        return
    q = [x.astype(np.float64) for x in p]
    c = (q[0] + q[1] + q[2]) / 3.0
    rad = np.sqrt(np.max([((x - c) ** 2).sum(1) for x in q], 0))
    scale = max(float(np.abs(np.concatenate(q)).max()), float(np.abs(o).max()), 1.0)
    rad = rad * (1 + 2.0 ** -16) + 2.0 ** -16 * scale
    n_b = (n_t + block - 1) // block
    first = np.arange(n_b) * block
    cb = np.add.reduceat(c, first, 0) / np.diff(np.append(first, n_t))[:, None]
    rb = np.maximum.reduceat(np.sqrt(((c - np.repeat(cb, block, 0)[:n_t]) ** 2).sum(1)) + rad, first) * (1 + 2.0 ** -16)
    oo, dd = o.astype(np.float64), d.astype(np.float64)
    dn = np.sqrt((dd * dd).sum(1))
    dd = dd / dn[:, None]
    tm = t_max.astype(np.float64) * dn
    step = max(1, chunk // max(n_b, 1))
    for a in range(0, n_r, step):
        s = slice(a, min(a + step, n_r))
        bi, ri = np.nonzero(_near_spheres(cb[:, None], rb[:, None], oo[None, s], dd[None, s], tm[None, s]))
        ri = ri + a
        ti = (bi[:, None] * block + np.arange(block)[None, :]).ravel()
        ri = np.repeat(ri, block)
        keep = ti < n_t
        ti, ri = ti[keep], ri[keep]
        near = _near_spheres(c[ti], rad[ti], oo[ri], dd[ri], tm[ri])
        yield ri[near], ti[near]


class Closest:
    """Per ray: t (the minimum accepted t, +inf if none), prim (the lowest id at that t, INVALID_ID if none), n_ties, and the
    tie pairs (tie_ray, tie_prim) with their (tie_u, tie_v) as the float32 test computes them (their t is the ray's t)."""

    def __init__(self, n):
        self.t = np.full(n, np.inf, F)
        self.prim = np.full(n, INVALID_ID, np.uint32)
        self.n_ties = np.zeros(n, np.int64)
        self.n_accepted = np.zeros(n, np.int64)


def closest(tris, rays, t_min=None, t_max=None, prefilter=None):
    o, d, lo, hi = ray_arrays(rays, t_min, t_max)
    p = tri_points(tris)
    if prefilter is None:
        prefilter = len(tris) > 256
    acc, pairs = [], []
    for r, ti in candidate_pairs(p, o, d, hi, prefilter):
        ok, u, v, t = triangle_test(o[r], d[r], p[0][ti], p[1][ti], p[2][ti], lo[r], hi[r])
        acc.append((r[ok], ti[ok], t[ok], u[ok], v[ok]))
        if prefilter:
            pairs.append((r, ti))
    out = reduce_accepted(len(o), acc)
    out.pairs = pairs or None                   # the prefilter's pairs, which classify() tests again in float64
    return out


def reduce_accepted(n, acc):
    """The Closest of n rays from the accepted (ray, prim, t, u, v) arrays of acc."""
    out = Closest(n)
    if acc:
        r, ti, t, u, v = (np.concatenate(x) for x in zip(*acc))
    else:
        r, ti, t, u, v = np.zeros(0, np.int64), np.zeros(0, np.uint32), np.zeros(0, F), np.zeros(0, F), np.zeros(0, F)
    ti = ti.astype(np.uint32)
    np.minimum.at(out.t, r, t)
    np.add.at(out.n_accepted, r, 1)
    tie = t == out.t[r]
    np.add.at(out.n_ties, r[tie], 1)
    out.tie_ray, out.tie_prim, out.tie_u, out.tie_v = r[tie], ti[tie], u[tie], v[tie]
    np.minimum.at(out.prim, r[tie], ti[tie])
    return out


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).view(np.uint8)).hexdigest()


def select(ref, part):
    """The Closest of the rays ref[part] (tie pairs left out)."""
    out = Closest(0)
    out.pairs = None
    out.t, out.prim, out.n_ties, out.n_accepted = ref.t[part], ref.prim[part], ref.n_ties[part], ref.n_accepted[part]
    return out


def any_hit(tris, rays, t_min=None, t_max=None, prefilter=None):
    """Occlusion: the ray accepts some triangle in [t_min, t_max]."""
    return closest(tris, rays, t_min, t_max, prefilter).n_accepted > 0


def restate(tris, rays, prims, t_min=None, t_max=None):
    """The float32 test of ray i against triangle prims[i] alone -> accepted, u, v, t."""
    o, d, lo, hi = ray_arrays(rays, t_min, t_max)
    p = [x[prims.astype(np.int64)] for x in tri_points(tris)]
    return triangle_test(o, d, p[0], p[1], p[2], lo, hi)


def parents(nodes):
    """Parent node of every node of a reference-layout tree (-1 for the root and unreachable nodes), and the leaf of every
    triangle."""
    count = nodes["num_primitives_axis"] >> 16
    par = np.full(len(nodes), -1, np.int64)
    inner = np.flatnonzero(count == 0)
    par[inner + 1] = inner
    par[nodes["offset"][inner].astype(np.int64)] = inner
    leaf_of = np.full(int((nodes["offset"].astype(np.int64) + count)[count > 0].max()), -1, np.int64)
    for k in np.flatnonzero(count > 0):
        leaf_of[nodes["offset"][k]: nodes["offset"][k] + count[k]] = k
    return par, leaf_of


def near_box_face(nodes, o, d, t, prim):
    """Rays (rows) whose point o + t d (float64) lies within 2^-20 (relative to the coordinates involved) of a face of a box on
    the root-to-leaf path of triangle prim, or outside such a box (a box that does not hold its triangle is not rounding: it
    is reported as not near, so that the miss fails)."""
    par, leaf_of = parents(nodes)
    x = o.astype(np.float64) + t.astype(np.float64)[:, None] * d.astype(np.float64)
    sc = np.maximum(np.abs(o.astype(np.float64)), np.abs(x))
    near = np.zeros(len(o), bool)
    outside = np.zeros(len(o), bool)
    node = leaf_of[prim.astype(np.int64)]
    live = node >= 0
    while live.any():
        k = node[live]
        lo = nodes["bounds_min"][k, :3].astype(np.float64); hi = nodes["bounds_max"][k, :3].astype(np.float64)
        xx, s = x[live], sc[live]
        tol_lo = EPS * np.maximum(s, np.abs(lo)); tol_hi = EPS * np.maximum(s, np.abs(hi))
        near[live] |= ((np.abs(xx - lo) <= tol_lo) | (np.abs(xx - hi) <= tol_hi)).any(1)
        outside[live] |= ((xx < lo - tol_lo) | (xx > hi + tol_hi)).any(1)
        node[live] = par[k]
        live = node >= 0
    return near & ~outside


def pair_classes(p, o, d, lo, hi, r, ti, marginal_t, sign=None):
    """The float64 evaluation of the (ray r, triangle ti) pairs (sign as triangle_test's): lowers marginal_t (the smallest t of a
    test that float32 might decide either way) per ray and -> the pairs that hit without doubt as (r, t, ti)."""
    q1, q2, q3 = (x[ti].astype(np.float64) for x in p)
    oo, dd = o[r].astype(np.float64), d[r].astype(np.float64)
    with np.errstate(all="ignore"):
        e1, e2 = q2 - q1, q3 - q1
        pvec = _cross(dd, e2); det = _dot(e1, pvec)
        tvec = oo - q1; qvec = _cross(tvec, e1)
        u = _dot(tvec, pvec) / det; v = _dot(dd, qvec) / det; t = _dot(e2, qvec) / det
        nrm = lambda a: np.sqrt((a * a).sum(-1))
        size = nrm(tvec) + nrm(e1) + nrm(e2)
        err = np.maximum(1.0, size * size * nrm(dd) / np.abs(det))        # conditioning of u and v
        m = np.minimum(np.minimum(u, v), 1.0 - u - v)
        t_tol = EPS * np.maximum(np.abs(t), err * nrm(e2) / np.maximum(nrm(dd), 1e-300))
        det_tol = EPS * nrm(e1) * nrm(pvec) + EPS * 1e-8
        cdet = det if sign is None else det * float(sign)
        hit = (cdet >= 1e-8) & (m >= 0) & (t >= lo[r]) & (t <= hi[r])
        shaky = (np.abs(cdet - 1e-8) <= det_tol) | (np.abs(m) <= EPS * err) | (np.abs(t - lo[r]) <= t_tol) | \
                (np.abs(t - hi[r]) <= t_tol) | ~np.isfinite(t)
    cand = shaky & (cdet > -det_tol)
    np.minimum.at(marginal_t, r[cand], np.where(np.isfinite(t[cand]), t[cand], -np.inf))
    h = hit & ~shaky
    return r[h], t[h], ti[h]


def ray_classes(n, hits, marginal_t, box):
    """-> (class per ray, f64 nearest prim per ray) from pair_classes' hits and marginal_t, and the near_box_face rays."""
    if hits:
        rr, tt, pp = (np.concatenate(x) for x in zip(*hits))
    else:
        rr, tt, pp = np.zeros(0, np.int64), np.zeros(0), np.zeros(0, np.uint32)
    order = np.lexsort((pp, tt, rr))
    rr, tt, pp = rr[order], tt[order], pp[order]
    first = np.ones(len(rr), bool); first[1:] = rr[1:] != rr[:-1]
    best = np.full(n, np.inf); second = np.full(n, np.inf); best_p = np.full(n, INVALID_ID, np.uint32)
    best[rr[first]], best_p[rr[first]] = tt[first], pp[first]
    nxt = np.flatnonzero(first) + 1
    nxt = nxt[(nxt < len(rr))]
    nxt = nxt[rr[nxt] == rr[nxt - 1]]
    second[rr[nxt]] = tt[nxt]
    with np.errstate(invalid="ignore"):
        near_tie = np.isfinite(second) & (second - best <= EPS * np.maximum(np.abs(best), 1e-30))
    near_edge = marginal_t <= np.where(np.isfinite(best), best * (1 + EPS) + EPS, np.inf)
    cls = np.zeros(n, np.int64)
    cls[near_tie] = 1
    cls[near_edge] = 2
    cls[box] = 3
    return cls, best_p


def classify(tris, rays, nodes, ref, t_min=None, t_max=None, prefilter=None):
    """-> (class index per ray into CLASSES, f64 nearest prim per ray (INVALID_ID if none)).  ref: closest() of the same rays."""
    o, d, lo, hi = ray_arrays(rays, t_min, t_max)
    p = tri_points(tris)
    if prefilter is None:
        prefilter = len(tris) > 256
    n = len(o)
    marginal_t = np.full(n, np.inf)
    hits = [pair_classes(p, o, d, lo, hi, r, ti, marginal_t)
            for r, ti in (ref.pairs if getattr(ref, "pairs", None) is not None else candidate_pairs(p, o, d, hi, prefilter))]
    hit32 = ref.prim != INVALID_ID
    box = np.zeros(n, bool)
    box[hit32] = near_box_face(nodes, o[hit32], d[hit32], ref.t[hit32], ref.prim[hit32])
    return ray_classes(n, hits, marginal_t, box)


def verdict(tris, rays, nodes, prim, bc, t, where, t_min=None, t_max=None, ref=None, cls=None, allow_box=0.01):
    """Checks a traversal's hits (prim, bc (n, 2), t) against the brute force; -> report {class: count, 'box_misses': n}.
    allow_box: the fraction of rays on which a miss or a farther hit may occur (near_box_face rays only)."""
    if ref is None:
        ref = closest(tris, rays, t_min, t_max)
    if cls is None:
        cls = classify(tris, rays, nodes, ref, t_min, t_max)[0]
    prim = np.asarray(prim, np.uint32)
    hit = prim != INVALID_ID
    return judge(restate(tris, rays[hit], prim[hit], t_min, t_max), prim, bc, t, where, ref, cls, allow_box)


def judge(restated, prim, bc, t, where, ref, cls, allow_box):
    """verdict() on the hits' restated tests (accepted, u, v, t of every reported hit, in order)."""
    prim = np.asarray(prim, np.uint32)
    hit = prim != INVALID_ID
    ok, u, v, tt = restated
    bad = np.flatnonzero(hit)[~ok]
    assert bad.size == 0, (where, "hit not accepted by the restated test", bad[:8].tolist(), prim[bad[:8]].tolist())
    got = np.ascontiguousarray(np.stack([bc[hit, 0], bc[hit, 1], t[hit]], 1), F).view(np.uint32)
    want = np.ascontiguousarray(np.stack([u, v, tt], 1), F).view(np.uint32)
    bad = np.flatnonzero(hit)[(got != want).any(1)]
    assert bad.size == 0, (where, "hit bits differ from the restated test", bad[:8].tolist())
    closest_ok = np.where(hit, np.asarray(t, F) == ref.t, ref.prim == INVALID_ID)
    wrong = np.flatnonzero(~closest_ok)
    not_box = wrong[cls[wrong] != 3]
    assert not_box.size == 0, (where, "not the closest hit", [(int(i), int(prim[i]), float(t[i]), int(ref.prim[i]), float(ref.t[i]),
                                                            CLASSES[cls[i]]) for i in not_box[:8]])
    assert wrong.size <= allow_box * len(prim), (where, "box-face misses", wrong.size, len(prim))
    rep = {c: int((cls == i).sum()) for i, c in enumerate(CLASSES)}
    rep["ties"] = int((ref.n_ties > 1).sum())
    rep["box_misses"] = int(wrong.size)
    return rep
