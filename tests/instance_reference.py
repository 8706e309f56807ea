"""
The brute force of tests/trace_reference.py for instanced scenes: it knows nothing about the top-level tree, the world boxes or the
meshes' trees.  Per instance i (mesh m, object-to-world M):

- W and sign(det M) from tests/instance_tree_model.inverse (the independent restatement of rt_instances.h's inverse);
- the ray in object space as the traversal computes it, float32 with no contraction: o' = ((w0 o.x + w1 o.y) + w2 o.z) + w3 per row,
  d' the same without w3, and t_min / t_max unchanged;
- every triangle of m tested with trace_reference.triangle_test, culling on det * sign (u, v and t still divide by det).

closest(): the minimum accepted t over every instance; the tie set is every (instance, triangle) pair accepted at that t, reported
as virtual ids (base_i + triangle).  any_hit(): some pair is accepted.  classify(): near_tie and near_edge as trace_reference's,
evaluated in each instance's object space; near_box_face only for the boxes of the hit triangle's root-to-leaf path in its mesh's
own tree, evaluated with the object-space ray.  A miss caused by an instance's world box or a top-level box is never excused.
verdict(): a reported virtual id is tested again in its instance's object space and its (u, v, t) bits must match.

The rays reach a mesh only through a float64 world-space prefilter (the line within the instance's bounding sphere, mapped by M
and padded by 2^-10 of the scene's scale, far beyond the rounding of the ray transform), and then trace_reference.candidate_pairs
in object space; neither drops a pair that could be accepted.
"""
import numpy as np

from raytracing_b200.layouts import INVALID_ID
from tests import instance_tree_model as tree_model
from tests import trace_reference as R

F = np.float32


def object_rays(w, o, d):
    """o, d (n, 3) float32 -> the object-space ray of the traversal under W (3, 4) float32."""
    w = np.asarray(w, F)
    oo = np.stack([((w[k, 0] * o[:, 0] + w[k, 1] * o[:, 1]) + w[k, 2] * o[:, 2]) + w[k, 3] for k in range(3)], 1)
    dd = np.stack([(w[k, 0] * d[:, 0] + w[k, 1] * d[:, 1]) + w[k, 2] * d[:, 2] for k in range(3)], 1)
    return np.ascontiguousarray(oo, F), np.ascontiguousarray(dd, F)


class Scene:
    """meshes: dicts with "triangles" (and "nodes", read by classify() only); mesh_ids, transforms (n, 3, 4) as rt_set_instances
    takes them."""

    def __init__(self, meshes, mesh_ids, transforms):
        self.meshes = meshes
        self.ids = np.asarray(mesh_ids, np.int64)
        self.mats = np.asarray(transforms, F).reshape(-1, 3, 4)
        self.points = [R.tri_points(m["triangles"]) for m in meshes]
        self.inst = []
        base = 0
        for m, k in zip(self.mats, self.ids):
            w, sign = tree_model.inverse(m)
            p = [x.astype(np.float64) for x in self.points[k]]
            c = (p[0] + p[1] + p[2]) / 3.0
            rad = np.sqrt(np.max([((x - c) ** 2).sum(1) for x in p], 0))
            a = m[:, :3].astype(np.float64)
            lo, hi = (c - rad[:, None]).min(0), (c + rad[:, None]).max(0)
            centre = (lo + hi) / 2.0
            r_obj = np.sqrt((((hi - lo) / 2.0) ** 2).sum())
            self.inst.append({"w": w, "sign": sign, "base": base, "mesh": int(k), "centre": a @ centre + m[:, 3],
                              "radius": np.linalg.norm(a, 2) * r_obj})
            base += len(meshes[k]["triangles"])
        self.n_virtual = base

    def base_of(self, prim):
        """-> instance index of each virtual id (the last base <= prim)."""
        bases = np.array([i["base"] for i in self.inst], np.int64)
        return np.searchsorted(bases, np.asarray(prim, np.int64), side="right") - 1

    def _near(self, i, o, d, hi):
        """Rows of rays whose world line passes near instance i's bounding sphere."""
        inst = self.inst[i]
        oo, dd = o.astype(np.float64), d.astype(np.float64)
        scale = max(float(np.abs(oo).max(initial=0.0)), float(np.abs(inst["centre"]).max()) + inst["radius"], 1.0)
        dn = np.sqrt((dd * dd).sum(1))
        return np.flatnonzero(R._near_spheres(inst["centre"][None], inst["radius"] + 2.0 ** -10 * scale, oo, dd / dn[:, None],
                                              hi.astype(np.float64) * dn))

    def pairs(self, rays, t_min=None, t_max=None):
        """Yields (instance, object-space o, d (of the selected rows), t_min, t_max, rows, candidate (row index, triangle) pairs)."""
        o, d, lo, hi = R.ray_arrays(rays, t_min, t_max)
        for i, inst in enumerate(self.inst):
            rows = self._near(i, o, d, hi)
            if rows.size == 0:
                continue
            oo, dd = object_rays(inst["w"], o[rows], d[rows])
            p = self.points[inst["mesh"]]
            for r, ti in R.candidate_pairs(p, oo, dd, hi[rows], len(p[0]) > 256):
                yield i, oo, dd, lo[rows], hi[rows], rows, r, ti

    def closest(self, rays, t_min=None, t_max=None):
        acc = []
        for i, oo, dd, lo, hi, rows, r, ti in self.pairs(rays, t_min, t_max):
            inst = self.inst[i]
            p = self.points[inst["mesh"]]
            ok, u, v, t = R.triangle_test(oo[r], dd[r], p[0][ti], p[1][ti], p[2][ti], lo[r], hi[r], sign=inst["sign"])
            acc.append((rows[r[ok]], (inst["base"] + ti[ok]).astype(np.uint32), t[ok], u[ok], v[ok]))
        out = R.reduce_accepted(len(rays), acc)
        out.pairs = None
        return out

    def any_hit(self, rays, t_min=None, t_max=None):
        return self.closest(rays, t_min, t_max).n_accepted > 0

    def restate(self, rays, prims, t_min=None, t_max=None):
        """The float32 test of ray k against virtual id prims[k] alone, in its instance's object space -> accepted, u, v, t."""
        o, d, lo, hi = R.ray_arrays(rays, t_min, t_max)
        prims = np.asarray(prims, np.int64)
        out = [np.zeros(len(prims), bool)] + [np.zeros(len(prims), F) for _ in range(3)]
        which = self.base_of(prims)
        for i in np.unique(which):
            sel = np.flatnonzero(which == i)
            inst = self.inst[i]
            oo, dd = object_rays(inst["w"], o[sel], d[sel])
            p = [x[prims[sel] - inst["base"]] for x in self.points[inst["mesh"]]]
            res = R.triangle_test(oo, dd, p[0], p[1], p[2], lo[sel], hi[sel], sign=inst["sign"])
            for k in range(4):
                out[k][sel] = res[k]
        return tuple(out)

    def classify(self, rays, ref, t_min=None, t_max=None):
        """-> (class per ray into trace_reference.CLASSES, f64 nearest virtual id per ray).  ref: closest() of the same rays."""
        n = len(rays)
        marginal_t = np.full(n, np.inf)
        hits = []
        for i, oo, dd, lo, hi, rows, r, ti in self.pairs(rays, t_min, t_max):
            inst = self.inst[i]
            marg = np.full(len(rows), np.inf)
            rr, tt, pp = R.pair_classes(self.points[inst["mesh"]], oo, dd, lo, hi, r, ti, marg, sign=inst["sign"])
            np.minimum.at(marginal_t, rows, marg)
            hits.append((rows[rr], tt, (inst["base"] + pp).astype(np.uint32)))
        box = np.zeros(n, bool)
        hit = np.flatnonzero(ref.prim != INVALID_ID)
        which = self.base_of(ref.prim[hit])
        o, d, _, _ = R.ray_arrays(rays, t_min, t_max)
        for i in np.unique(which):
            sel = hit[which == i]
            inst = self.inst[i]
            oo, dd = object_rays(inst["w"], o[sel], d[sel])
            box[sel] = R.near_box_face(self.meshes[inst["mesh"]]["nodes"], oo, dd, ref.t[sel], ref.prim[sel] - np.uint32(inst["base"]))
        return R.ray_classes(n, hits, marginal_t, box)

    def mesh_lost(self, model, rays, got_t, ref):
        """Per ray: the brute force's closest hit is one that its instance's mesh tree, traced alone (model.trace_mesh) with the
        object-space ray and t_max lowered to got_t (the traversal's final t, +inf for a miss), does not find either: a loss to
        the rounding of the mesh's own boxes, which the traversal of the same ray through a flat scene shares.  Any other loss is
        the top level's."""
        o, d, lo, hi = R.ray_arrays(rays)
        lost = np.zeros(len(rays), bool)
        hit = np.flatnonzero(ref.prim != INVALID_ID)
        which = self.base_of(ref.prim[hit])
        for i in np.unique(which):
            sel = hit[which == i]
            inst = self.inst[i]
            oo, dd = object_rays(inst["w"], o[sel], d[sel])
            r = np.zeros(len(sel), rays.dtype)
            r["origin"][:, :3], r["origin"][:, 3] = oo, lo[sel]
            r["direction"][:, :3], r["direction"][:, 3] = dd, np.minimum(hi[sel], np.asarray(got_t, F)[sel])
            h = model.trace_mesh(inst["mesh"], r, inst["sign"])
            lost[sel] = h["t"] != ref.t[sel]
        return lost

    def verdict(self, rays, prim, bc, t, where, t_min=None, t_max=None, ref=None, cls=None, allow_box=0.01, lost=None):
        """trace_reference.verdict for instanced hits (virtual ids).  lost (mesh_lost()): when given, it decides which rays may miss
        or hit farther instead of the near_box_face class."""
        if ref is None:
            ref = self.closest(rays, t_min, t_max)
        if cls is None:
            cls = self.classify(rays, ref, t_min, t_max)[0]
        if lost is not None:
            cls = np.where(lost, 3, np.where(cls == 3, 0, cls))
        prim = np.asarray(prim, np.uint32)
        hit = prim != INVALID_ID
        return R.judge(self.restate(rays[hit], prim[hit], t_min, t_max), prim, np.asarray(bc), np.asarray(t), where, ref, cls, allow_box)
