"""
Designed scenes for the brute-force traversal checks (tests/trace_reference.py): trees at the 64-entry stack limit, exact distance
ties, hits on shared edges and vertices and at t = 0, the det cut, flat boxes and rays on their planes.  Every scene has one white
diffuse material, CornellBox's directional light and a constant environment, so that it uploads.  The geometry is placed on the
float32 bounce-0 rays of a pinhole camera, which do not depend on the scene (Oracle.generate_rays gives the device's).
"""
import numpy as np

from oracle.orcbind import Oracle
from raytracing_b200 import hostapi
from raytracing_b200.camera import default_camera
from raytracing_b200.layouts import INVALID_ID as INVALID
from raytracing_b200.layouts import MATERIAL_DT, NODE_DT, RAY_DT, TRIANGLE_DT
from tests.helpers import scene
from tests import lbvh_model
from tests.refit_model import refit

F = np.float32
W, H = 64, 48


def axis_camera(w, h, position, front, up):
    """A camera whose every primary ray is exactly `front`: fov 0 and no aperture, axes filled in by hand (default_camera goes
    through float32 sin/cos of pi/2 and never gives an exact axis)."""
    cam = default_camera(w, h)
    cam["position"][:3] = position; cam["front"][:3] = front; cam["up"][:3] = up; cam["fov"] = 0.0
    return cam


def triangles(p1, p2, p3, part=0):
    """TRIANGLE_DT records from (n, 3) vertex arrays; material 0.  `part` goes into every texture coordinate's u, which the
    untextured material never reads, so that a test can tell the parts of a scene apart after the SAH builder reorders them."""
    p1, p2, p3 = (np.asarray(p, F).reshape(-1, 3) for p in (p1, p2, p3))
    t = np.zeros(len(p1), TRIANGLE_DT)
    for v, p in (("v1", p1), ("v2", p2), ("v3", p3)):
        t[v]["position"][:, :3] = p
        t[v]["normal"][:, :3] = (0, 0, 1)
        t[v]["texcoord"][:, 0] = part
    return t


def part_of(tris):
    """The `part` of every triangle (see triangles())."""
    return tris["v1"]["texcoord"][:, 0].astype(np.int64)


STRIP, FAN, AT_CAMERA, EDGE_ON, GRAZED_WALL, U_ONE = 1, 2, 3, 4, 5, 6


def make_scene(tris, nodes=None):
    """A complete scene dict over tris: the host SAH tree (which reorders the triangles) unless nodes (leaf order) is given."""
    sc = dict(scene("CornellBox"))
    if nodes is None:
        tris, nodes, _ = hostapi.build_bvh(tris)
    mat = np.zeros(1, MATERIAL_DT)
    mat["diffuse_albedo"] = 0xFFC8C8C8                 # white diffuse; every texture index byte 0xFF (none)
    mat["specular_albedo"] = 0xFF000000
    mat["roughness_metalness"] = 0xFF00FF80
    mat["ior_emission_idx_transparency"] = 0xFFFFFF26
    info = np.array(sc["scene_info"], copy=True); info["emissive_count"] = 0
    sc.update(triangles=tris, nodes=nodes, materials=mat, emissive=np.zeros(0, "<u4"), scene_info=info,
              env=np.full_like(sc["env"], 0.25))
    return sc


def camera_rays(cam, w=W, h=H):
    return Oracle(make_scene(triangles([0, 0, 0], [1, 0, 0], [1, 1, 0]))).generate_rays(cam, w, h)


# ------------------------------------------------------------------------------------------------ depth at the stack limit
def chain(levels):
    """A caller-supplied tree with `levels` interior nodes (depth levels + 1) over levels + 1 nested triangles facing the default
    camera: interior node k (preorder k) has the next interior node as its first child and a leaf as its second; the last one has two
    leaves.  All split axes are y and every camera ray has d.y > 0, so the near child is the first (the subtree) under the literal
    rule (ray_sign[axis]) and the fast rule alike, and a ray through the innermost triangle defers one leaf at every level.
    Triangle j lies at y = 0.2 + 0.03 j, tilted by 0.02 in y so that its box has thickness, and shrinks with j."""
    m = levels
    j = np.arange(m + 1, dtype=F)
    y = F(0.2) + F(0.03) * j
    s = F(1.2) - F(0.015) * j
    x0, z0 = np.zeros_like(s), np.full_like(s, F(1.0))
    tris = triangles(np.stack([x0 - 3 * s, y, z0 - s], 1), np.stack([x0 + s, y, z0 - s], 1), np.stack([x0 + s, y + F(0.02), z0 + 3 * s], 1))
    nodes = np.zeros(2 * m + 1, NODE_DT)
    nodes["num_primitives_axis"][:m] = 1                                   # interior, split axis y
    nodes["offset"][:m - 1] = 2 * m + 1 - np.arange(1, m)                  # second child of node k - 1: the leaf of triangle k - 1
    nodes["offset"][m - 1] = m + 1
    leaf_tri = np.concatenate([[m - 1, m], np.arange(m - 2, -1, -1)])      # nodes m, m + 1 (the last pair), then the deferred leaves
    nodes["offset"][m:] = leaf_tri
    nodes["num_primitives_axis"][m:] = 1 << 16
    return make_scene(tris, refit(nodes, tris))


def geometric_chain(n):
    """The 1.5^k chain of test_ploc_cpu (one PLOC merge per triangle), facing a camera above it that looks down (-z)."""
    from tests.test_ploc_cpu import geometric_chain as gc
    return make_scene(gc(n))


def chain_camera(w=W, h=H):
    cam = axis_camera(w, h, (0.55, 0.2, 1.0), (0.0, 0.0, -1.0), (0.0, 1.0, 0.0))
    cam["fov"] = F(0.6)
    return cam


def lbvh_deep():
    """The key points of test_lbvh_cpu.morton_chain (halving distances along x, y, z in turn, and a block of equal codes at 0 whose
    ids 0, 1, 2, 4, ... chain in the id bits) as real triangles: v1 = c + (0, 1/4, 0), v2 = c + (1/4, 0, 0), v3 = c - (1/4, 1/4, 0),
    whose sum is exactly 3c, so the keys and the LBVH are morton_chain's.  They face -z: rays going up with d > 0 on every axis
    take the first child (lower keys) as the near one at every level, toward the equal-code block."""
    from tests.test_lbvh_cpu import morton_chain
    c = morton_chain()["v1"]["position"][:, :3].astype(F)
    a, b = np.array([0, 0.25, 0], F), np.array([0.25, 0, 0], F)
    tris = triangles(c + a, c + b, c - (a + b))
    return make_scene(tris, lbvh_model.build(tris)[0])             # uploaded in this order: the ids are part of the keys


def lbvh_camera(w=W, h=H):
    cam = axis_camera(w, h, (-0.25, -0.2, -1.0), (0.25, 0.2, 1.0), (0.0, 1.0, 0.0))
    cam["front"][:3] /= np.linalg.norm(cam["front"][:3])
    cam["up"][:3] = np.cross(np.cross(cam["front"][:3], [0, 1, 0]), cam["front"][:3]).astype(F)
    cam["up"][:3] /= np.linalg.norm(cam["up"][:3])
    cam["fov"] = F(0.5)
    return cam


def deferred_entries(nodes, o, d, fast=False):
    """The traversal of one ray without its triangle tests, which only shrink t_max: -> (maximum number of deferred entries on the
    stack, nodes visited).  fast=False: the literal rule (trace_literal / oracle.cpp TraceBvh: every visited node's box is tested
    and the far child is pushed unconditionally); fast=True: the rule of trace_fast (both children's boxes are tested at their
    parent, the far child is pushed only when both are hit), whose visited count is not compared with anything."""
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = F(1) / d.astype(F)
        sign = inv < 0

        def box(k):
            n = nodes[k]
            t0 = (n["bounds_min"][:3] - o) * inv; t1 = (n["bounds_max"][:3] - o) * inv
            lo = np.fmax(np.fmax(np.fmin(t0[0], t1[0]), np.fmin(t0[1], t1[1])), np.fmin(t0[2], t1[2]))
            hi = np.fmin(np.fmin(np.fmax(t0[0], t1[0]), np.fmax(t0[1], t1[1])), np.fmax(t0[2], t1[2]))
            return np.fmin(hi, F(1e30)) >= np.fmax(lo, F(0))
        stack, cur, best, visited = [], 0, 0, 0
        if fast and not box(0):
            return 0, 1
        while True:
            n = nodes[cur]
            visited += 1
            inner = (n["num_primitives_axis"] >> 16) == 0
            if inner and (fast or box(cur)):
                near_first = not sign[n["num_primitives_axis"] & 0xFFFF]
                near, far = (cur + 1, int(n["offset"])) if near_first else (int(n["offset"]), cur + 1)
                if not fast or box(near):
                    if not fast or box(far):
                        stack.append(far)
                    cur = near
                    best = max(best, len(stack))
                    continue
                if box(far):
                    cur = far
                    continue
            if not stack:
                return best, visited
            cur = stack.pop()


# ------------------------------------------------------------------------------------------------ ties, edges, walls
def quad_tris(x0, x1, z0, z1, y):
    """Two triangles on the plane y facing -y (CornellBox's back-wall winding)."""
    c = [(x0, z0), (x1, z0), (x1, z1), (x0, z1)]
    p = [[(c[i][0], y, c[i][1]) for i in k] for k in ((0, 1, 2), (2, 3, 0))]
    return triangles(*[np.array([q[v] for q in p]) for v in range(3)])


def ties():
    """A wall of quads at y = 1 in front of the default camera, each triangle present twice (an exact copy) plus a coplanar copy
    shifted in the plane, and a second layer at y = 1.5 behind it: every hit on the wall ties in t with its copy, which the SAH
    builder puts in the same leaf or another one; flat leaf boxes give far-child entries equal to the hit distance."""
    out = []
    for i in range(6):
        for k in range(4):
            x0, z0 = F(-1.2 + 0.4 * i), F(0.2 + 0.4 * k)
            q = quad_tris(x0, x0 + F(0.4), z0, z0 + F(0.4), F(1.0))
            out += [q, q.copy(), quad_tris(x0 + F(0.1), x0 + F(0.5), z0 + F(0.1), z0 + F(0.5), F(1.0))]
    out.append(quad_tris(F(-2), F(2), F(-1), F(3), F(1.5)))
    return make_scene(np.concatenate(out))


def edges(cam, w=W, h=H):
    """Meshes whose vertices lie on the camera's float32 rays, facing the camera: a grid strip with a vertex on every third pixel
    ray at t between 1.5 and 1.8 (rays hit shared vertices and pass along shared edges), and fans of six triangles around a vertex
    on a ray.  Also a small triangle with a vertex at the camera, hit at t = 0 (u = v = 0) by every ray whose det >= 1e-8: its
    normal is tilted so that det crosses 1e-8 inside the image and only a corner of it, away from the strip and the fans, is
    covered; a triangle edge-on to the camera (rays parallel to its plane) and a back-facing quad."""
    rays = camera_rays(cam, w, h)
    o = rays["origin"][:, :3].reshape(h, w, 3); d = rays["direction"][:, :3].reshape(h, w, 3)
    out = []
    ys, xs = np.arange(1, h, 3), np.arange(1, w // 2, 3)
    t = F(1.5) + F(0.3) * ((xs[None, :] * 7 + ys[:, None] * 3) % 5).astype(F) / F(4)
    v = o[ys][:, xs] + t[..., None] * d[ys][:, xs]
    a, b, c, e = v[:-1, :-1].reshape(-1, 3), v[:-1, 1:].reshape(-1, 3), v[1:, :-1].reshape(-1, 3), v[1:, 1:].reshape(-1, 3)
    out += [triangles(a, b, c, STRIP), triangles(b, e, c, STRIP)]
    for py, px in ((10, 40), (24, 50), (37, 44)):
        ctr = o[py, px] + F(1.2) * d[py, px]
        ring = [ctr + F(0.08) * np.array([np.cos(k * np.pi / 3), 0, np.sin(k * np.pi / 3)], F) for k in range(7)]
        out += [triangles(ctr, ring[k], ring[k + 1], FAN) for k in range(6)]
    p0 = cam["position"][:3].astype(F)
    n = np.array(AT_CAMERA_NORMAL); n /= np.linalg.norm(n)
    s1 = np.cross(n, [0.0, 0.0, 1.0]); s1 /= np.linalg.norm(s1)
    s2 = np.cross(n, s1)                                     # s1 x s2 = n: det = dot(d, e2 x e1) = 1e-6 dot(d, n)
    out.append(triangles(p0, p0 + F(1e-3) * s2.astype(F), p0 + F(1e-3) * s1.astype(F), AT_CAMERA))
    out.append(triangles(p0 + np.array([0.3, 2.0, 0], F), p0 + np.array([0.6, 2.0, 0], F), p0 + np.array([0.45, 2.5, 0], F), EDGE_ON))
    bq = quad_tris(F(-2), F(2), F(-1), F(3), F(3.0))
    bq["v2"], bq["v3"] = bq["v3"].copy(), bq["v2"].copy()
    out.append(bq)
    return make_scene(np.concatenate(out))


AT_CAMERA_NORMAL = (-1.0, -1.5, 1.0)


def walls():
    """An axis-aligned room: floor, ceiling, back wall and a partition, all quads (flat leaf boxes), a wall in the plane z = 1
    (x in [0.2, 0.9]) and one in the plane y = -1, back-facing, so that the default camera at (0, -1, 1) starts on the planes of
    both and sees past them.  The axis camera's ray from (0.5, -0.5, 1) along +y runs inside the plane of the z = 1 wall across
    it, and meets a triangle whose second vertex, (0.5, 0.5, 1), lies inside the triangle's box: it hits there at t = 1 with
    u = 1 and v = 0 exactly.  (A vertex on a box plane would not do: a ray with zero direction components that starts on a plane
    of a box misses it under the reference's slab test.  For the same reason the back wall reaches x = 1.2: with x and z
    exchanged (swap_axes) no box on that ray's way then has a face in its plane z = 1.)"""
    def plane(axis, at, lo, hi, flip=False, part=0):
        other = [k for k in range(3) if k != axis]
        c = np.zeros((4, 3), F)
        c[:, axis] = at
        c[:, other] = [(lo[0], lo[1]), (hi[0], lo[1]), (hi[0], hi[1]), (lo[0], hi[1])]
        i = ((0, 2, 1), (2, 0, 3)) if flip else ((0, 1, 2), (2, 3, 0))
        return triangles(*[c[[k[v] for k in i]] for v in range(3)], part=part)
    out = [plane(1, 2.0, (-1, 0), (1.2, 2)), plane(1, -1.0, (-1, 0), (1, 2), True),
           plane(2, 0.0, (-1, -1), (1, 2)), plane(2, 2.0, (-1, -1), (1, 2), True),
           plane(2, 1.0, (0.2, -1), (0.9, 1.5), part=GRAZED_WALL),
           plane(0, 0.0, (0.3, 0.0), (1.5, 1.8)), plane(0, -0.5, (-1, 0.5), (2, 1.2), True),
           triangles([-0.5, 0.5, 0], [0.5, 0.5, 1], [1.5, 0.5, 3], U_ONE)]
    return make_scene(np.concatenate(out))


def swap_axes(tris):
    """The same triangles with x and z exchanged (wound back to face the same way): flat boxes become flat along another axis."""
    t = tris.copy()
    for vv in ("v1", "v2", "v3"):
        t[vv]["position"][:, :3] = tris[vv]["position"][:, [2, 1, 0]]
    t["v2"], t["v3"] = t["v3"].copy(), t["v2"].copy()
    return t


def shipped_rays(rays, n=2000, seed=0):
    """A seeded sample of n rays."""
    rng = np.random.default_rng(seed)
    return rays[np.sort(rng.choice(len(rays), min(n, len(rays)), replace=False))]


# name -> (scene, camera); the producers that apply are chosen by the tests
def case(name):
    if name == "chain64":
        return chain(63), default_camera(W, H)
    if name == "ploc64":
        return geometric_chain(64), chain_camera()
    if name == "lbvh_deep":
        return lbvh_deep(), lbvh_camera()
    if name == "ties":
        return ties(), default_camera(W, H)
    if name == "edges":
        cam = default_camera(W, H)
        return edges(cam), cam
    if name == "walls":
        return walls(), default_camera(W, H)
    if name == "walls_axis":
        return walls(), axis_camera(W, H, (0.5, -0.5, 1.0), (0.0, 1.0, 0.0), (0.0, 0.0, 1.0))
    return scene(name), scene(name).get("camera_pose", default_camera(W, H))


def reached(name, sc, rays, ref):
    """What a designed case is built to reach, from the brute force (closest()) of its bounce-0 rays -> {what: count of rays}.
    edges: hits on a shared vertex or edge of the strip or a fan (u == 0, v == 0 or u + v == 1 exactly), ties of several strip or
    fan triangles, hits at t == 0 on the triangle at the camera.  walls: hits at t == 0 and the triangles hit.  walls_axis: rays
    along the z = 1 wall's plane across the wall, and hits on the u = 1 vertex."""
    part = part_of(sc["triangles"])
    tie_part = part[ref.tie_prim.astype(np.int64)]
    if name == "edges":
        mesh = (tie_part == STRIP) | (tie_part == FAN)
        u, v = ref.tie_u, ref.tie_v
        on_edge = mesh & ((u == 0) | (v == 0) | (u + v == F(1)))
        return {"vertex_or_edge": len(np.unique(ref.tie_ray[on_edge])),
                "mesh_ties": int((np.bincount(ref.tie_ray[mesh], minlength=len(rays)) > 1).sum()),
                "t_zero": len(np.unique(ref.tie_ray[tie_part == AT_CAMERA]))}
    if name == "walls":
        return {"t_zero": int((ref.t == 0).sum()), "triangles_hit": len(np.unique(ref.prim[ref.prim != INVALID]))}
    if name == "walls_axis":
        o, d = rays["origin"][:, :3], rays["direction"][:, :3]
        along = (o[:, 2] == 1) & (d[:, 2] == 0) & (d[:, 0] == 0) & (o[:, 0] >= F(0.2)) & (o[:, 0] <= F(0.9))
        u_one = (tie_part == U_ONE) & (ref.tie_u == 1) & (ref.tie_v == 0)
        return {"along_grazed_wall": int(along.sum()), "u_one": len(np.unique(ref.tie_ray[u_one]))}
    return {}


# the least each case must reach on its 64 x 48 bounce-0 rays
REACH = {"edges": {"vertex_or_edge": 40, "mesh_ties": 10, "t_zero": 8}, "walls": {"triangles_hit": 6},
         "walls_axis": {"along_grazed_wall": W * H, "u_one": W * H}}


DESIGNED = ["chain64", "ploc64", "lbvh_deep", "ties", "edges", "walls", "walls_axis"]
SHIPPED = ["CornellBox", "ShaderBalls", "CornellBox_Dragon"]


def designed_rays(sc, n=1500, seed=3):
    """Rays that start on the planes of the scene's boxes, with direction components of exactly +0 and -0, and random rays from
    inside its box."""
    rng = np.random.default_rng(seed)
    nodes = sc["nodes"]
    planes = np.concatenate([nodes["bounds_min"][:, :3], nodes["bounds_max"][:, :3]])
    lo, hi = planes.min(0), planes.max(0)
    o = rng.uniform(lo, hi, (n, 3)).astype(F)
    pick = planes[rng.integers(0, len(planes), n)]
    axis = rng.integers(0, 3, n)
    o[np.arange(n), axis] = pick[np.arange(n), axis]                     # on a box plane
    d = rng.standard_normal((n, 3)).astype(F)
    d /= np.linalg.norm(d, axis=1, keepdims=True).astype(F)
    zero = rng.random((n, 3)) < 0.3
    d[zero] = np.where(rng.random(zero.sum()) < 0.5, F(0.0), F(-0.0))
    d[(d == 0).all(1), 1] = F(1.0)
    r = np.zeros(n, RAY_DT)
    r["origin"][:, :3] = o; r["direction"][:, :3] = d; r["direction"][:, 3] = F(20000.0)
    return r
