"""
CPU tests of the two-level traversal of instanced scenes against the brute force of tests/instance_reference.py, which ignores the
top-level tree, the world boxes and the meshes' trees.

- The brute force itself: one identity instance gives trace_reference.closest of the flat scene bit for bit, and a mirrored
  instance culls exactly the faces its flattened triangles cull.
- The CPU model's traversal (InstanceModel.trace_instanced, tests/instance_model.cpp im_trace, which the device equals bit for bit)
  meets the brute force's rules per ray, for closest hit and any hit, on the placements of test_gpu_instancing.placements_case,
  replicate()'s 183-copy field, and designed cases: a small, ill-conditioned instance seen from 1000 of its extents away, a mesh far
  from its object-space origin placed back near the world origin, coinciding instances (t ties across instances), a mesh whose tree
  is one leaf, exactly one instance and none.  Shadow rays end exactly on the closest hit (t_max = t: occluded) and just before it.

No miss is excused by an instance's world box or a top-level box: a lost hit is excused only when the mesh's own tree, traced alone
with the same object-space ray, loses it too (the rounding of the mesh's boxes, which a flat scene shares), on at most 1 % of the
rays.  The per-class counts are printed (pytest -s).
"""
import math

import numpy as np
import pytest

from oracle.orcbind import Oracle
from raytracing_b200 import hostapi, synthetic
from raytracing_b200.camera import default_camera
from raytracing_b200.layouts import INVALID_ID, RAY_DT
from tests import instance_reference as IR
from tests import trace_reference as R
from tests.helpers import bits, scene
from tests.instance_model import InstanceModel

EYE = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)
MAX_DIST = np.float32(20000.0)          # RT_MAX_RENDER_DIST: the t_max of every extension ray


def rot(axis, ang):
    c, s = math.cos(ang), math.sin(ang)
    r = np.eye(3)
    i, j = [(1, 2), (0, 2), (0, 1)][axis]
    r[i, i], r[i, j], r[j, i], r[j, j] = c, -s, s, c
    return r


def mat(r, t):
    out = np.zeros((3, 4), np.float32)
    out[:, :3] = r
    out[:, 3] = t
    return out


def as_mesh(sc):
    return {"triangles": sc["triangles"], "nodes": sc["nodes"]}


def camera_rays(shared, cam, w, h):
    rays = Oracle({**shared, "emissive": np.zeros(0, "<u4")}).generate_rays(cam, w, h)
    rays["origin"][:, 3] = 0.0
    rays["direction"][:, 3] = MAX_DIST
    return rays


def placements(sc):
    lo, hi = sc["nodes"]["bounds_min"][0, :3], sc["nodes"]["bounds_max"][0, :3]
    span = float((hi - lo).max())
    mats = [mat(np.eye(3), (0, 0, 0)),
            mat(rot(2, 0.7) @ rot(0, 0.3), (1.2 * span, 0, 0)),                      # rotated
            mat(np.diag([1.5, 0.6, 1.0]), (-1.2 * span, 0, 0)),                      # non-uniform scale
            mat(rot(2, 0.4) @ np.diag([-1.0, 1.0, 1.0]), (0, 1.2 * span, 0)),        # mirror
            mat(np.eye(3), (0, 1.2 * span, 0)),                                      # overlaps the mirror
            mat(np.eye(3), (0, 0, 0)),                                               # coincides with instance 0
            mat(0.2 * np.eye(3), (0.1 * span, 0.1 * span, 0))]                       # inside instance 0's box
    cam = default_camera(96, 64, position=(0.5 * (lo[0] + hi[0]), float(lo[1]) - 2.5 * span, float(hi[2]) + 0.8 * span), pitch=1.9)
    return np.stack(mats), cam


def far_camera_case(scale, yaw):
    """One CornellBox instance, M = scale * diag(3, 0.05, 1) Rx(0.4) (condition number about 60), seen from 1000 of its extents away
    with a narrow field of view, from the side given by yaw (about the world z axis).  Under a top-level box padded by 2^-20 of its
    coordinates alone, one hit of each of the two views below is lost: the rounding of the object-space ray outgrows the pad."""
    sc = scene("CornellBox")
    m = mat(scale * np.diag([3.0, 0.05, 1.0]) @ rot(0, 0.4), (0, 0, 0))
    lo, hi = sc["nodes"]["bounds_min"][0, :3].astype(np.float64), sc["nodes"]["bounds_max"][0, :3].astype(np.float64)
    corners = np.array([[(hi if c & 1 else lo)[0], (hi if c & 2 else lo)[1], (hi if c & 4 else lo)[2]] for c in range(8)])
    world = corners @ m[:, :3].astype(np.float64).T
    ext = float((world.max(0) - world.min(0)).max())
    centre = (world.max(0) + world.min(0)) / 2
    pitch = 1.5708
    front = np.array([math.cos(yaw) * math.sin(pitch), math.sin(yaw) * math.sin(pitch), math.cos(pitch)])
    cam = default_camera(96, 64, position=tuple(centre - 1000.0 * ext * front), yaw=yaw, pitch=pitch)
    cam["fov"] = np.float32(2.0 * math.atan(0.6 / 1000.0))
    return [as_mesh(sc)], sc, [0], m[None], cam


def offset_mesh_case():
    """A mesh whose coordinates lie 1000 of its extents from its object-space origin, placed back near the world origin by a
    rotation and a translation: the object-space ray is computed at that magnitude."""
    sc = scene("CornellBox")
    t = sc["triangles"].copy()
    lo, hi = sc["nodes"]["bounds_min"][0, :3], sc["nodes"]["bounds_max"][0, :3]
    shift = np.float32(1000.0 * float((hi - lo).max()))
    for v in ("v1", "v2", "v3"):
        t[v]["position"][:, 0] += shift
    ordered, nodes, _ = hostapi.build_bvh(t)
    r = rot(2, 0.3) @ rot(0, 0.2)
    m = mat(r, -(r @ np.array([float(shift), 0.0, 0.0])))
    cam = default_camera(96, 64, position=(0.0, -3.0, 1.0))
    return [{"triangles": ordered, "nodes": nodes}], sc, [0], m[None], cam


def single_leaf_case():
    """Two two-triangle meshes (CornellBox walls) whose trees are a single leaf, placed four times with rotations, one mirrored."""
    sc = scene("CornellBox")
    meshes = []
    for first in (0, 6):
        ordered, nodes, _ = hostapi.build_bvh(sc["triangles"][first: first + 2].copy())
        assert len(nodes) == 1
        meshes.append({"triangles": ordered, "nodes": nodes})
    mats = np.stack([mat(np.eye(3), (0, 0, 0)), mat(rot(2, 0.5), (0.3, 0.2, 0.1)), mat(rot(1, 0.2) @ np.diag([-1.0, 1.0, 1.0]), (-0.4, 0.1, 0)),
                     mat(0.5 * np.eye(3), (0.1, -0.3, 0.4))])
    return meshes, sc, [0, 1, 0, 1], mats, default_camera(96, 64)


def coinciding_case():
    sc = scene("CornellBox")
    mats = np.stack([EYE, EYE, mat(rot(2, 0.2), (0.1, 0, 0)), EYE])
    return [as_mesh(sc)], sc, [0, 0, 0, 0], mats, default_camera(96, 64)


def one_instance_case():
    sc = scene("ShaderBalls")
    m = mat(rot(2, 0.6) @ rot(1, 0.2) @ np.diag([1.2, 0.8, 1.0]), (0.3, -0.2, 0.1))
    return [as_mesh(sc)], sc, [0], m[None], default_camera(96, 64)


def zero_instances_case():
    sc = scene("CornellBox")
    return [as_mesh(sc)], sc, [], np.zeros((0, 3, 4), np.float32), default_camera(96, 64)


def placements_case(name):
    sc = scene(name)
    mats, cam = placements(sc)
    return [as_mesh(sc)], sc, [0] * len(mats), mats, cam


def field_case():
    fld = synthetic.instanced_field(scene("ShaderBalls"), copies=183, width=240, height=135)
    return fld["meshes"], fld["shared"], fld["mesh_ids"], fld["transforms"], fld["camera_pose"]


CASES = {"placements_CornellBox": lambda: placements_case("CornellBox"), "placements_ShaderBalls": lambda: placements_case("ShaderBalls"),
         "field": field_case, "far_ill_conditioned": lambda: far_camera_case(1.0, 4.675), "far_ill_conditioned_small": lambda: far_camera_case(1e-3, 1.625),
         "offset_mesh": offset_mesh_case, "coinciding": coinciding_case, "single_leaf": single_leaf_case, "one_instance": one_instance_case,
         "zero_instances": zero_instances_case}
SIZE = {"field": (240, 135)}
SAMPLE = {"field": 4000}
# A closest hit may be lost to the rounding of a box of its mesh's own tree, as in a flat scene (the mesh's tree traced alone with
# the same object-space ray loses it too: InstanceReference.mesh_lost); at most this share of the rays.  A loss the mesh's tree
# alone does not share is the top level's, and fails.
ALLOW_MESH_LOST = 0.01


def check_rays(model, ids, mats, ref_scene, rays, where, allow_box):
    """The model's closest and any-hit traversal of `rays` against the brute force -> the verdict's report."""
    ref = ref_scene.closest(rays)
    cls = ref_scene.classify(rays, ref)[0]
    hits = model.trace_instanced(ids, mats, rays)
    got_t = np.where(hits["primitive_id"] != INVALID_ID, hits["t"], np.float32(np.inf))
    lost = ref_scene.mesh_lost(model, rays, got_t, ref)
    rep = ref_scene.verdict(rays, hits["primitive_id"], hits["bc"], hits["t"], where, ref=ref, cls=cls, allow_box=allow_box, lost=lost)
    rep["mesh_lost"] = int(lost.sum())
    occ = model.trace_instanced(ids, mats, rays, any_hit=True)
    box = ref_scene.mesh_lost(model, rays, np.full(len(rays), np.inf, np.float32), ref)
    bad = np.flatnonzero(((occ == 0) != (ref.n_accepted > 0)) & ~box)
    assert bad.size == 0, (where, "any hit", bad[:8].tolist())
    return ref, box, rep


@pytest.mark.parametrize("name", sorted(CASES))
def test_model_meets_the_instanced_brute_force(name):
    meshes, shared, ids, mats, cam = CASES[name]()
    w, h = SIZE.get(name, (96, 64))
    rays = camera_rays(shared, cam, w, h)
    if name in SAMPLE:
        rays = rays[np.sort(np.random.default_rng(3).choice(len(rays), SAMPLE[name], replace=False))]
    model = InstanceModel(meshes, shared)
    ref_scene = IR.Scene(meshes, ids, mats)
    ref, box, rep = check_rays(model, ids, mats, ref_scene, rays, (name, "camera"), ALLOW_MESH_LOST)
    print(name, "camera", rep)
    if len(ids) == 0:
        assert (ref.prim == INVALID_ID).all()
    else:
        assert (ref.prim != INVALID_ID).sum() >= 100, (name, (ref.prim != INVALID_ID).sum())
    hit = np.flatnonzero(ref.prim != INVALID_ID)
    for t_max, blocked in ((ref.t[hit], True), (np.nextafter(ref.t[hit], np.float32(-1)), False)):
        shadow = rays[hit].copy()
        shadow["direction"][:, 3] = t_max
        want = ref_scene.any_hit(shadow)
        assert (want == blocked).all(), name
        occ = model.trace_instanced(ids, mats, shadow, any_hit=True)
        lost = ref_scene.mesh_lost(model, shadow, np.full(len(hit), np.inf, np.float32), R.select(ref, hit)) if blocked else np.zeros(len(hit), bool)
        bad = np.flatnonzero(((occ == 0) != want) & ~lost)
        assert bad.size == 0, (name, "shadow rays ending at t" if blocked else "shadow rays ending before t", bad[:8].tolist())


@pytest.mark.parametrize("name", ["CornellBox", "ShaderBalls"])
def test_identity_instance_equals_the_flat_brute_force(name):
    sc = scene(name)
    cam = sc.get("camera_pose", default_camera(96, 64))
    rays = camera_rays(sc, cam, 96, 64)
    if name == "ShaderBalls":
        rays = rays[::3]
    flat = R.closest(sc["triangles"], rays)
    inst = IR.Scene([as_mesh(sc)], [0], EYE[None]).closest(rays)
    assert np.array_equal(bits(inst.t), bits(flat.t)) and np.array_equal(inst.prim, flat.prim), name
    assert np.array_equal(inst.n_ties, flat.n_ties) and np.array_equal(inst.n_accepted, flat.n_accepted), name


def test_mirrored_instance_culls_the_faces_its_flattened_triangles_cull():
    """Per (ray, triangle) pair, det * sign(det M) in object space and det of the placed triangle in world space have the same
    sign wherever neither is within rounding of zero; the brute force's hits are the flattened triangles' hits."""
    sc = scene("CornellBox")
    m = mat(rot(2, 0.4) @ np.diag([-1.0, 1.0, 1.0]), (0.1, 0.2, 0.0))
    rays = camera_rays(sc, default_camera(48, 32), 48, 32)
    inst = IR.Scene([as_mesh(sc)], [0], m[None])
    w, sign = inst.inst[0]["w"], inst.inst[0]["sign"]
    assert sign == -1.0
    o, d, _, _ = R.ray_arrays(rays)
    oo, dd = IR.object_rays(w, o, d)
    p = R.tri_points(sc["triangles"])
    q = [((x[:, :1] * m[:, 0] + x[:, 1:2] * m[:, 1]) + x[:, 2:3] * m[:, 2]) + m[:, 3] for x in p]
    n_r, n_t = len(rays), len(p[0])
    r, ti = np.repeat(np.arange(n_r), n_t), np.tile(np.arange(n_t), n_r)
    det_obj = R._dot(p[1][ti] - p[0][ti], R._cross(dd[r], p[2][ti] - p[0][ti])).astype(np.float64) * sign
    det_world = R._dot(q[1][ti] - q[0][ti], R._cross(d[r], q[2][ti] - q[0][ti])).astype(np.float64)
    clear = (np.abs(det_obj) > 1e-4 * np.abs(det_obj).max()) & (np.abs(det_world) > 1e-4 * np.abs(det_world).max())
    assert clear.mean() > 0.5
    assert np.array_equal(det_obj[clear] > 0, det_world[clear] > 0)
    flat = R.closest(np.concatenate([sc["triangles"][:0], _placed(sc["triangles"], m)]), rays)
    ref = inst.closest(rays)
    same = ref.prim == flat.prim
    assert (ref.prim != INVALID_ID).any() and same.mean() >= 0.99, same.mean()


def _placed(tris, m):
    t = tris.copy()
    for v in ("v1", "v2", "v3"):
        p = t[v]["position"][:, :3]
        t[v]["position"][:, :3] = ((p[:, :1] * m[:, 0] + p[:, 1:2] * m[:, 1]) + p[:, 2:3] * m[:, 2]) + m[:, 3]
    return t
