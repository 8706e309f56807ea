"""
GPU tests (-m gpu) of instanced scenes (rt_upload_instanced_scene, rt_set_instances; include/rt_b200.h):
- one identity instance of a whole scene gives the flat upload's radiance, statistics and hit ids bit for bit on every schedule
  (per-phase graph and direct launches, overlap 0 / 1 / 2, PDL off, kernel timing, traversal counting, the stepwise calls and
  rt_integrate_samples), and a two-device context gives the single device's bits;
- rotated, non-uniformly scaled, mirrored and overlapping instances, and replicate()'s field, agree with their flattened triangles
  in hit depth and shading normal (the matrix arithmetic rounds differently from flattening, so not bit for bit);
- rt_set_instances between frames (count growing, shrinking, zero) gives the frames of a context that was given each list first;
- virtual ids: a hit's id names the instance and mesh triangle whose placed plane contains the hit point;
- object motion: the velocity AOV follows the previous transform of each instance;
- every rejected argument and unsupported call.
"""
import numpy as np
import pytest

from raytracing_b200 import capi, hostapi, synthetic
from raytracing_b200.camera import default_camera
from tests.helpers import bits, scene
from tests.test_gpu_parity import run_frame

pytestmark = pytest.mark.gpu

W, H, MB = 64, 48, 4
STAT_KEYS = ("n_ext", "n_miss", "n_shadow", "n_cont", "n_unoccluded", "n_emissive_hits")
RUNS = {
    "default": (),
    "phase_direct": ((capi.OPT_GRAPH, 0),),
    "overlap0": ((capi.OPT_OVERLAP, 0),),
    "overlap1": ((capi.OPT_OVERLAP, 1),),
    "no_pdl": ((capi.OPT_PDL, 0),),
    "timed": ((capi.OPT_KERNEL_TIMING, 1),),
    "counted": ((capi.OPT_COUNT_TRAVERSAL, 1),),
    "frame_kernel": ((capi.OPT_FRAME_KERNEL, 1),),
    "stepwise": (),
    "samples": (),
}
EYE = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)


def as_mesh(sc):
    return {"triangles": sc["triangles"], "nodes": sc["nodes"]}


def inst_ctx(meshes, shared, ids, mats, w=W, h=H, cam=None, options=(), devices=None):
    c = capi.Context(w, h, devices=devices)
    for k, v in options:
        c.set_option(k, v)
    c.upload_instanced_scene(meshes, shared)
    c.set_instances(ids, mats)
    c.set_camera(cam if cam is not None else shared.get("camera_pose", default_camera(w, h)))
    return c


def frame(c, run, mb=MB):
    c.reset()
    if run == "samples":
        c.integrate_samples(mb, 3)
    else:
        run_frame(c, run, mb)
    st = c.frame_stats()
    return bits(c.read_radiance()[..., :3]), {k: st[k][: mb + 1].copy() for k in STAT_KEYS + ("nodes_ext",)}


def primary_hits(c, w=W, h=H):
    c.reset(); c.generate_rays(); c.intersect(0)
    hits, pix = c.read_hits(0)
    prim = np.full(w * h, 0xFFFFFFFE, np.uint32); prim[pix] = hits["primitive_id"]
    return prim, hits, pix


@pytest.mark.parametrize("name", ["CornellBox", "ShaderBalls"])
def test_identity_instance_equals_flat_upload(name):
    sc = scene(name)
    cam = sc.get("camera_pose", default_camera(W, H))
    ref = capi.Context(W, H); ref.upload_scene(sc); ref.set_camera(cam)
    rad0, st0 = frame(ref, "default")
    radn, _ = frame(ref, "samples")
    prim0, _, _ = primary_hits(ref)
    ref.destroy()
    for run, opts in RUNS.items():
        c = inst_ctx([as_mesh(sc)], sc, [0], [EYE], cam=cam, options=opts)
        assert c.bvh_staging()[0] == 0
        rad, st = frame(c, run)
        assert np.array_equal(rad, radn if run == "samples" else rad0), (name, run)
        if run != "samples":
            for k in STAT_KEYS:
                assert np.array_equal(st[k], st0[k]), (name, run, k)
        if run == "counted":
            assert (st["nodes_ext"][:1] > 0).all()
        if run == "timed":
            kt = c.kernel_times()
            assert kt["trace_closest"][1] > 0 and kt["shade_queues"][1] > 0
        prim, _, _ = primary_hits(c)
        assert np.array_equal(prim, prim0), (name, run)
        c.destroy()


def test_two_devices_equal_one():
    sc = scene("CornellBox")
    mats = np.stack([EYE, EYE.copy()]); mats[1, 0, 3] = 0.3
    one = inst_ctx([as_mesh(sc)], sc, [0, 0], mats)
    two = inst_ctx([as_mesh(sc)], sc, [0, 0], mats, devices=[0, 0])
    a, sa = frame(one, "default"); b, sb = frame(two, "default")
    assert np.array_equal(a, b) and all(np.array_equal(sa[k], sb[k]) for k in STAT_KEYS)
    one.destroy(); two.destroy()


def placed(tris, m):
    """The triangles of a mesh placed by m (3x4), positions in float as shading computes M * p; normals by the inverse transpose."""
    t = tris.copy()
    m = np.asarray(m, np.float32)
    wt = np.linalg.inv(m[:, :3].astype(np.float64)).T.astype(np.float32)
    for v in ("v1", "v2", "v3"):
        p = t[v]["position"][:, :3]
        t[v]["position"][:, :3] = ((p[:, :1] * m[:, 0] + p[:, 1:2] * m[:, 1]) + p[:, 2:3] * m[:, 2]) + m[:, 3]
        t[v]["normal"][:, :3] = t[v]["normal"][:, :3] @ wt.T
    return t


def flattened(sc, parts):
    """A flat scene of the placed meshes [(triangles, m), ...] under a BVH of its own."""
    tris = np.concatenate([placed(t, m) for t, m in parts])
    ordered, nodes, _ = hostapi.build_bvh(tris)
    out = dict(sc); out["triangles"], out["nodes"] = ordered, nodes
    out["emissive"] = np.zeros(0, "<u4")
    return out


def aovs(c, mb=1):
    c.set_option(capi.OPT_AOV_ALWAYS, 1)
    c.reset(); c.integrate(mb)
    _, depth, normal, _ = c.read_aovs()
    return depth, normal


def assert_agrees_with_flattened(meshes, sc, ids, mats, cam, w, h, min_share=0.999):
    flat = flattened(sc, [(meshes[i]["triangles"], m) for i, m in zip(ids, mats)])
    c = inst_ctx(meshes, sc, ids, mats, w=w, h=h, cam=cam)
    f = capi.Context(w, h); f.upload_scene(flat); f.set_camera(cam)
    d0, n0 = aovs(c); d1, n1 = aovs(f)
    hit = (d0 < 1e30) | (d1 < 1e30)
    assert hit.mean() > 0.05
    same = (np.abs(d0 - d1) <= 1e-5 * np.maximum(np.abs(d1), 1e-30)) & (np.abs(n0[..., :3] - n1[..., :3]).max(-1) <= 1e-4)
    assert same[hit].mean() >= min_share, same[hit].mean()
    r0 = frame(c, "default")[0].view(np.float32); r1 = frame(f, "default")[0].view(np.float32)
    assert abs(r0.mean() - r1.mean()) <= 0.02 * abs(r1.mean())
    c.destroy(); f.destroy()


def rot(axis, ang):
    c, s = np.cos(ang), np.sin(ang)
    r = np.eye(3); i, j = [(1, 2), (0, 2), (0, 1)][axis]
    r[i, i], r[i, j], r[j, i], r[j, j] = c, -s, s, c
    return r


def test_rotated_scaled_mirrored_and_overlapping_instances():
    sc = scene("ShaderBalls")
    mesh = as_mesh(sc)
    lo, hi = sc["nodes"]["bounds_min"][0, :3], sc["nodes"]["bounds_max"][0, :3]
    span = float((hi - lo).max())
    def m(r, t):
        out = np.zeros((3, 4), np.float32); out[:, :3] = r; out[:, 3] = t; return out
    mats = [m(np.eye(3), (0, 0, 0)),
            m(rot(2, 0.7) @ rot(0, 0.3), (1.2 * span, 0, 0)),                        # rotated
            m(np.diag([1.5, 0.6, 1.0]), (-1.2 * span, 0, 0)),                        # non-uniform scale
            m(rot(2, 0.4) @ np.diag([-1.0, 1.0, 1.0]), (0, 1.2 * span, 0)),          # mirror
            m(np.eye(3), (0, 1.2 * span, 0)),                                        # overlaps the mirror
            m(np.eye(3), (0, 0, 0)),                                                 # coincides with instance 0: t ties
            m(0.2 * np.eye(3), (0.1 * span, 0.1 * span, 0))]                         # inside instance 0's box
    cam = default_camera(96, 64, position=(0.5 * (lo[0] + hi[0]), float(lo[1]) - 2.5 * span, float(hi[2]) + 0.8 * span), pitch=1.9)
    assert_agrees_with_flattened([mesh], sc, [0] * len(mats), mats, cam, 96, 64, min_share=0.995)


def test_instanced_field_against_flattened_field():
    base = scene("ShaderBalls")
    fld = synthetic.instanced_field(base, copies=8, width=120, height=68)
    tris, _ = synthetic.replicate(base["triangles"], 8)
    ordered, nodes, _ = hostapi.build_bvh(tris)
    flat = dict(base); flat["triangles"], flat["nodes"] = ordered, nodes; flat["emissive"] = np.zeros(0, "<u4")
    cam = fld["camera_pose"]
    c = inst_ctx(fld["meshes"], base, fld["mesh_ids"], fld["transforms"], w=120, h=68, cam=cam)
    f = capi.Context(120, 68); f.upload_scene(flat); f.set_camera(cam)
    d0, _ = aovs(c); d1, _ = aovs(f)
    hit = (d0 < 1e30) | (d1 < 1e30)
    close = np.abs(d0 - d1) <= 1e-5 * np.maximum(np.abs(d1), 1e-30)
    assert hit.mean() > 0.9 and close[hit].mean() >= 0.999
    c.destroy(); f.destroy()


def test_set_instances_between_frames():
    sc = scene("CornellBox")
    mesh = as_mesh(sc)
    rng = np.random.default_rng(5)
    lists = []
    for n in (3, 6, 2, 0, 6, 1):
        mats = np.repeat(EYE[None], n, 0)
        mats[:, :, 3] = rng.uniform(-0.6, 0.6, (n, 3))
        lists.append(mats)
    c = inst_ctx([mesh], sc, [0] * 3, lists[0])
    for mats in lists:
        c.set_instances([0] * len(mats), mats)
        got = frame(c, "default")
        fresh = inst_ctx([mesh], sc, [0] * len(mats), mats)
        want = frame(fresh, "default")
        fresh.destroy()
        assert np.array_equal(got[0], want[0]) and all(np.array_equal(got[1][k], want[1][k]) for k in STAT_KEYS), len(mats)
        if len(mats) == 0:
            assert got[1]["n_miss"][0] == got[1]["n_ext"][0] and got[1]["n_ext"][1] == 0
    c.destroy()


def test_virtual_ids_name_the_placed_triangle():
    sc = scene("CornellBox")
    n = len(sc["triangles"])
    mats = np.stack([EYE.copy(), EYE.copy()]); mats[1, :, :3] = rot(2, 0.5) * 0.5; mats[1, :, 3] = (0.2, 0.1, 0.3)
    c = inst_ctx([as_mesh(sc)], sc, [0, 0], mats)
    c.generate_rays(); c.intersect(0)
    hits, pix = c.read_hits(0)
    rays, rpix = c.read_rays(0)
    assert np.array_equal(pix, rpix)
    ok = hits["primitive_id"] != 0xFFFFFFFF
    prim = hits["primitive_id"][ok]
    assert prim.max() < 2 * n and (prim >= n).any() and (prim < n).any()
    o, d = rays["origin"][ok, :3].astype(np.float64), rays["direction"][ok, :3].astype(np.float64)
    x = o + d * hits["t"][ok, None]
    inst = (prim >= n).astype(int)
    t = sc["triangles"][prim - inst * n]
    for k, mi in enumerate(mats):
        sel = inst == k
        p = [placed(t[sel], mi)[v]["position"][:, :3].astype(np.float64) for v in ("v1", "v2", "v3")]
        nrm = np.cross(p[1] - p[0], p[2] - p[0]); nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
        assert np.abs(((x[sel] - p[0]) * nrm).sum(1)).max() < 1e-4
    c.destroy()


def test_object_motion_follows_the_previous_transform():
    sc = scene("CornellBox")
    mats = np.stack([EYE.copy(), EYE.copy()]); mats[1, :, :3] *= 0.3; mats[1, :, 3] = (0.1, 0.0, 0.2)
    c = inst_ctx([as_mesh(sc)], sc, [0, 0], mats, options=((capi.OPT_OBJECT_MOTION, 1), (capi.OPT_AOV, 4)))
    c.set_camera(default_camera(W, H))                   # previous camera = current: camera motion is zero
    c.reset(); c.integrate(1)
    v_first = c.read_aovs()[3]
    assert not v_first.any()                             # no earlier list: previous = current
    moved = mats.copy(); moved[1, 0, 3] += 0.05
    c.set_instances([0, 0], moved)
    c.reset(); c.integrate(1)
    v = c.read_aovs()[3]
    assert v.any()
    c.set_option(capi.OPT_OBJECT_MOTION, 0)
    c.reset(); c.integrate(1)
    assert not c.read_aovs()[3].any()
    c.set_option(capi.OPT_OBJECT_MOTION, 1)
    c.set_instances([0, 0], moved)                       # the same list again: no motion
    c.reset(); c.integrate(1)
    assert not c.read_aovs()[3].any()
    c.destroy()


def rc_of(fn):
    try:
        fn()
    except capi.RtError as e:
        return e.code
    return 0


def test_errors_and_unsupported_calls():
    sc = scene("CornellBox")
    mesh = as_mesh(sc)
    c = capi.Context(W, H)
    assert rc_of(lambda: c.set_instances([0], [EYE])) == -4            # no instanced scene yet
    c.upload_scene(sc)
    assert rc_of(lambda: c.set_instances([0], [EYE])) == -4            # a flat scene
    c.upload_instanced_scene([mesh], sc)
    bad = [EYE.copy() for _ in range(4)]
    bad[0][2, :3] = 0.0; bad[1][0, 0] = np.nan; bad[2][1, 3] = np.inf
    for b in bad[:3]:
        assert rc_of(lambda: c.set_instances([0], [b])) == -1
    assert rc_of(lambda: c.set_instances([1], [EYE])) == -1            # mesh out of range
    assert rc_of(lambda: c.update_triangles(sc["triangles"])) == -5
    assert rc_of(lambda: c.rebuild_bvh("linear")) == -5
    assert rc_of(lambda: c.rebuild_bvh("ploc")) == -5
    assert rc_of(lambda: c.read_bvh()) == -5
    assert rc_of(lambda: c.set_option(capi.OPT_EMITTER_SAMPLING, 1)) == -5
    c.set_option(capi.OPT_ENV_SAMPLING, 1)                              # environment sampling works
    c.set_instances([0], [EYE]); c.set_camera(default_camera(W, H)); c.reset(); c.integrate(2)
    c.upload_scene(sc)                                                  # back to flat: emitter sampling and updates work again
    c.set_option(capi.OPT_EMITTER_SAMPLING, 1)
    assert rc_of(lambda: c.upload_instanced_scene([mesh], sc)) == -5
    c.set_option(capi.OPT_EMITTER_SAMPLING, 0)
    bad_mesh = dict(mesh); bad_mesh["nodes"] = mesh["nodes"].copy(); bad_mesh["nodes"]["bounds_max"][0, 0] = np.inf
    assert rc_of(lambda: c.upload_instanced_scene([bad_mesh], sc)) == -1
    c.destroy()


# ---- bit for bit against the CPU model of the instanced frame (tests/instance_model.cpp)
def model_frame(model, ids, mats, cam, w, h, mb, prev=None):
    return model.render_instanced(ids, mats, cam, w, h, mb, prev=prev)


def assert_equals_model(c, model, ids, mats, cam, w, h, mb, where):
    rad, hits, st, _ = model_frame(model, ids, mats, cam, w, h, mb)
    for run in ("default", "overlap0", "stepwise"):
        if run == "overlap0":
            c.set_option(capi.OPT_OVERLAP, 0)
        got, gst = frame(c, run, mb)
        assert np.array_equal(got, bits(rad[..., :3])), (where, run)
        for k in STAT_KEYS:
            assert np.array_equal(gst[k], st[k][: mb + 1]), (where, run, k)
    c.set_option(capi.OPT_OVERLAP, 2)
    _, ghits, pix = primary_hits(c, w, h)
    want = hits[pix]
    assert np.array_equal(ghits["primitive_id"], want["primitive_id"]), where
    ok = want["primitive_id"] != 0xFFFFFFFF
    assert np.array_equal(bits(ghits["t"][ok]), bits(want["t"][ok])) and np.array_equal(bits(ghits["bc"][ok]), bits(want["bc"][ok])), where


def placements_case(sc):
    lo, hi = sc["nodes"]["bounds_min"][0, :3], sc["nodes"]["bounds_max"][0, :3]
    span = float((hi - lo).max())
    def m(r, t):
        out = np.zeros((3, 4), np.float32); out[:, :3] = r; out[:, 3] = t; return out
    mats = [m(np.eye(3), (0, 0, 0)),
            m(rot(2, 0.7) @ rot(0, 0.3), (1.2 * span, 0, 0)),
            m(np.diag([1.5, 0.6, 1.0]), (-1.2 * span, 0, 0)),
            m(rot(2, 0.4) @ np.diag([-1.0, 1.0, 1.0]), (0, 1.2 * span, 0)),
            m(np.eye(3), (0, 1.2 * span, 0)),
            m(np.eye(3), (0, 0, 0)),
            m(0.2 * np.eye(3), (0.1 * span, 0.1 * span, 0))]
    cam = default_camera(96, 64, position=(0.5 * (lo[0] + hi[0]), float(lo[1]) - 2.5 * span, float(hi[2]) + 0.8 * span), pitch=1.9)
    return np.stack(mats), cam


@pytest.mark.parametrize("name", ["CornellBox", "ShaderBalls"])
def test_placed_instances_equal_the_model(name):
    """Rotation, non-uniform scale, a mirror, an instance overlapping the mirror, one coinciding with instance 0 (t ties across
    instances) and one inside instance 0's box: radiance, statistics, primary ids, t and barycentrics bit for bit."""
    from tests.instance_model import InstanceModel
    sc = scene(name)
    mats, cam = placements_case(sc)
    ids = [0] * len(mats)
    model = InstanceModel([as_mesh(sc)], sc)
    c = inst_ctx([as_mesh(sc)], sc, ids, mats, w=96, h=64, cam=cam)
    assert_equals_model(c, model, ids, mats, cam, 96, 64, MB, name)
    c.destroy()


def test_set_instances_between_frames_equals_the_model():
    from tests.instance_model import InstanceModel
    sc = scene("ShaderBalls")
    mats, cam = placements_case(sc)
    model = InstanceModel([as_mesh(sc)], sc)
    c = inst_ctx([as_mesh(sc)], sc, [0] * 3, mats[:3], w=96, h=64, cam=cam)
    for sel in ([0, 1, 2, 3, 4, 5, 6], [6, 3], [], [1, 2, 3], [0, 1, 2, 3, 4, 5, 6, 0, 3]):
        m = mats[sel] if sel else np.zeros((0, 3, 4), np.float32)
        c.set_instances([0] * len(sel), m)
        assert_equals_model(c, model, [0] * len(sel), m, cam, 96, 64, 2, sel)
    c.destroy()


def test_instanced_field_equals_the_model():
    """replicate()'s 183-copy field as instances, 240 x 135, 4 bounces."""
    from tests.instance_model import InstanceModel
    fld = synthetic.instanced_field(scene("ShaderBalls"), copies=183, width=240, height=135)
    model = InstanceModel(fld["meshes"], fld["shared"])
    c = inst_ctx(fld["meshes"], fld["shared"], fld["mesh_ids"], fld["transforms"], w=240, h=135, cam=fld["camera_pose"])
    assert_equals_model(c, model, fld["mesh_ids"], fld["transforms"], fld["camera_pose"], 240, 135, 4, "field")
    c.destroy()


def test_velocity_equals_the_model():
    """The velocity AOV after lists that move, drop and re-list instances: each index's previous transform is its transform in the
    last earlier list that had it."""
    from tests.instance_model import InstanceModel
    sc = scene("CornellBox")
    model = InstanceModel([as_mesh(sc)], sc)
    cam = default_camera(W, H)
    base = np.stack([EYE.copy() for _ in range(3)])
    base[1, :, :3] *= 0.3; base[1, :, 3] = (0.1, 0.0, 0.2); base[2, :, :3] = rot(2, 0.3) * 0.25; base[2, :, 3] = (-0.3, 0.1, 0.1)
    c = inst_ctx([as_mesh(sc)], sc, [0] * 3, base, options=((capi.OPT_OBJECT_MOTION, 1), (capi.OPT_AOV, 4)), cam=cam)
    c.set_camera(cam)                                     # previous camera = current: the velocity is the objects' own motion
    history = {i: base[i] for i in range(3)}
    lists = [base.copy(), base[:1].copy(), base.copy()]   # moved, shrunk to one, re-listed (index 1 and 2 keep their older transform)
    lists[0][1, 0, 3] += 0.05; lists[0][2, 1, 3] -= 0.04
    lists[2][1, 2, 3] += 0.03
    for mats in lists:
        prev = np.stack([history.get(i, mats[i]) for i in range(len(mats))])
        c.set_instances([0] * len(mats), mats)
        c.reset(); c.integrate(1)
        v = c.read_aovs()[3]
        _, _, _, mv = model_frame(model, [0] * len(mats), mats, cam, W, H, 1, prev=prev)
        np.testing.assert_allclose(v, mv, rtol=0, atol=1e-6)
        assert np.array_equal(v != 0, mv != 0)
        for i in range(len(mats)):
            history[i] = mats[i]
    assert v.any()
    c.destroy()


def test_host_render_instanced_scene(tmp_path):
    """Render::UploadInstancedScene / SetInstances (the C++ layer): the scene's own triangles and tree as one mesh at identity render
    the flat upload's image bit for bit; a second, moved instance changes it as the same list does through the C ABI."""
    from tests.test_host import PROC_OBJ, make_env
    w, h, mb = 64, 48, 3
    env_path, _ = make_env(tmp_path, w=64, h=32)
    s = hostapi.HostScene(PROC_OBJ)
    s.add_directional_light((-0.6, -1.5, 3.5), (15, 10, 5))
    r = hostapi.HostRender(s, w, h, env_path)
    try:
        r.set_max_bounces(mb)
        r.render_frame()
        flat = r.image().copy()
        a = s.arrays(); a["nodes"] = r.nodes()
        mesh = {"triangles": a["triangles"], "nodes": a["nodes"]}
        r.upload_instanced_scene([mesh])
        r.set_instances([0], [EYE])
        r.request_reset(); r.render_frame()
        assert np.array_equal(bits(r.image()), bits(flat))
        mats = np.stack([EYE, EYE.copy()]); mats[1, :, 3] = (0.3, 0.2, 0.1)
        r.set_instances([0, 0], mats)
        r.request_reset(); r.render_frame()
        img = r.image().copy()
        assert not np.array_equal(bits(img), bits(flat))
        c = capi.Context(w, h)
        c.upload_instanced_scene([mesh], a); c.set_instances([0, 0], mats); c.set_camera(hostapi.default_camera(w, h))
        c.reset(); c.integrate(mb)
        assert np.array_equal(bits(c.resolve()), bits(img))
        c.destroy()
    finally:
        r.close(); s.close()
