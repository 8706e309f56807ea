"""
GPU tests (-m gpu) of mesh updates in instanced scenes (rt_update_mesh_triangles*, include/rt_b200.h):
- equivalence: after update_mesh_triangles(k, T'), a context renders what a fresh context renders that uploaded mesh k as (T', the
  refit of its nodes by tests/refit_model.py) and made the same set_instances call: radiance bits, statistics, primary hits and AOVs,
  on every schedule; an identity update also equals the context before it.  Cases: noise, a shear and a move; a mesh used by many
  instances (mirrored and coinciding ones among them), by one and by none; two meshes updated in turn; update, set_instances, update;
- one deforming case against the CPU instance model bit for bit;
- the device variant (uint8 and float32 tensors, dropped right after the call) equals the host variant;
- every error, each leaving the next frame as it was; graph replay after updates; object motion; two devices; the C++ layer.
"""
import numpy as np
import pytest

from raytracing_b200 import capi, hostapi, synthetic
from tests.helpers import bits, scene
from tests.refit_model import deform, refit
from tests.test_gpu_instancing import (EYE, MB, RUNS, STAT_KEYS, W, H, as_mesh, assert_equals_model, frame, inst_ctx, placements_case,
                                       primary_hits, rc_of)

pytestmark = pytest.mark.gpu


def updated(mesh, tris):
    """The mesh a fresh upload takes after an update: the new triangles and the refit of the mesh's own nodes."""
    return {"triangles": tris, "nodes": refit(mesh["nodes"], tris)}


def shear(tris, k=0.15):
    t = tris.copy()
    for v in ("v1", "v2", "v3"):
        p = t[v]["position"]
        p[:, 0] = p[:, 0] + np.float32(k) * p[:, 2]
    return t


def move(tris, d=(0.05, -0.03, 0.02)):
    t = tris.copy()
    for v in ("v1", "v2", "v3"):
        t[v]["position"][:, :3] += np.asarray(d, np.float32)
    return t


def outputs(c, run, w=W, h=H, mb=MB):
    """Radiance bits, statistics, primary hits (ids, t, barycentrics by pixel) and the four AOV planes of one frame."""
    rad, st = frame(c, run, mb)
    prim, hits, pix = primary_hits(c, w, h)
    order = np.argsort(pix)
    c.set_option(capi.OPT_AOV_ALWAYS, 1)
    c.reset(); c.integrate(1)
    aov = [bits(np.ascontiguousarray(a)) for a in c.read_aovs()]
    c.set_option(capi.OPT_AOV_ALWAYS, 0)
    return rad, st, prim, bits(hits["t"][order]), bits(hits["bc"][order]), aov


def assert_same(a, b, where):
    assert np.array_equal(a[0], b[0]), (where, "radiance")
    for k in STAT_KEYS:
        assert np.array_equal(a[1][k], b[1][k]), (where, k)
    for i, name in ((2, "ids"), (3, "t"), (4, "bc")):
        assert np.array_equal(a[i], b[i]), (where, name)
    for i in range(4):
        assert np.array_equal(a[5][i], b[5][i]), (where, "aov", i)


def two_mesh_field(w=W, h=H):
    """replicate()'s field with 6 copies: mesh 0 (the ShaderBalls model) under 6 rotated instances, mesh 1 (the ground) under one."""
    fld = synthetic.instanced_field(scene("ShaderBalls"), copies=6, width=w, height=h)
    return fld["meshes"], fld["shared"], list(fld["mesh_ids"]), fld["transforms"], fld["camera_pose"]


def check_against_fresh(meshes, shared, ids, mats, cam, updates, runs=("default",), w=W, h=H):
    """updates: [(mesh, triangles) | ("set", ids, mats)] applied in order to a context of (meshes, ids, mats), one per run; the fresh
    context of the final meshes and list must give the same outputs."""
    cur, ids_end, mats_end = list(meshes), ids, mats
    for u in updates:
        if u[0] == "set":
            ids_end, mats_end = u[1], u[2]
        else:
            cur[u[0]] = updated(cur[u[0]], u[1])
    for run in runs:
        opts = RUNS.get(run, ())
        c = inst_ctx(meshes, shared, ids, mats, w=w, h=h, cam=cam, options=opts)
        for u in updates:
            if u[0] == "set":
                c.set_instances(u[1], u[2])
            else:
                c.update_mesh_triangles(u[0], u[1])
        f = inst_ctx(cur, shared, ids_end, mats_end, w=w, h=h, cam=cam, options=opts)
        assert_same(outputs(c, run, w, h), outputs(f, run, w, h), run)
        c.destroy(); f.destroy()


def test_identity_update_equals_before_and_fresh_on_every_schedule():
    """ShaderBalls as one mesh under the placements of tests/test_gpu_instancing.py (rotated, scaled, mirrored, overlapping,
    coinciding, nested): an update with the mesh's own triangles changes no output, on every schedule."""
    sc = scene("ShaderBalls")
    mats, cam = placements_case(sc)
    mesh = as_mesh(sc)
    ids = [0] * len(mats)
    for run, opts in RUNS.items():
        c = inst_ctx([mesh], sc, ids, mats, w=96, h=64, cam=cam, options=opts)
        before = outputs(c, run, 96, 64)
        c.update_mesh_triangles(0, sc["triangles"])
        assert_same(outputs(c, run, 96, 64), before, run)
        c.destroy()


@pytest.mark.parametrize("kind", ["noise", "shear", "move"])
def test_deformed_mesh_equals_fresh_upload_on_every_schedule(kind):
    """One mesh under seven placements (a mirror and coinciding instances among them), deformed: every schedule gives the fresh
    upload's outputs."""
    sc = scene("ShaderBalls")
    mats, cam = placements_case(sc)
    mesh = as_mesh(sc)
    t = {"noise": lambda x: deform(x, "noise", seed=3), "shear": shear, "move": move}[kind](sc["triangles"])
    cur = updated(mesh, t)
    for run, opts in RUNS.items():
        c = inst_ctx([mesh], sc, [0] * len(mats), mats, w=96, h=64, cam=cam, options=opts)
        frame(c, run)                                         # the first frame captures the graph before the update
        c.update_mesh_triangles(0, t)
        f = inst_ctx([cur], sc, [0] * len(mats), mats, w=96, h=64, cam=cam, options=opts)
        assert_same(outputs(c, run, 96, 64), outputs(f, run, 96, 64), (kind, run))
        c.destroy(); f.destroy()


@pytest.mark.parametrize("users", ["many", "one", "none"])
def test_mesh_used_by_many_one_and_no_instances(users):
    meshes, shared, ids, mats, cam = two_mesh_field()
    if users == "none":                                       # the ground mesh unused: only the mesh is written
        ids, mats = ids[:-1], mats[:-1]
    k = 0 if users == "many" else 1
    t = move(meshes[k]["triangles"], (0.0, 0.0, 0.3)) if k == 1 else deform(meshes[0]["triangles"], "noise", seed=5)
    check_against_fresh(meshes, shared, ids, mats, cam, [(k, t)], runs=("default", "stepwise"))
    if users == "none":                                       # a later list that uses it sees the refit box
        c = inst_ctx(meshes, shared, ids, mats, cam=cam)
        c.update_mesh_triangles(1, t)
        full_ids, full_mats = two_mesh_field()[2:4]
        c.set_instances(full_ids, full_mats)
        cur = list(meshes); cur[1] = updated(meshes[1], t)
        f = inst_ctx(cur, shared, full_ids, full_mats, cam=cam)
        assert_same(outputs(c, "default"), outputs(f, "default"), "listed later")
        c.destroy(); f.destroy()


def test_two_meshes_in_turn_and_set_instances_between_updates():
    meshes, shared, ids, mats, cam = two_mesh_field()
    t0 = deform(meshes[0]["triangles"], "noise", seed=7)
    t1 = move(meshes[1]["triangles"], (0.0, 0.0, 0.2))
    check_against_fresh(meshes, shared, ids, mats, cam, [(0, t0), (1, t1)], runs=("default", "overlap1", "samples"))
    moved = mats.copy(); moved[:3, :, 3] += np.float32(0.4)
    t0b = shear(t0)
    upd = [(0, t0), ("set", ids[:3] + ids[-1:], np.concatenate([moved[:3], moved[-1:]])), (0, t0b)]
    check_against_fresh(meshes, shared, ids, mats, cam, upd, runs=("default", "phase_direct"))


def test_deformed_mesh_equals_the_model():
    from tests.instance_model import InstanceModel
    sc = scene("ShaderBalls")
    mats, cam = placements_case(sc)
    t = deform(sc["triangles"], "noise", seed=11)
    cur = updated(as_mesh(sc), t)
    ids = [0] * len(mats)
    c = inst_ctx([as_mesh(sc)], sc, ids, mats, w=96, h=64, cam=cam)
    c.update_mesh_triangles(0, t)
    assert_equals_model(c, InstanceModel([cur], sc), ids, mats, cam, 96, 64, MB, "deformed")
    c.destroy()


def tensors(t):
    import torch
    d = torch.from_numpy(t.view(np.uint8).reshape(len(t), 160).copy()).cuda()
    return {"u8": d, "f32": d.view(torch.float32)}


@pytest.mark.parametrize("src", ["u8", "f32"])
def test_device_variant_equals_host_variant(src):
    """The tensor is dropped right after the call while a frame is queued, and the allocator's next block of that size is filled
    with 0xFF at once."""
    import torch
    meshes, shared, ids, mats, cam = two_mesh_field()
    a = inst_ctx(meshes, shared, ids, mats, cam=cam)
    b = inst_ctx(meshes, shared, ids, mats, cam=cam)
    for seed in (1, 2):
        t = deform(meshes[0]["triangles"], "noise", seed=seed)
        a.update_mesh_triangles(0, t)
        b.reset(); b.integrate(MB)                            # keeps the render stream busy
        d = tensors(t)[src]
        b.update_mesh_triangles(0, d)
        del d
        junk = torch.full((len(t), 160), 255, dtype=torch.uint8, device="cuda")
        assert_same(outputs(a, "default"), outputs(b, "default"), (src, seed))
        del junk
    a.destroy(); b.destroy()


def test_errors_leave_frames_unchanged():
    import torch
    L = capi.load_library()
    sc = scene("CornellBox")
    mesh = as_mesh(sc)
    t = sc["triangles"]
    c = capi.Context(W, H)
    assert rc_of(lambda: c.update_mesh_triangles(0, t)) == -4          # no scene
    c.upload_scene(sc)
    assert rc_of(lambda: c.update_mesh_triangles(0, t)) == -4          # a flat scene
    assert rc_of(lambda: c.update_mesh_triangles(0, tensors(t)["u8"])) == -4
    c.destroy()
    mats = np.stack([EYE, EYE.copy()]); mats[1, :, 3] = (0.2, 0.1, 0.0)
    c = inst_ctx([mesh], sc, [0, 0], mats)
    before = outputs(c, "default")
    nan = t.copy(); nan["v2"]["position"][3, 1] = np.nan
    inf = t.copy(); inf["v3"]["position"][len(t) - 1, 2] = -np.inf
    pad_w = t.copy(); pad_w["v1"]["position"][:, 3] = np.nan               # the .w words are not positions
    buf = torch.zeros(len(t) * 160 + 16, dtype=torch.uint8, device="cuda")
    misaligned = buf[8: 8 + len(t) * 160].view(len(t), 160)
    cases = [
        ("mesh out of range", lambda: c.update_mesh_triangles(1, t), -1),
        ("count", lambda: c.update_mesh_triangles(0, t[:-1]), -1),
        ("null host", lambda: c._ck(L.rt_update_mesh_triangles(c.h, 0, None, len(t))), -1),
        ("null device", lambda: c._ck(L.rt_update_mesh_triangles_device(c.h, 0, None, len(t))), -1),
        ("host pointer to device variant", lambda: c._ck(L.rt_update_mesh_triangles_device(c.h, 0, t.ctypes.data, len(t))), -1),
        ("misaligned", lambda: c.update_mesh_triangles(0, misaligned), -1),
        ("nan host", lambda: c.update_mesh_triangles(0, nan), -1),
        ("inf host", lambda: c.update_mesh_triangles(0, inf), -1),
        ("nan device", lambda: c.update_mesh_triangles(0, tensors(nan)["u8"]), -1),
        ("inf device", lambda: c.update_mesh_triangles(0, tensors(inf)["f32"]), -1),
        ("flat update", lambda: c.update_triangles(t), -5),
    ]
    for name, fn, code in cases:
        assert rc_of(fn) == code, name
        assert_same(outputs(c, "default"), before, name)
    c.update_mesh_triangles(0, pad_w)                                   # accepted: mtlIndex, padding and .w are not read
    c.destroy()
    two = inst_ctx([mesh], sc, [0, 0], mats, devices=[0, 0])
    assert rc_of(lambda: two.update_mesh_triangles(0, tensors(t)["u8"])) == -5
    two.destroy()


def test_launches_count_as_misc():
    sc = scene("CornellBox")
    c = inst_ctx([as_mesh(sc)], sc, [0], [EYE], options=((capi.OPT_KERNEL_TIMING, 1),))
    c.kernel_times()
    before = c.launch_count()
    c.update_mesh_triangles(0, sc["triangles"])
    assert c.launch_count() - before == 2                               # records + refit
    c.update_mesh_triangles(0, tensors(sc["triangles"])["u8"])
    assert c.launch_count() - before == 5                               # check + records + refit
    assert c.kernel_times()["misc"][1] == 5
    c.destroy()


def test_graph_replay_after_updates_matches_direct_launches():
    meshes, shared, ids, mats, cam = two_mesh_field()
    g = inst_ctx(meshes, shared, ids, mats, cam=cam, options=((capi.OPT_GRAPH, 1),))
    d = inst_ctx(meshes, shared, ids, mats, cam=cam, options=((capi.OPT_GRAPH, 0),))
    for seed in (1, 2, 3):
        t = deform(meshes[0]["triangles"], "noise", seed=seed)
        for c in (g, d):
            c.reset(); c.integrate(MB)
            c.update_mesh_triangles(0, t)
        assert np.array_equal(frame(g, "default")[0], frame(d, "default")[0]), seed
    g.destroy(); d.destroy()


def test_object_motion_follows_mesh_updates():
    """The velocity AOV after mesh updates, with and without transform changes, against tests/mesh_motion_model.py fed the previous positions Q
    (the positions before the mesh's last update) and the previous transforms.  Without a mesh update the velocity is that of
    the parent's rule, and turning the option on changes no output."""
    from tests.mesh_motion_model import MeshMotionModel
    meshes, shared, ids, mats, cam = two_mesh_field()
    c = inst_ctx(meshes, shared, ids, mats, cam=cam)
    c.set_camera(cam)                                                   # previous camera = current: no camera motion
    plain = outputs(c, "default")
    c.set_option(capi.OPT_OBJECT_MOTION, 1)
    assert_same(outputs(c, "default"), plain, "option on, no update")
    c.set_option(capi.OPT_AOV, 4)
    q = [m["triangles"] for m in meshes]
    cur = [m["triangles"] for m in meshes]
    prev_m = mats.copy()
    steps = [(0, deform(cur[0], "noise", seed=2), None), (1, move(cur[1], (0.0, 0.0, 0.05)), None),
             (0, shear(cur[0]), mats + np.float32(0.01) * (np.arange(12).reshape(3, 4) % 2)), (None, None, None)]
    m_now = mats
    for k, t, new_mats in steps:
        if new_mats is not None:
            c.set_instances(ids, new_mats); prev_m = m_now; m_now = new_mats
        if k is not None:
            q = list(q); q[k] = cur[k]
            cur = list(cur); cur[k] = t
            c.update_mesh_triangles(k, t)
        c.reset(); c.integrate(1)
        v = c.read_aovs()[3]
        model = MeshMotionModel([updated(meshes[i], cur[i]) for i in range(2)], shared)
        qpos = np.concatenate([np.stack([x[s]["position"][:, :3] for s in ("v1", "v2", "v3")], axis=1) for x in q])
        _, _, _, mv = model.render_instanced(ids, m_now, cam, W, H, 1, prev=prev_m, prev_positions=qpos)
        np.testing.assert_allclose(v, mv, rtol=0, atol=1e-6)
        assert np.array_equal(v != 0, mv != 0)
        assert v.any()
    c.destroy()


def test_two_devices_equal_one():
    meshes, shared, ids, mats, cam = two_mesh_field()
    t = deform(meshes[0]["triangles"], "noise", seed=9)
    one = inst_ctx(meshes, shared, ids, mats, cam=cam)
    two = inst_ctx(meshes, shared, ids, mats, cam=cam, devices=[0, 0])
    for c in (one, two):
        c.update_mesh_triangles(0, t)
    a, sa = frame(one, "default"); b, sb = frame(two, "default")
    assert np.array_equal(a, b) and all(np.array_equal(sa[k], sb[k]) for k in STAT_KEYS)
    one.destroy(); two.destroy()


def test_host_render_update_mesh_triangles(tmp_path):
    """Render::UpdateMeshTriangles through hostapi gives the image the C ABI gives."""
    from tests.test_host import PROC_OBJ, make_env
    w, h, mb = 64, 48, 3
    env_path, _ = make_env(tmp_path, w=64, h=32)
    s = hostapi.HostScene(PROC_OBJ)
    s.add_directional_light((-0.6, -1.5, 3.5), (15, 10, 5))
    r = hostapi.HostRender(s, w, h, env_path)
    try:
        r.set_max_bounces(mb)
        r.render_frame()
        a = s.arrays(); a["nodes"] = r.nodes()
        mesh = {"triangles": a["triangles"], "nodes": a["nodes"]}
        mats = np.stack([EYE, EYE.copy()]); mats[1, :, 3] = (0.3, 0.2, 0.1)
        t = deform(a["triangles"], "noise", seed=4)
        r.upload_instanced_scene([mesh]); r.set_instances([0, 0], mats)
        r.update_mesh_triangles(0, t)
        r.request_reset(); r.render_frame()
        img = r.image().copy()
        c = capi.Context(w, h)
        c.upload_instanced_scene([mesh], a); c.set_instances([0, 0], mats); c.set_camera(hostapi.default_camera(w, h))
        c.update_mesh_triangles(0, t)
        c.reset(); c.integrate(mb)
        assert np.array_equal(bits(c.resolve()), bits(img))
        c.destroy()
    finally:
        r.close(); s.close()
