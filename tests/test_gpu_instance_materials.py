"""
GPU tests (-m gpu) of per-instance materials (rt_set_instance_materials, include/rt_b200.h).  The reference for nearly every case
is a fresh context of duplicated meshes: each instance with a row gets a private copy of its mesh whose triangles carry the
remapped mtlIndex, under the same transforms in the same order.  Compared: radiance bits, statistics, primary ids / t /
barycentrics, the albedo, depth, normal and velocity AOVs, and on the stepwise run the hits of every bounce.
- one identity instance with a row (red and green walls swapped, an untextured material onto a textured one and back) against the
  flat upload of the remapped triangles and the oracle on it, on every schedule, for CornellBox and a textured CornellBox;
- rotated, scaled, mirrored, coinciding and nested placements, and replicate()'s field: every instance with its own row, a subset
  without a row, identity rows (which also equal no assignment);
- emission through a row; the lifetime of the assignment (set_instances, mesh updates, reset, a second call, an upload, a clearing
  call, a growing table and graph replay); every error; object motion; two devices; the C++ layer.
"""
import numpy as np
import pytest

from raytracing_b200 import capi, hostapi, synthetic
from raytracing_b200.camera import default_camera
from tests.helpers import bits, scene
from tests.test_gpu_instanced_mesh_updates import assert_same, outputs, updated
from tests.test_gpu_instancing import EYE, MB, RUNS, STAT_KEYS, W, H, as_mesh, frame, inst_ctx, placements_case, rc_of

pytestmark = pytest.mark.gpu

INVALID = 0xFFFFFFFF
# CornellBox's 8 materials: 0 <-> 1 (in textured_cornell() 0 is untextured and 1 textured), 2 <-> 3 (the green and red walls)
SWAP = np.array([1, 0, 3, 2, 4, 5, 6, 7], np.uint32)


def remapped(tris, row):
    t = tris.copy()
    t["mtlIndex"] = np.asarray(row, np.uint32)[t["mtlIndex"]]
    return t


def row_of(of, i):
    r = of[i] if i < len(of) else None
    return None if r is None or int(r) in (-1, INVALID) else int(r)


def duplicated(meshes, ids, rows, of):
    """The meshes and ids of the equivalent scene: a private, remapped copy of its mesh for each instance with a row."""
    out, new_ids = list(meshes), [int(m) for m in ids]
    for i, m in enumerate(new_ids):
        r = row_of(of, i)
        if r is not None:
            out.append({"triangles": remapped(meshes[m]["triangles"], rows[r]), "nodes": meshes[m]["nodes"]})
            new_ids[i] = len(out) - 1
    return out, new_ids


def dup_ctx(meshes, shared, ids, mats, rows, of, **kw):
    m, i = duplicated(meshes, ids, rows, of)
    return inst_ctx(m, shared, i, mats, **kw)


def row_ctx(meshes, shared, ids, mats, rows, of, **kw):
    c = inst_ctx(meshes, shared, ids, mats, **kw)
    c.set_instance_materials(rows, of)
    return c


def bounce_hits(c, mb=MB):
    """The stepwise frame with every bounce's hits read after its rt_intersect: [(pixels, hit bytes) by pixel] per bounce."""
    c.reset(); c.generate_rays()
    out = []
    for b in range(mb + 1):
        c.intersect(b)
        h, pix = c.read_hits(b)
        o = np.argsort(pix, kind="stable")
        out.append((pix[o].copy(), h[o].tobytes()))
        if b == 0:
            c.compute_aovs()
        c.shade_miss(b); c.clear_outgoing_counter(b); c.clear_shadow_counter(); c.shade_hits(b); c.intersect_shadow(); c.accumulate_direct()
    c.advance_sample_count()
    return out


def assert_equivalent(c, ref, run="default", w=W, h=H, where=()):
    assert_same(outputs(c, run, w, h), outputs(ref, run, w, h), where)
    if run == "stepwise":
        for b, (x, y) in enumerate(zip(bounce_hits(c), bounce_hits(ref))):
            assert np.array_equal(x[0], y[0]) and x[1] == y[1], (where, "bounce", b)


# ---- 1. one identity instance with a row against the flat upload of the remapped triangles and the oracle
@pytest.mark.parametrize("name", ["CornellBox", "textured"])
def test_identity_instance_equals_remapped_flat_upload_and_oracle(name):
    from oracle.orcbind import Oracle
    from tests.scenes_extra import textured_cornell
    sc = textured_cornell() if name == "textured" else scene(name)
    cam = default_camera(W, H)
    flat = dict(sc); flat["triangles"] = remapped(sc["triangles"], SWAP)
    orad, _, ost = Oracle(flat).render(cam, W, H, MB)
    f = capi.Context(W, H); f.upload_scene(flat); f.set_camera(cam)
    want = outputs(f, "default")
    want_n = frame(f, "samples")[0]
    want_hits = bounce_hits(f)
    f.destroy()
    assert np.array_equal(want[0], bits(orad[..., :3]))
    for k in STAT_KEYS:
        assert np.array_equal(want[1][k], ost[k][: MB + 1]), k
    plain = inst_ctx([as_mesh(sc)], sc, [0], [EYE], cam=cam)
    assert not np.array_equal(frame(plain, "default")[0], want[0])      # the row changes the image
    plain.destroy()
    for run, opts in RUNS.items():
        c = row_ctx([as_mesh(sc)], sc, [0], [EYE], [SWAP], [0], cam=cam, options=opts)
        got = outputs(c, run)
        if run == "samples":                                            # three samples; their statistics are summed
            assert np.array_equal(got[0], want_n), (name, run)
            got = want[:2] + got[2:]
        assert_same(got, want, (name, run))
        if run == "stepwise":
            for b, (x, y) in enumerate(zip(bounce_hits(c), want_hits)):
                assert np.array_equal(x[0], y[0]) and x[1] == y[1], (name, "bounce", b)
        c.destroy()


# ---- 2. placements and the field against duplicated meshes
def placement_rows(kind, n, n_mat, seed=3):
    rng = np.random.default_rng(seed)
    ident = np.arange(n_mat, dtype=np.uint32)
    if kind == "own":
        return np.stack([rng.permutation(n_mat) for _ in range(n)]).astype(np.uint32), list(range(n))
    if kind == "subset":
        rows = np.stack([rng.permutation(n_mat) for _ in range(3)]).astype(np.uint32)
        return rows, [0, -1, 1, None, 2, -1, 0][:n]
    return np.stack([ident, ident]), [0, 1, 0, 1, 0, 1, 0][:n]


@pytest.mark.parametrize("kind", ["own", "subset", "identity"])
def test_placements_equal_duplicated_meshes(kind):
    sc = scene("ShaderBalls")
    mats, cam = placements_case(sc)
    ids = [0] * len(mats)
    rows, of = placement_rows(kind, len(mats), len(sc["materials"]))
    for run in ("default", "stepwise"):
        c = row_ctx([as_mesh(sc)], sc, ids, mats, rows, of, w=96, h=64, cam=cam, options=RUNS[run])
        ref = dup_ctx([as_mesh(sc)], sc, ids, mats, rows, of, w=96, h=64, cam=cam, options=RUNS[run])
        assert_equivalent(c, ref, run, 96, 64, (kind, run))
        if kind == "identity":                                          # an identity row equals no assignment at all
            plain = inst_ctx([as_mesh(sc)], sc, ids, mats, w=96, h=64, cam=cam, options=RUNS[run])
            assert_same(outputs(c, run, 96, 64), outputs(plain, run, 96, 64), (kind, run, "no assignment"))
            plain.destroy()
        c.destroy(); ref.destroy()


def test_field_equals_duplicated_meshes():
    """replicate()'s field (48 copies and the ground): every instance its own permutation of the materials, the ground without."""
    base = scene("ShaderBalls")
    fld = synthetic.instanced_field(base, copies=48, width=160, height=90)
    ids, mats, cam = fld["mesh_ids"], fld["transforms"], fld["camera_pose"]
    rng = np.random.default_rng(11)
    rows = np.stack([rng.permutation(len(base["materials"])) for _ in range(48)]).astype(np.uint32)
    of = list(range(48)) + [-1]
    c = row_ctx(fld["meshes"], base, ids, mats, rows, of, w=160, h=90, cam=cam)
    ref = dup_ctx(fld["meshes"], base, ids, mats, rows, of, w=160, h=90, cam=cam)
    assert_equivalent(c, ref, "default", 160, 90, "field")
    plain = inst_ctx(fld["meshes"], base, ids, mats, w=160, h=90, cam=cam)
    assert not np.array_equal(frame(c, "default")[0], frame(plain, "default")[0])
    c.destroy(); ref.destroy(); plain.destroy()


# ---- 3. emission through a row
def test_row_onto_the_emissive_material():
    sc = scene("CornellBox")
    light = int(np.flatnonzero(sc["materials"]["emission"] != 0)[0])
    row = np.arange(len(sc["materials"]), dtype=np.uint32); row[2] = light          # the green wall glows
    mats = np.stack([EYE, EYE.copy()]); mats[1, :, :3] *= 0.4; mats[1, :, 3] = (0.2, -0.1, 0.3)
    for run in ("default", "stepwise"):
        c = row_ctx([as_mesh(sc)], sc, [0, 0], mats, [row], [0, -1], options=RUNS[run])
        ref = dup_ctx([as_mesh(sc)], sc, [0, 0], mats, [row], [0, -1], options=RUNS[run])
        plain = inst_ctx([as_mesh(sc)], sc, [0, 0], mats, options=RUNS[run])
        assert_equivalent(c, ref, run, where=run)
        got, base = frame(c, run)[1]["n_emissive_hits"], frame(plain, run)[1]["n_emissive_hits"]
        assert got[0] > base[0], run
        c.destroy(); ref.destroy(); plain.destroy()


# ---- 4. lifetime
def translated_lists(seed=5):
    rng = np.random.default_rng(seed)
    out = []
    for n in (3, 6, 2, 0, 9, 1):
        m = np.repeat(EYE[None], n, 0)
        m[:, :, 3] = rng.uniform(-0.6, 0.6, (n, 3))
        out.append(m)
    return out


def test_assignment_survives_set_instances_by_index():
    """Lists that grow past the buffer's capacity, shrink, go to zero and re-list: index i uses the row given for i, and indices
    beyond the assignment (4 and up) keep their mesh's materials."""
    sc = scene("CornellBox")
    rows = np.stack([SWAP, np.roll(np.arange(8, dtype=np.uint32), 3)])
    of = [1, -1, 0, 1]
    lists = translated_lists()
    c = inst_ctx([as_mesh(sc)], sc, [0] * 3, lists[0])
    c.set_instance_materials(rows, of)
    for mats in lists:
        c.set_instances([0] * len(mats), mats)
        ref = dup_ctx([as_mesh(sc)], sc, [0] * len(mats), mats, rows, of)
        assert_equivalent(c, ref, where=len(mats))
        ref.destroy()
    c.destroy()


def test_assignment_survives_mesh_updates_and_reset():
    from tests.refit_model import deform
    meshes_fld = synthetic.instanced_field(scene("ShaderBalls"), copies=6, width=W, height=H)
    meshes, shared, ids, mats, cam = meshes_fld["meshes"], meshes_fld["shared"], list(meshes_fld["mesh_ids"]), meshes_fld["transforms"], meshes_fld["camera_pose"]
    rng = np.random.default_rng(2)
    n_mat = len(shared["materials"])
    rows = np.stack([rng.permutation(n_mat) for _ in range(3)]).astype(np.uint32)
    of = [0, 1, -1, 2, 0, 1, 2]
    t = deform(meshes[0]["triangles"], "noise", seed=3)
    cur = list(meshes); cur[0] = updated(meshes[0], t)
    for run in ("default", "overlap1"):
        c = row_ctx(meshes, shared, ids, mats, rows, of, cam=cam, options=RUNS[run])
        frame(c, run)
        c.update_mesh_triangles(0, t)
        c.reset()
        ref = dup_ctx(cur, shared, ids, mats, rows, of, cam=cam, options=RUNS[run])
        assert_equivalent(c, ref, run, where=run)
        c.destroy(); ref.destroy()


def test_second_call_replaces_and_upload_or_empty_call_clears():
    sc = scene("CornellBox")
    mats = np.stack([EYE, EYE.copy(), EYE.copy()]); mats[1, :, 3] = (0.3, 0.1, 0.0); mats[2, :, :3] *= 0.5
    a_rows, a_of = [SWAP], [0, 0, 0]
    b_rows, b_of = np.stack([np.roll(np.arange(8, dtype=np.uint32), 1), SWAP]), [None, 1]
    c = row_ctx([as_mesh(sc)], sc, [0] * 3, mats, a_rows, a_of)
    c.set_instance_materials(b_rows, b_of)
    ref = dup_ctx([as_mesh(sc)], sc, [0] * 3, mats, b_rows, b_of)
    assert_equivalent(c, ref, where="replaced")
    ref.destroy()
    plain = inst_ctx([as_mesh(sc)], sc, [0] * 3, mats)
    want = outputs(plain, "default")
    plain.destroy()
    c.set_instance_materials([], [])
    assert_same(outputs(c, "default"), want, "cleared by an empty call")
    c.set_instance_materials(b_rows, b_of)
    c.upload_instanced_scene([as_mesh(sc)], sc)
    c.set_instances([0] * 3, mats)
    assert_same(outputs(c, "default"), want, "cleared by an upload")
    c.destroy()


def test_growing_table_recaptures_the_graph():
    sc = scene("CornellBox")
    mats = np.stack([EYE, EYE.copy()]); mats[1, :, 3] = (0.25, 0.0, 0.1)
    perm = lambda k: np.roll(np.arange(8, dtype=np.uint32), k)
    steps = [([SWAP], [0, 0]), (np.stack([perm(1), perm(2), SWAP]), [2, 1]), (np.stack([perm(3), SWAP]), [1, 0]),
             (np.stack([perm(k) for k in range(9)]), [8, 5])]
    g = inst_ctx([as_mesh(sc)], sc, [0, 0], mats, options=((capi.OPT_GRAPH, 1),))
    d = inst_ctx([as_mesh(sc)], sc, [0, 0], mats, options=((capi.OPT_GRAPH, 0),))
    frame(g, "default"); frame(d, "default")                            # the graph is captured before the first table exists
    for rows, of in steps:
        for c in (g, d):
            c.set_instance_materials(rows, of)
        got = frame(g, "default")
        assert np.array_equal(got[0], frame(d, "default")[0]), len(rows)
        ref = dup_ctx([as_mesh(sc)], sc, [0, 0], mats, rows, of)
        want = frame(ref, "default")
        ref.destroy()
        assert np.array_equal(got[0], want[0]) and all(np.array_equal(got[1][k], want[1][k]) for k in STAT_KEYS), len(rows)
    g.destroy(); d.destroy()


# ---- 5. errors
def test_errors_leave_the_next_frame_unchanged():
    L = capi.load_library()
    sc = scene("CornellBox")
    c = capi.Context(W, H)
    assert rc_of(lambda: c.set_instance_materials([SWAP], [0])) == -4   # no scene
    c.upload_scene(sc)
    assert rc_of(lambda: c.set_instance_materials([SWAP], [0])) == -4   # a flat scene
    c.destroy()
    mats = np.stack([EYE, EYE.copy()]); mats[1, :, 3] = (0.2, 0.1, 0.0)
    c = row_ctx([as_mesh(sc)], sc, [0, 0], mats, [SWAP], [0, -1])
    before = outputs(c, "default")
    row = np.ascontiguousarray(SWAP); of = np.zeros(2, np.uint32)
    high = SWAP.copy(); high[4] = 8
    cases = [
        ("null remaps", lambda: c._ck(L.rt_set_instance_materials(c.h, None, 1, of.ctypes.data, 2))),
        ("null remap_of_instance", lambda: c._ck(L.rt_set_instance_materials(c.h, row.ctypes.data, 1, None, 2))),
        ("entry >= n_materials", lambda: c.set_instance_materials([SWAP, high], [0, 1])),
        ("row out of range", lambda: c.set_instance_materials([SWAP], [0, 1])),
        ("row 0xFFFFFFFE", lambda: c.set_instance_materials([SWAP], [0xFFFFFFFE])),
        ("2^32 entries", lambda: c._ck(L.rt_set_instance_materials(c.h, row.ctypes.data, (1 << 32) // 8, of.ctypes.data, 2))),
        ("2^32 - 1 entries and more", lambda: c._ck(L.rt_set_instance_materials(c.h, row.ctypes.data, 0xFFFFFFFF, of.ctypes.data, 2))),
    ]
    for name, fn in cases:
        assert rc_of(fn) == -1, name
        assert_same(outputs(c, "default"), before, name)
    assert rc_of(lambda: c.set_option(capi.OPT_EMITTER_SAMPLING, 1)) == -5
    assert_same(outputs(c, "default"), before, "emitter sampling refused")
    c.destroy()


# ---- 6. object motion
def test_velocity_with_rows_equals_velocity_without():
    sc = scene("CornellBox")
    cam = default_camera(W, H)
    mats = np.stack([EYE.copy() for _ in range(3)]); mats[1, :, :3] *= 0.3; mats[1, :, 3] = (0.1, 0.0, 0.2); mats[2, :, 3] = (-0.3, 0.1, 0.1)
    moved = mats.copy(); moved[1, 0, 3] += 0.05; moved[2, 1, 3] -= 0.04
    opts = ((capi.OPT_OBJECT_MOTION, 1), (capi.OPT_AOV, 4))
    vel = []
    for rows, of in (([SWAP], [0, 0, -1]), ([], [])):
        c = row_ctx([as_mesh(sc)], sc, [0] * 3, mats, rows, of, cam=cam, options=opts)
        c.set_camera(cam)
        c.set_instances([0] * 3, moved)
        c.reset(); c.integrate(1)
        vel.append(bits(np.ascontiguousarray(c.read_aovs()[3])))
        c.destroy()
    assert np.array_equal(vel[0], vel[1]) and vel[0].any()


# ---- 7. fan-out
def test_two_devices_equal_one():
    sc = scene("CornellBox")
    mats = np.stack([EYE, EYE.copy()]); mats[1, 0, 3] = 0.3
    one = row_ctx([as_mesh(sc)], sc, [0, 0], mats, [SWAP], [None, 0])
    two = row_ctx([as_mesh(sc)], sc, [0, 0], mats, [SWAP], [None, 0], devices=[0, 0])
    a, sa = frame(one, "default"); b, sb = frame(two, "default")
    assert np.array_equal(a, b) and all(np.array_equal(sa[k], sb[k]) for k in STAT_KEYS)
    one.destroy(); two.destroy()


def test_host_render_set_instance_materials(tmp_path):
    """Render::SetInstanceMaterials through hostapi gives the image the C ABI gives."""
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
        rows = [np.arange(len(a["materials"]), dtype=np.uint32)[::-1]]
        r.upload_instanced_scene([mesh]); r.set_instances([0, 0], mats)
        r.request_reset(); r.render_frame()
        plain = r.image().copy()
        r.set_instance_materials(rows, [-1, 0])
        r.request_reset(); r.render_frame()
        img = r.image().copy()
        assert not np.array_equal(bits(img), bits(plain))
        c = capi.Context(w, h)
        c.upload_instanced_scene([mesh], a); c.set_instances([0, 0], mats); c.set_camera(hostapi.default_camera(w, h))
        c.set_instance_materials(rows, [-1, 0])
        c.reset(); c.integrate(mb)
        assert np.array_equal(bits(c.resolve()), bits(img))
        c.destroy()
    finally:
        r.close(); s.close()
