"""The host half of instanced scenes (raytracing_b200/csrc/rt_instances.h) against the restatement in tests/instance_tree_model.py:
the world-to-object matrices, the world boxes and the top-level records, on random placements, equal centroids, one instance,
mirrored and scaled matrices, and the rejected lists."""
import ctypes as C
import math
import os
import subprocess
import tempfile

import numpy as np
import pytest

from tests import instance_tree_model as model

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def lib():
    so = os.path.join(tempfile.gettempdir(), f"libinstance_tree_host_{os.getpid()}.so")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-I" + os.path.join(REPO, "include"),
                    "-I" + os.path.join(REPO, "raytracing_b200", "csrc"), "-o", so, os.path.join(HERE, "instance_tree_host.cpp")], check=True)
    L = C.CDLL(so)
    L.inst_prepare.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                               C.c_void_p, C.POINTER(C.c_uint32), C.c_void_p, C.POINTER(C.c_int), C.c_char_p, C.c_int]
    yield L
    os.remove(so)


def prepare(L, mats, mesh_ids, mesh_boxes, mesh_tris):
    mats = np.ascontiguousarray(mats, np.float32).reshape(-1, 12)
    ids = np.ascontiguousarray(mesh_ids, np.uint32)
    mb = np.ascontiguousarray(mesh_boxes, np.float32).reshape(-1, 6)
    mt = np.ascontiguousarray(mesh_tris, np.uint32)
    n = len(ids)
    rec = np.zeros((max(n, 1), 32), np.float32); boxes = np.zeros((max(n, 1), 6), np.float32)
    records = np.zeros((max(n - 1, 1), 16), np.float32); root = np.zeros(6, np.float32)
    nrec, ref = C.c_uint32(), C.c_int()
    err = C.create_string_buffer(256)
    ok = L.inst_prepare(mats.ctypes.data, ids.ctypes.data, n, mb.ctypes.data, mt.ctypes.data, len(mt), rec.ctypes.data, boxes.ctypes.data,
                        records.ctypes.data, C.byref(nrec), root.ctypes.data, C.byref(ref), err, 256)
    if not ok:
        return None, err.value.decode()
    return {"rec": rec[:n], "boxes": boxes[:n], "records": records[:nrec.value], "root": root, "root_ref": ref.value}, ""


def rot(axis, ang):
    c, s = math.cos(ang), math.sin(ang)
    r = np.eye(3)
    i, j = [(1, 2), (0, 2), (0, 1)][axis]
    r[i, i], r[i, j], r[j, i], r[j, j] = c, -s, s, c
    return r


def placements(rng, n, mirror=False, scale=False):
    out = np.zeros((n, 3, 4), np.float32)
    for k in range(n):
        r = rot(0, rng.uniform(0, 6.3)) @ rot(1, rng.uniform(0, 6.3)) @ rot(2, rng.uniform(0, 6.3))
        if scale:
            r = r @ np.diag(rng.uniform(0.1, 10.0, 3))
        if mirror and k % 2:
            r = r @ np.diag([-1.0, 1.0, 1.0])
        out[k, :, :3] = r
        out[k, :, 3] = rng.uniform(-100, 100, 3)
    return out


def check(L, mats, ids, mesh_boxes, mesh_tris):
    got, err = prepare(L, mats, ids, mesh_boxes, mesh_tris)
    assert got is not None, err
    mb = np.asarray(mesh_boxes, np.float32).reshape(-1, 6)
    boxes = np.array([model.world_box(m, mb[i, :3], mb[i, 3:]) for m, i in zip(mats, ids)], np.float32)
    assert np.array_equal(got["boxes"].view(np.uint32), boxes.view(np.uint32))
    base = np.concatenate([[0], np.cumsum(np.asarray(mesh_tris, np.int64)[ids])[:-1]]).astype(np.uint32)
    assert np.array_equal(got["rec"][:, 27].view(np.uint32), base)
    for k, m in enumerate(mats):
        w, sign = model.inverse(m)
        np.testing.assert_allclose(got["rec"][k, :12].reshape(3, 4), w, rtol=2e-7, atol=1e-30)
        np.testing.assert_array_equal(got["rec"][k, 12:24], np.asarray(m, np.float32).reshape(12))
        assert got["rec"][k, 28] == sign
    recs, root, ref = model.tree(boxes)
    assert got["root_ref"] == ref
    assert np.array_equal(got["root"].view(np.uint32), root.view(np.uint32))
    assert np.array_equal(got["records"].view(np.uint32), recs.view(np.uint32))
    return got


MESH_BOXES = [[-1, -2, -0.5, 1, 2, 3.5], [0, 0, 0, 10, 0.1, 5]]
MESH_TRIS = [1000, 2]


@pytest.mark.parametrize("n", [1, 2, 3, 7, 64, 184, 1000])
def test_random_placements(lib, n):
    rng = np.random.default_rng(n)
    mats = placements(rng, n)
    ids = rng.integers(0, 2, n)
    got = check(lib, mats, ids, MESH_BOXES, MESH_TRIS)
    if n == 1:
        assert got["root_ref"] == ~0 and len(got["records"]) == 0
    else:
        assert len(got["records"]) == n - 1


@pytest.mark.parametrize("kind", ["mirror", "scale"])
def test_mirrored_and_scaled(lib, kind):
    rng = np.random.default_rng(7)
    mats = placements(rng, 50, mirror=kind == "mirror", scale=kind == "scale")
    got = check(lib, mats, np.zeros(50, np.uint32), MESH_BOXES, MESH_TRIS)
    signs = got["rec"][:, 28]
    if kind == "mirror":
        assert np.array_equal(signs, np.where(np.arange(50) % 2, -1.0, 1.0).astype(np.float32))
    else:
        assert np.all(signs == 1.0)


def test_equal_centroids(lib):
    """Coincident instances: every split ties, so the instance id orders them."""
    m = np.zeros((9, 3, 4), np.float32)
    m[:, :, :3] = np.eye(3)
    m[::3, :, 3] = 5.0                    # three groups of equal centroids
    got = check(lib, m, np.zeros(9, np.uint32), MESH_BOXES, MESH_TRIS)
    leaves = sorted(~int(r) for r in got["records"][:, 12:14].view(np.int32).ravel() if r < 0)
    assert leaves == list(range(9))


def test_box_contains_transformed_mesh(lib):
    """Every corner of the mesh box, transformed in float, lies inside the instance's world box."""
    rng = np.random.default_rng(3)
    mats = placements(rng, 20, scale=True)
    got = check(lib, mats, np.zeros(20, np.uint32), MESH_BOXES, MESH_TRIS)
    lo, hi = np.float32(MESH_BOXES[0][:3]), np.float32(MESH_BOXES[0][3:])
    for m, b in zip(mats, got["boxes"]):
        for c in range(8):
            p = np.array([(hi if c & 1 else lo)[0], (hi if c & 2 else lo)[1], (hi if c & 4 else lo)[2]], np.float32)
            q = ((m[:, 0] * p[0] + m[:, 1] * p[1]) + m[:, 2] * p[2]) + m[:, 3]
            assert np.all(q >= b[:3]) and np.all(q <= b[3:])


@pytest.mark.parametrize("bad", ["singular", "nan", "inf", "mesh"])
def test_rejected(lib, bad):
    m = np.zeros((2, 3, 4), np.float32)
    m[:, :, :3] = np.eye(3)
    ids = np.zeros(2, np.uint32)
    if bad == "singular":
        m[1, 2, :3] = 0.0
    elif bad == "nan":
        m[1, 0, 3] = np.nan
    elif bad == "inf":
        m[1, 1, 1] = np.inf
    else:
        ids[1] = 2
    got, err = prepare(lib, m, ids, MESH_BOXES, MESH_TRIS)
    assert got is None and "instance 1" in err


def test_id_space(lib):
    """The virtual ids must stay below 0xFFFFFFFF."""
    m = np.zeros((2, 3, 4), np.float32)
    m[:, :, :3] = np.eye(3)
    assert prepare(lib, m, [0, 0], MESH_BOXES[:1], [0x7FFFFFFF])[0] is not None
    got, err = prepare(lib, np.concatenate([m, m[:1]]), [0, 0, 0], MESH_BOXES[:1], [0x7FFFFFFF])
    assert got is None and "2^32" in err


# ---- the CPU model of the instanced frame (tests/instance_model.cpp)
EYE = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)


@pytest.mark.parametrize("name", ["CornellBox", "ShaderBalls"])
def test_model_identity_instance_equals_oracle(name):
    """One identity instance of the whole scene: W = M = I leaves every ray, position and normal unchanged (x * 1 + 0 * y + ...
    equals x except that -0 becomes +0, which changes no comparison here) and the top-level box culls nothing, so the model's frame
    is the oracle's bit for bit."""
    from oracle.orcbind import Oracle
    from raytracing_b200.camera import default_camera
    from tests.helpers import bits, scene
    from tests.instance_model import InstanceModel
    sc = scene(name)
    w, h, mb = 96, 64, 4
    cam = sc.get("camera_pose", default_camera(w, h))
    m = InstanceModel([{"triangles": sc["triangles"], "nodes": sc["nodes"]}], sc)
    for sample in (0, 5):
        rad, hits, st, _ = m.render_instanced([0], [EYE], cam, w, h, mb, sample_idx=sample)
        orad, ohits, ost = Oracle(sc).render(cam, w, h, mb, sample_idx=sample)
        assert np.array_equal(bits(rad[..., :3]), bits(orad[..., :3])), (name, sample)
        for k in ("n_ext", "n_miss", "n_shadow", "n_cont", "n_unoccluded", "n_emissive_hits"):
            assert np.array_equal(st[k][: mb + 1], ost[k][: mb + 1]), (name, k)
        assert np.array_equal(hits["primitive_id"], ohits["primitive_id"].ravel())


def field_ids(base, copies):
    """-> (the instanced field, the flattened field, the flat primitive id -> virtual id map).  Triangle k * n + j of replicate() is
    copy k's base triangle j; the builders reorder triangles, so each keeps its source index in padding[0]."""
    from raytracing_b200 import hostapi, synthetic
    t = base["triangles"].copy()
    n = len(t)
    t["padding"][:, 0] = np.arange(n)
    base = dict(base, triangles=t)
    fld = synthetic.instanced_field(base, copies=copies, width=240, height=135)
    tris, _ = synthetic.replicate(t, copies)
    tris["padding"][: copies * n, 0] += (np.arange(copies * n) // n * n).astype(np.uint32)
    tris["padding"][copies * n:, 0] = copies * n + np.arange(2)
    ordered, nodes, _ = hostapi.build_bvh(tris)
    flat = dict(base, triangles=ordered, nodes=nodes, emissive=np.zeros(0, "<u4"))
    pos = np.empty(n, np.int64); pos[fld["meshes"][0]["triangles"]["padding"][:, 0]] = np.arange(n)
    src = ordered["padding"][:, 0].astype(np.int64)
    g = fld["meshes"][1]["triangles"]["v2"]["position"]
    gpos = [int(np.nonzero((g == tris[copies * n + k]["v2"]["position"]).all(1))[0][0]) for k in range(2)]
    virt = np.where(src < copies * n, (src // n) * n + pos[src % n], copies * n + np.take(gpos, np.clip(src - copies * n, 0, 1)))
    return fld, flat, virt.astype(np.uint32)


@pytest.mark.slow
def test_model_field_against_flattened_field():
    """replicate()'s 183-copy field (10 M triangles flattened) at 240 x 135: the model's instanced frame against the oracle's frame of
    the flattened triangles.  Primary hit ids agree on >= 99.9 % of the pixels, t within 1e-5 relative where they agree, and the mean
    radiance within the noise of the frame."""
    from oracle.orcbind import Oracle
    from tests.helpers import scene
    from tests.instance_model import InstanceModel
    fld, flat, virt = field_ids(scene("ShaderBalls"), 183)
    cam = fld["camera_pose"]
    m = InstanceModel(fld["meshes"], fld["shared"])
    rad, hits, _, _ = m.render_instanced(fld["mesh_ids"], fld["transforms"], cam, 240, 135, 2)
    orad, ohits, _ = Oracle(flat).render(cam, 240, 135, 2)
    op = ohits["primitive_id"].ravel()
    want = np.where(op == 0xFFFFFFFF, 0xFFFFFFFF, virt[np.minimum(op, len(virt) - 1)])
    same = hits["primitive_id"] == want
    assert same.mean() >= 0.999, same.mean()
    both = same & (want != 0xFFFFFFFF)
    np.testing.assert_allclose(hits["t"][both], ohits["t"].ravel()[both], rtol=1e-5)
    a, b = rad[..., :3].astype(np.float64), orad[..., :3].astype(np.float64)
    assert abs(a.mean() - b.mean()) <= 3 * b.std() / np.sqrt(b.size)
