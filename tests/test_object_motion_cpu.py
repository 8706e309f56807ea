"""
CPU tests of the object-motion model (tests/motion_model.cpp, the rule stated at RT_OPT_OBJECT_MOTION in include/rt_b200.h): with
the previous positions equal to the current ones it is the oracle's GenerateAOV bit for bit; on a scene built here, a quad that
moves along the camera's right axis reports the analytic screen shift, and the temporal denoiser's reprojection fed with it takes
its history from the quad's old footprint (camera-only motion vectors take it from the same pixel).
"""
import math

import numpy as np
import pytest

from oracle.orcbind import Oracle
from raytracing_b200 import hostapi
from raytracing_b200.camera import default_camera
from raytracing_b200.layouts import TRIANGLE_DT
from tests.helpers import bits, scene
from tests.motion_model import MotionModel, positions
from tests.refit_model import refit

W, H = 64, 48


@pytest.mark.parametrize("name", ["CornellBox", "ShaderBalls", "CornellBox_Dragon"])
def test_unchanged_positions_give_the_oracle_aovs(name):
    """Q = the current positions: all four planes equal orc_aovs bit for bit, with a camera that moved since the previous one."""
    sc = scene(name)
    cam = default_camera(W, H)
    prev_cam = default_camera(W, H, position=(0.05, -1.02, 1.01), yaw=1.55)
    m = MotionModel(sc)
    want = Oracle(sc).aovs(cam, prev_cam, W, H, sample_idx=3)
    got = m.mv_aovs(sc["triangles"], cam, prev_cam, W, H, sample_idx=3)
    for g, w in zip(got, want):
        assert np.array_equal(bits(g), bits(w))
    assert np.any(got[3] != 0)


def quad(x0, x1, y, z0, z1, mtl):
    """Two triangles spanning [x0, x1] x [z0, z1] in the plane at y, facing -y (towards the default camera)."""
    t = np.zeros(2, dtype=TRIANGLE_DT)
    corners = [((x0, y, z0), (x1, y, z0), (x1, y, z1)), ((x0, y, z0), (x1, y, z1), (x0, y, z1))]
    for i, tri in enumerate(corners):
        for v, p in zip(("v1", "v2", "v3"), tri):
            t[i][v]["position"][:3] = p
            t[i][v]["normal"][:3] = (0.0, -1.0, 0.0)
        t[i]["mtlIndex"] = mtl
    return t


def known_answer_scene():
    """A backdrop 4 units in front of the default camera and a 0.6 x 0.6 quad 2 units in front of it, with a different untextured
    material; the materials, lights and environment are CornellBox's.  -> (scene dict, mask of the quad's triangles)."""
    base = scene("CornellBox")
    mats = base["materials"]
    plain = [i for i in range(len(mats)) if (mats["diffuse_albedo"][i] >> 24) == 0xFF and mats["emission"][i] == mats["emission"][0]]
    back = plain[0]
    front = next(i for i in plain if mats["diffuse_albedo"][i] != mats["diffuse_albedo"][back])
    soup = np.concatenate([quad(-5.0, 5.0, 3.0, -3.0, 5.0, back), quad(-0.3, 0.3, 1.0, 0.7, 1.3, front)])
    tris, nodes, _ = hostapi.build_bvh(soup)
    return {**base, "triangles": tris, "nodes": nodes, "emissive": np.zeros(0, "<u4")}, tris["mtlIndex"] == front


def translated(sc, mask, dx):
    t = sc["triangles"].copy()
    for v in ("v1", "v2", "v3"):
        t[v]["position"][mask, 0] += np.float32(dx)
    return {**sc, "triangles": t, "nodes": refit(sc["nodes"], t)}


def history_source(o, velocity, depth, prev_depth):
    """The pixel whose previous radiance orc_temporal_accumulation blends into each pixel (-1: none): the previous radiance
    encodes pixel i as i + 1, the current radiance is 0, so the result is 0.9 * (source + 1)."""
    prev = np.zeros((H, W, 4), "<f4")
    prev[..., 0] = (np.arange(W * H, dtype=np.float32) + 1).reshape(H, W)
    out = o.temporal_accumulation(np.zeros((H, W, 4), "<f4"), prev, depth, prev_depth, velocity)
    return np.rint(out[..., 0] / np.float32(0.9)).astype(np.int64).ravel() - 1


def test_translated_quad_known_answer_and_reprojection():
    sc, mask = known_answer_scene()
    dx = 0.3
    moved = translated(sc, mask, dx)
    cam = default_camera(W, H)
    m = MotionModel(moved)
    al, de, _, ve = m.mv_aovs(positions(sc["triangles"]), cam, cam, W, H)
    old_al, old_de, _, _ = Oracle(sc).aovs(cam, cam, W, H)

    # the quad's pixels: those whose albedo differs from the backdrop's (the corner pixel sees the backdrop)
    backdrop = al[0, 0, :3]
    on_quad = np.any(al[..., :3] != backdrop, axis=-1)
    was_quad = np.any(old_al[..., :3] != backdrop, axis=-1)
    assert 20 < on_quad.sum() < W * H // 4 and 20 < was_quad.sum() < W * H // 4
    interior = on_quad.copy()
    interior[1:-1, 1:-1] &= on_quad[:-2, 1:-1] & on_quad[2:, 1:-1] & on_quad[1:-1, :-2] & on_quad[1:-1, 2:]
    interior[[0, -1], :] = False; interior[:, [0, -1]] = False
    assert interior.sum() >= 20

    # analytic screen shift: dx / (2 z tan(fov / 2) aspect), z the quad's depth along the camera's front axis
    front = cam["front"][:3].astype(np.float64); pos = cam["position"][:3].astype(np.float64)
    z = float(np.dot(np.array([0.0, 1.0, 1.0]) - pos, front))
    want = dx / (2.0 * z * math.tan(0.5 * float(cam["fov"])) * float(cam["aspect_ratio"]))
    assert np.abs(ve[interior][:, 0] - want).max() <= 1e-6
    assert np.abs(ve[interior][:, 1]).max() <= 1e-6
    assert np.all(ve[~on_quad] == 0)                         # the backdrop does not move and neither does the camera

    # the temporal denoiser's reprojection: the model's velocity fetches from the old footprint, camera-only from the same pixel
    o = Oracle(moved)
    src = history_source(o, ve, de, old_de)
    idx = np.flatnonzero(interior)
    assert np.all(src[idx] >= 0) and np.all(was_quad.ravel()[src[idx]])
    assert np.any(~was_quad.ravel()[idx])                    # the shift moved the quad off some of its old pixels
    _, _, _, cam_only = o.aovs(cam, cam, W, H)
    assert np.all(cam_only == 0)
    src0 = history_source(o, cam_only, de, de)
    assert np.array_equal(src0[idx], idx)
