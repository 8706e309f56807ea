"""
CPU checks of mesh updates in instanced scenes (rt_update_mesh_triangles*, include/rt_b200.h): the null-context checks of the two
entry points, and the velocity model of deforming meshes (tests/mesh_motion_model.cpp: the previous mesh positions Q of object
motion on the primary hits of tests/instance_model.cpp's frame): with Q equal to the current positions it reproduces the instance
model's velocity bit for bit (replicate()'s field and a mirrored instance), and with Q moved by an offset its velocity is that of
the instance's previous transform moved by the offset.
"""
import ctypes as C

import numpy as np
import pytest

from raytracing_b200 import capi
from raytracing_b200.layouts import TRIANGLE_DT

EYE = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)


def test_entry_points_reject_a_null_context():
    L = capi.load_library()
    t = np.zeros(1, dtype=TRIANGLE_DT)
    assert L.rt_update_mesh_triangles(None, 0, t.ctypes.data, 1) == -1
    assert L.rt_update_mesh_triangles_device(None, 0, None, 1) == -1


def positions(meshes):
    """The current positions of the concatenated meshes as Q: (n, 3, 3)."""
    t = np.concatenate([m["triangles"] for m in meshes])
    return np.stack([t[v]["position"][:, :3] for v in ("v1", "v2", "v3")], axis=1).astype(np.float32)


def assert_same_frame(a, b):
    """(radiance, primary hits, statistics[, velocity]) equal bit for bit."""
    for x, y in zip(a, b):
        assert x.shape == y.shape and x.tobytes() == y.tobytes()


def field(copies=8, w=120, h=68):
    from raytracing_b200 import synthetic
    from tests.helpers import scene
    return synthetic.instanced_field(scene("ShaderBalls"), copies=copies, width=w, height=h)


def test_model_with_current_positions_reproduces_the_field():
    """replicate()'s field (8 copies and the ground): radiance, primary hits, statistics and velocity with Q = the current positions
    equal the model's output without Q, with and without moved previous transforms."""
    from tests.mesh_motion_model import MeshMotionModel
    fld = field()
    m = MeshMotionModel(fld["meshes"], fld["shared"])
    ids, mats, cam = fld["mesh_ids"], fld["transforms"], fld["camera_pose"]
    prev = mats.copy(); prev[:, :, 3] += np.float32(0.02)
    q = positions(fld["meshes"])
    for pv in (None, prev):
        a = m.render_instanced(ids, mats, cam, 120, 68, 2, prev=pv)
        b = m.render_instanced(ids, mats, cam, 120, 68, 2, prev=pv, prev_positions=q)
        assert_same_frame(a, b)
        assert (a[3] != 0).any() == (pv is not None)


def test_model_with_current_positions_reproduces_a_mirrored_instance():
    from tests.helpers import scene
    from tests.mesh_motion_model import MeshMotionModel
    from raytracing_b200.camera import default_camera
    sc = scene("CornellBox")
    mesh = {"triangles": sc["triangles"], "nodes": sc["nodes"]}
    m = MeshMotionModel([mesh], sc)
    mats = np.stack([EYE.copy(), EYE.copy()])
    mats[1, :, :3] = np.diag([-0.5, 0.5, 0.5]); mats[1, :, 3] = (0.2, -0.1, 0.3)
    prev = mats.copy(); prev[1, 1, 3] += np.float32(0.03)
    cam = default_camera(64, 48)
    a = m.render_instanced([0, 0], mats, cam, 64, 48, 3, prev=prev)
    b = m.render_instanced([0, 0], mats, cam, 64, 48, 3, prev=prev, prev_positions=positions([mesh]))
    assert_same_frame(a, b)
    assert (a[3] != 0).any()


def test_model_moved_positions_equal_a_moved_transform():
    """Q = P + d under M_prev = M = I moves the previous point as M_prev = translation by d does with Q = P: the velocities agree to
    the rounding of the two sums, and the radiance and hits do not depend on Q."""
    from tests.helpers import scene
    from tests.mesh_motion_model import MeshMotionModel
    from raytracing_b200.camera import default_camera
    sc = scene("CornellBox")
    mesh = {"triangles": sc["triangles"], "nodes": sc["nodes"]}
    m = MeshMotionModel([mesh], sc)
    d = np.array([0.03, -0.02, 0.01], np.float32)
    cam = default_camera(64, 48)
    moved = EYE.copy(); moved[:, 3] = d
    a = m.render_instanced([0], [EYE], cam, 64, 48, 1, prev=[moved])
    b = m.render_instanced([0], [EYE], cam, 64, 48, 1, prev=[EYE], prev_positions=positions([mesh]) + d)
    assert_same_frame(a[:3], b[:3])
    assert (b[3] != 0).mean() > 0.5
    np.testing.assert_allclose(b[3], a[3], rtol=0, atol=1e-5)


def test_model_rejects_a_wrong_position_count():
    from tests.helpers import scene
    from tests.mesh_motion_model import MeshMotionModel
    from raytracing_b200.camera import default_camera
    sc = scene("CornellBox")
    m = MeshMotionModel([{"triangles": sc["triangles"], "nodes": sc["nodes"]}], sc)
    with pytest.raises(ValueError):
        m.render_instanced([0], [EYE], default_camera(8, 8), 8, 8, 1, prev_positions=np.zeros((1, 3, 3), np.float32))
