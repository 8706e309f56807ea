"""
GPU tests (-m gpu) of the 4-wide octant tables that scenes staged whole in shared memory traverse (RT_OPT_OCTANT_BVH,
rt_octant.h): radiance bits, frame statistics and primary hits with the option on equal those with it off on every schedule,
the unmerged per-phase kernels included, and rt_integrate_samples; after rt_update_triangles, rt_rebuild_bvh and
rt_rebuild_bvh_ploc; and for an uploaded tree that fails only the nesting guard (a collapsed child whose box does not contain
its children), whose CTAs must all take the binary traversal.
"""
import numpy as np
import pytest

from oracle.orcbind import Oracle
from raytracing_b200.camera import default_camera
from tests.helpers import bits, scene
from tests.scenes_extra import closed_cornell, many_lights_scene, single_leaf_scene, textured_cornell
from tests.test_gpu_octant_bvh import assert_on_equals_off, failing_records

pytestmark = pytest.mark.gpu

W, H, MB = 64, 48, 4
RUNS = ("frame", "phase_graph", "phase_direct", "timed", "stepwise", "samples")
SMALL = {"CornellBox": lambda: scene("CornellBox"), "textured": textured_cornell, "closed": closed_cornell, "many_lights": many_lights_scene,
         "leaf1": lambda: single_leaf_scene(1), "leaf3": lambda: single_leaf_scene(3)}


def off_axis_camera(w, h):
    return default_camera(w, h, position=(0.4, -1.5, 0.7), yaw=1.8, pitch=1.45, aperture=0.03, focus_distance=2.0)


@pytest.mark.parametrize("name", sorted(SMALL))
def test_small_scenes_on_every_schedule(name):
    rad, _, prim = assert_on_equals_off(SMALL[name](), off_axis_camera(W, H), W, H, MB, name, runs=RUNS)
    assert (prim != 0xFFFFFFFF).any() and rad.any()


@pytest.mark.parametrize("kind", ["update", "rebuild", "ploc"])
def test_after_geometry_updates(kind):
    sc = scene("CornellBox")
    rng = np.random.default_rng(11)
    t = sc["triangles"].copy()
    for v in ("v1", "v2", "v3"):
        t[v]["position"][:, :3] += rng.uniform(-0.04, 0.04, (len(t), 3)).astype("<f4")

    def prepare(c):
        c.update_triangles(t)
        if kind != "update":
            c.rebuild_bvh("linear" if kind == "rebuild" else "ploc")
    assert_on_equals_off(sc, off_axis_camera(W, H), W, H, MB, kind, runs=("frame", "phase_graph", "timed", "stepwise"), prepare=prepare)


def test_tree_that_fails_only_the_nesting_guard():
    """The root's first child (node 1, interior: collapsed into the root's wide node) gets a box that no longer contains its
    children.  Every record still passes rt_oct_record_ok, so only rt_wide_nests stops the CTAs from using the tables; the
    binary traversal tests the shrunken box and skips the triangles outside it, where a wide step that skipped that test would
    find them.  Option 1 must give option 0's bits, which the oracle on the same tree confirms."""
    sc = dict(scene("CornellBox"))
    nodes = sc["nodes"].copy()
    assert (nodes["num_primitives_axis"][[0, 1, 2]] >> 16 == 0).all()
    nodes["bounds_max"][1, 0] = 0.0; nodes["bounds_max"][1, 2] = 0.3
    sc["nodes"] = nodes
    seen = []

    def prepare(c):
        seen.append(len(failing_records(c.read_bvh()[1])))
    rad, _, _ = assert_on_equals_off(sc, default_camera(W, H), W, H, MB, "nesting", runs=("frame", "phase_graph", "timed", "stepwise"),
                                     prepare=prepare)
    assert seen and max(seen) == 0
    orad, _, _ = Oracle(sc).render(default_camera(W, H), W, H, MB)
    assert np.array_equal(rad[..., :3], bits(orad[..., :3]))
    full, _, _ = Oracle(scene("CornellBox")).render(default_camera(W, H), W, H, MB)
    assert not np.array_equal(bits(full[..., :3]), bits(orad[..., :3]))      # the shrunken box changes the image
