"""
GPU tests (-m gpu) of RT_OPT_OCTANT_BVH: scenes staged whole in shared memory traverse per-octant copies of the interior records
(rt_octant.h).  Radiance bits, frame statistics and primary hits with the option on equal those with it off on every schedule
and rt_integrate_samples, and rt_bvh_staging reports the mode each arm ran: small scenes, a root-leaf tree, scenes on both sides
of the size limit, rays with direction components of exactly 0 that start on box planes (the per-ray guard), trees with a
non-finite or inverted box (the per-CTA guard), and trees after rt_update_triangles and rt_rebuild_bvh.
"""
import numpy as np
import pytest

from raytracing_b200 import capi, hostapi
from oracle.orcbind import Oracle
from raytracing_b200.camera import default_camera
from tests.helpers import bits, scene
from tests.scenes_extra import closed_cornell, many_lights_scene, single_leaf_scene, textured_cornell
from tests.test_gpu_parity import run_frame, schedule_ctx
from tests.trace_cases import axis_camera

pytestmark = pytest.mark.gpu

W, H, MB = 64, 48, 4
RUNS = ("frame", "phase_graph", "phase_direct", "stepwise", "samples")


def staged_bytes(nodes, n_tris, tables=True):
    """Dynamic shared memory of a scene staged whole: canonical records + triangle records (+ 8 tables + the flag word)."""
    n_rec = max(int(((nodes["num_primitives_axis"] >> 16) == 0).sum()), 1)
    return n_rec * 64 + n_tris * 48 + (n_rec * 8 * 64 + 16 if tables else 0)


def subset_scene(n_tris):
    """The first n_tris triangles of ShaderBalls under a BVH of their own."""
    sc = dict(scene("ShaderBalls"))
    ordered, nodes, _ = hostapi.build_bvh(sc["triangles"][:n_tris].copy())
    sc["triangles"], sc["nodes"] = ordered, nodes
    sc["emissive"] = np.zeros(0, dtype="<u4")
    info = np.array(sc["scene_info"], copy=True); info["emissive_count"] = 0
    sc["scene_info"] = info
    return sc


def render(c, run, mb, w, h):
    c.reset()
    if run == "samples":
        c.integrate_samples(mb, 3)
    else:
        run_frame(c, run, mb)
    out = [bits(c.read_radiance()), c.frame_stats().tobytes()]
    c.generate_rays(); c.intersect(0)
    hits, pix = c.read_hits(0)
    prim = np.full(w * h, 0xFFFFFFFE, np.uint32); prim[pix] = hits["primitive_id"]
    return out + [prim]


def assert_on_equals_off(sc, cam, w, h, mb, where, runs=RUNS, prepare=None, mode_on=3):
    """Every run with the option 0 and 1 (each first in a context of its own, then switched in the same context) gives the same
    bits; the staging mode is 1 with the option off and mode_on with it on (3: the tables fit)."""
    for run in runs:
        got = []
        for octant in (0, 1):
            c = schedule_ctx("frame" if run == "samples" else run, sc, cam, w, h, ((capi.OPT_OCTANT_BVH, octant),))
            if prepare:
                c.reset(); run_frame(c, run if run != "samples" else "frame", mb)        # stages (and captures) the tree of the upload first
                prepare(c)
            for opt in (octant, 1 - octant):
                c.set_option(capi.OPT_OCTANT_BVH, opt)
                assert c.bvh_staging()[0] == (mode_on if opt else 1), (where, run, opt)
                got.append(render(c, run, mb, w, h))
            c.destroy()
        for other in got[1:]:
            assert np.array_equal(got[0][0], other[0]) and got[0][1] == other[1] and np.array_equal(got[0][2], other[2]), (where, run)
    return got[0]


@pytest.mark.parametrize("name", ["CornellBox", "textured", "closed", "many_lights", "leaf1", "leaf3"])
def test_small_scenes_on_every_schedule(name):
    sc = {"CornellBox": lambda: scene("CornellBox"), "textured": textured_cornell, "closed": closed_cornell, "many_lights": many_lights_scene,
          "leaf1": lambda: single_leaf_scene(1), "leaf3": lambda: single_leaf_scene(3)}[name]()
    assert staged_bytes(sc["nodes"], len(sc["triangles"])) <= 40 * 1024
    rad, _, prim = assert_on_equals_off(sc, default_camera(W, H), W, H, MB, name)
    assert (prim != 0xFFFFFFFF).any() and rad.any()


def test_both_sides_of_the_size_limit():
    sizes = {n: staged_bytes(subset_scene(n)["nodes"], n) for n in range(40, 140, 5)}
    under = max(n for n, b in sizes.items() if b <= 40 * 1024)
    over = min(n for n, b in sizes.items() if b > 40 * 1024)
    assert staged_bytes(subset_scene(over)["nodes"], over, tables=False) <= 40 * 1024       # still staged whole, without the tables
    cam = scene("ShaderBalls").get("camera_pose", default_camera(W, H))
    for n, mode in ((under, 3), (over, 1)):
        assert_on_equals_off(subset_scene(n), cam, W, H, 3, ("subset", n), runs=("frame", "phase_graph"), mode_on=mode)


@pytest.mark.parametrize("view", ["+y", "+x", "-z"])
def test_direction_components_of_exactly_zero(view):
    """Primary rays parallel to an axis that start exactly on planes of the tree's boxes: two reciprocal direction components are
    infinite and 0 * inf = NaN occurs in the slab test, where the ordered test would decide differently from the pairwise one
    (tests/test_octant_slab_cpu.py).  Such rays must run the pairwise step; later bounces are ordinary rays."""
    sc = scene("CornellBox")
    w, h = 33, 17
    position, front, up = {"+y": ((0.04, -1.0, 1.2), (0, 1, 0), (0, 0, 1)), "+x": ((-0.9, 0.13, 0.6), (1, 0, 0), (0, 0, 1)),
                           "-z": ((0.25, -0.05, 1.9), (0, 0, -1), (0, 1, 0))}[view]
    cam = axis_camera(w, h, position, front, up)
    orc = Oracle(sc)
    rays = orc.generate_rays(cam, w, h)
    o, d = rays["origin"][:, :3], rays["direction"][:, :3]
    with np.errstate(divide="ignore"):
        infinite = ~np.isfinite(np.float32(1) / d)
    assert (infinite.sum(1) == 2).all()
    planes = np.concatenate([sc["nodes"]["bounds_min"][1:, :3], sc["nodes"]["bounds_max"][1:, :3]])      # the child boxes of the records
    on_plane = (o[:, None, :] == planes[None, :, :]) & infinite[:, None, :]
    assert on_plane.any((1, 2)).all()                                    # every primary ray meets 0 * inf at some record
    assert_on_equals_off(sc, cam, w, h, 3, ("axis", view))
    rad, _, prim = assert_on_equals_off(sc, cam, w, h, 3, ("axis", view), runs=("phase_graph",))
    orad, ohits, ost = orc.render(cam, w, h, 3)
    assert np.array_equal(prim, ohits["primitive_id"]) and (prim != 0xFFFFFFFF).all()
    assert np.array_equal(rad[..., :3], bits(orad[..., :3])) and ost["n_ext"][2] > 0


def failing_records(rec):
    """Indices of the traversal records (rt_read_bvh) that rt_oct_record_ok rejects: a non-finite plane or min > max."""
    lo = np.concatenate([rec[:, 0:3], rec[:, 6:9]], 1); hi = np.concatenate([rec[:, 3:6], rec[:, 9:12]], 1)
    with np.errstate(invalid="ignore"):
        ok = (lo <= hi) & np.isfinite(lo) & np.isfinite(hi)
    return np.nonzero(~ok.all(1))[0]


@pytest.mark.parametrize("kind", ["inverted_upload", "nan_upload", "inf_vertex"])
def test_trees_that_fail_the_record_guard(kind):
    """A record with an inverted or non-finite box: every CTA finds it while building the tables and runs the pairwise step
    on the canonical records for all its rays (the mode is still 3: the decision is taken on the device).  With the infinite
    vertex a hit distance becomes NaN, where the staged traversal and the literal one part ways: only the former equals option 0."""
    sc = dict(scene("CornellBox"))
    t = None
    if kind == "inf_vertex":        # the refit's max keeps +inf (its min / max drop a NaN vertex, so a NaN never reaches a box)
        t = sc["triangles"].copy(); t["v3"]["position"][9, 2] = np.inf
    else:                           # the upload copies the caller's boxes as they are
        nodes = sc["nodes"].copy()
        k = 1 + int(np.nonzero((nodes["num_primitives_axis"][1:] >> 16) == 0)[0][0])          # an interior child
        if kind == "inverted_upload":
            nodes["bounds_min"][k, 0], nodes["bounds_max"][k, 0] = nodes["bounds_max"][k, 0], nodes["bounds_min"][k, 0]
        else:
            nodes["bounds_max"][k, 1] = np.nan
        sc["nodes"] = nodes
    seen = []

    def prepare(c):
        if t is not None:
            c.update_triangles(t)
        seen.append(len(failing_records(c.read_bvh()[1])))
    assert_on_equals_off(sc, default_camera(W, H), W, H, MB, kind, runs=("frame", "phase_graph", "stepwise"), prepare=prepare)
    assert seen and min(seen) > 0


@pytest.mark.parametrize("kind", ["flat", "nan", "rebuild"])
def test_after_geometry_updates(kind):
    sc = scene("CornellBox")
    t = sc["triangles"].copy()
    if kind == "flat":          # twelve triangles squashed into one plane: leaf boxes with min == max on z
        z = t["v1"]["position"][:, 2].min()
        for v in ("v1", "v2", "v3"):
            t[v]["position"][12:24, 2] = z
    elif kind == "nan":         # one NaN vertex: the refit's min / max drop it, the boxes stay finite; the triangle never hits
        t["v2"]["position"][7, 1] = np.nan
    else:
        rng = np.random.default_rng(3)
        for v in ("v1", "v2", "v3"):
            t[v]["position"][:, :3] += rng.uniform(-0.05, 0.05, (len(t), 3)).astype("<f4")

    def prepare(c):
        c.update_triangles(t)
        if kind == "rebuild":
            c.rebuild_bvh()
    assert_on_equals_off(sc, default_camera(W, H), W, H, MB, kind, runs=("frame", "phase_graph", "stepwise"), prepare=prepare)
