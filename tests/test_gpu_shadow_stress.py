"""
GPU tests (-m gpu) of the any-hit loop on the 4-wide octant tables (trace_fast<true, false, 3>: k_trace_both<3>,
k_shadow_accumulate<false, 3>) on shadow rays built to stress it.  Each scene is rendered on the per-phase schedules and the
one-kernel frame with RT_OPT_OCTANT_BVH on (the table walk where the tables are staged) and off (the binary SMEM 1 loop): radiance
bits, the frame statistics (n_shadow and n_unoccluded per bounce) and the primary hits must be equal, and equal the oracle's.

- cloud: small triangles of both facings scattered through the box, so that a shadow ray reaches many leaves before its first
  hit, or none; the floor and walls under the cloud mix, in one warp, rays that reach no leaf with rays that reach several.
- wall light: point lights on the back wall's plane, so that unoccluded rays end exactly where that wall is, at t_max.
- axis lights: directional lights along +z and in the x = 0 plane, so that every shadow ray has direction components of exactly
  0 and starts on box planes (the floor's, the walls'): the per-ray guard must send them to the SMEM 1 loop.
"""
import numpy as np
import pytest

from oracle.orcbind import Oracle
from raytracing_b200 import capi, hostapi
from raytracing_b200.camera import default_camera
from tests.helpers import bits, scene
from tests.test_gpu_octant_bvh import assert_on_equals_off, staged_bytes

pytestmark = pytest.mark.gpu

W, H, MB = 96, 64, 4
RUNS = ("phase_graph", "phase_direct", "timed", "frame")


def with_lights(sc, lights):
    sc = dict(sc)
    out = np.zeros(len(lights), dtype=sc["lights"].dtype)
    for i, (kind, origin, rad) in enumerate(lights):
        out[i]["origin"][:3] = origin; out[i]["radiance"][:3] = rad; out[i]["type"] = kind
    sc["lights"] = out
    info = np.array(sc["scene_info"], copy=True); info["analytic_light_count"] = len(out)
    sc["scene_info"] = info
    return sc


def cloud_scene(n=48, seed=3):
    """CornellBox with n small triangles (edge about 0.12, random orientation) inside the box, under a BVH of its own."""
    sc = dict(scene("CornellBox"))
    tris = sc["triangles"]
    rng = np.random.default_rng(seed)
    extra = np.repeat(tris[[4]], n).copy()
    centre = rng.uniform((-0.8, -0.8, 0.3), (0.8, 0.8, 1.7), (n, 3)).astype("<f4")
    for v in ("v1", "v2", "v3"):
        extra[v]["position"][:, :3] = centre + rng.uniform(-0.08, 0.08, (n, 3)).astype("<f4")
    e1 = extra["v2"]["position"][:, :3] - extra["v1"]["position"][:, :3]
    e2 = extra["v3"]["position"][:, :3] - extra["v1"]["position"][:, :3]
    nrm = np.cross(e1, e2); nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    for v in ("v1", "v2", "v3"):
        extra[v]["normal"][:, :3] = nrm
    ordered, nodes, _ = hostapi.build_bvh(np.concatenate([tris, extra]))
    sc["triangles"], sc["nodes"] = ordered, nodes
    emissive_mtl = tris["mtlIndex"][sc["emissive"]]
    sc["emissive"] = np.flatnonzero(np.isin(ordered["mtlIndex"], emissive_mtl)).astype("<u4")
    return sc


def directional(d):
    d = np.asarray(d, np.float32)
    return d / np.float32(np.sqrt((d * d).sum(dtype=np.float32)))


SCENES = {
    "cloud": lambda: cloud_scene(),
    "cloud_point_lights": lambda: with_lights(cloud_scene(seed=7), [(0, (0.1, 0.2, 1.9), (4.0, 4.0, 4.0)), (0, (-0.5, -0.5, 0.5), (3.0, 1.0, 1.0)),
                                                                    (1, directional((-0.156, -0.389, 0.908)), (1.0, 1.0, 1.0))]),
    "wall_light": lambda: with_lights(scene("CornellBox"), [(0, (0.3, 1.0, 1.2), (5.0, 5.0, 5.0)), (0, (-0.25, 1.0, 0.75), (2.0, 3.0, 4.0))]),
    "axis_lights": lambda: with_lights(cloud_scene(seed=11), [(1, (0.0, 0.0, 1.0), (2.0, 2.0, 2.0)), (1, directional((0.0, -0.6, 0.8)), (1.0, 2.0, 1.0))]),
}


def off_axis_camera(w, h):
    return default_camera(w, h, position=(0.4, -1.5, 0.7), yaw=1.8, pitch=1.45, aperture=0.03, focus_distance=2.0)


@pytest.mark.parametrize("name", sorted(SCENES))
def test_shadow_rays_on_the_tables_equal_the_binary_loop_and_the_oracle(name):
    sc = SCENES[name]()
    assert staged_bytes(sc["nodes"], len(sc["triangles"])) <= 40 * 1024          # the octant tables are staged (mode 3)
    for cam in (default_camera(W, H), off_axis_camera(W, H)):
        rad, stats, prim = assert_on_equals_off(sc, cam, W, H, MB, name, runs=RUNS)
        orad, _, ost = Oracle(sc).render(cam, W, H, MB)
        assert np.array_equal(rad[..., :3], bits(orad[..., :3])), name
        st = np.frombuffer(stats, dtype=capi.FRAME_STATS_DT)[0]
        for k in ("n_shadow", "n_unoccluded"):
            assert np.array_equal(st[k][: MB + 1], ost[k][: MB + 1]), (name, k)
        shadow, unocc = int(st["n_shadow"][: MB + 1].sum()), int(st["n_unoccluded"][: MB + 1].sum())
        assert 0 < unocc < shadow, (name, shadow, unocc)                      # both outcomes occur
