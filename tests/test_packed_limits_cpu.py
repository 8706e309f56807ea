"""
Scene builders for the tests of the packed queue words at their limits (tests/test_gpu_packed_limits.py), and the oracle-side
checks that make those scenes discriminating.  CPU only.

A shadow ray toward directional light l < 255 stores the light's index in the high byte of its sA word and no sB plane: the shadow
pass reads the direction and t_max from light_rec[2 l].  From index 255 on the byte is 0xFF and sB is stored.  The light lists
here are built so that reading another light's record, light 0's above all (the byte that 256 << 24 wraps to), changes which
shadow rays are unoccluded, not only the radiance they carry: lights 0 .. 252 shine through the closed ceiling of the box (always
occluded), lights from 253 on through its open side toward the camera (mostly unoccluded).
"""
import numpy as np
import pytest

from oracle.orcbind import Oracle
from raytracing_b200 import hostapi
from raytracing_b200.camera import default_camera
from tests.helpers import bits, scene
from tests.test_shadow_records_and_bsdf import with_lights

F = np.float32
LIGHT_COUNTS = (254, 255, 256, 257, 300)
POINT_AT = (100, 150, 200, 252, 270)         # point lights (three-plane records); 0 .. 44 and 253 .. 256 stay directional
OPEN_FROM = 253                              # first light that shines through the open side


def unit(d):
    d = np.asarray(d, F)
    return d / F(np.sqrt((d * d).sum(dtype=F)))


def light_list(n):
    """n analytic lights: (type, origin, radiance).  Directional lights below OPEN_FROM point up through the ceiling with slightly
    different directions; from OPEN_FROM on they point out of the open side (y < 0), half of them a little up and half a little
    down, so that floor and ceiling points both spawn shadow rays toward them, with origin lengths from 0.5 to 2.4 (t_max 1e4 ..
    4.8e4).  A few point lights sit inside the box."""
    out = []
    for l in range(n):
        if l in POINT_AT:
            out.append((0, (0.5 * np.sin(l), 0.4 * np.cos(l), 1.0 + 0.3 * np.sin(3 * l)), (2.0 + l % 3, 2.0, 1.0 + l % 5)))
        elif l < OPEN_FROM:
            out.append((1, unit((0.3 * np.sin(l), 0.2 * np.cos(l) - 0.3, 1.0)), (1.0, 0.9, 0.8)))
        else:
            k = l - OPEN_FROM
            d = unit((0.25 * np.sin(k), -1.0, 0.3 if k % 2 else -0.3)) * F(0.5 + 0.1 * (k % 20))
            out.append((1, d, (0.4 + 0.1 * (k % 7), 0.3 + 0.05 * (k % 11), 0.6)))
    return out


def light_scene(n):
    return with_lights(scene("CornellBox"), light_list(n))


def aliased_scene(n, how):
    """light_scene(n) with every light from index 255 on replaced by light 0 (how = "zero") or by light l & 0xFF (how = "byte"),
    keeping the count: what a shadow pass that read the light byte of those records would render."""
    lights = light_list(n)
    for l in range(255, n):
        lights[l] = lights[0] if how == "zero" else lights[l & 0xFF]
    return with_lights(scene("CornellBox"), lights)


def edge_origin_scene():
    """Directional lights whose records come out of unusual origins: non-unit, axis-aligned (exact zeros), so small that t_max is
    tiny but finite (every shadow ray unoccluded), (0, 0, 0) (NaN direction), and so large that origin * RT_MAX_RENDER_DIST or its
    squared length overflows; one point light keeps a three-plane record among them."""
    return with_lights(scene("CornellBox"), [
        (1, (0.3, -2.0, 0.9), (1.0, 0.8, 0.6)),              # non-unit
        (1, (0.0, -1.0, 0.0), (0.5, 0.5, 0.5)),              # axis-aligned: floor and ceiling get cos = 0
        (1, (0.0, 0.0, 3.0), (0.7, 0.6, 0.5)),               # axis-aligned, through the ceiling
        (1, (-1.0, 0.0, 0.0), (0.3, 0.6, 0.9)),              # axis-aligned, through a side wall
        (1, (1e-18, -3e-18, 1e-18), (0.9, 0.9, 0.2)),        # t_max ~ 7e-14: nothing occludes
        (1, (0.0, 0.0, 0.0), (1.0, 1.0, 1.0)),               # NaN direction, t_max 0
        (1, (1e36, -2e36, 1e36), (1.0, 0.2, 0.2)),           # origin * 20000 = inf
        (1, (1e20, -3e20, 0.0), (0.2, 1.0, 0.2)),            # finite product, squared length inf
        (0, (0.2, 0.3, 1.5), (2.0, 2.0, 2.0)),
    ])


def wall_scene():
    """One diffuse triangle (the back wall's material) in the plane y = 1, facing the default camera and filling its view at any
    aspect up to 3:1 with no edge in sight (a ray through an edge shared by two triangles can miss both), lit by a directional
    light from the camera's side: every primary ray hits, and nearly every hit spawns an unoccluded shadow ray and a continuation
    ray, which leaves the scene."""
    sc = dict(scene("CornellBox"))
    tris = sc["triangles"][[4]].copy()
    tris["v1"]["position"][:, :3] = (-20.0, 1.0, -20.0)
    tris["v2"]["position"][:, :3] = (20.0, 1.0, -20.0)
    tris["v3"]["position"][:, :3] = (0.0, 1.0, 40.0)
    for v in ("v1", "v2", "v3"):
        tris[v]["normal"][:, :3] = (0.0, -1.0, 0.0)
    ordered, nodes, _ = hostapi.build_bvh(tris)
    sc["triangles"], sc["nodes"] = ordered, nodes
    sc["emissive"] = np.zeros(0, dtype="<u4")
    info = np.array(sc["scene_info"], copy=True); info["emissive_count"] = 0
    sc["scene_info"] = info
    return with_lights(sc, [(1, unit((0.2, -1.0, 0.4)), (1.0, 1.0, 1.0))])


W, H, MB = 96, 64, 4


def render(sc, samples=2):
    o = Oracle(sc)
    acc = np.zeros((H, W, 4), "<f4")
    cam = default_camera(W, H)
    n_shadow = n_unocc = 0
    for s in range(samples):
        acc, _, st = o.render(cam, W, H, MB, sample_idx=s, radiance=acc, want_hits=False)
        n_shadow += int(st["n_shadow"][: MB + 1].sum()); n_unocc += int(st["n_unoccluded"][: MB + 1].sum())
    return acc, n_shadow, n_unocc


def test_light_lists_put_directional_lights_at_the_byte_boundary():
    for n in LIGHT_COUNTS:
        sc = light_scene(n)
        assert len(sc["lights"]) == n and int(np.asarray(sc["scene_info"]["analytic_light_count"]).ravel()[0]) == n
        types = sc["lights"]["type"]
        assert all(types[l] == 1 for l in (253, 254, 255, 256) if l < n), n
        assert (types == 0).sum() >= 4 and (types == 1).sum() > 240, n


@pytest.mark.parametrize("l", (255, 256, 257, 299))
def test_high_lights_disagree_with_their_aliases_at_most_shading_points(l):
    """For most primary hits where light l spawns a shadow ray, tracing it with the direction and t_max of light 0 or of light
    l & 0xFF gives the other verdict."""
    sc = light_scene(300)
    o = Oracle(sc)
    cam = default_camera(W, H)
    _, hits, _ = o.render(cam, W, H, 0)
    rays = o.generate_rays(cam, W, H)
    hit = hits["primitive_id"] != 0xFFFFFFFF
    assert hit.mean() > 0.9
    # a point just in front of each primary hit (its shading point, less the offset along the normal)
    origin = rays["origin"][hit][:, :3] + rays["direction"][hit][:, :3] * (hits["t"][hit] * F(0.999))[:, None]

    def occluded(k):
        typ, d, _ = light_list(300)[k]
        assert typ == 1
        q = np.zeros(len(origin), dtype=rays.dtype)
        q["origin"][:, :3] = origin
        q["direction"][:, :3] = unit(d)
        q["direction"][:, 3] = F(np.sqrt((np.asarray(d, F) ** 2).sum())) * F(20000.0)      # t_max
        flags, _ = o.trace(q, any_hit=True)
        return flags != 0
    v = occluded(l)
    for alias in {0, l & 0xFF} - {l}:
        assert (v != occluded(alias)).mean() > 0.5, (l, alias)


@pytest.mark.parametrize("n", (256, 257, 300))
def test_aliased_light_records_change_the_unoccluded_count(n):
    """What the GPU tests compare: a shadow pass that read light 0's record, or light l & 0xFF's, for the lights from 255 on
    would change n_unoccluded, and the radiance, against the scene as built."""
    acc, n_shadow, n_unocc = render(light_scene(n))
    assert n_shadow > 0 and 0 < n_unocc < n_shadow
    for how in ("zero", "byte") if n > 256 else ("zero",):
        aacc, _, a_unocc = render(aliased_scene(n, how))
        assert a_unocc != n_unocc, (n, how)
        assert not np.array_equal(bits(aacc[..., :3]), bits(acc[..., :3])), (n, how)


def test_edge_origin_scene_renders_finite_and_sees_the_tiny_light():
    """The oracle's per-hit length / normalize of the edge origins: the tiny-origin light is unoccluded wherever it is sampled,
    the NaN and overflowed ones spawn no shadow ray (their cos is NaN or 0), and no pixel goes NaN."""
    acc, n_shadow, n_unocc = render(edge_origin_scene())
    assert np.isfinite(acc[..., :3]).all()
    assert 0 < n_unocc < n_shadow


def test_wall_scene_spawns_a_shadow_and_a_continuation_ray_per_pixel():
    sc = wall_scene()
    for w, h in ((64, 64), (96, 32)):
        _, _, st = Oracle(sc).render(default_camera(w, h), w, h, 1, want_hits=False)
        n = w * h
        assert (st["n_ext"][0], st["n_miss"][0], st["n_shadow"][0], st["n_cont"][0], st["n_unoccluded"][0]) == (n, 0, n, n, n)
        assert st["n_miss"][1] == n and st["n_shadow"][1] == 0
