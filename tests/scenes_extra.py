"""Small synthetic scene variants for edge-case tests (built from the CornellBox fixture)."""
import numpy as np

from raytracing_b200.layouts import TEXTURE_DT
from tests.helpers import scene


def textured_cornell(seed=5):
    """CornellBox with image textures on every slot the reference supports (material.h:251-264): diffuse albedo, specular
    albedo, roughness, metalness, emission, transparency — random RGBA8 texels, random per-vertex texture coordinates
    (also negative / > 1: the lookup wraps, material.h:322-323)."""
    rng = np.random.default_rng(seed)
    sc = dict(scene("CornellBox"))
    texs, texels = [], []
    for (w, h) in [(16, 16), (7, 5), (32, 8), (3, 9)]:
        texs.append((len(np.concatenate(texels)) if texels else 0, w, h, 0))
        t = rng.integers(0, 256, size=(w * h, 4), dtype=np.uint32)
        t[:, 3] = 255
        texels.append((t[:, 0] | (t[:, 1] << 8) | (t[:, 2] << 16) | (t[:, 3] << 24)).astype("<u4"))
    sc["textures"] = np.array(texs, dtype=TEXTURE_DT)
    sc["texels"] = np.concatenate(texels)
    tris = sc["triangles"].copy()
    for v in ("v1", "v2", "v3"):
        tris[v]["texcoord"][:, :2] = rng.uniform(-1.5, 2.5, size=(len(tris), 2)).astype(np.float32)
    sc["triangles"] = tris
    mats = sc["materials"].copy()
    n = len(mats)
    pick = lambda: rng.integers(0, len(texs), size=n).astype(np.uint32)
    on = lambda p: rng.random(n) < p
    def set_idx(word, shift, idx, mask):
        cur = (word >> shift) & 0xFF
        new = np.where(mask, idx, cur).astype(np.uint32)
        return (word & ~(np.uint32(0xFF) << np.uint32(shift))) | (new << np.uint32(shift))
    mats["diffuse_albedo"] = set_idx(mats["diffuse_albedo"], 24, pick(), on(0.7))
    mats["specular_albedo"] = set_idx(mats["specular_albedo"], 24, pick(), on(0.5))
    mats["roughness_metalness"] = set_idx(mats["roughness_metalness"], 8, pick(), on(0.5))
    mats["roughness_metalness"] = set_idx(mats["roughness_metalness"], 24, pick(), on(0.5))
    mats["ior_emission_idx_transparency"] = set_idx(mats["ior_emission_idx_transparency"], 8, pick(), on(0.4))
    mats["ior_emission_idx_transparency"] = set_idx(mats["ior_emission_idx_transparency"], 24, pick(), on(0.3))
    sc["materials"] = mats
    return sc


def single_leaf_scene(n_tris=1):
    """A BVH whose root is a leaf (1..4 triangles): the traversal's root-leaf path."""
    from raytracing_b200 import hostapi
    sc = dict(scene("CornellBox"))
    tris = sc["triangles"][[4, 5, 0, 1][:n_tris]].copy()          # back wall / ceiling quads
    ordered, nodes, _ = hostapi.build_bvh(tris)
    assert len(nodes) == 1 and (nodes["num_primitives_axis"][0] >> 16) == n_tris or n_tris > 2
    sc["triangles"], sc["nodes"] = ordered, nodes
    sc["emissive"] = np.zeros(0, dtype="<u4")
    info = np.array(sc["scene_info"], copy=True); info["emissive_count"] = 0
    sc["scene_info"] = info
    return sc


def closed_cornell():
    """CornellBox with its open side (the plane y = -1 of the default camera) closed by a quad of the back wall's material,
    facing into the box.  Primary rays leave through its back face (culled, trace_bvh.cl:37); every later ray stays inside, so
    paths only end when a sampled direction has pdf 0.  With no Russian roulette in the reference, their throughput decays
    through the subnormal range over a few hundred bounces.  The default light is directional: its shadow rays are always
    occluded, so the shadow-ray count of a bounce is the number of hits whose light sample is still non-zero."""
    from raytracing_b200 import hostapi
    sc = dict(scene("CornellBox"))
    tris = sc["triangles"]
    quad = tris[[4, 5]].copy()                                       # back wall (y = +1), material of the back wall
    quad["v1"]["position"][:, :3] = [(1.0, -1.0, 0.0), (-1.0, -1.0, 2.0)]
    quad["v2"]["position"][:, :3] = [(-1.0, -1.0, 0.0), (1.0, -1.0, 2.0)]
    quad["v3"]["position"][:, :3] = [(-1.0, -1.0, 2.0), (1.0, -1.0, 0.0)]
    for v in ("v1", "v2", "v3"):
        quad[v]["normal"][:, :3] = (0.0, 1.0, 0.0)
    ordered, nodes, _ = hostapi.build_bvh(np.concatenate([tris, quad]))
    sc["triangles"], sc["nodes"] = ordered, nodes
    emissive_mtl = tris["mtlIndex"][sc["emissive"]]                 # the ceiling light's triangles, now in leaf order
    sc["emissive"] = np.flatnonzero(np.isin(ordered["mtlIndex"], emissive_mtl)).astype("<u4")
    return sc


def many_lights_scene(name="CornellBox"):
    """The fixture with five analytic lights — two directional, three point lights inside the box (light.h:30-65: uniform
    pick, 1/d^2 fall-off, shadow rays that stop at the light)."""
    sc = dict(scene(name))
    lights = np.zeros(5, dtype=sc["lights"].dtype)
    lights[0] = sc["lights"][0]
    d = np.array([0.3, 0.2, 0.93], dtype=np.float32); d /= np.float32(np.sqrt((d * d).sum(dtype=np.float32)))
    lights[1]["origin"][:3] = d; lights[1]["radiance"][:3] = (2.0, 3.0, 6.0); lights[1]["type"] = 1
    for i, (pos, rad) in enumerate([((0.0, 0.0, 1.6), (3.0, 3.0, 3.0)), ((-0.6, 0.3, 0.4), (5.0, 1.0, 0.5)), ((0.7, -0.4, 1.0), (0.5, 2.0, 6.0))]):
        lights[2 + i]["origin"][:3] = pos; lights[2 + i]["radiance"][:3] = rad; lights[2 + i]["type"] = 0
    sc["lights"] = lights
    info = np.array(sc["scene_info"], copy=True); info["analytic_light_count"] = len(lights)
    sc["scene_info"] = info
    return sc
