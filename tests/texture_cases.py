"""
Scenes for the edges of the textured-material path (material.h:251-264,319-369; rt_device.cuh sample_texture / unpack_material),
no GPU needed to build them:

- chart_scene(): a grid of camera-facing quads, one material each, on the plane y = 1 in front of the default camera.  Rows are
  texture shapes (1x1, 1x7, 7x1, 7x5, 256x256, 4096x1, a 3x4 at index 253 and a 2048x2048 at index 254, placed last in the
  texel array beyond 2^24 words), columns are texture-coordinate edges (exact integers and their float32 neighbours, -1e-9,
  +-2^23, +-2^24, +-1e30, NaN, +-inf); one more row puts a texture on each slot alone and on all six at once.  A tiny triangle
  with a vertex at the camera's position is hit at t = 0 with barycentrics (0, 0), so its vertex weights u = v = 0 meet
  infinite texture coordinates and interpolate to NaN.
- ladder_scene(): one quad per emission exponent byte 0..255 in three variants (untextured; a 1x1 white emission texture, which
  forces the per-hit decode; random bytes in every other field), diffuse, specular and transparency 0.
- write_textured_obj(): an OBJ + MTL whose materials use map_Kd, map_Ks, map_Pr, map_Pm, map_Ke and map_d on small PNGs.
"""
import os

import numpy as np

from raytracing_b200.camera import default_camera
from raytracing_b200.layouts import MATERIAL_DT, TEXTURE_DT, TRIANGLE_DT
from tests.helpers import scene

NONE = 0xFF
F32 = np.float32

# texture-coordinate edges: name -> (u centre, u half-spread, v centre, v half-spread); the per-vertex coordinates are the
# centre -/+ the spread at the quad's corners, so the interpolated coordinates sweep the float32 values around the centre
EDGES = {
    "wide": (0.5, 0.6, 0.5, 0.6),            # the whole texture and a wrap on each side
    "zero": (0.0, 0.0, 0.0, 4e-7),           # u exactly 0 (every product is 0); v around 0, both signs
    "one": (1.0, 6e-7, 1.0, 6e-7),
    "minus_one": (-1.0, 6e-7, -1.0, 6e-7),
    "three": (3.0, 1.5e-6, -2.0, 1.5e-6),
    "tiny_negative": (-1e-9, 0.0, -1e-9, 0.0),    # u - floor(u) rounds to 1.0: the clamp
    "2^23": (2.0 ** 23, 3.0, -(2.0 ** 23), 3.0),
    "2^24": (2.0 ** 24, 6.0, -(2.0 ** 24), 6.0),
    "1e30": (1e30, 0.0, -1e30, 0.0),
    "nan": (float("nan"), 0.0, 0.5, 0.0),
    "inf": (float("inf"), 0.0, float("-inf"), 0.0),
}
# texture index -> (width, height); the indices 6..252 in between are 2x3 fillers
SHAPES = {0: (1, 1), 1: (1, 7), 2: (7, 1), 3: (7, 5), 4: (256, 256), 5: (4096, 1), 253: (3, 4), 254: (2048, 2048)}
N_TEXTURES = 255
LAST_START = (1 << 24) + 4099            # data_start of texture 254; the words before it that no texture covers stay 0
SLOTS = ("diffuse", "specular", "roughness", "metalness", "emission", "transparency")
CHART_W, CHART_H = 200, 150


def rgb_word(r, g, b, idx=NONE):
    return (int(r) | int(g) << 8 | int(b) << 16 | int(idx) << 24) & 0xFFFFFFFF


def material(diffuse=(0, 0, 0), specular=(0, 0, 0), emission=(0, 0, 0, 0), roughness=128, metalness=0, ior=38, transparency=255,
             tex=None):
    """A packed material (shared_structures.h:75-81); tex: {slot: texture index}."""
    t = dict.fromkeys(SLOTS, NONE)
    t.update(tex or {})
    m = np.zeros((), MATERIAL_DT)
    m["diffuse_albedo"] = rgb_word(*diffuse, t["diffuse"])
    m["specular_albedo"] = rgb_word(*specular, t["specular"])
    m["emission"] = rgb_word(*emission[:3], emission[3])
    m["roughness_metalness"] = (roughness | t["roughness"] << 8 | metalness << 16 | t["metalness"] << 24) & 0xFFFFFFFF
    m["ior_emission_idx_transparency"] = (ior | t["emission"] << 8 | transparency << 16 | t["transparency"] << 24) & 0xFFFFFFFF
    return m


def quad(x0, x1, z0, z1, mtl, uv, y=1.0):
    """Two triangles on the plane y facing -y (the default camera), wound as CornellBox's back wall; uv: the corners' texture
    coordinates in the order (x0, z0), (x1, z0), (x1, z1), (x0, z1)."""
    t = np.zeros(2, TRIANGLE_DT)
    c = [(x0, z0), (x1, z0), (x1, z1), (x0, z1)]
    for k, corners in enumerate(((0, 1, 2), (2, 3, 0))):
        for v, ci in zip(("v1", "v2", "v3"), corners):
            t[k][v]["position"][:3] = (c[ci][0], y, c[ci][1])
            t[k][v]["normal"][:3] = (0.0, -1.0, 0.0)
            t[k][v]["texcoord"][:2] = uv[ci]
    t["mtlIndex"] = mtl
    return t


def edge_uv(edge):
    cu, su, cv, sv = EDGES[edge]
    return [(cu - su, cv - sv), (cu + su, cv - sv), (cu + su, cv + sv), (cu - su, cv + sv)]


def texel_words(start, n):
    """Distinct RGB per texel of a texture (an odd multiplier is a bijection modulo 2^24), alpha 255."""
    i = np.arange(n, dtype=np.uint64) + np.uint64(start)
    return ((i * np.uint64(2654435761) + np.uint64(0x5A17)) & np.uint64(0xFFFFFF)).astype("<u4") | np.uint32(0xFF000000)


def chart_textures():
    """-> (TEXTURE_DT records, texel words): N_TEXTURES textures, index 254 last beyond 2^24 words."""
    recs = np.zeros(N_TEXTURES, TEXTURE_DT)
    start = 0
    for i in range(N_TEXTURES - 1):
        w, h = SHAPES.get(i, (2, 3))
        recs[i] = (start, w, h, 0)
        start += w * h
    w, h = SHAPES[254]
    assert start <= LAST_START
    recs[254] = (LAST_START, w, h, 0)
    texels = np.zeros(LAST_START + w * h, "<u4")
    for r in recs:
        texels[r["data_start"]: r["data_start"] + r["width"] * r["height"]] = texel_words(r["data_start"], r["width"] * r["height"])
    return recs, texels


def finish(tris, mats, textures, texels):
    """A complete scene dict: host BVH, CornellBox's directional light and environment, the emissive triangles listed."""
    from raytracing_b200 import hostapi
    sc = dict(scene("CornellBox"))
    ordered, nodes, _ = hostapi.build_bvh(np.concatenate(tris))
    mats = np.array(mats, dtype=MATERIAL_DT)
    emissive = np.flatnonzero((mats["emission"] & 0xFFFFFF)[ordered["mtlIndex"]] != 0).astype("<u4")
    info = np.array(sc["scene_info"], copy=True); info["emissive_count"] = len(emissive)
    sc.update(triangles=ordered, nodes=nodes, materials=mats, textures=np.asarray(textures, TEXTURE_DT),
              texels=np.ascontiguousarray(texels, "<u4"), emissive=emissive, scene_info=info)
    return sc


def _cells(n_cols, n_rows, x_half, z_half, fill=0.8):
    """Quad extents on a regular grid centred on the default camera's axis (x = 0, z = 1)."""
    cw, ch = 2.0 * x_half / n_cols, 2.0 * z_half / n_rows
    out = {}
    for r in range(n_rows):
        for c in range(n_cols):
            x0, z0 = -x_half + c * cw, 1.0 - z_half + r * ch
            mx, mz = cw * (1 - fill) / 2, ch * (1 - fill) / 2
            out[r, c] = (x0 + mx, x0 + cw - mx, z0 + mz, z0 + ch - mz)
    return out


CHART_ROWS = (0, 1, 2, 3, 4, 5, 253, 254)          # one row of diffuse-textured quads per texture shape, the slot row on top


def zero_weight_triangle(mtl, w, h, px=8.5, py=8.5):
    """A triangle with v1 at the default camera's position and edges of about 1e-4: every ray from the camera within a few
    degrees of its normal has det just above the 1e-8 cut (trace_bvh.cl) and hits it at t = 0 with u = v = 0, so v2 and v3 weigh
    exactly 0 — against texture coordinates +inf and -inf.  The normal points at pixel (px, py), a corner the chart leaves empty."""
    cam = default_camera(w, h)
    o = cam["position"][:3].astype(np.float64)
    ang = np.tan(0.5 * float(cam["fov"]))
    x = (px / w * 2 - 1) * ang * float(cam["aspect_ratio"]); y = (py / h * 2 - 1) * ang
    front, up = cam["front"][:3].astype(np.float64), cam["up"][:3].astype(np.float64)
    right = np.cross(front, up)
    d = x * right + y * up + front; d /= np.linalg.norm(d)
    a = np.cross(d, up); a /= np.linalg.norm(a)
    b = np.cross(a, d)                          # e1 x e2 = a x b = -d: the rays along d are front-facing
    s = np.sqrt(1e-8 / np.cos(np.radians(5.0)))    # det = s^2 cos(angle to d) > 1e-8 within about 5 degrees
    t = np.zeros(1, TRIANGLE_DT)
    for v, p in (("v1", o), ("v2", o + s * a), ("v3", o + s * b)):
        t[0][v]["position"][:3] = p
        t[0][v]["normal"][:3] = -d
    t[0]["v1"]["texcoord"][:2] = (0.25, 0.75)
    t[0]["v2"]["texcoord"][:2] = (float("inf"), 0.5)
    t[0]["v3"]["texcoord"][:2] = (0.5, float("-inf"))
    t["mtlIndex"] = mtl
    return t


def chart_scene(tile=1):
    """The texture chart (module docstring), tile x tile copies side by side for large frames (chart_camera(tile))."""
    textures, texels = chart_textures()
    rng = np.random.default_rng(17)
    edges = list(EDGES)
    n_cols, n_rows = len(edges) + 1, len(CHART_ROWS) + 1
    mats, tris = [], []

    def add(m, cell, uv):
        mats.append(m)
        tris.append(quad(*cell, len(mats) - 1, uv))

    rgb = lambda: tuple(int(x) for x in rng.integers(0, 256, 3))
    for ty in range(tile):
        for tx in range(tile):
            cells = _cells(n_cols, n_rows, 2.0, 1.45)
            shift = lambda c: (c[0] + 4.0 * (tx - (tile - 1) / 2), c[1] + 4.0 * (tx - (tile - 1) / 2),
                               c[2] + 2.9 * (ty - (tile - 1) / 2), c[3] + 2.9 * (ty - (tile - 1) / 2))
            for r, tex in enumerate(CHART_ROWS):
                for c, edge in enumerate(edges):
                    add(material(diffuse=rgb(), specular=rgb(), roughness=int(rng.integers(0, 256)), tex={"diffuse": tex}),
                        shift(cells[r, c + 1]), edge_uv(edge))
            # the slot row: each slot alone, then all six; every other quad of the row an edge of its own
            r = len(CHART_ROWS)
            for c, slots in enumerate([(s,) for s in SLOTS] + [SLOTS] * 5):
                tex = {s: int(CHART_ROWS[(c + k) % len(CHART_ROWS)]) for k, s in enumerate(slots)}
                m = material(diffuse=rgb(), specular=rgb(), emission=rgb() + (128,), roughness=int(rng.integers(0, 256)),
                             metalness=int(rng.integers(0, 256)), transparency=int(rng.integers(128, 256)), tex=tex)
                add(m, shift(cells[r, c]), edge_uv(edges[(3 * c) % len(edges)]))
            for r in range(len(CHART_ROWS)):       # column 0: untextured references
                add(material(diffuse=rgb(), specular=rgb()), shift(cells[r, 0]), edge_uv("wide"))
    if tile == 1:
        mats.append(material(diffuse=(200, 100, 50), tex={"diffuse": 3}))
        tris.append(zero_weight_triangle(len(mats) - 1, CHART_W, CHART_H))
    return finish(tris, mats, textures, texels)


def chart_camera(w, h, tile=1):
    """The default camera, moved back so that tile x tile charts fill the frame."""
    return default_camera(w, h, position=(0.0, 1.0 - 2.0 * tile, 1.0))


# ------------------------------------------------------------------------------------------------------------ emission ladder
LADDER_COLS, LADDER_ROWS = 32, 24
LADDER_W, LADDER_H = 256, 192
VARIANTS = ("untextured", "per_hit", "random")


def ladder_mantissas(e):
    """RGB mantissa bytes of exponent byte e: 0, 1, 128 and 255 in every channel across the ladder."""
    vals = (0, 1, 128, 255, 37, 200)
    return vals[e % 6], vals[(e + 2) % 6], vals[(e + 4) % 6] if e % 5 else 255


def ladder_scene(exponents=range(256), variants=VARIANTS, floor=False):
    """One quad per (variant, exponent byte) on a 32 x 24 grid (the first 256 cells untextured, the next 256 with the 1x1 white
    emission texture, the last 256 with random bytes in every non-texture field and the white emission texture); diffuse and
    specular albedo and transparency 0 in the first two variants (a primary hit's radiance is then its emission alone:
    the specular lobe's Fresnel term does not vanish with the specular albedo, a pass-through material's BSDF does).  floor: a white diffuse floor in front of the ladder, lit by it."""
    rng = np.random.default_rng(23)
    textures = np.zeros(1, TEXTURE_DT); textures[0] = (0, 1, 1, 0)
    texels = np.array([0xFFFFFFFF], "<u4")
    cells = _cells(LADDER_COLS, LADDER_ROWS, 2.0, 1.45, fill=0.7)
    mats, tris, where = [], [], {}
    for vi, variant in enumerate(VARIANTS):
        if variant not in variants:
            continue
        for e in exponents:
            mant = ladder_mantissas(e)
            if variant == "random":
                b = [int(x) for x in rng.integers(0, 256, 8)]
                m = material(diffuse=b[0:3], specular=b[3:6], emission=mant + (e,), roughness=b[6], metalness=b[7],
                             ior=int(rng.integers(0, 256)), transparency=int(rng.integers(0, 256)), tex={"emission": 0})
            else:
                # transparency 0: the BSDF is 0 (material.h:134), so the light sample adds nothing to the emission
                m = material(emission=mant + (e,), roughness=200, metalness=0, transparency=0,
                             tex={"emission": 0} if variant == "per_hit" else None)
            mats.append(m)
            k = vi * 256 + e
            cell = cells[k // LADDER_COLS, k % LADDER_COLS]
            tris.append(quad(*cell, len(mats) - 1, [(0.5, 0.5)] * 4))
            where[len(mats) - 1] = (variant, e)
    if floor:
        mats.append(material(diffuse=(230, 230, 230), roughness=255))
        t = quad(-2.2, 2.2, -0.4, 1.0, len(mats) - 1, [(0.0, 0.0)] * 4)
        for k in range(2):                   # rotate onto the plane z = -0.5, facing +z, from y = -0.4 to y = 1
            for v in ("v1", "v2", "v3"):
                x, _, y = t[k][v]["position"][:3]
                t[k][v]["position"][:3] = (x, y, -0.5)
                t[k][v]["normal"][:3] = (0.0, 0.0, 1.0)
            t[k]["v2"], t[k]["v3"] = t[k]["v3"].copy(), t[k]["v2"].copy()
        tris.append(t)
    sc = finish(tris, mats, textures, texels)
    sc["ladder"] = where
    return sc


def emission_f64(word):
    """ldexp(mantissa, e - 136) of an RGBE word, per channel, in float64 (exact in float32 for every byte)."""
    e = (int(word) >> 24) - 136
    return np.array([np.ldexp(float((int(word) >> s) & 0xFF), e) for s in (0, 8, 16)])


# ------------------------------------------------------------------------------------------------------------ textured OBJ
OBJ_MAPS = ("map_Kd", "map_Ks", "map_Pr", "map_Pm", "map_Ke", "map_d")
OBJ_IMAGES = {"t1x1.png": (1, 1), "t1x7.png": (7, 1), "t7x1.png": (1, 7), "t7x5.png": (5, 7), "t16.png": (16, 16), "t3x9.png": (9, 3)}


def write_textured_obj(directory, seed=11):
    """Six quads facing the default camera, each with one map_* key (and the last with all six) on small PNGs of distinct
    texels; texture coordinates sweep integers, their neighbours and -1e-9.  -> the OBJ path."""
    from PIL import Image
    rng = np.random.default_rng(seed)
    names = sorted(OBJ_IMAGES)
    for n in names:
        h, w = OBJ_IMAGES[n]
        px = rng.permutation(256 ** 2)[: w * h]
        img = np.stack([px & 0xFF, px >> 8, rng.integers(0, 256, w * h), np.full(w * h, 255)], 1).astype(np.uint8)
        Image.fromarray(img.reshape(h, w, 4)).save(os.path.join(directory, n))
    with open(os.path.join(directory, "edges.mtl"), "w") as f:
        for i, key in enumerate(OBJ_MAPS):
            f.write(f"newmtl m{i}\nKd 0.6 0.5 0.4\nKs 0.3 0.3 0.3\nKe 0.4 0.3 0.2\nPr 0.4\nPm 0.2\nNi 1.5\n{key} {names[i]}\n")
        f.write("newmtl all\nKd 1 1 1\nKs 1 1 1\nKe 1 1 1\nPr 1\nPm 1\n")
        for i, key in enumerate(OBJ_MAPS):
            f.write(f"{key} {names[(i + 2) % len(names)]}\n")
    uvs = [(-1e-9, -1e-9), (1.0, 1.0), (1.0000001, 0.99999994), (2.0, -1.0), (0.5, 0.5), (-3.0, 3.0)]
    with open(os.path.join(directory, "edges.obj"), "w") as f:
        f.write("mtllib edges.mtl\nvn 0 -1 0\n")
        for u, v in uvs:
            f.write("vt %.9g %.9g\n" % (u, v))
        k = 0
        for i, m in enumerate(list(range(len(OBJ_MAPS))) + ["all"]):
            x0 = -1.7 + 0.5 * i
            f.write(f"v {x0:.4f} 1 0.4\nv {x0 + 0.45:.4f} 1 0.4\nv {x0 + 0.45:.4f} 1 1.6\nv {x0:.4f} 1 1.6\n")
            f.write("usemtl %s\n" % (m if m == "all" else "m%d" % m))
            t = [(i + j) % len(uvs) + 1 for j in range(4)]
            f.write("f %d/%d/1 %d/%d/1 %d/%d/1 %d/%d/1\n" % (k + 1, t[0], k + 2, t[1], k + 3, t[2], k + 4, t[3]))
            k += 4
    return os.path.join(directory, "edges.obj")


def obj_scene(directory):
    """The textured OBJ through the host loader and BVH builder, under CornellBox's environment, with one directional light."""
    from raytracing_b200 import hostapi, scene_io
    s = hostapi.HostScene(write_textured_obj(directory))
    s.add_directional_light((-0.3, -0.8, 1.0), (6, 6, 6)); s.build_bvh()
    env, env_w, env_h = scene_io.load_env()
    s.finalize(env=env, env_width=env_w, env_height=env_h)
    a = s.arrays(); s.close()
    return a


# ------------------------------------------------------------------------------------------------------------ albedo restatement
POW_EXPONENT = float(F32(2.2))


def primary_texcoords(sc, prim, bc):
    """Interpolated texture coordinates of primary hits as hit_surface.cl:95-96 computes them in float32 (left to right, no
    FMA), and the same in float64 from the same barycentrics.  -> (uv32 (n, 2), uv64 (n, 2)) for hits (prim != invalid)."""
    tri = sc["triangles"][prim]
    u, v = bc[:, 0].astype(F32), bc[:, 1].astype(F32)
    with np.errstate(all="ignore"):
        w0 = ((F32(1.0) - u).astype(F32) - v).astype(F32)
        t = [tri[k]["texcoord"][:, :2].astype(F32) for k in ("v1", "v2", "v3")]
        uv32 = ((t[0] * w0[:, None]).astype(F32) + (t[1] * u[:, None]).astype(F32)).astype(F32) + (t[2] * v[:, None]).astype(F32)
        u64, v64 = u.astype(np.float64), v.astype(np.float64)
        uv64 = t[0] * (1.0 - u64 - v64)[:, None] + t[1] * u64[:, None] + t[2] * v64[:, None]
    return uv32.astype(F32), uv64


def texel_lookup(uv, width, height):
    """material.h:319-369 in the precision of uv: wrap, flip, scale, NaN guard, clamp.  -> (tx, ty) int64 arrays."""
    dt = uv.dtype.type
    with np.errstate(all="ignore"):
        f = (uv - np.floor(uv)).astype(dt)
        fy = (dt(1.0) - f[:, 1]).astype(dt)
        sx, sy = (f[:, 0] * width.astype(dt)).astype(dt), (fy * height.astype(dt)).astype(dt)
        tx = np.where(np.isnan(sx), 0, np.trunc(np.nan_to_num(sx))).astype(np.int64)
        ty = np.where(np.isnan(sy), 0, np.trunc(np.nan_to_num(sy))).astype(np.int64)
    return np.clip(tx, 0, width - 1), np.clip(ty, 0, height - 1)


def albedo_restatement(sc, prim, bc):
    """The albedo AOV of primary hits (aov.cl:106): untextured diffuse rgb / 255 in float32; textured, the texel the float32 rule
    picks as (texel / 255)^2.2 in float64.  -> (albedo (n, 3) float64, textured mask, f32 texel (n,) index, f64 texel index,
    uv32)."""
    n = len(prim)
    hit = prim != 0xFFFFFFFF
    out = np.zeros((n, 3)); textured = np.zeros(n, bool)
    idx32 = np.full(n, -1, np.int64); idx64 = np.full(n, -1, np.int64); uv32 = np.zeros((n, 2), F32)
    p = prim[hit].astype(np.int64)
    word = sc["materials"]["diffuse_albedo"][sc["triangles"]["mtlIndex"][p]]
    tex = (word >> 24).astype(np.int64)
    rgb = np.stack([((word >> s) & 0xFF).astype(F32) / F32(255.0) for s in (0, 8, 16)], 1).astype(F32)
    a = rgb.astype(np.float64)
    on = tex != NONE
    uv_hit32, uv_hit64 = primary_texcoords(sc, p[on], bc[hit][on])
    t = sc["textures"][tex[on]]
    w, h, start = t["width"].astype(np.int64), t["height"].astype(np.int64), t["data_start"].astype(np.int64)
    tx, ty = texel_lookup(uv_hit32, w, h)
    i32 = start + ty * w + tx
    tx64, ty64 = texel_lookup(uv_hit64, w, h)
    d = sc["texels"][i32]
    c = np.stack([((d >> s) & 0xFF).astype(F32) / F32(255.0) for s in (0, 8, 16)], 1).astype(F32)
    a[on] = np.power(c.astype(np.float64), POW_EXPONENT)
    out[hit] = a; textured[np.flatnonzero(hit)[on]] = True
    idx32[np.flatnonzero(hit)[on]] = i32; idx64[np.flatnonzero(hit)[on]] = start + ty64 * w + tx64
    uv32[np.flatnonzero(hit)[on]] = uv_hit32
    return out, textured, idx32, idx64, uv32


def ulp_distance(got32, want64):
    """|got - want| in units of the float32 spacing at want (0 where both are 0)."""
    want32 = want64.astype(F32)
    spacing = np.spacing(np.abs(want32)).astype(np.float64)
    return np.abs(got32.astype(np.float64) - want64) / spacing


def edge_of_pixel(sc, prim, edges=EDGES):
    """Name of the chart column (coordinate edge) each primary hit lies in, from the hit quad's corner coordinates; '' elsewhere."""
    out = np.full(len(prim), "", dtype=object)
    hit = prim != 0xFFFFFFFF
    tri = sc["triangles"][prim[hit].astype(np.int64)]
    corners = np.stack([tri[k]["texcoord"][:, :2] for k in ("v1", "v2", "v3")], 1)
    for name in edges:
        uvs = np.array(edge_uv(name), F32)
        m = np.all([np.any(np.all((corners == c) | (np.isnan(corners) & np.isnan(c)), -1), 1) for c in uvs[:3]], 0)
        out[np.flatnonzero(hit)[m]] = name
    return out
