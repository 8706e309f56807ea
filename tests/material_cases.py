"""
Scenes for the shading pass across the packed material space (material.h:132-241; rt_device.cuh evaluate_material, sample_bxdf,
tangent_frame; rt_kernels.cu shade_hit), no GPU needed to build them:

- chart_scene(): 1 711 camera-facing cells on a 48 x 36 grid, one material each: every value 0..255 of roughness, metalness, ior
  and transparency on a coloured base with both lobes weighted; the diffuse and specular channels at 0, 1, 127, 128, 254, 255 one
  at a time; a cross grid of roughness x metalness x ior x transparency bytes; black/black (a NaN lobe pdf), black diffuse under
  a white metal, white/white.  variant "per_hit" points every emission slot at a 1x1 white texture, which forces the per-hit
  decode (unpack_material) without changing any value; variant "grazing" gives every cell vertex normals perpendicular to the
  view of its centre, so n.i crosses 0 and the RT_EPS clamp inside each cell.
- normal_scene(): cells whose vertex normals are zero at one or all vertices, flipped, scaled by 1e-3, 1e3, 1e-20 and 1e-23,
  perpendicular to the view, and with n.x at the float32 neighbours of tangent_frame's 0.001 switch.
- lights_scene(): roughness-0 and near-delta cells under a directional light exactly grazing them (n.l == 0) and at the float
  neighbours of grazing, one below the horizon, a point light on the cells' plane and one at the camera, where a triangle with
  a vertex at the camera is hit at t = 0 (the light at the hit: infinite radiance and normalize(0)).
- mirror_scene(): a narrow-field camera on roughness-0 cells under a directional light at the mirror direction of its axis, so
  that n.h == 1 (ggx_d's 0/0) at a block of pixels.

Plus numpy restatements that do not depend on the oracle: the kRandom draws (wang_hash chains, rt_device.cuh:45-77), the primary
hit's float32 position and shading normal, what each bounce-0 pixel reaches (reach()), and a float64 restatement of
evaluate_material and sample_bxdf (f64_direct(), f64_sky()) with switches for the negative controls.
"""
import numpy as np

from raytracing_b200.camera import default_camera
from raytracing_b200.layouts import LIGHT_DT, TEXTURE_DT
from tests.texture_cases import _cells, finish, material, quad

F32 = np.float32
EPS = float(F32(1e-3))                      # RT_EPS
CHART_COLS, CHART_ROWS = 48, 36
CHART_W, CHART_H = 240, 180
BASE = dict(diffuse=(180, 120, 60), specular=(90, 160, 220), roughness=128, metalness=40, ior=38, transparency=255)
CHANNEL_VALUES = (0, 1, 127, 128, 254, 255)
CROSS = dict(roughness=(0, 1, 2, 3, 4, 25, 128, 254, 255), metalness=(0, 1, 127, 128, 254, 255), ior=(0, 1, 25, 26, 38, 255),
             transparency=(127, 128))
WHITE_TEX = np.array([(0, 1, 1, 0)], TEXTURE_DT), np.array([0xFFFFFFFF], "<u4")


def chart_materials():
    """-> [(packed material, tag)]: tag = (group, detail) for the REACH tables and the known-answer report."""
    out = []
    for field in ("roughness", "metalness", "ior", "transparency"):
        for v in range(256):
            out.append((material(**dict(BASE, **{field: v})), ("sweep_" + field, v)))
    for lobe in ("diffuse", "specular"):
        for ch in range(3):
            for v in CHANNEL_VALUES:
                rgb = list(BASE[lobe]); rgb[ch] = v
                out.append((material(**dict(BASE, **{lobe: tuple(rgb)})), ("channel_" + lobe, (ch, v))))
    for r in CROSS["roughness"]:
        for m in CROSS["metalness"]:
            for i in CROSS["ior"]:
                for t in CROSS["transparency"]:
                    out.append((material(**dict(BASE, roughness=r, metalness=m, ior=i, transparency=t)), ("cross", (r, m, i, t))))
    out.append((material(**dict(BASE, diffuse=(0, 0, 0), specular=(0, 0, 0), metalness=0)), ("black_black", 0)))
    out.append((material(**dict(BASE, diffuse=(0, 0, 0), specular=(255, 255, 255), metalness=255)), ("black_white_metal", 0)))
    out.append((material(**dict(BASE, diffuse=(255, 255, 255), specular=(255, 255, 255))), ("white_white", 0)))
    return out


def per_hit(m):
    """The emission slot of a packed material pointed at texture 0 (the 1x1 white texel): every value stays the same."""
    m = m.copy()
    m["ior_emission_idx_transparency"] = (int(m["ior_emission_idx_transparency"]) & ~0xFF00) & 0xFFFFFFFF
    return m


def set_normals(t, normals):
    """Vertex normals of a quad's two triangles; normals: the corners' normals in quad()'s corner order."""
    for k, corners in enumerate(((0, 1, 2), (2, 3, 0))):
        for v, ci in zip(("v1", "v2", "v3"), corners):
            t[k][v]["normal"][:3] = normals[ci]
    return t


def perpendicular_to_view(cell, cam_pos=(0.0, -1.0, 1.0)):
    """A unit normal perpendicular to the direction from the camera to the cell's centre, in the plane of that direction and z."""
    c = np.array([(cell[0] + cell[1]) / 2, 1.0, (cell[2] + cell[3]) / 2]) - np.array(cam_pos)
    d = c / np.linalg.norm(c)
    n = np.array([0.0, 0.0, 1.0]) - d[2] * d
    return tuple(n / np.linalg.norm(n))


def chart_scene(variant="untextured", tile=1):
    """The material chart (module docstring); tile x tile copies side by side for large frames (chart_camera(tile))."""
    mats_tags = chart_materials()
    cells = _cells(CHART_COLS, CHART_ROWS, 2.0, 1.45, fill=0.85)
    order = sorted(cells)
    mats, tris, tags = [], [], []
    for ty in range(tile):
        for tx in range(tile):
            dx, dz = 4.0 * (tx - (tile - 1) / 2), 2.9 * (ty - (tile - 1) / 2)
            for k, (m, tag) in enumerate(mats_tags):
                c = cells[order[k]]
                cell = (c[0] + dx, c[1] + dx, c[2] + dz, c[3] + dz)
                mats.append(per_hit(m) if variant == "per_hit" else m); tags.append(tag)
                t = quad(*cell, len(mats) - 1, [(0.5, 0.5)] * 4)
                if variant == "grazing":
                    set_normals(t, [perpendicular_to_view(cell)] * 4)
                tris.append(t)
    sc = finish(tris, mats, *WHITE_TEX)
    sc["tags"] = tags
    return sc


def chart_camera(w, h, tile=1):
    return default_camera(w, h, position=(0.0, 1.0 - 2.0 * tile, 1.0))


def with_lights(sc, lights):
    """sc with its analytic lights replaced; lights: [(kind, (x, y, z), (r, g, b))], kind 'point' (position) or 'directional'
    (direction towards the light)."""
    sc = dict(sc)
    arr = np.zeros(len(lights), LIGHT_DT)
    for k, (kind, xyz, rgb) in enumerate(lights):
        arr[k]["origin"][:3] = xyz; arr[k]["radiance"][:3] = rgb
        arr[k]["type"] = 0 if kind == "point" else 1
    info = np.array(sc["scene_info"], copy=True); info["analytic_light_count"] = len(lights)
    sc.update(lights=arr, scene_info=info)
    return sc


def with_sky(sc, rgb):
    """sc under a constant 1x1 environment of value rgb."""
    sc = dict(sc)
    sc["env"] = np.array(list(rgb) + [1.0], "<f4"); sc["env_width"] = sc["env_height"] = 1
    return sc


# light kinds of LightRec: RT_LIGHT_TYPE_POINT 0, directional 1 (include/rt_types.h)
KA_LIGHT = ("directional", (-0.3, -0.8, 0.5), (3.0, 2.5, 2.0))
SKY_C = (0.75, 1.25, 0.5)


def direct_frame_scene(variant="untextured"):
    """Known answer (a): max_bounces 0, one directional light, a black sky."""
    return with_sky(with_lights(chart_scene(variant), [KA_LIGHT]), (0.0, 0.0, 0.0))


def sky_frame_scene(variant="untextured"):
    """Known answer (b): max_bounces 1, a light of radiance 0, a constant 1x1 sky SKY_C."""
    return with_sky(with_lights(chart_scene(variant), [("directional", KA_LIGHT[1], (0.0, 0.0, 0.0))]), SKY_C)


# ------------------------------------------------------------------------------------------------------------ normal panel
NX_ULPS = (-3, -2, -1, 0, 1, 2, 3)


def normal_cases():
    """name -> corner normals (quad() corner order) or 'perpendicular'."""
    d = (0.0, -1.0, 0.0)
    cases = {"zero_one_vertex": [(0.0, 0.0, 0.0), d, d, d], "zero_all": [(0.0, 0.0, 0.0)] * 4, "flipped": [(0.0, 1.0, 0.0)] * 4,
             "scaled_1e-3": [(0.0, -1e-3, 0.0)] * 4, "scaled_1e3": [(0.0, -1e3, 0.0)] * 4,
             "scaled_1e-20": [(0.0, -1e-20, 0.0)] * 4, "scaled_1e-23": [(0.0, -1e-23, 0.0)] * 4, "perpendicular": "perpendicular"}
    for sign in (1, -1):
        for k in NX_ULPS:
            x = F32(0.001)
            for _ in range(abs(k)):
                x = np.nextafter(x, F32(np.inf) if k > 0 else F32(0))
            y = float(F32(-np.sqrt(1.0 - float(x) ** 2)))
            cases["nx_%+d_%s" % (k, "pos" if sign > 0 else "neg")] = [(sign * float(x), y, 0.0)] * 4
    return cases


def normal_scene():
    cases = normal_cases()
    cells = _cells(6, 4, 2.0, 1.45, fill=0.85)
    order = sorted(cells)
    mats, tris, tags = [], [], []
    for k, (name, nrm) in enumerate(cases.items()):
        mats.append(material(**dict(BASE, roughness=128 if k % 2 == 0 else 200))); tags.append(("normal", name))
        cell = cells[order[k]]
        t = quad(*cell, len(mats) - 1, [(0.5, 0.5)] * 4)
        set_normals(t, [perpendicular_to_view(cell)] * 4 if nrm == "perpendicular" else nrm)
        tris.append(t)
    sc = finish(tris, mats, *WHITE_TEX)
    sc["tags"] = tags
    return sc


# ------------------------------------------------------------------------------------------------------------ light placements
CAM_POS = (0.0, -1.0, 1.0)
TINY = float(np.nextafter(F32(0), F32(1)))
LIGHTS = [("directional", (1.0, 0.0, 0.0), (4.0, 4.0, 4.0)),          # exactly grazing: n.l == 0
          ("directional", (1.0, -TINY, 0.0), (4.0, 4.0, 4.0)),        # its float neighbours: just above the horizon ...
          ("directional", (1.0, TINY, 0.0), (4.0, 4.0, 4.0)),         # ... and just below
          ("directional", (1.0, -1e-7, 0.0), (4.0, 4.0, 4.0)),
          ("directional", (0.2, 0.9, 0.3), (4.0, 4.0, 4.0)),          # below the horizon
          ("point", (0.31, 1.0, 1.17), (2.0, 2.0, 2.0)),              # on the cells' plane
          ("point", CAM_POS, (2.0, 2.0, 2.0))]                        # at the camera
LIGHT_CELLS = [dict(BASE, roughness=0, metalness=0), dict(BASE, roughness=0, metalness=255), dict(BASE, roughness=1),
               dict(BASE, roughness=3), dict(BASE, roughness=128), dict(BASE, transparency=0)]
LIGHTS_W, LIGHTS_H = 128, 96


def camera_triangle(cam, w, h, mtl, px=6.5, py=6.5):
    """tests/texture_cases.zero_weight_triangle for camera `cam`: v1 at the camera's position, hit at t = 0 with u = v = 0 (so at
    exactly the camera's position) by the rays around pixel (px, py)."""
    from raytracing_b200.layouts import TRIANGLE_DT
    o = cam["position"][:3].astype(np.float64)
    ang = np.tan(0.5 * float(cam["fov"]))
    x = (px / w * 2 - 1) * ang * float(cam["aspect_ratio"]); y = (py / h * 2 - 1) * ang
    front, up = cam["front"][:3].astype(np.float64), cam["up"][:3].astype(np.float64)
    d = x * np.cross(front, up) + y * up + front; d /= np.linalg.norm(d)
    a = np.cross(d, up); a /= np.linalg.norm(a)
    b = np.cross(a, d)
    s = np.sqrt(1e-8 / np.cos(np.radians(3.0)))
    t = np.zeros(1, TRIANGLE_DT)
    for v, p in (("v1", o), ("v2", o + s * a), ("v3", o + s * b)):
        t[0][v]["position"][:3] = p
        t[0][v]["normal"][:3] = -d
    t["mtlIndex"] = mtl
    return t


def lights_scene():
    cells = _cells(3, 2, 2.0, 1.45, fill=0.9)
    mats, tris, tags = [], [], []
    for k, kw in enumerate(LIGHT_CELLS):
        mats.append(material(**kw)); tags.append(("light_cell", k))
        tris.append(quad(*cells[sorted(cells)[k]], len(mats) - 1, [(0.5, 0.5)] * 4))
    mats.append(material(**dict(BASE, roughness=0))); tags.append(("camera_triangle", 0))
    tris.append(camera_triangle(default_camera(LIGHTS_W, LIGHTS_H), LIGHTS_W, LIGHTS_H, len(mats) - 1))
    sc = with_lights(finish(tris, mats, *WHITE_TEX), LIGHTS)
    sc["tags"] = tags
    return sc


MIRROR_W, MIRROR_H = 96, 72
MIRROR_FOV = 0.004


def mirror_camera(w=MIRROR_W, h=MIRROR_H):
    cam = default_camera(w, h)
    cam["fov"] = F32(MIRROR_FOV)
    return cam


def mirror_scene():
    """Roughness-0 cells (dielectric left, white metal right) filling the narrow view; a directional light at the mirror
    direction of the camera's axis about the cells' normal (0, -1, 0)."""
    f = mirror_camera()["front"][:3].astype(np.float64)
    mats = [material(**dict(BASE, roughness=0, metalness=0)), material(**dict(BASE, roughness=0, metalness=255))]
    tris = [quad(-0.5, 0.0, 0.5, 1.5, 0, [(0.5, 0.5)] * 4), quad(0.0, 0.5, 0.5, 1.5, 1, [(0.5, 0.5)] * 4)]
    sc = with_lights(finish(tris, mats, *WHITE_TEX), [("directional", (f[0], -f[1], f[2]), (5.0, 5.0, 5.0))])
    sc["tags"] = [("mirror", 0), ("mirror", 1)]
    return sc


# ------------------------------------------------------------------------------------------------------------ restatements
def wang_hash(x):
    x = np.asarray(x, np.uint32)
    with np.errstate(over="ignore"):
        x = (x ^ np.uint32(61)) ^ (x >> np.uint32(16))
        x = x + (x << np.uint32(3))
        x = x ^ (x >> np.uint32(4))
        x = x * np.uint32(0x27D4EB2D)
        x = x ^ (x >> np.uint32(15))
    return x.astype(np.uint32)


def k_random(w, h, sample, bounce, typ):
    """kRandom draw of every pixel (rt_device.cuh:66-77, sampling.h:64-82), float32 (h * w,)."""
    px = np.tile(np.arange(w, dtype=np.uint32), h); py = np.repeat(np.arange(h, dtype=np.uint32), w)
    with np.errstate(over="ignore"):
        seed = wang_hash(px)
        seed = wang_hash(seed + wang_hash(py))
        seed = wang_hash(seed + wang_hash(np.full_like(px, sample)))
        s = wang_hash(seed + wang_hash(np.uint32(bounce * 5 + typ)))
    return (s.astype(F32) * F32(2.3283064365386963e-10)).astype(F32)


LAYER, U, V, LIGHT = 1, 2, 3, 4


def _dot32(a, b):
    return ((a[..., 0] * b[..., 0]).astype(F32) + (a[..., 1] * b[..., 1]).astype(F32)).astype(F32) + (a[..., 2] * b[..., 2]).astype(F32)


def _normalize32(a):
    with np.errstate(all="ignore"):
        inv = (F32(1.0) / np.sqrt(_dot32(a, a).astype(F32))).astype(F32)
        return (a * inv[..., None]).astype(F32)


def primary_surface(sc, prim, bc):
    """Float32 position and shading normal of primary hits as shade_hit computes them (rt_kernels.cu:148-150, no FMA)."""
    tri = sc["triangles"][prim.astype(np.int64)]
    u, v = bc[:, 0].astype(F32), bc[:, 1].astype(F32)
    w0 = ((F32(1.0) - u).astype(F32) - v).astype(F32)

    def interp(f):
        a = [tri[k][f][:, :3].astype(F32) for k in ("v1", "v2", "v3")]
        return (((a[0] * w0[:, None]).astype(F32) + (a[1] * u[:, None]).astype(F32)).astype(F32) + (a[2] * v[:, None]).astype(F32)).astype(F32)
    with np.errstate(all="ignore"):
        return interp("position"), _normalize32(interp("normal"))


def decode(sc, prim):
    """The float32 material of each hit's triangle (build_mat_rec's decode), as float64 arrays."""
    m = sc["materials"][sc["triangles"]["mtlIndex"][prim.astype(np.int64)]]
    b = lambda word, s: ((m[word] >> s) & 0xFF).astype(F32)
    rgb = lambda word: np.stack([(b(word, s) / F32(255.0)).astype(F32) for s in (0, 8, 16)], 1).astype(np.float64)
    return {"diffuse": rgb("diffuse_albedo"), "specular": rgb("specular_albedo"),
            "roughness": (b("roughness_metalness", 0) / F32(255.0)).astype(F32).astype(np.float64),
            "metalness": (b("roughness_metalness", 16) / F32(255.0)).astype(F32).astype(np.float64),
            "ior_byte": b("ior_emission_idx_transparency", 0).astype(np.float64),
            "ior": (b("ior_emission_idx_transparency", 0) / F32(25.5)).astype(F32).astype(np.float64),
            "transparency": (b("ior_emission_idx_transparency", 16) / F32(255.0)).astype(F32).astype(np.float64),
            "transparency_byte": b("ior_emission_idx_transparency", 16).astype(np.int64)}


def primary_view(sc, cam, w, h, hits, sample=0):
    """Per covered pixel of sample `sample`: pixel index, float32 position, normal, incoming direction (-ray direction, from the
    oracle's ray generation), the hit's material (decode) and its tag."""
    from oracle.orcbind import Oracle
    prim, bc = hits["primitive_id"], hits["bc"]
    px = np.flatnonzero(prim != 0xFFFFFFFF)
    rays = Oracle(sc).generate_rays(cam, w, h, sample)
    pos, nrm = primary_surface(sc, prim[px], bc[px])
    inc = (-rays["direction"][px, :3]).astype(F32)
    mtl = sc["triangles"]["mtlIndex"][prim[px].astype(np.int64)]
    return {"px": px, "pos": pos, "n": nrm, "i": inc, "m": decode(sc, prim[px]), "mtl": mtl,
            "tag": [sc["tags"][k] for k in mtl]}


def reach(sc, view, w, h, sample=0):
    """What each covered bounce-0 pixel reaches, from the float32 restatement and the kRandom draws: -> {branch: count}."""
    m, n, i = view["m"], view["n"], view["i"]
    px = view["px"]
    s1 = k_random(w, h, sample, 0, LAYER)[px]
    alpha = (m["roughness"].astype(F32) * m["roughness"].astype(F32)).astype(F32)
    with np.errstate(all="ignore"):
        spec_pdf, _ = lobe_pdfs(m, n.astype(np.float64), i.astype(np.float64))
    passing = m["transparency"] < 0.5
    black = np.array([t[0] == "black_black" for t in view["tag"]])
    out = {"pass_through": int(passing.sum()),
           "delta_lobe": int((~passing & (alpha <= F32(1e-4)) & (s1 <= spec_pdf)).sum()),
           "nan_lobe_pdf": int((~passing & np.isnan(spec_pdf)).sum()),
           "black_black": int(black.sum()),
           "tangent_axis_y": int((np.abs(n[:, 0]) > F32(0.001)).sum()),
           "tangent_axis_x": int((np.abs(n[:, 0]) <= F32(0.001)).sum()),
           "tangent_at_switch": int((np.abs(n[:, 0]) == F32(0.001)).sum()),
           "tangent_above_switch_4ulp": int(((np.abs(n[:, 0]) > F32(0.001)) & (np.abs(n[:, 0]) <= F32(0.001) + 4 * np.spacing(F32(0.001)))).sum()),
           "tangent_below_switch_4ulp": int(((np.abs(n[:, 0]) < F32(0.001)) & (np.abs(n[:, 0]) >= F32(0.001) - 4 * np.spacing(F32(0.001)))).sum()),
           "nan_normal": int(np.isnan(n).any(1).sum())}
    with np.errstate(all="ignore"):
        ndi = _dot32(n, i)
    out["n.i<0"] = int((ndi < 0).sum())
    out["n.i_at_eps_clamp"] = int(((ndi >= 0) & (ndi < F32(EPS))).sum())
    out["|n.i|<1e-5"] = int((np.abs(ndi) < 1e-5).sum())
    # the light each pixel samples and what its shading sees (rt_device.cuh light_sample, rt_kernels.cu:266-283)
    lights = sc["lights"]
    sl = k_random(w, h, sample, 0, LIGHT)[px]
    idx = np.clip((sl * F32(len(lights))).astype(F32).astype(np.int64), 0, len(lights) - 1)
    o = np.zeros_like(i)
    with np.errstate(all="ignore"):
        for k, l in enumerate(lights):
            sel = idx == k
            if l["type"] == 0:
                o[sel] = _normalize32((l["origin"][:3].astype(F32) - view["pos"][sel]).astype(F32))
            else:
                v = (l["origin"][:3].astype(F32) * F32(20000.0)).astype(F32)
                d2 = ((v[0] * v[0]).astype(F32) + (v[1] * v[1]).astype(F32) + (v[2] * v[2]).astype(F32)).astype(F32)
                o[sel] = (v * (F32(1.0) / np.sqrt(d2)).astype(F32)).astype(F32)
        cos_l = np.where(np.isnan(_dot32(o, n)), F32(0), np.maximum(_dot32(o, n), F32(0)))
        hv = _normalize32((i + o).astype(F32))
        ndh = _dot32(n, hv)
    out["cos_l==0_skip"] = int((cos_l == 0).sum())
    out["n.h==1"] = int((ndh == F32(1.0)).sum())
    out["n.h==1_at_alpha_0"] = int(((ndh == F32(1.0)) & (alpha == 0) & ~passing & (cos_l > 0)).sum())
    out["light_at_hit"] = int(((idx >= 0) & np.isnan(o).all(1)).sum())
    return out


# ---------------------------------------------------------------------------------------------- float64 BSDF (material.h:132-241)
CONTROLS = ("alpha_is_roughness", "diffuse_without_fresnel", "ior_over_25", "pass_through_le_128")


def _luma(c):
    return c[:, 0] * 0.299 + c[:, 1] * 0.587 + c[:, 2] * 0.114


def _params(m, control=None):
    r = m["roughness"]
    alpha = r if control == "alpha_is_roughness" else r * r
    ior = m["ior_byte"] / 25.0 if control == "ior_over_25" else m["ior"]
    f0d = ((ior - 1.0) / (ior + 1.0)) ** 2
    met = m["metalness"][:, None]
    f0 = f0d[:, None] + (m["specular"] - f0d[:, None]) * met
    passing = m["transparency_byte"] <= 128 if control == "pass_through_le_128" else m["transparency"] < 0.5
    return alpha, f0, met, passing


def lobe_pdfs(m, n, i, control=None):
    """sample_bxdf's lobe weights (material.h:185-212) in float64: -> (specular_pdf, diffuse_pdf)."""
    alpha, f0, met, _ = _params(m, control)
    diff = (1.0 - met) * m["diffuse"]
    spec_alb = m["specular"] + (1.0 - m["specular"]) * met
    ndi = np.sum(n * i, 1)
    fres = (f0 + (1.0 - f0) * (1.0 - ndi)[:, None] ** 5) * spec_alb
    sw = _luma(spec_alb * fres)
    dw = _luma(diff * ((1.0 - fres) if control != "diffuse_without_fresnel" else 1.0))
    return sw / (sw + dw), dw / (sw + dw)


def _unit(a):
    return a / np.linalg.norm(a, axis=1, keepdims=True)


def ggx_d(alpha, ndh):
    a2 = alpha * alpha
    return a2 / np.pi / (ndh * ndh * (a2 - 1.0) + 1.0) ** 2


def v_smith(ndi, ndo, alpha):
    a2 = alpha * alpha
    return 0.5 / (ndo * np.sqrt((-ndi * a2 + ndi) * ndi + a2) + ndi * np.sqrt((-ndo * a2 + ndo) * ndo + a2))


def evaluate_f64(m, n, i, o, control=None):
    """EvaluateMaterial (material.h:132-169) in float64 for float32 inputs n, i, o (n, 3)."""
    alpha, f0, met, passing = _params(m, control)
    h = _unit(i + o)
    ndi, ndo = np.maximum(np.sum(n * i, 1), EPS), np.maximum(np.sum(n * o, 1), EPS)
    ndh, hdo = np.maximum(np.sum(n * h, 1), EPS), np.maximum(np.sum(h * o, 1), EPS)
    fres = f0 + (1.0 - f0) * (1.0 - hdo)[:, None] ** 5
    spec = ggx_d(alpha, ndh) * v_smith(ndi, ndo, alpha)
    diff = (1.0 - met) * m["diffuse"] / np.pi
    out = fres * spec[:, None] + (diff if control == "diffuse_without_fresnel" else (1.0 - fres) * diff)
    out[passing] = 0.0
    return out


def f64_direct(view, light=KA_LIGHT, control=None):
    """Known answer (a): L * brdf * cos_l per covered pixel (pdf 1: one light), float64; 0 where cos_l <= 0."""
    v = (np.array(light[1], F32) * F32(20000.0)).astype(F32)
    o = np.broadcast_to((v / np.linalg.norm(v.astype(np.float64))), view["i"].shape)
    n, i = view["n"].astype(np.float64), view["i"].astype(np.float64)
    cos_l = np.maximum(np.sum(o * n, 1), 0.0)
    with np.errstate(all="ignore"):
        out = np.array(light[2])[None, :] * evaluate_f64(view["m"], n, i, o, control) * cos_l[:, None]
    out[cos_l == 0] = 0.0
    return out


def tangent_frame(n, n32x):
    axis = np.where((np.abs(n32x) > F32(0.001))[:, None], [0.0, 1.0, 0.0], [1.0, 0.0, 0.0])
    t = _unit(np.cross(axis, n))
    return t, np.cross(n, t)


def f64_sky(view, w, h, sample=0, sky=SKY_C, control=None):
    """Known answer (b): sky * bxdf / pdf of the direction sample_bxdf draws from the pixel's kRandom draws, float64.
    -> (value (n, 3), spawned (n,) bool, |s1 - specular_pdf| (n,): the distance of the lobe choice from its boundary, n.o of
    the sampled direction (n,), whether the GGX lobe was sampled (n,))."""
    m, px = view["m"], view["px"]
    n, i = view["n"].astype(np.float64), view["i"].astype(np.float64)
    s1 = k_random(w, h, sample, 0, LAYER)[px].astype(np.float64)
    sx = k_random(w, h, sample, 0, U)[px].astype(np.float64); sy = k_random(w, h, sample, 0, V)[px].astype(np.float64)
    alpha, f0, met, passing = _params(m, control)
    diff = (1.0 - met) * m["diffuse"]
    spec_alb = m["specular"] + (1.0 - m["specular"]) * met
    ndi = np.sum(n * i, 1)
    with np.errstate(all="ignore"):
        fres = (f0 + (1.0 - f0) * (1.0 - ndi)[:, None] ** 5) * spec_alb
        sp, dp = lobe_pdfs(m, n, i, control)
        phi = 2.0 * np.pi * sx
        t, b = tangent_frame(n, view["n"][:, 0])
        spec = s1 <= sp
        # specular: delta (alpha <= 1e-4) or GGX
        delta = alpha <= float(F32(1e-4))
        cos_t = 1.0 / np.sqrt(1.0 + alpha * alpha * sy / (1.0 - sy))
        sin_t = np.sqrt(np.maximum(0.0, 1.0 - cos_t * cos_t))
        wh = _unit(b * (np.cos(phi) * sin_t)[:, None] + t * (np.sin(phi) * sin_t)[:, None] + n * cos_t[:, None])
        wh = np.where(delta[:, None], n, wh)
        o_s = -i + 2.0 * np.sum(i * wh, 1)[:, None] * wh           # reflect(-i, wh)
        ndo_s = np.sum(n * o_s, 1)
        ndh = np.sum(n * wh, 1)
        D = ggx_d(alpha, ndh)
        G = v_smith(ndi, ndo_s, alpha)
        ratio_ggx = fres * (G * np.maximum(ndo_s, 0.0) * 4.0 * np.sum(wh * o_s, 1) / (ndh * sp))[:, None]
        ratio_delta = fres * (np.maximum(ndo_s, 0.0) / ndo_s / sp)[:, None]
        pdf_spec = np.where(delta, sp, D * ndh / (4.0 * np.sum(wh * o_s, 1)) * sp)
        # diffuse
        ct = np.sqrt(1.0 - sy)
        o_d = _unit(b * (np.cos(phi) * np.sqrt(sy))[:, None] + t * (np.sin(phi) * np.sqrt(sy))[:, None] + n * ct[:, None])
        pdf_diff = ct / np.pi * dp
        dfac = 1.0 if control == "diffuse_without_fresnel" else (1.0 - fres)
        ratio_diff = dfac * diff * (np.maximum(np.sum(o_d * n, 1), 0.0) / (ct * dp))[:, None]
        value = np.where(spec[:, None], np.where(delta[:, None], ratio_delta, ratio_ggx), ratio_diff)
        pdf = np.where(spec, pdf_spec, pdf_diff)
        ndo = np.where(spec, ndo_s, np.sum(o_d * n, 1))
    spawned = pdf > 0
    value = np.where(spawned[:, None], value, 0.0)
    value[passing] = 1.0; spawned[passing] = True
    return np.array(sky)[None, :] * value, spawned, np.abs(s1 - sp), ndo, spec & ~delta & ~passing
