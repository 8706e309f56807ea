"""
Synthetic "Bistro-scale" scene of BASELINE.json configs[4] / SURVEY 8(d) C5: K copies of the ShaderBalls triangles
(183 copies = 10 026 570 triangles) on a 14 x 14 grid (first K cells), pitch = 1.1 x the model's XY extent, every copy
rotated about Z by an angle drawn from the LCG x = 1103515245 x + 12345 (seed 1234), same 13 materials and the
reference's directional light, built directly as a Triangle[] (no OBJ round trip).  The copies stand on one ground
quad (2 triangles, the model's first material) that extends one pitch beyond the field: without it two thirds of the
field is empty space between the models and most camera rays leave the scene at once (round 1: 83 % of the primary
rays missed).  The BVH is built on the host by raytracing_b200/host/bvh.cpp (the build stays on the host, north_star).
The camera is raised and pulled back so that the whole grid is in view and more than 90 % of the primary rays hit
geometry; its exact pose is part of the returned scene dict (key "camera_pose").
"""
import math

import numpy as np

from .camera import default_camera
from .layouts import TRIANGLE_DT


def replicate(base_triangles: np.ndarray, copies: int = 183, grid: int = 14, seed: int = 1234, ground: bool = True):
    """Returns (triangles[copies * n (+ 2 ground triangles)], (xmin, xmax, ymin, ymax, zmax) of the whole field)."""
    t = np.ascontiguousarray(base_triangles, dtype=TRIANGLE_DT)
    pos = np.stack([t[v]["position"][:, :3] for v in ("v1", "v2", "v3")], axis=1).astype(np.float64)      # n,3,3
    nrm = np.stack([t[v]["normal"][:, :3] for v in ("v1", "v2", "v3")], axis=1).astype(np.float64)
    lo, hi = pos.reshape(-1, 3).min(0), pos.reshape(-1, 3).max(0)
    centre = (lo + hi) * 0.5
    pitch = 1.1 * max(hi[0] - lo[0], hi[1] - lo[1])
    out = np.zeros(copies * len(t) + (2 if ground else 0), dtype=TRIANGLE_DT)
    x = seed
    for k in range(copies):
        x = (1103515245 * x + 12345) & 0xFFFFFFFF
        ang = (x / 4294967296.0) * 2.0 * math.pi
        c, s = math.cos(ang), math.sin(ang)
        rot = np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])
        cell = np.array([(k % grid) * pitch, (k // grid) * pitch, 0.0])
        p = (pos - centre * [1, 1, 0]) @ rot.T + cell
        n = nrm @ rot.T
        blk = out[k * len(t):(k + 1) * len(t)]
        blk.view(np.uint8)[:] = t.view(np.uint8)               # (a record-wise copy of a structured array is ~20x slower)
        for j, v in enumerate(("v1", "v2", "v3")):
            blk[v]["position"][:, :3] = p[:, j].astype(np.float32)
            blk[v]["normal"][:, :3] = n[:, j].astype(np.float32)
    bounds = _field_ground(out[copies * len(t):] if ground else None, lo, hi, pitch, copies, grid, t["mtlIndex"][0])
    return out, bounds


def _field_ground(g, lo, hi, pitch, copies, grid, mtl):
    """The field's bounds (xmin, xmax, ymin, ymax, zmax); writes the ground quad into g (2 triangles) unless g is None."""
    rows = (copies + grid - 1) // grid
    half = pitch * 0.5
    bounds = (-half, (min(copies, grid) - 1) * pitch + half, -half, (rows - 1) * pitch + half, float(hi[2]))
    if g is not None:
        gx0, gx1, gy0, gy1 = bounds[0] - pitch, bounds[1] + pitch, bounds[2] - pitch, bounds[3] + pitch
        gz = float(lo[2]) - 0.01 * float(hi[2] - lo[2])           # just below the lowest vertex of the models
        corners = np.array([[gx0, gy0, gz], [gx1, gy0, gz], [gx1, gy1, gz], [gx0, gy1, gz]], dtype=np.float32)
        for tri, idx in zip(g, ((0, 1, 2), (0, 2, 3))):               # counter-clockwise seen from above: front face up
            for v, k in zip(("v1", "v2", "v3"), idx):
                tri[v]["position"][:3] = corners[k]
                tri[v]["normal"][:3] = (0.0, 0.0, 1.0)
        g["mtlIndex"] = mtl
    return bounds


def field_camera(width: int, height: int, bounds, pitch_angle: float = 2.2689) -> np.ndarray:
    """Camera above the near rows of the field (5 % into it, 5 % of its depth above the models) looking 40 degrees down
    along it (yaw = pi/2 as the default camera, pitch = pi/2 + 40 deg): the horizon lies above the top of the frame and
    the wide horizontal field of view stays over the ground quad, so ~96 % of the primary rays end on a model or on the
    ground (oracle, 240x135: 3.2 rays per pixel at 8 bounces against 4.2 for the single ShaderBalls model)."""
    xmin, xmax, ymin, ymax, zmax = bounds
    depth = ymax - ymin
    position = ((xmin + xmax) * 0.5, ymin + 0.05 * depth, 0.05 * depth + zmax)
    return default_camera(width, height, position=position, pitch=pitch_angle)


def bistro_scale_scene(base_scene: dict, copies: int = 183, width: int = 1920, height: int = 1080) -> dict:
    """Full scene dict (arrays in the reference layout) with the BVH built by the host builder."""
    from . import hostapi
    tris, bounds = replicate(base_scene["triangles"], copies)
    ordered, nodes, depth = hostapi.build_bvh(tris)
    scene = dict(base_scene)
    scene["triangles"], scene["nodes"] = ordered, nodes
    mats = np.ascontiguousarray(base_scene["materials"])
    emis = (mats["emission"][ordered["mtlIndex"]] >> 24) != 0          # RGBE exponent byte 0 <=> no emission (scene.cpp:87-103)
    scene["emissive"] = np.nonzero(emis)[0].astype("<u4")
    info = np.array(base_scene["scene_info"], copy=True)
    info["emissive_count"] = len(scene["emissive"])
    scene["scene_info"] = info
    scene["camera_pose"] = field_camera(width, height, bounds)
    scene["bvh_depth"] = depth
    return scene



def instanced_field(base_scene: dict, copies: int = 183, grid: int = 14, seed: int = 1234, width: int = 1920, height: int = 1080) -> dict:
    """replicate()'s field as an instanced scene (Context.upload_instanced_scene / set_instances): the base model as mesh 0, the
    ground quad as mesh 1, and copies + 1 instances with replicate()'s placements (the rotation about Z and the grid cell as one
    matrix rounded to float; the ground at identity).  Each mesh's BVH comes from the host builder.  Keys: meshes, shared (the
    base scene, for its materials, lights, textures and environment), mesh_ids, transforms (n, 3, 4), camera_pose."""
    from . import hostapi
    t = np.ascontiguousarray(base_scene["triangles"], dtype=TRIANGLE_DT)
    pos = np.stack([t[v]["position"][:, :3] for v in ("v1", "v2", "v3")], axis=1).astype(np.float64)
    lo, hi = pos.reshape(-1, 3).min(0), pos.reshape(-1, 3).max(0)
    centre = (lo + hi) * 0.5
    pitch = 1.1 * max(hi[0] - lo[0], hi[1] - lo[1])
    ground = np.zeros(2, dtype=TRIANGLE_DT)
    bounds = _field_ground(ground, lo, hi, pitch, copies, grid, t["mtlIndex"][0])
    meshes = []
    for tris in (t, ground):
        ordered, nodes, _ = hostapi.build_bvh(tris)
        meshes.append({"triangles": ordered, "nodes": nodes})
    transforms = np.zeros((copies + 1, 3, 4), dtype=np.float32)
    x = seed
    for k in range(copies):
        x = (1103515245 * x + 12345) & 0xFFFFFFFF
        ang = (x / 4294967296.0) * 2.0 * math.pi
        c, s = math.cos(ang), math.sin(ang)
        rot = np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])
        cell = np.array([(k % grid) * pitch, (k // grid) * pitch, 0.0])
        transforms[k, :, :3] = rot
        transforms[k, :, 3] = cell - rot @ (centre * [1, 1, 0])
    transforms[copies, :, :3] = np.eye(3)
    return {"meshes": meshes, "shared": base_scene, "mesh_ids": np.array([0] * copies + [1], dtype="<u4"), "transforms": transforms,
            "camera_pose": field_camera(width, height, bounds)}
