"""
ctypes binding of raytracing_b200/librt_host.so: the C++ host side (Scene loader, SAH BVH builder,
Integrator / CUDAPathTraceIntegrator, headless Render with RenderBackend::kCUDA) through the small C
façade in host/host_capi.cpp.  Used by tests and bench.py; the C++ classes are the real interface.
"""
import ctypes as C
import os

import numpy as np

from .layouts import CAMERA_DT, NODE_DT, SCENE_ARRAYS, TRIANGLE_DT

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "librt_host.so")
_lib = None


def load_library():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'`")
    # The BVH builder's OpenMP tasks leave workers idle at the top of the tree; spinning idle workers (libgomp's default) cost
    # 3x on shared hosts.  Only effective if this is the process's first OpenMP user (the policy is read when libgomp starts).
    os.environ.setdefault("OMP_WAIT_POLICY", "passive")
    L = C.CDLL(LIB_PATH)
    L.rth_last_error.restype = C.c_char_p
    L.rth_scene_load.restype = C.c_void_p
    L.rth_scene_load.argtypes = [C.c_char_p, C.c_float, C.c_int]
    L.rth_scene_free.argtypes = [C.c_void_p]
    L.rth_scene_add_directional_light.argtypes = [C.c_void_p] + [C.c_float] * 6
    L.rth_scene_add_point_light.argtypes = [C.c_void_p] + [C.c_float] * 6
    L.rth_scene_build_bvh.argtypes = [C.c_void_p]
    L.rth_scene_finalize_hdr.argtypes = [C.c_void_p, C.c_char_p]
    L.rth_scene_finalize_image.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32]
    L.rth_scene_query.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    L.rth_bvh_build.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_size_t), C.POINTER(C.c_uint32)]
    L.rth_default_camera.argtypes = [C.c_uint32, C.c_uint32, C.c_void_p]
    L.rth_obj_parse_number.argtypes = [C.c_char_p, C.POINTER(C.c_double)]
    L.rth_render_create.restype = C.c_void_p
    L.rth_render_create.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_char_p, C.c_int, C.c_int]
    L.rth_render_free.argtypes = [C.c_void_p]
    L.rth_render_set_max_bounces.argtypes = [C.c_void_p, C.c_uint32]
    L.rth_render_set_samples_per_frame.argtypes = [C.c_void_p, C.c_uint32]
    L.rth_render_set_adaptive_sampling.argtypes = [C.c_void_p, C.c_float, C.c_uint32]
    L.rth_render_set_spatial_denoiser.argtypes = [C.c_void_p, C.c_uint32, C.c_float, C.c_float, C.c_float]
    L.rth_render_set_emitter_sampling.argtypes = [C.c_void_p, C.c_int]
    L.rth_render_set_environment_sampling.argtypes = [C.c_void_p, C.c_int]
    L.rth_render_set_object_motion.argtypes = [C.c_void_p, C.c_int]
    L.rth_render_set_light_selection.argtypes = [C.c_void_p, C.c_float, C.c_float, C.c_float]
    L.rth_render_update_triangles.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.rth_render_rebuild_bvh.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
    L.rth_render_upload_instanced_scene.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint32]
    L.rth_render_set_instances.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
    L.rth_render_update_mesh_triangles.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t]
    L.rth_render_set_instance_materials.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]
    L.rth_render_rebuild_bvh_ploc.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
    L.rth_render_active_pixels.argtypes = [C.c_void_p, C.POINTER(C.c_uint32)]
    L.rth_render_enable_white_furnace.argtypes = [C.c_void_p, C.c_int]
    L.rth_render_set_sampler.argtypes = [C.c_void_p, C.c_int]
    L.rth_render_set_sampler_tables.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.rth_render_frame.argtypes = [C.c_void_p]
    L.rth_render_request_reset.argtypes = [C.c_void_p]
    L.rth_render_nodes.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]
    L.rth_render_image.restype = C.POINTER(C.c_float)
    L.rth_render_image.argtypes = [C.c_void_p]
    L.rth_render_context.restype = C.c_void_p
    L.rth_render_context.argtypes = [C.c_void_p]
    _lib = L
    return L


class HostError(RuntimeError):
    pass


def _err(L):
    return HostError(L.rth_last_error().decode())


def default_camera(width, height):
    cam = np.zeros((), dtype=CAMERA_DT)
    load_library().rth_default_camera(width, height, cam.ctypes.data)
    return cam


def obj_parse_number(text: str):
    """A number token as the OBJ reader reads it (the reference loader's digit accumulation, not strtod); None = not a number."""
    v = C.c_double()
    return v.value if load_library().rth_obj_parse_number(text.encode(), C.byref(v)) else None


def build_bvh(triangles):
    """Host SAH build over a triangle array -> (triangles in leaf order, LinearBVHNode[], max depth)."""
    L = load_library()
    src = np.ascontiguousarray(triangles, dtype=TRIANGLE_DT)
    t = np.empty(src.shape, dtype=TRIANGLE_DT)
    t.view(np.uint8)[:] = src.view(np.uint8)                   # byte copy: numpy copies structured records field by field otherwise
    nodes = np.empty(2 * t.shape[0], dtype=NODE_DT)          # a binary tree over n leaves has at most 2n - 1 nodes
    n, depth = C.c_size_t(), C.c_uint32()
    if L.rth_bvh_build(t.ctypes.data, t.shape[0], nodes.ctypes.data, C.byref(n), C.byref(depth)) != 0:
        raise _err(L)
    return t, nodes[: n.value], depth.value


class HostScene:
    """rt_host::Scene (+ an rt_host::Bvh) behind a handle."""

    def __init__(self, obj_path, scale=1.0, flip_yz=False):
        self.L = load_library()
        self.h = self.L.rth_scene_load(obj_path.encode(), scale, int(flip_yz))
        if not self.h:
            raise _err(self.L)

    def add_directional_light(self, d, rgb): self.L.rth_scene_add_directional_light(self.h, *map(float, d), *map(float, rgb))
    def add_point_light(self, p, rgb): self.L.rth_scene_add_point_light(self.h, *map(float, p), *map(float, rgb))

    def build_bvh(self):
        if self.L.rth_scene_build_bvh(self.h) != 0:
            raise _err(self.L)

    def finalize(self, env_path=None, env=None, env_width=0, env_height=0):
        if env_path is not None:
            if self.L.rth_scene_finalize_hdr(self.h, env_path.encode()) != 0:
                raise _err(self.L)
        else:
            e = np.ascontiguousarray(env, dtype="<f4")
            self.L.rth_scene_finalize_image(self.h, e.ctypes.data, env_width, env_height)

    def arrays(self) -> dict:
        out = {}
        for i, (name, dt) in enumerate(SCENE_ARRAYS):
            p, n, e0, e1 = C.c_void_p(), C.c_size_t(), C.c_uint32(), C.c_uint32()
            self.L.rth_scene_query(self.h, i, C.byref(p), C.byref(n), C.byref(e0), C.byref(e1))
            nbytes = n.value * dt.itemsize
            buf = (C.c_char * nbytes).from_address(p.value) if nbytes else b""
            out[name] = np.frombuffer(bytes(buf), dtype=dt).copy()
            if name == "env":
                out["env_width"], out["env_height"] = e0.value, e1.value
        return out

    def close(self):
        if self.h:
            self.L.rth_scene_free(self.h)
            self.h = None


def scene_from_arrays(scene: dict):
    """HostScene holding a scene dump (dict of arrays in the reference layout): the C++ Scene as it is after Load() and the
    Add*Light calls (bench/test plumbing; the triangles are copied)."""
    from .layouts import LIGHT_DT, MATERIAL_DT, TEXTURE_DT, TRIANGLE_DT
    hs = HostScene.__new__(HostScene)
    hs.L = load_library()
    hs.L.rth_scene_from_arrays.restype = C.c_void_p
    hs.L.rth_scene_from_arrays.argtypes = [C.c_void_p, C.c_size_t] * 5
    t = np.ascontiguousarray(scene["triangles"], dtype=TRIANGLE_DT); m = np.ascontiguousarray(scene["materials"], dtype=MATERIAL_DT)
    li = np.ascontiguousarray(scene["lights"], dtype=LIGHT_DT); tx = np.ascontiguousarray(scene["textures"], dtype=TEXTURE_DT)
    te = np.ascontiguousarray(scene["texels"], dtype="<u4")
    hs.h = hs.L.rth_scene_from_arrays(t.ctypes.data, len(t), m.ctypes.data, len(m), li.ctypes.data, len(li), tx.ctypes.data, len(tx), te.ctypes.data, len(te))
    if not hs.h:
        raise _err(hs.L)
    return hs


class HostRender:
    """rt_host::Render(width, height, RenderBackend::kCUDA, scene): builds the BVH, finalizes the scene, creates the
    CUDAPathTraceIntegrator and uploads, like Render::Render in the reference (render.cpp:38-83)."""

    SCHEDULES = {"frame": 0, "fused": 1, "stepwise": 2}

    def __init__(self, scene: HostScene, width, height, env_path, device=0, stepwise=False, devices=None, schedule=None):
        """devices = [d0, d1, ...] (or [] for every CUDA device of the node): one CUDAPathTraceIntegrator over several GPUs
        (rt_create_multi).  schedule: "frame" (default: Integrate() submits the whole frame with one call), "fused" (two
        kernels per bounce as the virtuals arrive), "stepwise" (one kernel per virtual)."""
        self.L = scene.L
        self.width, self.height = width, height
        sched = self.SCHEDULES[schedule] if schedule else (2 if stepwise else 0)
        if env_path is None:
            raise ValueError("env_path is required (use HostRender.with_env_image for a decoded environment image)")
        if devices is not None:
            self.L.rth_render_create_multi.restype = C.c_void_p
            self.L.rth_render_create_multi.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_char_p, C.POINTER(C.c_int), C.c_uint32, C.c_int]
            arr = (C.c_int * max(len(devices), 1))(*devices)
            self.h = self.L.rth_render_create_multi(scene.h, width, height, env_path.encode(), arr, len(devices), sched)
        else:
            self.h = self.L.rth_render_create(scene.h, width, height, env_path.encode(), device, int(stepwise))
        if not self.h:
            raise _err(self.L)
        if devices is None and schedule:
            self.set_schedule(schedule)

    @classmethod
    def with_env_image(cls, scene: HostScene, width, height, env_rgba, env_width, env_height, devices, schedule="frame"):
        """Render over `devices` with the environment image handed over decoded (RGBA32F rows)."""
        self = cls.__new__(cls)
        self.L = scene.L
        self.width, self.height = width, height
        self.L.rth_render_create_env.restype = C.c_void_p
        self.L.rth_render_create_env.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(C.c_int), C.c_uint32, C.c_int]
        env = np.ascontiguousarray(env_rgba, dtype="<f4")
        arr = (C.c_int * max(len(devices), 1))(*devices)
        self.h = self.L.rth_render_create_env(scene.h, width, height, env.ctypes.data, env_width, env_height, arr, len(devices), cls.SCHEDULES[schedule])
        if not self.h:
            raise _err(self.L)
        return self

    def set_camera(self, cam):
        c = np.ascontiguousarray(cam)
        self.L.rth_render_set_camera.argtypes = [C.c_void_p, C.c_void_p]
        self.L.rth_render_set_camera(self.h, c.ctypes.data)

    def set_schedule(self, schedule):
        self.L.rth_render_set_schedule.argtypes = [C.c_void_p, C.c_int]
        self.L.rth_render_set_schedule(self.h, self.SCHEDULES[schedule])

    def set_max_bounces(self, b):
        if self.L.rth_render_set_max_bounces(self.h, b) != 0:
            raise _err(self.L)

    def set_samples_per_frame(self, n):
        """Progressive samples accumulated by one render_frame() (Render::SetSamplesPerFrame); needs the "frame" schedule for n > 1."""
        if self.L.rth_render_set_samples_per_frame(self.h, n) != 0:
            raise _err(self.L)

    def set_adaptive_sampling(self, max_error, min_samples=2):
        """Render::SetAdaptiveSampling: pixels stop tracing once they have settled; applies from the next render_frame()."""
        if self.L.rth_render_set_adaptive_sampling(self.h, float(max_error), int(min_samples)) != 0:
            raise _err(self.L)

    def set_spatial_denoiser(self, iterations, sigma_color=0.0, sigma_normal=0.0, sigma_depth=0.0):
        """Render::SetSpatialDenoiser: edge-avoiding a-trous filter (0 = off .. 5 passes) on the image of every later render_frame()."""
        if self.L.rth_render_set_spatial_denoiser(self.h, int(iterations), float(sigma_color), float(sigma_normal), float(sigma_depth)) != 0:
            raise _err(self.L)

    def set_emitter_sampling(self, on):
        """Render::SetEmitterSampling: next-event estimation on the emissive triangles too (MIS); applies from the next render_frame()."""
        if self.L.rth_render_set_emitter_sampling(self.h, int(bool(on))) != 0:
            raise _err(self.L)

    def set_object_motion(self, on):
        """Render::SetObjectMotion: motion vectors (AOV view 4, the temporal denoiser) follow update_triangles as well as the camera."""
        if self.L.rth_render_set_object_motion(self.h, int(bool(on))) != 0:
            raise _err(self.L)

    def set_environment_sampling(self, on):
        """Render::SetEnvironmentSampling: next-event estimation on the environment map too (MIS); applies from the next render_frame()."""
        if self.L.rth_render_set_environment_sampling(self.h, int(bool(on))) != 0:
            raise _err(self.L)

    def set_light_selection(self, analytic=1.0, emitters=1.0, environment=1.0):
        """Render::SetLightSelection: relative weights of the light kind drawn at each vertex; applies from the next render_frame()."""
        if self.L.rth_render_set_light_selection(self.h, float(analytic), float(emitters), float(environment)) != 0:
            raise _err(self.L)

    def update_triangles(self, triangles):
        """Render::UpdateTriangles: the scene's triangles in leaf order with new positions, normals and texcoords; the BVH is refit
        on the device.  Keeps the accumulation (request_reset() starts over)."""
        t = np.ascontiguousarray(triangles, dtype=TRIANGLE_DT)
        if self.L.rth_render_update_triangles(self.h, t.ctypes.data, t.shape[0]) != 0:
            raise _err(self.L)

    def upload_instanced_scene(self, meshes):
        """Render::UploadInstancedScene: meshes = a list of dicts with "triangles" (leaf order) and "nodes" (the mesh's own array);
        the scene's materials, lights and environment are shared."""
        tris = np.concatenate([np.ascontiguousarray(m["triangles"], dtype=TRIANGLE_DT) for m in meshes])
        nodes = np.concatenate([np.ascontiguousarray(m["nodes"], dtype=NODE_DT) for m in meshes])
        desc = np.zeros((len(meshes), 4), dtype="<u8")
        t0 = n0 = 0
        for k, m in enumerate(meshes):
            desc[k] = (t0, len(m["triangles"]), n0, len(m["nodes"]))
            t0 += len(m["triangles"]); n0 += len(m["nodes"])
        if self.L.rth_render_upload_instanced_scene(self.h, tris.ctypes.data, len(tris), nodes.ctypes.data, len(nodes), desc.ctypes.data,
                                                    len(meshes)) != 0:
            raise _err(self.L)

    def set_instances(self, mesh_ids, transforms):
        """Render::SetInstances: mesh_ids[i] placed by the row-major 3x4 transforms[i]."""
        from .capi import INSTANCE_DT
        ids = np.ascontiguousarray(mesh_ids, dtype="<u4").reshape(-1)
        rec = np.zeros(len(ids), dtype=INSTANCE_DT)
        rec["object_to_world"] = np.ascontiguousarray(transforms, dtype="<f4").reshape(-1, 12)
        rec["mesh"] = ids
        if self.L.rth_render_set_instances(self.h, rec.ctypes.data if len(rec) else None, len(rec)) != 0:
            raise _err(self.L)

    def update_mesh_triangles(self, mesh, triangles):
        """Render::UpdateMeshTriangles: mesh `mesh` of the instanced scene in its leaf order with new positions, normals and
        texcoords; its tree is refit on the device.  Keeps the accumulation (request_reset() starts over)."""
        t = np.ascontiguousarray(triangles, dtype=TRIANGLE_DT)
        if self.L.rth_render_update_mesh_triangles(self.h, int(mesh), t.ctypes.data, t.shape[0]) != 0:
            raise _err(self.L)

    def set_instance_materials(self, remaps, remap_of_instance):
        """Render::SetInstanceMaterials: remaps (n_remaps, n_materials) rows, remap_of_instance the row of each instance index
        (-1 / None: its mesh's own materials), as capi.Context.set_instance_materials.  Keeps the accumulation."""
        from .capi import instance_material_arrays
        rows, of = instance_material_arrays(remaps, remap_of_instance)
        if self.L.rth_render_set_instance_materials(self.h, rows.ctypes.data if rows.size else None, rows.shape[0],
                                                    of.ctypes.data if of.size else None, len(of)) != 0:
            raise _err(self.L)

    def rebuild_bvh(self, method="linear"):
        """Render::RebuildBvh: a tree over the current triangles, built on the device, by method "linear" (BvhBuild::kLinear) or
        "ploc" (BvhBuild::kPloc); -> the new node count (2n - 1).  Keeps the accumulation (request_reset() starts over)."""
        fn = {"linear": self.L.rth_render_rebuild_bvh, "ploc": self.L.rth_render_rebuild_bvh_ploc}.get(method)
        if fn is None:
            raise ValueError("rebuild_bvh: method must be 'linear' or 'ploc', not %r" % (method,))
        n = C.c_uint64()
        if fn(self.h, C.byref(n)) != 0:
            raise _err(self.L)
        return n.value

    def active_pixels(self):
        """Render::ActivePixels: pixels that trace the next sample."""
        n = C.c_uint32()
        if self.L.rth_render_active_pixels(self.h, C.byref(n)) != 0:
            raise _err(self.L)
        return n.value

    def enable_white_furnace(self, e):
        if self.L.rth_render_enable_white_furnace(self.h, int(e)) != 0:
            raise _err(self.L)

    def set_blue_noise(self, e):
        if self.L.rth_render_set_sampler(self.h, int(e)) != 0:
            raise _err(self.L)

    def set_blue_noise_tables(self, sobol, scrambling, ranking):
        t = [np.ascontiguousarray(a, dtype=np.int32) for a in (sobol, scrambling, ranking)]
        if self.L.rth_render_set_sampler_tables(self.h, *[a.ctypes.data for a in t]) != 0:
            raise _err(self.L)

    def render_frame(self):
        if self.L.rth_render_frame(self.h) != 0:
            raise _err(self.L)

    def request_reset(self): self.L.rth_render_request_reset(self.h)

    def image(self):
        p = self.L.rth_render_image(self.h)
        return np.ctypeslib.as_array(p, shape=(self.height, self.width, 4)).copy()

    def nodes(self):
        p, n = C.c_void_p(), C.c_size_t()
        self.L.rth_render_nodes(self.h, C.byref(p), C.byref(n))
        buf = (C.c_char * (n.value * NODE_DT.itemsize)).from_address(p.value)
        return np.frombuffer(bytes(buf), dtype=NODE_DT).copy()

    def context_handle(self): return self.L.rth_render_context(self.h)

    def close(self):
        if self.h:
            self.L.rth_render_free(self.h)
            self.h = None
