"""
ctypes binding of raytracing_b200/librt_b200.so — the C ABI declared in include/rt_b200.h.
Thin on purpose: one method per entry point, numpy arrays in the reference's byte layouts
(raytracing_b200/layouts.py) in and out.  Fails loudly when the CUDA library is missing;
there is no CPU fallback.
"""
import ctypes as C
import os

import numpy as np

from .layouts import (CAMERA_DT, HIT_DT, LIGHT_DT, MATERIAL_DT, NODE_DT, RAY_DT, SCENE_INFO_DT, TEXTURE_DT, TRIANGLE_DT)

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("RT_B200_LIB", os.path.join(HERE, "librt_b200.so"))   # override: tuning variants
MAX_BOUNCES = 255

OPT_WHITE_FURNACE, OPT_SAMPLER, OPT_AOV, OPT_DENOISER = 0, 1, 2, 3
BN_SOBOL_COUNT, BN_TILE_COUNT = 65536, 131072
OPT_COUNT_TRAVERSAL, OPT_KERNEL_TIMING, OPT_TRAVERSAL = 16, 17, 18
OPT_AOV_ALWAYS, OPT_SMEM_BVH, OPT_OVERLAP, OPT_GRAPH, OPT_PDL, OPT_FRAME_KERNEL, OPT_PRESENT, OPT_FRAME_THREADS, OPT_TOP_SMEM = 21, 22, 23, 24, 25, 26, 27, 28, 29
KERNEL_CLASSES = ["raygen", "intersect", "miss", "hit", "intersect_shadow", "accumulate", "extend_shade",
                  "shadow_accumulate", "resolve", "aov", "misc", "trace_closest", "shade_queues", "trace_both"]

# every symbol include/rt_b200.h declares
SYMBOLS = ["rt_create", "rt_destroy", "rt_last_error", "rt_set_partition", "rt_upload_scene", "rt_set_camera", "rt_set_option",
           "rt_upload_sampler_tables",
           "rt_reset", "rt_advance_sample_count", "rt_generate_rays", "rt_intersect", "rt_compute_aovs", "rt_shade_miss",
           "rt_clear_outgoing_counter", "rt_clear_shadow_counter", "rt_shade_hits", "rt_intersect_shadow",
           "rt_accumulate_direct", "rt_denoise", "rt_copy_history", "rt_resolve", "rt_resolve_async", "rt_resolve_wait", "rt_resolve_gathered", "rt_resolve_gathered_async", "rt_extend_shade", "rt_shadow_accumulate",
           "rt_integrate", "rt_integrate_samples", "rt_sync", "rt_read_hits", "rt_read_rays", "rt_read_radiance", "rt_read_frame_stats",
           "rt_read_sample_count", "rt_read_aovs", "rt_kernel_times", "rt_launch_count", "rt_local_pixel_count",
           "rt_radiance_device_ptr", "rt_stream_handle",
           "rt_create_multi", "rt_device_count", "rt_gather_radiance", "rt_host_register", "rt_host_unregister", "rt_math_eval",
           "rt_gather_buffer", "rt_ipc_export", "rt_ipc_open", "rt_set_gather_target", "rt_gather_wait",
           "rt_set_adaptive_sampling", "rt_read_pixel_samples", "rt_read_active_pixels", "rt_set_spatial_denoiser"]


class RtSceneDesc(C.Structure):
    _fields_ = [("triangles", C.c_void_p), ("n_triangles", C.c_uint64),
                ("nodes", C.c_void_p), ("n_nodes", C.c_uint64),
                ("materials", C.c_void_p), ("n_materials", C.c_uint64),
                ("lights", C.c_void_p), ("n_lights", C.c_uint64),
                ("textures", C.c_void_p), ("n_textures", C.c_uint64),
                ("texture_data", C.c_void_p), ("n_texture_data", C.c_uint64),
                ("emissive_indices", C.c_void_p), ("n_emissive", C.c_uint64),
                ("env_image", C.c_void_p), ("env_width", C.c_uint32), ("env_height", C.c_uint32),
                ("scene_info", C.c_uint32 * 4)]


FRAME_STATS_DT = np.dtype([(k, "<u4", MAX_BOUNCES + 1) for k in ("n_ext", "n_miss", "n_emissive_hits", "n_shadow", "n_cont", "n_unoccluded")] +
                          [(k, "<u8", MAX_BOUNCES + 1) for k in ("nodes_ext", "tris_ext", "nodes_shadow", "tris_shadow")])


class RtError(RuntimeError):
    def __init__(self, code, message):
        super().__init__(f"rt_b200 error {code}: {message}")
        self.code = code


_lib = None


def load_library():
    """Loads librt_b200.so (no compute). Raises if the CUDA extension has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU fallback for the render path)")
    L = C.CDLL(LIB_PATH)
    L.rt_last_error.restype = C.c_char_p
    L.rt_last_error.argtypes = [C.c_void_p]
    L.rt_create.argtypes = [C.c_uint32, C.c_uint32, C.c_int, C.POINTER(C.c_void_p)]
    L.rt_set_partition.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
    L.rt_upload_scene.argtypes = [C.c_void_p, C.POINTER(RtSceneDesc)]
    L.rt_set_camera.argtypes = [C.c_void_p, C.c_void_p]
    L.rt_set_option.argtypes = [C.c_void_p, C.c_int, C.c_uint32]
    L.rt_upload_sampler_tables.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    for name in ("rt_destroy", "rt_reset", "rt_advance_sample_count", "rt_generate_rays", "rt_compute_aovs", "rt_clear_shadow_counter",
                 "rt_intersect_shadow", "rt_accumulate_direct", "rt_denoise", "rt_copy_history", "rt_sync"):
        getattr(L, name).argtypes = [C.c_void_p]
    for name in ("rt_intersect", "rt_shade_miss", "rt_clear_outgoing_counter", "rt_shade_hits", "rt_extend_shade",
                 "rt_shadow_accumulate", "rt_integrate"):
        getattr(L, name).argtypes = [C.c_void_p, C.c_uint32]
    L.rt_integrate_samples.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
    L.rt_resolve.argtypes = [C.c_void_p, C.c_void_p]
    L.rt_resolve_async.argtypes = [C.c_void_p, C.c_void_p]
    L.rt_resolve_wait.argtypes = [C.c_void_p]
    L.rt_resolve_gathered.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
    L.rt_resolve_gathered_async.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
    L.rt_read_hits.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32)]
    L.rt_read_rays.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32)]
    L.rt_read_radiance.argtypes = [C.c_void_p, C.c_void_p]
    L.rt_read_frame_stats.argtypes = [C.c_void_p, C.c_void_p]
    L.rt_read_sample_count.argtypes = [C.c_void_p, C.POINTER(C.c_uint32)]
    L.rt_read_aovs.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.rt_kernel_times.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.rt_launch_count.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
    L.rt_local_pixel_count.argtypes = [C.c_void_p, C.POINTER(C.c_uint32)]
    L.rt_radiance_device_ptr.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]
    L.rt_stream_handle.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
    L.rt_create_multi.argtypes = [C.c_uint32, C.c_uint32, C.POINTER(C.c_int), C.c_uint32, C.POINTER(C.c_void_p)]
    L.rt_device_count.argtypes = [C.POINTER(C.c_int)]
    L.rt_gather_radiance.argtypes = [C.c_void_p]
    L.rt_host_register.argtypes = [C.c_void_p, C.c_uint64]
    L.rt_host_unregister.argtypes = [C.c_void_p]
    L.rt_math_eval.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]
    L.rt_gather_buffer.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    L.rt_ipc_export.argtypes = [C.c_void_p, C.c_void_p]
    L.rt_ipc_open.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]
    L.rt_set_gather_target.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    L.rt_gather_wait.argtypes = [C.c_void_p]
    L.rt_set_adaptive_sampling.argtypes = [C.c_void_p, C.c_float, C.c_uint32]
    L.rt_read_pixel_samples.argtypes = [C.c_void_p, C.c_void_p]
    L.rt_read_active_pixels.argtypes = [C.c_void_p, C.POINTER(C.c_uint32)]
    L.rt_set_spatial_denoiser.argtypes = [C.c_void_p, C.c_uint32, C.c_float, C.c_float, C.c_float]
    _lib = L
    return L


class Context:
    """One render context (== one CLPathTraceIntegrator + CLContext in the reference) on one GPU."""

    def __init__(self, width: int, height: int, device: int = 0, rank: int = 0, world: int = 1, devices=None):
        """devices = [d0, d1, ...]: ONE context over several GPUs of the node (rt_create_multi: device i renders rank i of a
        len(devices)-way scanline partition, every call fans out inside the library); otherwise a single-device context,
        optionally one rank of a partition driven from outside (one process per GPU)."""
        self.lib = load_library()
        self.width, self.height = width, height
        h = C.c_void_p()
        if devices is not None:
            arr = (C.c_int * len(devices))(*devices)
            rc = self.lib.rt_create_multi(width, height, arr, len(devices), C.byref(h))
        else:
            rc = self.lib.rt_create(width, height, device, C.byref(h))
        if rc != 0:
            raise RtError(rc, self.lib.rt_last_error(None).decode())
        self.h = h
        self.rank, self.world = rank, world
        self.devices = list(devices) if devices is not None else None
        if world != 1:
            self._ck(self.lib.rt_set_partition(self.h, rank, world))
        self._keep = None

    def gather_radiance(self):
        self._ck(self.lib.rt_gather_radiance(self.h))

    # ---- fused gather over peer memory (rt_gather_buffer .. rt_gather_wait)
    def gather_buffer(self):
        """-> (device pointer, slab stride in bytes, total bytes) of the gathered-radiance buffer this context owns."""
        p, st, tot = C.c_void_p(), C.c_uint64(), C.c_uint64()
        self._ck(self.lib.rt_gather_buffer(self.h, C.byref(p), C.byref(st), C.byref(tot)))
        return p.value, st.value, tot.value

    def ipc_open(self, handle: bytes):
        buf = C.create_string_buffer(bytes(handle), 64)
        p = C.c_void_p()
        self._ck(self.lib.rt_ipc_open(self.h, buf, C.byref(p)))
        return p.value

    def set_gather_target(self, base, stride_bytes=0):
        self._ck(self.lib.rt_set_gather_target(self.h, C.c_void_p(base) if base else None, stride_bytes))

    def gather_wait(self):
        self._ck(self.lib.rt_gather_wait(self.h))

    def _ck(self, rc):
        if rc != 0:
            raise RtError(rc, self.lib.rt_last_error(self.h).decode())

    def destroy(self):
        if self.h:
            self.lib.rt_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass

    # ---- Integrator public interface
    def upload_scene(self, scene: dict):
        a = {
            "triangles": np.ascontiguousarray(scene["triangles"], dtype=TRIANGLE_DT),
            "nodes": np.ascontiguousarray(scene["nodes"], dtype=NODE_DT),
            "materials": np.ascontiguousarray(scene["materials"], dtype=MATERIAL_DT),
            "lights": np.ascontiguousarray(scene["lights"], dtype=LIGHT_DT),
            "textures": np.ascontiguousarray(scene["textures"], dtype=TEXTURE_DT),
            "texels": np.ascontiguousarray(scene["texels"], dtype="<u4"),
            "emissive": np.ascontiguousarray(scene["emissive"], dtype="<u4"),
            "env": np.ascontiguousarray(scene["env"], dtype="<f4"),
        }
        d = RtSceneDesc()
        d.triangles, d.n_triangles = a["triangles"].ctypes.data, a["triangles"].shape[0]
        d.nodes, d.n_nodes = a["nodes"].ctypes.data, a["nodes"].shape[0]
        d.materials, d.n_materials = a["materials"].ctypes.data, a["materials"].shape[0]
        d.lights, d.n_lights = a["lights"].ctypes.data, a["lights"].shape[0]
        d.textures, d.n_textures = (a["textures"].ctypes.data if a["textures"].size else None), a["textures"].shape[0]
        d.texture_data, d.n_texture_data = (a["texels"].ctypes.data if a["texels"].size else None), a["texels"].shape[0]
        d.emissive_indices, d.n_emissive = (a["emissive"].ctypes.data if a["emissive"].size else None), a["emissive"].shape[0]
        d.env_image, d.env_width, d.env_height = a["env"].ctypes.data, int(scene["env_width"]), int(scene["env_height"])
        info = np.ascontiguousarray(scene["scene_info"], dtype=SCENE_INFO_DT).view("<u4").ravel()
        for i in range(4):
            d.scene_info[i] = int(info[i])
        self._ck(self.lib.rt_upload_scene(self.h, C.byref(d)))

    def set_camera(self, cam):
        c = np.ascontiguousarray(cam, dtype=CAMERA_DT)
        self._ck(self.lib.rt_set_camera(self.h, c.ctypes.data))

    def set_option(self, key, value): self._ck(self.lib.rt_set_option(self.h, key, int(value)))

    def upload_sampler_tables(self, sobol, scrambling, ranking):
        """The blue-noise sampler's tables (utils/blue_noise_sampler.hpp in the reference); then set_option(OPT_SAMPLER, 1)."""
        t = [np.ascontiguousarray(a, dtype=np.int32) for a in (sobol, scrambling, ranking)]
        if [a.size for a in t] != [BN_SOBOL_COUNT, BN_TILE_COUNT, BN_TILE_COUNT]:
            raise ValueError("sampler tables must have 65536, 131072 and 131072 entries")
        self._ck(self.lib.rt_upload_sampler_tables(self.h, *[a.ctypes.data for a in t]))

    # ---- Integrator protected steps
    def reset(self): self._ck(self.lib.rt_reset(self.h))
    def advance_sample_count(self): self._ck(self.lib.rt_advance_sample_count(self.h))
    def generate_rays(self): self._ck(self.lib.rt_generate_rays(self.h))
    def intersect(self, bounce): self._ck(self.lib.rt_intersect(self.h, bounce))
    def compute_aovs(self): self._ck(self.lib.rt_compute_aovs(self.h))
    def shade_miss(self, bounce): self._ck(self.lib.rt_shade_miss(self.h, bounce))
    def clear_outgoing_counter(self, bounce): self._ck(self.lib.rt_clear_outgoing_counter(self.h, bounce))
    def clear_shadow_counter(self): self._ck(self.lib.rt_clear_shadow_counter(self.h))
    def shade_hits(self, bounce): self._ck(self.lib.rt_shade_hits(self.h, bounce))
    def intersect_shadow(self): self._ck(self.lib.rt_intersect_shadow(self.h))
    def accumulate_direct(self): self._ck(self.lib.rt_accumulate_direct(self.h))
    def extend_shade(self, bounce): self._ck(self.lib.rt_extend_shade(self.h, bounce))
    def shadow_accumulate(self, bounce): self._ck(self.lib.rt_shadow_accumulate(self.h, bounce))
    def integrate(self, max_bounces): self._ck(self.lib.rt_integrate(self.h, max_bounces))

    def integrate_samples(self, max_bounces, n_samples):
        """n_samples consecutive frames of integrate(max_bounces) in one call (rt_integrate_samples): the same bits, the frame
        statistics summed over the samples."""
        self._ck(self.lib.rt_integrate_samples(self.h, max_bounces, n_samples))

    def sync(self): self._ck(self.lib.rt_sync(self.h))

    # ---- adaptive sampling
    def set_adaptive_sampling(self, max_error, min_samples=2):
        """Stop tracing pixels whose resolved luminance has a standard error <= max_error after >= min_samples samples
        (rt_set_adaptive_sampling); max_error 0 turns it off.  Takes effect at the next reset()."""
        self._ck(self.lib.rt_set_adaptive_sampling(self.h, float(max_error), int(min_samples)))

    def pixel_samples(self):
        """-> (h, w) uint32: every local pixel's sample count (rows of other ranks left zero)."""
        out = np.zeros((self.height, self.width), dtype="<u4")
        self._ck(self.lib.rt_read_pixel_samples(self.h, out.ctypes.data))
        return out

    def active_pixels(self):
        """Pixels that will trace the next sample (all local pixels when adaptive sampling is off)."""
        n = C.c_uint32()
        self._ck(self.lib.rt_read_active_pixels(self.h, C.byref(n)))
        return n.value

    # ---- spatial denoiser
    def set_spatial_denoiser(self, iterations, sigma_color=0.0, sigma_normal=0.0, sigma_depth=0.0):
        """Edge-avoiding a-trous filter on the shaded colour of resolve() / resolve_async() (rt_set_spatial_denoiser): iterations
        0 (off) .. 5, guided by the last frame's normal and depth; a sigma of 0 drops its term."""
        self._ck(self.lib.rt_set_spatial_denoiser(self.h, int(iterations), float(sigma_color), float(sigma_normal), float(sigma_depth)))

    def integrate_stepwise(self, max_bounces):
        """The schedule of Integrator::Integrate (integrator.cpp:35-51), one call per reference virtual."""
        self.generate_rays()
        for b in range(max_bounces + 1):
            self.intersect(b)
            if b == 0:
                self.compute_aovs()
            self.shade_miss(b)
            self.clear_outgoing_counter(b)
            self.clear_shadow_counter()
            self.shade_hits(b)
            self.intersect_shadow()
            self.accumulate_direct()
        self.advance_sample_count()

    def resolve(self, out=None):
        if out is None:
            out = np.zeros((self.height, self.width, 4), dtype="<f4")
        self._ck(self.lib.rt_resolve(self.h, out.ctypes.data))
        return out

    def resolve_async(self, out):
        """out: pinned/contiguous (h, w, 4) float32 host array that stays alive and untouched until resolve_wait()."""
        self._ck(self.lib.rt_resolve_async(self.h, out.ctypes.data))

    def resolve_wait(self): self._ck(self.lib.rt_resolve_wait(self.h))

    def resolve_gathered(self, slabs_device_ptr, slab_stride_bytes, out=None, wait=True):
        """Rank 0 of a multi-GPU frame: resolve the gathered slabs (device pointer, one slab per rank) into the whole host image."""
        if out is None:
            out = np.zeros((self.height, self.width, 4), dtype="<f4")
        fn = self.lib.rt_resolve_gathered if wait else self.lib.rt_resolve_gathered_async
        self._ck(fn(self.h, C.c_void_p(slabs_device_ptr), int(slab_stride_bytes), out.ctypes.data))
        return out

    # ---- taps
    def local_pixel_count(self):
        n = C.c_uint32()
        self._ck(self.lib.rt_local_pixel_count(self.h, C.byref(n)))
        return n.value

    def read_hits(self, bounce):
        cap = self.local_pixel_count()
        hits = np.zeros(cap, dtype=HIT_DT)
        pix = np.zeros(cap, dtype="<u4")
        n = C.c_uint32()
        self._ck(self.lib.rt_read_hits(self.h, bounce, hits.ctypes.data, pix.ctypes.data, C.byref(n)))
        return hits[: n.value], pix[: n.value]

    def read_rays(self, bounce):
        cap = self.local_pixel_count()
        rays = np.zeros(cap, dtype=RAY_DT)
        pix = np.zeros(cap, dtype="<u4")
        n = C.c_uint32()
        self._ck(self.lib.rt_read_rays(self.h, bounce, rays.ctypes.data, pix.ctypes.data, C.byref(n)))
        return rays[: n.value], pix[: n.value]

    def read_radiance(self, out=None):
        if out is None:
            out = np.zeros((self.height, self.width, 4), dtype="<f4")
        self._ck(self.lib.rt_read_radiance(self.h, out.ctypes.data))
        return out

    def frame_stats(self):
        st = np.zeros((), dtype=FRAME_STATS_DT)
        self._ck(self.lib.rt_read_frame_stats(self.h, st.ctypes.data))
        return st

    def denoise(self): self._ck(self.lib.rt_denoise(self.h))
    def copy_history(self): self._ck(self.lib.rt_copy_history(self.h))

    def read_aovs(self):
        """-> albedo[h,w,4], depth[h,w], normal[h,w,4], velocity[h,w,2] (rows of other ranks left zero)."""
        al = np.zeros((self.height, self.width, 4), "<f4"); de = np.zeros((self.height, self.width), "<f4")
        no = np.zeros((self.height, self.width, 4), "<f4"); ve = np.zeros((self.height, self.width, 2), "<f4")
        self._ck(self.lib.rt_read_aovs(self.h, al.ctypes.data, de.ctypes.data, no.ctypes.data, ve.ctypes.data))
        return al, de, no, ve

    def sample_count(self):
        n = C.c_uint32()
        self._ck(self.lib.rt_read_sample_count(self.h, C.byref(n)))
        return n.value

    def kernel_times(self):
        ms = np.zeros(len(KERNEL_CLASSES), dtype="<f4")
        nl = np.zeros(len(KERNEL_CLASSES), dtype="<u4")
        self._ck(self.lib.rt_kernel_times(self.h, ms.ctypes.data, nl.ctypes.data))
        return {k: (float(ms[i]), int(nl[i])) for i, k in enumerate(KERNEL_CLASSES)}

    def launch_count(self):
        n = C.c_uint64()
        self._ck(self.lib.rt_launch_count(self.h, C.byref(n)))
        return n.value

    def radiance_device_ptr(self):
        p, b = C.c_void_p(), C.c_uint64()
        self._ck(self.lib.rt_radiance_device_ptr(self.h, C.byref(p), C.byref(b)))
        return p.value, b.value

    def stream_handle(self):
        p = C.c_void_p()
        self._ck(self.lib.rt_stream_handle(self.h, C.byref(p)))
        return p.value


def device_count() -> int:
    n = C.c_int()
    load_library().rt_device_count(C.byref(n))
    return n.value


def host_register(array) -> None:
    """Page-locks a numpy array's memory (the image handed to Context.resolve) — rt_host_register."""
    rc = load_library().rt_host_register(array.ctypes.data, array.nbytes)
    if rc != 0:
        raise RtError(rc, load_library().rt_last_error(None).decode())


def host_unregister(array) -> None:
    load_library().rt_host_unregister(array.ctypes.data)


MATH_FUNCTIONS = {"sin": 0, "cos": 1, "tan": 2, "atan2": 3, "acos": 4, "pow": 5, "fmin": 6, "fmax": 7, "rsqrt": 8, "div": 9, "exp": 10}


def math_eval(fn: str, a, b=None, device: int = 0):
    """include/rt_math.h function `fn` evaluated on the device (rt_math_eval)."""
    a = np.ascontiguousarray(a, dtype="<f4")
    b = np.ascontiguousarray(np.zeros_like(a) if b is None else b, dtype="<f4")
    out = np.zeros_like(a)
    rc = load_library().rt_math_eval(device, MATH_FUNCTIONS[fn], a.ctypes.data, b.ctypes.data, out.ctypes.data, a.size)
    if rc != 0:
        raise RtError(rc, load_library().rt_last_error(None).decode())
    return out


def ipc_export(dev_ptr: int) -> bytes:
    """64-byte CUDA IPC handle of a device allocation (rt_ipc_export)."""
    buf = C.create_string_buffer(64)
    rc = load_library().rt_ipc_export(C.c_void_p(dev_ptr), buf)
    if rc != 0:
        raise RtError(rc, load_library().rt_last_error(None).decode())
    return buf.raw
