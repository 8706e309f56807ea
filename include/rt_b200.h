/*
 * rt_b200.h — C ABI of the H100 (sm_90a) wavefront path-tracing backend.
 *
 * This shim takes the place of the reference's OpenCL wrapper layer
 *   /root/reference/src/gpu_wrappers/cl_context.hpp:37-99  (CLContext / CLKernel)
 * underneath an `Integrator` subclass (src/integrator/integrator.hpp:34-100); the C++
 * class that forwards the reference's virtual steps to these entry points is
 * raytracing_b200/host/cuda_pt_integrator.hpp.  Plain C: pointers, sizes, PODs from
 * rt_types.h (byte-identical to kernels/common/shared_structures.h); no torch, no CUDA
 * types.  Every function returns 0 on success or a negative RtStatus; the message is
 * available from rt_last_error().  No exception crosses this boundary (the reference
 * throws CLException from ThrowIfFailed, utils/cl_exception.hpp:117-123; the C++
 * integrator wrapper re-throws std::runtime_error to keep caller behaviour).
 *
 * Ownership (as the reference: CL_MEM_COPY_HOST_PTR, cl_pt_integrator.cpp:387-451):
 * rt_upload_scene copies; the caller keeps every host pointer before and after; all
 * device memory belongs to the context; read-backs go to caller-allocated memory.
 *
 * Threading/ordering (as the reference: ONE in-order queue, cl_context.cpp:89): one
 * caller thread per context; all step calls are asynchronous launches on one CUDA
 * stream; rt_resolve / rt_read_* / rt_sync are the synchronisation points.
 */
#ifndef RT_B200_H
#define RT_B200_H

#include <stdint.h>
#include "rt_types.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct rt_ctx rt_ctx;

typedef enum RtStatus {
    RT_OK = 0,
    RT_ERR_INVALID_ARGUMENT = -1,
    RT_ERR_CUDA = -2,            /* a CUDA runtime call or kernel failed */
    RT_ERR_NO_DEVICE = -3,       /* no usable CUDA device: there is NO CPU fallback */
    RT_ERR_NOT_READY = -4,       /* scene or camera not set yet */
    RT_ERR_UNSUPPORTED = -5
} RtStatus;

/* Inputs of Integrator::UploadGPUData (cl_pt_integrator.cpp:373-456): the seven Scene
 * arrays (scene/scene.hpp:45-53), SceneInfo and AccelerationStructure::GetNodes()
 * (acceleration_structure.hpp:31-38).  triangles[] must already be in BVH leaf order
 * (Bvh::BuildCPU reorders them, bvh.cpp:52).  Empty arrays: pointer may be NULL. */
typedef struct RtSceneDesc {
    const RtTriangle* triangles;        uint64_t n_triangles;      /* >= 1 */
    const RtLinearBVHNode* nodes;       uint64_t n_nodes;          /* >= 1 */
    const RtPackedMaterial* materials;  uint64_t n_materials;      /* >= 1 */
    const RtLight* lights;              uint64_t n_lights;         /* >= 1 (light.h:46 divides by the count) */
    const RtTexture* textures;          uint64_t n_textures;
    const uint32_t* texture_data;       uint64_t n_texture_data;
    const uint32_t* emissive_indices;   uint64_t n_emissive;       /* uploaded, never sampled (light.h:30-65) */
    const float* env_image;             uint32_t env_width, env_height;   /* RGBA32F rows, first row = v 0 */
    RtSceneInfo scene_info;
} RtSceneDesc;

/* rt_set_option keys: the Integrator setters (integrator.hpp:45-53) */
typedef enum RtOption {
    RT_OPT_WHITE_FURNACE = 0,   /* EnableWhiteFurnace(bool)                          */
    RT_OPT_SAMPLER = 1,         /* SetSamplerType: 0 = kRandom, 1 = kBlueNoise (after rt_upload_sampler_tables) */
    RT_OPT_AOV = 2,             /* SetAOV: 0 shaded colour, 1 albedo, 2 depth, 3 normal, 4 motion vectors (view used by rt_resolve) */
    RT_OPT_DENOISER = 3,        /* EnableDenoiser(bool): temporal accumulation (single-GPU only) */
    RT_OPT_COUNT_TRAVERSAL = 16,/* 1: kernels also count BVH nodes visited / triangles tested (slower; for
                                   the algorithmic-bytes figure of the roofline)     */
    RT_OPT_KERNEL_TIMING = 17,  /* 1: bracket every launch with CUDA events on the context's stream */
    RT_OPT_TRAVERSAL = 18,      /* 0: literal reference-order traversal on the reference node layout,
                                   1: child-box node layout (default); results are bit-identical */
    RT_OPT_AOV_ALWAYS = 21,     /* 1: produce the AOV buffers every frame even with the shaded-colour view (the reference always
                                   does; here they are skipped unless a view or the denoiser needs them) */
    RT_OPT_SMEM_BVH = 22,       /* 1 (default): scenes whose traversal records fit 40 KB are staged into shared memory by a TMA
                                   bulk copy at the start of every traversal kernel; 0: always fetch through L1 */
    RT_OPT_OVERLAP = 23,        /* how the shadow pass of bounce b overlaps the closest-hit traversal of bounce b+1 (they are independent):
                                   2 (default): rt_shadow_accumulate(b) is deferred and runs inside the traversal kernel of
                                      rt_extend_shade(b+1) (one persistent kernel drains both queues); any other call that needs
                                      its result launches it on its own first;
                                   1: on a second stream, concurrently with the traversal kernel;
                                   0: everything in call order on one in-order stream */
    RT_OPT_GRAPH = 24,          /* 1 (default): rt_integrate replays the frame as one CUDA graph (captured on first use, re-captured when an
                                   option, the scene or the partition changes; the camera and sample index are a node-parameter update) */
    RT_OPT_PDL = 25,            /* 1 (default): the traversal and shading kernels of a frame are chained by programmatic dependent launch
                                   (a kernel's CTAs start and stage the BVH while the previous kernel drains) */
    RT_OPT_FRAME_KERNEL = 26,   /* how rt_integrate runs a frame.  1: ONE persistent kernel in which every CTA is an independent
                                   wavefront over its own pixels (queue cursors in shared memory, no global atomics, no launch
                                   boundaries); 0: one kernel per phase (graph replay / PDL chain as configured above);
                                   2 (default): the one-kernel frame for partitions of up to 7168 pixels per SM (0.95 M pixels,
                                   under half a 1080p frame, on an H100's 132 SMs), per-phase kernels for larger ones.  Results are bit-identical.
                                   rt_integrate_samples: 1 also selects the regenerating frame kernel (one launch per call), which is
                                   bit-identical but measured slower than n one-kernel frames on scenes traversed through L1 (up to
                                   29 % on ShaderBalls, DESIGN.md section 4); 0 and 2 run n frames of rt_integrate's schedule */
    RT_OPT_PRESENT = 27,        /* multi-device contexts, rt_resolve: 0 (default) parallel read-back of every device's rows,
                                   1 gather to devices[0] over NVLink, resolve and read back there */
    RT_OPT_FRAME_THREADS = 28,  /* threads per CTA of the one-kernel frame: 0 (default) by partition size, else a multiple of 32 <= 1024 */
    RT_OPT_TOP_SMEM = 29        /* scenes whose traversal records do not fit shared memory: number of top-of-tree interior records
                                   (breadth-first, 64 B each, <= 640 = 40 KB) that every traversal CTA stages with one TMA bulk copy;
                                   0 (default) = none.  Results are bit-identical */
} RtOption;

#define RT_MAX_BOUNCES 255u     /* bounce index range supported per frame (reference GUI: 0..5) */
#define RT_MAX_REGEN_SAMPLES (1u << 24)   /* n_samples limit of rt_integrate_samples on the regenerating kernel (RT_OPT_FRAME_KERNEL 1) */

/* Per-bounce device counters of the last rt_integrate / rt_integrate_samples call (index = bounce, 0..max_bounces); a
 * multi-sample call returns the element-wise sums over its samples. */
typedef struct RtFrameStats {
    uint32_t n_ext[RT_MAX_BOUNCES + 1];        /* rays entering closest-hit traversal (ray_counter, trace_bvh.cl:116) */
    uint32_t n_miss[RT_MAX_BOUNCES + 1];
    uint32_t n_emissive_hits[RT_MAX_BOUNCES + 1];
    uint32_t n_shadow[RT_MAX_BOUNCES + 1];     /* shadow rays spawned (shadow_ray_counter, hit_surface.cl:138) */
    uint32_t n_cont[RT_MAX_BOUNCES + 1];       /* continuation rays spawned (hit_surface.cl:173)   */
    uint32_t n_unoccluded[RT_MAX_BOUNCES + 1];
    uint64_t nodes_ext[RT_MAX_BOUNCES + 1];    /* only with RT_OPT_COUNT_TRAVERSAL: reference-order node visits */
    uint64_t tris_ext[RT_MAX_BOUNCES + 1];
    uint64_t nodes_shadow[RT_MAX_BOUNCES + 1];
    uint64_t tris_shadow[RT_MAX_BOUNCES + 1];
} RtFrameStats;

/* Kernel classes for rt_kernel_times (RT_OPT_KERNEL_TIMING). */
typedef enum RtKernelClass {
    RT_K_RAYGEN = 0, RT_K_INTERSECT = 1, RT_K_MISS = 2, RT_K_HIT = 3, RT_K_INTERSECT_SHADOW = 4,
    RT_K_ACCUMULATE = 5, RT_K_EXTEND_SHADE = 6, RT_K_SHADOW_ACCUMULATE = 7, RT_K_RESOLVE = 8,
    RT_K_AOV = 9, RT_K_MISC = 10, RT_K_TRACE_CLOSEST = 11, RT_K_SHADE_QUEUES = 12, RT_K_TRACE_BOTH = 13,
    RT_K_CLASS_COUNT = 14
} RtKernelClass;

/* ---- lifetime ------------------------------------------------------------------ */
/* Replaces CLContext ctor + CLPathTraceIntegrator ctor (cl_context.cpp:47-94,
 * cl_pt_integrator.cpp:188-259): binds CUDA device `device`, allocates every per-pixel
 * buffer for a width x height render.  Fails with RT_ERR_NO_DEVICE if there is no GPU. */
int rt_create(uint32_t width, uint32_t height, int device, rt_ctx** out_ctx);
/* One context over several devices of the node — replaces CLContext's device enumeration
 * (gpu_wrappers/cl_context.cpp:64-89, where the reference lists every device and uses one): devices[i] renders
 * rank i of an n-way scanline partition (row y -> device y % n), scene replicated.  The caller stays
 * single-threaded; every call below fans out to the devices, which work concurrently (all steps are
 * asynchronous enqueues).  rt_resolve presents the WHOLE image: by default every device copies its rows
 * into the caller's image over its own PCIe link (page-lock it with rt_host_register); with
 * RT_OPT_PRESENT = 1 the radiance slabs are first gathered to devices[0] over NVLink (rt_gather_radiance,
 * the frame's one collective) and resolved there.  The stepwise taps (rt_read_hits, rt_read_rays), raw device
 * pointers and the temporal denoiser are single-device only.  n_devices == 1 is rt_create. */
int rt_create_multi(uint32_t width, uint32_t height, const int* devices, uint32_t n_devices, rt_ctx** out_ctx);
int rt_device_count(int* out_count);
int rt_destroy(rt_ctx* ctx);
/* Last error text of this context (ctx == NULL: of the last failed rt_create). */
const char* rt_last_error(const rt_ctx* ctx);

/* Multi-GPU image partition (new capability; the reference is single-device,
 * cl_context.cpp:64,86,89): this context renders only the scanlines y with
 * y % world == rank.  pixel_idx stays global, so RNG and results are unchanged.
 * Must be called before the first frame; (0,1) = whole image. */
int rt_set_partition(rt_ctx* ctx, uint32_t rank, uint32_t world);

/* ---- Integrator public interface ------------------------------------------------ */
int rt_upload_scene(rt_ctx* ctx, const RtSceneDesc* scene);     /* UploadGPUData, cl_pt_integrator.cpp:373-456 */
int rt_set_camera(rt_ctx* ctx, const RtCamera* camera);         /* SetCameraData,  cl_pt_integrator.cpp:365-371 */
int rt_set_option(rt_ctx* ctx, int key, uint32_t value);
/* The three tables of the blue-noise sampler (SamplerType::kBlueNoise, kernels/common/sampling.h:40-61).  The OpenCL
 * backend creates its buffers from the arrays of utils/blue_noise_sampler.hpp (cl_pt_integrator.cpp:222-235); the
 * caller passes the same arrays here: sobol_256spp_256d[RT_BN_SOBOL_COUNT], scramblingTile[RT_BN_TILE_COUNT],
 * rankingTile[RT_BN_TILE_COUNT].  Copied; ranking entries must lie in 0..255 (they are XORed into a sobol row index).
 * One deviation is defined here: the reference indexes rankingTile with the un-wrapped sample dimension
 * (sampling.h:50), which reads up to 247 entries past the end of the table for the last tile pixels once the dimension
 * exceeds 7 (undefined in the reference); such reads return 0. */
int rt_upload_sampler_tables(rt_ctx* ctx, const int32_t* sobol_256spp_256d, const int32_t* scrambling_tile, const int32_t* ranking_tile);

/* ---- Integrator protected steps, one call per virtual (integrator.hpp:55-71), same
 *      order contract as Integrator::Integrate (integrator.cpp:27-59) ----------------- */
int rt_reset(rt_ctx* ctx);                                      /* Reset: sample counter = 0 (unless denoiser), radiance = 0 */
int rt_advance_sample_count(rt_ctx* ctx);                       /* AdvanceSampleCount */
int rt_generate_rays(rt_ctx* ctx);                              /* GenerateRays   -> raygeneration.cl:65-139 */
int rt_intersect(rt_ctx* ctx, uint32_t bounce);                 /* IntersectRays  -> trace_bvh.cl:99-211 */
int rt_compute_aovs(rt_ctx* ctx);                               /* ComputeAOVs    -> aov.cl:44-110 (done inside the bounce-0 shading pass) */
int rt_shade_miss(rt_ctx* ctx, uint32_t bounce);                /* ShadeMissedRays -> miss.cl:41-77 */
int rt_clear_outgoing_counter(rt_ctx* ctx, uint32_t bounce);    /* ClearOutgoingRayCounter (counters are per bounce here: no-op) */
int rt_clear_shadow_counter(rt_ctx* ctx);                       /* ClearShadowRayCounter   (no-op, same reason) */
int rt_shade_hits(rt_ctx* ctx, uint32_t bounce);                /* ShadeSurfaceHits -> hit_surface.cl:30-186 */
int rt_intersect_shadow(rt_ctx* ctx);                           /* IntersectShadowRays -> trace_bvh.cl -D SHADOW_RAYS */
int rt_accumulate_direct(rt_ctx* ctx);                          /* AccumulateDirectSamples -> accumulate_direct_samples.cl:27-53 */
int rt_denoise(rt_ctx* ctx);                                    /* Denoise -> denoiser.cl:27-79 */
int rt_copy_history(rt_ctx* ctx);                               /* CopyHistoryBuffers, cl_pt_integrator.cpp:670-675 */
/* ResolveRadiance (resolve_radiance.cl:31-86) into a HOST RGBA32F image of width*height float4 (full image
 * rows; rows of other ranks are left untouched); dst may be NULL to resolve on the device only.  Blocks
 * (the reference's only Finish(), cl_pt_integrator.cpp:677-684). */
int rt_resolve(rt_ctx* ctx, float* dst_rgba);
/* Multi-device contexts: copies every device's radiance slab to devices[0] over NVLink (peer copies on the
 * devices' own streams; devices[0]'s stream waits for them) — the single collective of the frame. */
int rt_gather_radiance(rt_ctx* ctx);
/* Page-lock / release a caller-owned host buffer (the image given to rt_resolve) so that device->host copies into
 * it are asynchronous and the devices of a multi-device context read back in parallel. */
int rt_host_register(void* ptr, uint64_t bytes);
int rt_host_unregister(void* ptr);

/* Fused gather over peer memory — the frame's one collective done by the frame kernel itself (new capability).  The presenting
 * rank allocates a buffer of `world` slabs (stride = rows_max * width * 16 bytes, the layout rt_resolve_gathered reads) followed
 * by one completion flag per rank (rt_gather_buffer); every rank points its context at it (rt_set_gather_target: the owner with
 * its own pointer, ranks in other processes with the mapping rt_ipc_open returns for the 64-byte handle of rt_ipc_export, contexts
 * of a multi-device context through peer access — RT_OPT_PRESENT 1 does all of this).  From then on rt_integrate also delivers the
 * frame: the one-kernel frame stores a pixel's radiance into its rank's slab over NVLink the moment the pixel's path ends (the
 * transfer is spread over the frame), the per-phase schedule copies its slab at the end; then the rank's flag is set to its frame
 * number.  rt_gather_wait on the presenting context makes its stream wait for all flags; rt_resolve_gathered(buffer, stride)
 * presents. */
int rt_gather_buffer(rt_ctx* ctx, void** dev_ptr, uint64_t* stride_bytes, uint64_t* total_bytes);
int rt_ipc_export(const void* dev_ptr, void* handle64);
int rt_ipc_open(rt_ctx* ctx, const void* handle64, void** dev_ptr);
int rt_set_gather_target(rt_ctx* ctx, void* base, uint64_t stride_bytes);
int rt_gather_wait(rt_ctx* ctx);

/* Parity tap for include/rt_math.h (the elementary functions shared with the oracle): out[i] = f(a[i], b[i]) evaluated on
 * `device`; host pointers, blocking.  fn: 0 sin, 1 cos, 2 tan, 3 atan2(a, b), 4 acos, 5 pow(a, b), 6 fmin, 7 fmax,
 * 8 1 / sqrt(a), 9 a / b, 10 rt_expf(a). */
int rt_math_eval(int device, int fn, const float* a, const float* b, float* out, uint64_t n);

/* Pipelined read-back for frame loops: resolve on the render stream, device->host copy on a second stream (overlaps the
 * next frame's kernels).  dst must stay untouched until rt_resolve_wait() returns. */
int rt_resolve_async(rt_ctx* ctx, float* dst_rgba);
int rt_resolve_wait(rt_ctx* ctx);

/* Multi-GPU presentation on the rank that gathered the frame (new capability; SURVEY 8e: the resolve reads through the
 * scanline map).  `slabs` is a DEVICE pointer on this context's GPU to `world` radiance slabs, rank r's at
 * slabs + r * slab_stride_bytes, each holding that rank's rows (its local row k is image row r + k * world) as
 * width float4 per row — the layout rt_radiance_device_ptr exposes and the NCCL gather delivers.  Resolves the
 * shaded colour of the WHOLE width x height image (resolve_radiance.cl:80-84: radiance / sample_count, x/(1+x),
 * alpha 1) on the render stream and copies it to dst_rgba.  rt_resolve_gathered blocks; the _async variant copies on
 * the read-back stream like rt_resolve_async (rt_resolve_wait).  AOV views and the denoiser are single-GPU only. */
int rt_resolve_gathered(rt_ctx* ctx, const void* slabs, uint64_t slab_stride_bytes, float* dst_rgba);
int rt_resolve_gathered_async(rt_ctx* ctx, const void* slabs, uint64_t slab_stride_bytes, float* dst_rgba);

/* ---- fused steps (same per-pixel results, fewer passes over HBM) ------------------ */
int rt_extend_shade(rt_ctx* ctx, uint32_t bounce);              /* IntersectRays + ShadeMissedRays + ShadeSurfaceHits */
int rt_shadow_accumulate(rt_ctx* ctx, uint32_t bounce);         /* IntersectShadowRays + AccumulateDirectSamples */
/* With RT_OPT_OVERLAP = 2 (default) the work of rt_shadow_accumulate(b) is submitted with the traversal of the next
 * rt_extend_shade, or by the next call that depends on it: every step / resolve / read / rt_sync /
 * rt_advance_sample_count does that, so the device state after each call is what in-order execution gives. */
/* GenerateRays + (max_bounces+1) x {extend_shade, shadow_accumulate} + AdvanceSampleCount, i.e. the body of
 * Integrator::Integrate between Reset() and ResolveRadiance(). */
int rt_integrate(rt_ctx* ctx, uint32_t max_bounces);
/* n_samples consecutive frames of rt_integrate(ctx, max_bounces) in one call.  The results are bit-identical to calling
 * rt_integrate n_samples times: the radiance of every pixel, the sample count (n_samples higher), the AOV buffers (the last
 * sample's values), the resolved image of every view and, once the call completes, the fused-gather slab.  rt_read_frame_stats
 * returns the per-bounce counters summed over the call's samples.  With a gather target set, the completion flag is signalled
 * once per call.
 * With RT_OPT_FRAME_KERNEL = 1 (and neither RT_OPT_KERNEL_TIMING nor RT_OPT_COUNT_TRAVERSAL) the call is ONE launch of the
 * regenerating frame kernel: when a pixel's path ends, its CTA starts that pixel's next sample in the next traversal round.  It
 * carries a path's sample offset in 24 bits: n_samples > RT_MAX_REGEN_SAMPLES is RT_ERR_INVALID_ARGUMENT there.
 * Otherwise, the default included, the frame rt_integrate would run is run n_samples times (measured on H100, the regenerating
 * kernel is not faster at any partition size; DESIGN.md section 4); the fused gather is pushed by the last frame only.
 * n_samples == 1 is rt_integrate.  The stepwise taps (rt_read_rays, rt_read_hits) find no rays of a multi-sample call that ran
 * the one-kernel frame, and the last frame's rays after one that ran the per-phase frames.
 * Errors, checked before anything is enqueued: RT_ERR_INVALID_ARGUMENT for n_samples == 0, a sample count that would wrap
 * uint32_t, or max_bounces > RT_MAX_BOUNCES; RT_ERR_UNSUPPORTED for n_samples > 1 with the
 * temporal denoiser on (it runs once per sample).  Multi-device contexts fan out like rt_integrate. */
int rt_integrate_samples(rt_ctx* ctx, uint32_t max_bounces, uint32_t n_samples);

/* ---- adaptive sampling (new capability) ----------------------------------------------------------------------------------
 * Stop tracing pixels whose image has settled.  While it is on, a frame traces primary rays only for the ACTIVE local pixels; a
 * path is otherwise unchanged (its sample index is still the context's sample count), so a pixel that stops after n samples holds
 * exactly the radiance and AOVs that n frames give it.  After every sample (rt_advance_sample_count, every frame of rt_integrate
 * and rt_integrate_samples) each active pixel, now at n samples, updates its estimate of the standard error of its resolved
 * (Reinhard) luminance and stops when
 *     Y = luma(radiance) = (x * 0.299f + y * 0.587f) + z * 0.114f (float), then in double:
 *     y = Y - Y_prev;  Q += y * y;  Y_prev = Y;  m = Y / n;  v = max(Q / n - m * m, 0);  e = sqrt(v / n) / ((1 + m) * (1 + m))
 *     stop iff n >= min_samples and e <= max_error                         (NaN never stops)
 * max_error is in display units (0.002 is about half an 8-bit step).  A stopped pixel keeps its sample count, radiance and AOVs and
 * stays stopped until the next rt_reset.  After an rt_reset, an active pixel's sample count always equals rt_read_sample_count.
 *
 * max_error > 0 (finite) and min_samples >= 2 turn it on; max_error == 0 turns it off (min_samples is ignored); anything else is
 * RT_ERR_INVALID_ARGUMENT.  The setting takes effect at the next rt_reset (like the Integrator's SetMaxBounces -> RequestReset);
 * until then the previous one stays.  rt_reset with it on makes every local pixel active with a sample count of 0; so does
 * rt_set_partition, which clears the radiance but not the context's sample count (the sample index continues; call rt_reset to
 * start over, after which every active pixel's count equals the sample count again).  The per-pixel state (about 20 bytes per pixel) exists only while it is on.
 * With it on: rt_resolve / rt_resolve_async divide the shaded colour by each pixel's own sample count (the AOV views are
 * unchanged); n_ext[0] of rt_read_frame_stats counts the pixels active at the start of the frame; rt_integrate_samples always
 * runs n frames of rt_integrate's schedule (never the regenerating kernel).  Multi-device contexts fan out: every device decides
 * for its own rows, with the same result as one device.
 * RT_ERR_UNSUPPORTED, whichever of the two calls comes second: the temporal denoiser, a fused-gather target
 * (rt_set_gather_target), RT_OPT_PRESENT 1 on a multi-device context, and rt_resolve_gathered[_async]. */
int rt_set_adaptive_sampling(rt_ctx* ctx, float max_error, uint32_t min_samples);
/* Every local pixel's sample count as a full width*height uint32 image (rows of other ranks untouched).  Off: sample_count everywhere. */
int rt_read_pixel_samples(rt_ctx* ctx, uint32_t* counts);
/* Pixels that will trace the next sample (blocking; summed over the devices of a multi-device context).  Off: the local pixel count. */
int rt_read_active_pixels(rt_ctx* ctx, uint32_t* n_active);

/* ---- spatial denoiser (new capability) -----------------------------------------------------------------------------------
 * An edge-avoiding a-trous wavelet filter (Dammertz et al. 2010) on the shaded-colour view of rt_resolve / rt_resolve_async (the
 * host image and the device resolve target), guided by the bounce-0 AOVs of the last frame rendered.  The accumulation is never
 * touched: radiance, sample counts, AOVs, frame statistics and the AOV views 1-4 are what they are with the filter off.
 * iterations 0 = off; 1..5 passes with tap spacing s = 2^i, i = 0 .. iterations-1.  The input of pass 0 is the image k_resolve
 * produces (Reinhard colour in display units, from radiance / sample count, the per-pixel counts of adaptive sampling, or the
 * radiance alone under the temporal denoiser); pass i maps image c to image c', all in float (no contraction):
 *     kc = 1 / (sigma_color * sigma_color) * 2^i,  kn = 1 / (sigma_normal * sigma_normal),  kz = 1 / (sigma_depth * z_p)   (0 if sigma 0)
 *     centre p: if c_p is not finite, the colour term uses c_p = 0 and kc = 0 for this pixel
 *     for ty = -2..2, tx = -2..2 (row by row): q = p + s * (tx, ty); skip q outside the image and q whose colour is not finite;
 *         dc = (dr*dr + dg*dg) + db*db of c_p - c_q;  dn = the same of n_p - n_q (shading normal xyz);  dz = |z_p - z_q| (depth)
 *         term(d, k) = (k > 0 and d > 0) ? d * k : 0;   D = (term(dc, kc) + term(dn, kn)) + term(dz, kz)
 *         w = (h[ty] * h[tx]) * rt_expf(-D),  h = (1/16, 1/4, 3/8, 1/4, 1/16)
 *         if w > 0: W += w; S += w * c_q (per channel)
 *     c'_p = S / W per channel if W > 0, else c_p; alpha 1.
 * A sigma of 0 drops its term; a NaN or inf pixel never spreads, and a pixel with no usable tap keeps its value.
 * Turning the filter on makes frames produce the AOVs (as an AOV view or the temporal denoiser do; the captured frame graph is
 * re-captured).  rt_resolve / rt_resolve_async return RT_ERR_NOT_READY until a frame has written every local pixel's AOVs with the
 * filter (or another AOV consumer) on: after turning it on, and, with adaptive sampling, until the first frame after an rt_reset.
 * Two colour planes and one guide record (16 bytes each per pixel) are allocated while it is on.  Its launches count under
 * RT_K_RESOLVE.  RT_ERR_INVALID_ARGUMENT: iterations > 5, a negative or non-finite sigma.  RT_ERR_UNSUPPORTED, whichever call comes
 * second: a multi-device context, rt_set_partition with world > 1, and rt_resolve_gathered[_async]. */
int rt_set_spatial_denoiser(rt_ctx* ctx, uint32_t iterations, float sigma_color, float sigma_normal, float sigma_depth);

/* ---- parity / measurement taps ---------------------------------------------------- */
int rt_sync(rt_ctx* ctx);
/* Hits of the rays currently in the incoming queue of `bounce` after rt_intersect(bounce): n = live rays;
 * hits[i] and pixel_indices[i] for ray slot i (caller provides room for rt_local_pixel_count entries). */
int rt_read_hits(rt_ctx* ctx, uint32_t bounce, RtHit* hits, uint32_t* pixel_indices, uint32_t* n_out);
/* Incoming rays of `bounce` (reference Ray layout) + pixel indices. */
int rt_read_rays(rt_ctx* ctx, uint32_t bounce, RtRay* rays, uint32_t* pixel_indices, uint32_t* n_out);
/* Radiance accumulator as a full width*height float4 image (rows owned by other ranks untouched). */
int rt_read_radiance(rt_ctx* ctx, float* dst_rgba);
int rt_read_frame_stats(rt_ctx* ctx, RtFrameStats* out);
int rt_read_sample_count(rt_ctx* ctx, uint32_t* out);
/* AOV buffers of the local pixels as full-image arrays: albedo float4, depth float, normal float4, velocity float2 */
int rt_read_aovs(rt_ctx* ctx, float* albedo_rgba, float* depth, float* normal_rgba, float* velocity_xy);
/* Accumulated milliseconds and launch counts per RtKernelClass since the last call (RT_OPT_KERNEL_TIMING). */
int rt_kernel_times(rt_ctx* ctx, float* ms_per_class, uint32_t* launches_per_class);
/* Number of kernels launched by this context since creation. */
int rt_launch_count(rt_ctx* ctx, uint64_t* out);

/* Device-side access for the multi-GPU gather (torch.distributed/NCCL works on device pointers):
 * the local radiance slab is local_rows x width float4, local row r = image row rank + r*world. */
int rt_local_pixel_count(rt_ctx* ctx, uint32_t* out);
int rt_radiance_device_ptr(rt_ctx* ctx, void** out_ptr, uint64_t* out_bytes);
/* The render stream.  Work a caller enqueues on it sees the complete frame after rt_integrate or
 * rt_advance_sample_count (which close the frame in stream order). */
int rt_stream_handle(rt_ctx* ctx, void** out_cuda_stream);

#ifdef __cplusplus
}
#endif

#endif /* RT_B200_H */
