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
    const RtTexture* textures;          uint64_t n_textures;       /* each RtTexture: data_start + width * height <= 2^31 (texels
                                                                      are indexed in int); rt_upload_scene refuses any other */
    const uint32_t* texture_data;       uint64_t n_texture_data;
    const uint32_t* emissive_indices;   uint64_t n_emissive;       /* triangle ids; sampled only with RT_OPT_EMITTER_SAMPLING 1 */
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
    RT_OPT_FRAME_KERNEL = 26,   /* how rt_integrate, and every frame of rt_integrate_samples, runs a frame.  1: ONE persistent kernel
                                   in which every CTA is an independent wavefront over its own pixels (queue cursors in shared
                                   memory, no global atomics, no launch boundaries); 0: one kernel per phase (graph replay / PDL
                                   chain as configured above); 2 (default): the one-kernel frame for partitions of up to 7168
                                   pixels per SM (0.95 M pixels, under half a 1080p frame, on an H100's 132 SMs), per-phase
                                   kernels for larger ones.  Results are bit-identical */
    RT_OPT_PRESENT = 27,        /* multi-device contexts, rt_resolve: 0 (default) parallel read-back of every device's rows,
                                   1 gather to devices[0] over NVLink, resolve and read back there */
    RT_OPT_FRAME_THREADS = 28,  /* threads per CTA of the one-kernel frame: 0 (default) by partition size, else a multiple of 32 <= 1024 */
    RT_OPT_TOP_SMEM = 29,       /* scenes whose traversal records do not fit shared memory: number of top-of-tree interior records
                                   (breadth-first, 64 B each, <= 640 = 40 KB) that every traversal CTA stages with one TMA bulk copy;
                                   0 (default) = none.  Results are bit-identical */
    RT_OPT_EMITTER_SAMPLING = 30, /* 0 (default): emissive triangles add light only when a BSDF-sampled ray hits them; 1: next-event
                                   estimation on the emissive triangles too, combined with BSDF sampling by MIS (the rule is stated
                                   in the emitter-sampling block below; the image converges to the same expectation) */
    RT_OPT_ENV_SAMPLING = 31,   /* 0 (default): the environment map adds light only when a BSDF-sampled ray misses; 1: next-event
                                   estimation on the environment map too, combined with BSDF sampling by MIS (the environment-sampling
                                   block below; the image converges to the same expectation) */
    RT_OPT_OCTANT_BVH = 32,     /* 1 (default): a scene staged whole into shared memory (RT_OPT_SMEM_BVH) whose interior records fit
                                   eight more times within the same 40 KB is traversed through per-direction-octant copies of
                                   the records that every CTA builds after staging: the box test needs no pairwise min/max and
                                   no near/far selection (the per-phase kernels; the one-kernel frame keeps the canonical records).
                                   0: the canonical records only.  Results are bit-identical */
    RT_OPT_OBJECT_MOTION = 33   /* 0 (default): the motion-vector AOV follows the camera only (as the reference's); 1: it also follows
                                   rt_update_triangles* (the object-motion block below) */
} RtOption;

#define RT_MAX_BOUNCES 255u     /* bounce index range supported per frame (reference GUI: 0..5) */

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
 * The frame rt_integrate would run is run n_samples times; the fused gather is pushed by the last frame only.
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
 * unchanged); n_ext[0] of rt_read_frame_stats counts the pixels active at the start of the frame.  Multi-device contexts fan out:
 * every device decides for its own rows, with the same result as one device.
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

/* ---- emitter sampling (new capability): rt_set_option(ctx, RT_OPT_EMITTER_SAMPLING, 1) ------------------------------------
 * Next-event estimation on the emissive triangles, combined with BSDF sampling by multiple importance sampling (power heuristic).
 * The estimator has the expectation of the option off; only the noise changes.  All float, no contraction, in the order written.
 * Emitter table (raytracing_b200/csrc/rt_emitters.h), a pure function of the upload: the emitters are emissive_indices (leaf-ordered
 * triangle ids, upload order); A_t = 0.5f * sqrtf((cx*cx + cy*cy) + cz*cz), c = cross(p2 - p1, p3 - p1); w_t = A_t * luma(E_t), E_t the
 * material's constant emission, luma = (r*0.299f + g*0.587f) + b*0.114f, non-finite or negative w_t -> 0; cdf[i] = S_i / S_n (running
 * float sum in list order), cdf[n-1] = 1; pmf_i = cdf[i] - cdf[i-1]; pdfA[t] = (P_e * pmf_i) / A_t where pmf_i > 0, else 0 (and 0 off
 * the list).  P_e = 0 if S_n is not finite and > 0 or in white-furnace mode (the frame is then bit-identical to the option off);
 * 1 if every analytic light has zero radiance; else 0.5.  (Those are the default weights of rt_set_light_selection; the light-kind
 * block below states P_e and the analytic divisor for any weights and with environment sampling.)
 * At a hit of bounce b < max_bounces (the last max_bounces passed to rt_integrate / rt_integrate_samples; the stepwise steps, which
 * are not told max_bounces, use the value of the most recent such call, RT_MAX_BOUNCES before any), with kRandom draws r_k = hash(dimension 0x10000 + 4*b + k) whatever
 * the sampler:
 *     emitter iff P_e == 1 or r_0 < P_e;  else the analytic light sample of the option off, divided by (1 - P_e)
 *     emitter: i = first entry with cdf[i] > min(r_1, 0x1.fffffep-1), t = list[i]; s = sqrtf(r_2);
 *              y = (p1*(1-s) + p2*(s*(1-r_3))) + p3*(s*r_3); Le = emission of t's material at the same barycentrics' uv;
 *              o = position + geometry_normal * EPS; v = y - o; d2 = dot(v, v); d = sqrtf(d2); w = normalize(v);
 *              cos_e = -dot(w, n_t) (geometric normal of t); nothing if cos_e <= 0;  p_l = pdfA[t] * d2 / cos_e;
 *              g, p_b = the BSDF that sample_bxdf integrates and its non-delta lobe density for w (rt_device.cuh bxdf_eval_sampled;
 *              0 for pass-through materials, no specular term for alpha <= 1e-4 or where the specular sampler has no density:
 *              n.h <= 0 or h.o <= 0, h = normalize(i + w));
 *              sample = ((T * g) * Le) * (mis(p_l, p_b) / p_l), mis(p, q) = 1 / (1 + (q/p)^2) (NaN -> 0); shadow ray from o along w,
 *              t_max = 0.999f * d, spawned iff p_l > 0 and dot(sample, sample) > 0
 *     the continuation ray carries p_b of its direction (0 after a delta lobe: a pass-through or an alpha <= 1e-4 specular sample)
 * At a BSDF hit of an emitter with carried p_b > 0 and pdfA[prim] > 0: emission * mis(p_b, p_l), p_l = pdfA[prim] * dot(x - o, x - o) /
 * -dot(dir, n_prim) (x the hit, o the ray's origin); otherwise the emission of the option off.  At b = max_bounces nothing changes.
 * With the option on, an emissive index >= n_triangles or listed twice is RT_ERR_INVALID_ARGUMENT (at rt_upload_scene, or at
 * rt_set_option when the scene is already uploaded); values other than 0 and 1 too.  The setting applies from the next frame and keeps
 * the accumulation.  Stepwise callers: a frame driven through the step calls samples emitters at every bounce below that value, so
 * a caller whose last step bounce is below it gets emitter light from its last vertex, which BSDF sampling never adds (its
 * continuation is not traced): its image converges to a brighter value than with the option off.  Call rt_integrate (or
 * rt_integrate_samples) with the same max_bounces once before driving the steps.
 * Device memory: 4 B per triangle and 8 B per emitter while it is on. */

/* ---- environment sampling (new capability): rt_set_option(ctx, RT_OPT_ENV_SAMPLING, 1) --------------------------------------
 * Next-event estimation on the environment map, combined with BSDF sampling by MIS (power heuristic, as for emitters); same
 * expectation as the option off.  All float, no contraction, in the order written; sin / cos / atan2 / acos are rt_math.h's.
 * Environment table (raytracing_b200/csrc/rt_envmap.h), a pure function of the uploaded image (w x h texels) and the flags:
 *     W_ij = luma(texel i of row j) * sin(pi * ((j + 0.5f) / h)), a luma that is not finite and >= 0 counting as 0;
 *     marginal CDF over the row sums and one conditional CDF per row, running float sums, last entry 1;
 *     T = the sum of the row sums; p_uv(i, j) = ((w * h) * W_ij) / T; table[i, j] = P_v * p_uv(i, j).
 *     Active iff T is finite and > 0, the option is on and white-furnace mode is off; else the frame is that of the option off.
 * p_v(dir) = table[cell of dir] / (2pi^2 * sqrtf(max(1 - z*z, 0))), the cell holding sample_sky's texture coordinates
 * (cx = (atan2(x, y) + pi) / 2pi, cy = acos(z) / pi, wrapped to [0, 1), times w / h, truncated); one function for both sides.
 * At a hit of bounce b < max_bounces (as for emitters) that draws the environment kind (below):
 *     row j = first marginal entry > min(r_1, 0x1.fffffep-1), column i = first entry of row j > min(r_2, 0x1.fffffep-1), r_1..r_3 the
 *     emitter draws of the bounce and r_4 = hash(dimension 0x20000 + b) (kRandom whatever the sampler); u = (i + r_3) / w,
 *     v = (j + r_4) / h; phi = u * 2pi - pi, theta = v * pi; dir = (sin theta sin phi, sin theta cos phi, cos theta);
 *     Le = sample_sky(dir) (what a miss adds); g, p_b as for emitters; sample = ((T * g) * Le) * (mis(p_v, p_b) / p_v) with
 *     p_v = p_v(dir); shadow ray from position + geometry_normal * EPS along dir, t_max = RT_MAX_RENDER_DIST (unoccluded exactly
 *     where a continuation ray would miss), spawned iff p_v > 0 and dot(sample, sample) > 0.
 * A continuation ray that misses with carried p_b > 0 while the table is active adds (sky * T) * mis(p_b, p_v(dir)); every other miss
 * (primary rays, after a delta lobe, with the table inactive) is unchanged.  Values other than 0 and 1 are RT_ERR_INVALID_ARGUMENT.
 * The setting applies from the next frame and keeps the accumulation.  Device memory while it is active: 8 B per texel + 4 B per row,
 * built from the device copy of the image.  As for emitters, the stepwise steps use the last max_bounces, and rt_integrate_samples
 * runs n frames of rt_integrate's schedule.
 *
 * ---- light-kind selection: rt_set_light_selection(ctx, analytic, emitters, environment) ------------------------------------------
 * Relative weights of the light kind drawn at each vertex while emitter or environment sampling is active; default (1, 1, 1).
 * A kind's weight counts only while the kind is active (analytic: an analytic light has non-zero radiance; emitters: the emitter
 * table is active; environment: the environment table is active), else it is 0: w_a, w_e, w_v.  S = (w_a + w_e) + w_v,
 * P_e = w_e / S, P_v = w_v / S (pdfA of the emitter table uses this P_e).  With r_0 = hash(dimension 0x10000 + 4*b):
 *     emitter iff P_e >= 1 or r_0 < P_e;  else environment iff the environment table is active and (w_a == 0 or r_0 < P_e + P_v);
 *     else the analytic light sample of the options off, divided by (1 - (P_e + P_v)).
 * With RT_OPT_ENV_SAMPLING 0 and the default weights this is the emitter rule above bit for bit (P_e = 0.5 or 1); with both options
 * off nothing is drawn and the frame is the reference's.  A weight that is not finite or <= 0, or a sum that is not finite, is
 * RT_ERR_INVALID_ARGUMENT (a zero weight on an active kind would bias the estimator).  Applies from the next frame, keeps the
 * accumulation, and works with either option alone. */
int rt_set_light_selection(rt_ctx* ctx, float analytic, float emitters, float environment);

/* ---- geometry updates (new capability): animated geometry without a BVH rebuild ------------------------------------------------
 * triangles[i] replaces uploaded triangle i, in the leaf order rt_upload_scene received; n_triangles must equal the upload's count.
 * Positions, normals and texcoords are taken from the new array; mtlIndex and the padding words are not read (materials and the
 * emitter list stay those of the upload).  Every derived record becomes what rt_upload_scene derives from the new array
 * (rt_bvh_layout.h): wtris p1 / e1 / e2, tri_shade, tris_ref (the RtFloat3 .w words included); the end-of-leaf flags are kept.
 * The BVH keeps its topology and is refit: min(a, b) = (b < a) ? b : a and max(a, b) = (a < b) ? b : a (std::min / std::max as the
 * reference's Bounds3 uses them), per component.  A leaf box starts at min = FLT_MAX, max = -FLT_MAX and folds, for each of its
 * triangles in leaf order, tb = Union(Bounds3(p1, p2), p3) (Triangle::GetBounds) by box = Union(box, tb); an interior box is
 * Union(first child, second child).  The same boxes go into the nodes (xyz of bounds_min / bounds_max; their .w words, the offsets,
 * counts, split axes and padding are kept) and into the child slots of the parent's traversal record.  With unchanged positions
 * the boxes equal the builder's as float values (it folds over primitives rather than children, so only the sign of a zero can
 * differ, which no comparison of the traversal can tell apart).  Non-finite coordinates are not rejected (rt_upload_scene does not
 * reject them either); the comparisons above define their boxes too.
 * Ordering: the update is enqueued on the render stream after everything submitted before it (a shadow pass deferred by
 * RT_OPT_OVERLAP 2 is launched first, the second stream of RT_OPT_OVERLAP 1 is joined) and is asynchronous; the next frame sees the
 * new geometry.  The buffers keep their sizes and addresses, so a captured frame graph stays valid.  The accumulation is kept, as
 * for a camera move: call rt_reset.  Motion vectors stay camera-only (as in the reference) unless RT_OPT_OBJECT_MOTION is on (the
 * object-motion block below), which lets the velocity AOV and the temporal denoiser follow the update.  The sort-key origin of the sorted shading pass stays the upload's root-box centre (ray order, not results).
 * rt_update_triangles reads the caller's array before it returns, through a pinned staging buffer of at most 2 x 32 MB (allocated
 * at the first call) whose copies overlap the record kernel.  rt_update_triangles_device reads `device_triangles` (RtTriangle
 * layout, 16-byte aligned device memory of the context's device, else RT_ERR_INVALID_ARGUMENT) on the render stream: the caller
 * orders its producer before the call (rt_stream_handle) and keeps the buffer unchanged until the next blocking call.
 * Emitter sampling: while it is on, the emitter table's areas are rebuilt from the new positions (read back from the device), which
 * makes the call block; otherwise that happens when the option is turned on.  The environment table and the analytic lights are
 * unaffected.  The first update builds a refit map (parent and record slot per node, the leaf list, an arrival counter per node:
 * about 14 bytes per node, read from the device copy of the nodes, blocking) that lives until the next rt_upload_scene.
 * Errors: RT_ERR_NOT_READY before an upload; RT_ERR_INVALID_ARGUMENT for a count mismatch or a null pointer; RT_ERR_UNSUPPORTED for
 * rt_update_triangles_device on a multi-device context (rt_update_triangles fans out like rt_upload_scene).  The launches count
 * under RT_K_MISC (RT_OPT_KERNEL_TIMING) and in rt_launch_count. */
int rt_update_triangles(rt_ctx* ctx, const RtTriangle* triangles, uint64_t n_triangles);
int rt_update_triangles_device(rt_ctx* ctx, const void* device_triangles, uint64_t n_triangles);

/* ---- object motion vectors (new capability): rt_set_option(ctx, RT_OPT_OBJECT_MOTION, 1) ------------------------------------------
 * The velocity AOV of a bounce-0 hit follows the triangle's own motion as well as the camera's.  While the option is on, the context
 * keeps the previous positions Q[t] = (q1, q2, q3) of every triangle t, in upload (leaf) order:
 *     rt_upload_scene: Q = the uploaded positions;
 *     switching the option from 0 to 1 after an upload: Q = the current positions (those of the last update, if any);
 *     rt_update_triangles, rt_update_triangles_device: Q = every triangle's positions before the call, then the new ones are written
 *     (in render-stream order, like the update itself);
 *     unchanged by rt_rebuild_bvh, rt_rebuild_bvh_ploc, frames, rt_reset and camera changes (none of them moves a triangle).
 * This mirrors the camera rule, where the previous camera is that of the previous rt_set_camera call: an animation that updates
 * once per frame gets the motion of that frame; one that stops updating keeps the last update's motion until its next update.
 * A bounce-0 hit on triangle t at barycentrics (u, v), w0 = 1 - u - v, all float without contraction, in the order written:
 *     position = (p1 * w0 + p2 * u) + p3 * v;  prev = (q1 * w0 + q2 * u) + q3 * v;
 *     velocity = project_screen(position, camera) - project_screen(prev, previous camera)   (aov.cl's projection, as with it off)
 * With Q equal to the current positions, prev is position bit for bit and so is the velocity of the option off: turning the option on
 * changes no output until the next update.  Misses, the albedo, depth and normal AOVs, radiance, statistics and every other view
 * are unchanged; the temporal denoiser keeps its rule and reads these motion vectors; a pixel stopped by adaptive sampling keeps the
 * AOVs of its last traced sample.  Values other than 0 and 1 are RT_ERR_INVALID_ARGUMENT.
 * Device memory while the option is on and a scene is uploaded: 48 B per triangle (tris_ref's layout; 2.5 MB on CornellBox_Dragon,
 * 481 MB on Synthetic10M), allocated when the option is turned on after an upload or at an upload with it on, freed when it is
 * turned off.  If the allocation fails the call returns RT_ERR_CUDA and the option is off (an upload then leaves no scene).  Turning
 * the option on or off re-captures the frame graph; updates with it on move no buffer, so a captured graph stays valid.  An update
 * launches the same kernels with the option on (its record kernel also copies the old positions: about 96 B more per triangle).
 * Multi-device contexts fan out: each device keeps its own Q. */
/* Parity tap: the device's reference-layout nodes (n_nodes entries of the current tree: the upload's, or 2n - 1 after
 * rt_rebuild_bvh) and, if records != NULL, the traversal records
 * (16 floats per interior record, rt_bvh_layout.h; one zero record for a single-leaf tree); *n_records is set whenever n_records
 * != NULL (call with records == NULL to size the buffer).  Either pointer may be NULL.  Blocking.  Single-device contexts only. */
int rt_read_bvh(rt_ctx* ctx, RtLinearBVHNode* nodes, float* records, uint64_t* n_records);

/* ---- BVH rebuild (new capability): a fresh tree over the current triangles, built on the device ---------------------------------
 * Replaces the BVH by a linear BVH (one triangle per leaf, in Morton order) over the device copy of the positions: the upload's
 * triangles or those of the last rt_update_triangles*.  For geometry that has deformed far enough that a refit tree traces slowly
 * (DESIGN.md section 4 measures where that happens); nothing is copied from or to the host.  The rule, with n triangles and every
 * operation in float without contraction, in the order written:
 *  1. Key point s = (p1 + p2) + p3 per component.  The quantization box lo / hi of an axis is the min / max over the finite s of
 *     that axis (min and max are exact, so only the sign of a zero depends on the reduction order, which changes no code).
 *  2. Per axis: k = 1024.0f / (hi - lo) if hi > lo, else 0 (also when no s of the axis is finite); for a finite s, x = (s - lo) * k
 *     and q = 1023 if x >= 1023, trunc(x) if x > 0, else 0 (so a NaN x gives 0); a non-finite s gives q = 0.
 *  3. Code: bit j of qx goes to bit 3j + 2, of qy to 3j + 1, of qz to 3j (30 bits).  Key = (uint64(code) << 32) | triangle id; the
 *     keys are distinct, so their ascending order is unique.
 *  4. Topology: the binary radix tree of the sorted keys.  A range [a, b] of sorted keys with a < b splits after the unique i at
 *     which the highest bit h where key[a] and key[b] differ flips; the first child holds the lower keys.  Split axis: with
 *     m = h - 32, 2 - (m mod 3) if h >= 32, else 0 (equal codes, split by id).  Each level uses up at least one of the 30 + 31 key
 *     bits, so the depth is at most 62 levels (n < 2^31, the upload's limit), under the 64-entry traversal stack: nothing checks
 *     it at run time.
 *  5. Nodes in the reference layout, depth-first preorder (first child = node + 1, second child = `offset`): a leaf has offset =
 *     its triangle id and num_primitives_axis = 1 << 16; an interior node has offset = its second child and num_primitives_axis =
 *     its split axis; the .w words and the padding are 0; n = 1 gives a single leaf.  Triangles are not reordered, so primitive
 *     ids, emissive_indices, the leaf order rt_update_triangles expects and every AOV keep their meaning.  The boxes follow the
 *     refit rule of the geometry-update block exactly.
 *  6. The derived records are what rt_upload_scene derives from these nodes (rt_bvh_layout.h build_layout): the traversal
 *     records in its order (the first min(n - 1, 1024) interior nodes breadth-first, then the rest depth-first), the root
 *     reference and the breadth-first prefix length, and the wtris end-of-leaf flags, now all 1.  tris_ref, tri_shade and the
 *     materials are untouched.
 * Frames after a rebuild are those of the same triangles with these nodes uploaded; against the previous tree, results can differ
 * only where two triangles tie in t (the closest-hit traversal keeps the first found) or where a ray meets a triangle with a
 * non-finite coordinate (its test can report t = NaN, and what follows depends on the visiting order with any tree).  The accumulation is kept: call rt_reset
 * when the geometry moved.  The rebuild also builds the refit map, so a later rt_update_triangles* refits the rebuilt topology
 * without its blocking map build; rt_upload_scene returns to the uploaded tree.  State derived from the tree (shared-memory
 * staging of small trees, the RT_OPT_TOP_SMEM prefix) follows the new tree; the sort-key origin of the sorted shading pass stays
 * the upload's root-box centre, as after an update.  The light tables are unaffected (ids and positions do not change).
 * Ordering: enqueued on the render stream like an update (a deferred shadow pass is launched first, the second stream is joined).
 * The first rebuild after an upload replaces the nodes, records and refit map (2n - 1 nodes, max(n - 1, 1) records) and allocates
 * the build temporaries: it blocks, and the frame graph is re-captured.  Later rebuilds reuse all of them in place: they are
 * asynchronous and a captured frame graph stays valid.
 * Device memory while a rebuilt tree is live: nodes 48 B x (2n - 1) and records 64 B x (n - 1) in place of the upload's, the refit
 * map 12 B x (2n - 1) + 4 B x n, and temporaries of 32 B per triangle plus the radix sort's scratch.
 * n_nodes, if not NULL, is set to the new node count 2n - 1.  Multi-device contexts fan out: each device builds the same tree.
 * Errors: RT_ERR_NOT_READY before an upload.  The launches count under RT_K_MISC (RT_OPT_KERNEL_TIMING) and in rt_launch_count
 * (the radix sort counts as one). */
int rt_rebuild_bvh(rt_ctx* ctx, uint64_t* n_nodes);

/* ---- BVH rebuild at SAH quality (new capability): parallel locally-ordered clustering (PLOC), built on the device ---------------
 * Replaces the BVH, like rt_rebuild_bvh, by a tree over the device copy of the positions with one triangle per leaf, built by
 * PLOC (Meister & Bittner 2018): a slower build than rt_rebuild_bvh's, for a tree that traces about as fast as the SAH tree of
 * the upload (DESIGN.md section 4, "PLOC rebuild").  Which one pays off depends on how many frames the tree serves, which only
 * the caller knows.  The rule, with n triangles and every operation in float without contraction, in the order written; min and
 * max are the refit rule's, Union(A, B) is min(A.lo, B.lo), max(A.hi, B.hi) per component (order-sensitive for NaN and zeros):
 *  1. Initial clusters: the triangles in the ascending key order of rt_rebuild_bvh steps 1-3, each with the refit rule's leaf
 *     box of its triangle, at positions 0 .. c - 1 (c = n).
 *  2. Distance: A(lo, hi) = (ex*ey + ey*ez) + ez*ex with e = hi - lo, and A = +inf unless A >= 0 and finite (NaN, inf, inverted
 *     boxes).  For positions i < j, d(i, j) = d(j, i) = A(Union(box_i, box_j)), the lower position first.
 *  3. Nearest neighbour: nn(i) = the j != i in [i - R, i + R] with 0 <= j < c and the smallest d(i, j).  Ties go to the smaller
 *     gap |j - i|, then to the pair whose lower position is even, then to the smaller j.  (Ties to the smallest j alone would chain
 *     a run of equal boxes, such as coincident triangles, one merge per iteration and one level per triangle; this order pairs
 *     the run off in neighbours, halving it.)  R = RT_PLOC_RADIUS.
 *  4. Merge: i and j = nn(i) merge iff nn(j) = i.  The new cluster, an interior node, takes position min(i, j) with box
 *     Union(box_lower, box_higher); the other position is removed and the list compacted in order.  Steps 2-4 repeat until one
 *     cluster is left.  Distance and the tie order together order the pairs totally, so the first pair in that order is mutual:
 *     each iteration merges at least one pair.
 *  5. Each interior node (lower-position cluster L, higher H): cL = L.lo + L.hi, cH = H.lo + H.hi, delta_a = |cH_a - cL_a|; the
 *     axis starts at 0, becomes 1 if delta_1 > delta_axis, then 2 if delta_2 > delta_axis (NaN compares false); the first child
 *     is H iff cH_axis < cL_axis, else L.  The split axis is that axis.
 *  6. Nodes, records, end-of-leaf flags and boxes follow rt_rebuild_bvh steps 5-6 (depth-first preorder, a leaf's offset is its
 *     triangle id, boxes by the refit rule); the cluster boxes only steer the build.  Triangles are not reordered, so primitive
 *     ids, emissive_indices, the leaf order rt_update_triangles expects, the AOVs and the light tables keep their meaning.
 * The depth is not bounded by the rule (a chain of triangles whose extent grows geometrically merges one triangle per
 * iteration): a tree deeper than 64 levels (root = 1; the 64-entry traversal stack) gives RT_ERR_UNSUPPORTED and writes
 * nothing: the tree, records, refit map, shared-memory staging and a captured frame graph stay as they were.  rt_rebuild_bvh
 * always succeeds on the same triangles.
 * Memory: the tree group of rt_rebuild_bvh (either call allocates it, the other reuses it, so a context can alternate between
 * the two builds) plus the clustering temporaries, allocated all-or-nothing at the first call of this function after an upload:
 * about 97 bytes per triangle (the cluster list and its compaction target 64, the interior nodes 20, the parent links 8, the
 * neighbours and flags 5) and the compaction's scratch.  If no rebuild of either kind has run since the upload, the call also
 * allocates the tree group as rt_rebuild_bvh does and re-captures the frame graph (once the tree is known to fit); after that,
 * calls of either build move no buffer, so a captured graph stays valid.
 * Blocking: the host reads the cluster count after each iteration (about 50-70 for 50 000 triangles) and the depth flag before
 * anything of the tree is written.  Ordering, fan-out over multi-device contexts, n_nodes and what frames see afterwards are as
 * for rt_rebuild_bvh.  Errors: RT_ERR_NOT_READY before an upload, RT_ERR_UNSUPPORTED for the depth.  The launches count under
 * RT_K_MISC and in rt_launch_count: 9 + 3 per iteration for n > 1 (the sort and each compaction count as one), 2 for n = 1. */
#define RT_PLOC_RADIUS 16
int rt_rebuild_bvh_ploc(rt_ctx* ctx, uint64_t* n_nodes);

/* ---- instanced scenes (new capability): placed copies of shared meshes, traced through a two-level BVH ---------------------------
 * The scene kind is decided by the upload call: rt_upload_scene makes a flat scene, rt_upload_instanced_scene an instanced one; each
 * replaces whatever scene came before.  Nothing changes for flat scenes.
 * Meshes: scene->triangles and scene->nodes are the concatenation of the meshes; mesh k owns triangles [first_triangle,
 * first_triangle + n_triangles) in its own leaf order and nodes [first_node, first_node + n_nodes), a Bvh::BuildCPU array whose
 * offsets are relative to the mesh's own arrays.  Every mesh gets the records rt_upload_scene would derive from it alone
 * (rt_bvh_layout.h), concatenated.  Materials, textures, lights and the environment are shared.  emissive_indices is ignored.
 * Every mesh range must lie inside the arrays and each mesh's root box must be finite (else RT_ERR_INVALID_ARGUMENT).
 * Instances: rt_set_instances replaces the whole list (0 instances is legal: every ray misses).  RtInstance.object_to_world is M,
 * row-major 3x4.  The context computes W = M^-1 in double and rounds it to float, and rejects the whole call with
 * RT_ERR_INVALID_ARGUMENT (the previous list stays) if an instance's matrix is not finite or singular (det == 0 in double), its
 * mesh index is out of range, or the virtual triangle ids reach RT_INVALID_ID.  A negative determinant (a mirror) is allowed.
 * The top-level tree and the world boxes follow the rule of raytracing_b200/csrc/rt_instances.h.
 * Virtual triangle ids: instance i covers [base_i, base_i + n_triangles(mesh_i)), base = the prefix sum in instance order, so
 * RtHit.primitive_id, rt_read_hits and the statistics read as for the flattened scene.
 * Traversal: the top-level tree with the slab test, near/far order and deferred-child stack of the flat traversal, every top-level
 * box widened on each side by the ray's slack e = max(|o.x|, |o.y|, |o.z|) * a + b, with (a, b) computed by rt_set_instances from
 * the largest condition number ||A||_inf ||A^-1||_inf of the list, the world boxes and the translations (rt_instances.h states
 * the rule and its bound): a top-level box never culls a hit that the mesh's own tree finds for the object-space ray, for any |o|,
 * any condition number and t <= RT_MAX_RENDER_DIST (where e overflows every box passes); at an instance
 * the ray goes to object space, all float without contraction: o' = ((W0*o.x + W1*o.y) + W2*o.z) + W3 per row, d' = (W0*d.x + W1*d.y)
 * + W2*d.z; d' is not renormalised, so t is the same parameter in both spaces, and the mesh's tree is traced with the shared
 * t_max as a flat scene's (a later equal-t hit replaces the earlier, across instances too), except that the back-face test reads
 * det * sign(det M): a mirrored instance culls the faces its flattened triangles would.  Any-hit rays stop at the first hit.
 * Shading: the object-space position p as for flat scenes, then position = M * p (same row order as o'); the shading normal is
 * normalize(W^T * n) with n the interpolated vertex normal, the geometric normal normalize(W^T * n_g) * sign(det M); texture
 * coordinates, materials and emission are those of the mesh triangle (materials through the instance's row, if
 * rt_set_instance_materials gave it one).  With W = M = identity a frame equals that of the meshes
 * uploaded flat, except where a signed zero or a NaN coordinate meets the matrix arithmetic (0 * x, -0 + 0).
 * Object motion (RT_OPT_OBJECT_MOTION): the previous transform M_prev of instance index i is its transform in the last earlier
 * rt_set_instances (since the upload) whose list had index i, or its current one if none had; the velocity AOV of a bounce-0 hit is
 * project(M * p) - project(M_prev * q), all float as the shading position, with q the hit's point on the mesh triangle's previous
 * positions (the mesh-update block below; q = p until the mesh's first rt_update_mesh_triangles*).
 * Schedules: always the per-phase kernels (RT_OPT_FRAME_KERNEL has no effect), nothing staged (rt_bvh_staging reports mode 0;
 * RT_OPT_SMEM_BVH, RT_OPT_TOP_SMEM, RT_OPT_OCTANT_BVH and RT_OPT_TRAVERSAL have no effect).  Overlap modes, graphs, PDL, kernel
 * timing, traversal counting, the stepwise calls and rt_integrate_samples work.  Traversal counting counts each top-level box
 * tested once (the root, and both children of every top-level interior node visited) plus the mesh nodes the flat count would.
 * The sort-key origin of the shading pass (ray order only) is the top-level root box centre as of the last rt_set_instances that
 * grew the instance buffer.
 * Ordering: rt_set_instances is enqueued on the render stream like rt_update_triangles (a deferred shadow pass is launched first);
 * a captured frame graph stays valid while the instance count does not exceed the buffer's capacity (it grows to at least twice
 * its size when a list exceeds it).
 * RT_ERR_UNSUPPORTED on an instanced scene: rt_update_triangles*, rt_rebuild_bvh, rt_rebuild_bvh_ploc, rt_read_bvh and
 * RT_OPT_EMITTER_SAMPLING 1 (whichever call comes second).  RT_ERR_NOT_READY: rt_set_instances without an instanced scene.
 * Multi-device contexts fan out both calls. */
typedef struct RtMeshDesc { uint64_t first_triangle, n_triangles, first_node, n_nodes; } RtMeshDesc;
typedef struct RtInstance { float object_to_world[12]; uint32_t mesh; uint32_t padding[3]; } RtInstance;
int rt_upload_instanced_scene(rt_ctx* ctx, const RtSceneDesc* scene, const RtMeshDesc* meshes, uint32_t n_meshes);
int rt_set_instances(rt_ctx* ctx, const RtInstance* instances, uint32_t n_instances);

/* ---- mesh updates in instanced scenes (new capability): deform one shared mesh in place, its tree refit on the device ----------
 * triangles[i] replaces triangle first_triangle + i of mesh `mesh` (RtMeshDesc of the upload), in the mesh's own leaf order;
 * n_triangles must equal the mesh's count.  The mesh's records (tris_ref, wtris, tri_shade) become what the upload derives, as
 * rt_update_triangles defines them: mtlIndex and the padding are not read, the materials and end-of-leaf flags are kept.  The
 * mesh's tree keeps its topology and is refit by the refit rule of the geometry-update block, over the mesh's nodes only; no other
 * mesh's records are touched.  The refit root box is read back (32 bytes, so both variants block once for it) and becomes the
 * mesh's root box: if an instance of the current list uses the mesh, the top-level tree is rebuilt from it by rt_set_instances'
 * rule (raytracing_b200/csrc/rt_instances.h) for the current list, and only the header and the top-level records are rewritten.
 * The instance records (W, M, bases), the previous transforms of object motion and the sort-key origin of the shading pass stay
 * as they were.  So every output of a later frame is, bit for bit, that of rt_upload_instanced_scene with the refit nodes and the
 * new triangles followed by the same rt_set_instances; only the order of the continuation rays may differ.  If no instance uses
 * the mesh, only the mesh is written.
 * Object motion (RT_OPT_OBJECT_MOTION): the context keeps the previous positions Q of every mesh triangle, by the flat rule of the
 * object-motion block: Q = the positions before the last rt_update_mesh_triangles* of that mesh, the current ones after an upload
 * and after turning the option on; rt_set_instances, frames, rt_reset and camera changes leave Q alone.  The velocity AOV of a
 * bounce-0 hit on mesh triangle t of instance i at barycentrics (u, v), w0 = 1 - u - v, all float as the shading position:
 *     q = (q1 * w0 + q2 * u) + q3 * v;  velocity = project(M_i * p) - project(M_prev,i * q)
 * With Q equal to the current positions, q is the object-space hit point p bit for bit: nothing changes until a mesh update.
 * Memory: 48 B per mesh triangle while the option is on.
 * Validation: a position coordinate (xyz of v1, v2, v3) that is not finite is RT_ERR_INVALID_ARGUMENT and nothing is written
 * (the upload refuses a mesh root box that is not finite).  rt_update_mesh_triangles checks on the host;
 * rt_update_mesh_triangles_device runs a check kernel and reads back its flag (blocking) before anything is written.
 * Ordering and buffers as for rt_update_triangles: a deferred shadow pass is launched first and the update is enqueued on the
 * render stream; no buffer moves, so a captured frame graph stays valid; the refit kernels never trigger dependent launches.
 * rt_update_mesh_triangles reads the caller's array before it returns, through rt_update_triangles' staging (at most 2 x 32 MB,
 * allocated at the first host update of either kind); rt_update_mesh_triangles_device reads `device_triangles` (RtTriangle
 * layout, 16-byte aligned device memory of the context's device) on the render stream, and the caller keeps it unchanged until
 * the call returns.  The first update of a mesh builds its refit map (blocking; 12 B per node and 4 B per leaf of the mesh, plus
 * one 4-byte flag for the device variant), which lives until the next upload.
 * Errors: RT_ERR_NOT_READY without an instanced scene (none, or a flat one); RT_ERR_INVALID_ARGUMENT for a mesh index out of
 * range, a count mismatch, a null pointer or a position that is not finite, and for the device variant a pointer that is not
 * 16-byte aligned device memory of the context's device; RT_ERR_UNSUPPORTED for rt_update_mesh_triangles_device on a
 * multi-device context (rt_update_mesh_triangles fans out).  The launches count under RT_K_MISC (RT_OPT_KERNEL_TIMING) and in
 * rt_launch_count.  rt_update_triangles*, the rebuilds and rt_read_bvh stay RT_ERR_UNSUPPORTED on instanced scenes. */
int rt_update_mesh_triangles(rt_ctx* ctx, uint32_t mesh, const RtTriangle* triangles, uint64_t n_triangles);
int rt_update_mesh_triangles_device(rt_ctx* ctx, uint32_t mesh, const void* device_triangles, uint64_t n_triangles);

/* ---- per-instance materials in instanced scenes (new capability): each instance of a shared mesh shades with its own materials --
 * Rows: `remaps` holds n_remaps rows of n_materials entries (n_materials = the upload's material count); row r maps scene
 * material m to remaps[r * n_materials + m].  remap_of_instance[i] is the row of instance index i; RT_INVALID_ID, and every index
 * >= n_instances, keeps the mesh's own materials.
 * Rule: a hit on mesh triangle t of instance i with row r is shaded with material remaps[r * n_materials + t.mtlIndex] wherever
 * the frame reads t.mtlIndex: the BSDF, the textured flag (whether texture coordinates are interpolated), the texture lookups
 * (with the triangle's own texture coordinates), the emission and the n_emissive_hits count, and the albedo AOV.  Traversal,
 * virtual ids, geometry, normals, depth, motion vectors, the light tables and the sort-key origin are unchanged.  So every output
 * of a frame (radiance, statistics, the hits of every bounce, every AOV) equals, bit for bit, the frame of the same instanced scene
 * uploaded with a private copy of its mesh for each instance that has a row, whose triangles carry the remapped mtlIndex, under
 * the same transforms in the same order.
 * Lifetime: the assignment is indexed by instance index and replaced whole by each call.  rt_set_instances keeps it (instance i
 * of a later list uses the row given for index i, as the previous transforms of object motion are kept per index), and so do
 * rt_update_mesh_triangles* and rt_reset; rt_upload_scene and rt_upload_instanced_scene clear it, and so does a call with
 * n_remaps = n_instances = 0.
 * Device side: the row offset r * n_materials (or RT_INVALID_ID) is a word of each instance record; the rows live in a table of
 * their own (4 B per entry, allocated at the first call that needs it and freed by the next upload).  The shading pass of an
 * instanced scene makes one dependent 4-byte load per hit of an instance with a row; flat scenes run the code they ran before.
 * Ordering and buffers as for rt_set_instances: a deferred shadow pass is launched first and the copies are enqueued on the
 * render stream; the call returns once both host arrays have been read.  The table grows to at least twice its size when a
 * call needs more entries than it holds, the only case that re-captures a frame graph; otherwise no buffer moves.
 * Errors, each leaving the next frame as it was: RT_ERR_NOT_READY without an instanced scene (none, or a flat one);
 * RT_ERR_INVALID_ARGUMENT for a null pointer with a non-zero count, a row entry >= n_materials, a remap_of_instance entry that is
 * neither < n_remaps nor RT_INVALID_ID, or n_remaps * n_materials >= 2^32 - 1 (row offsets fit 32 bits and stay distinct from
 * RT_INVALID_ID).  Multi-device contexts fan out.  RtInstance, flat scenes and RT_OPT_EMITTER_SAMPLING (still RT_ERR_UNSUPPORTED
 * on instanced scenes) are unchanged; RtInstance.padding stays without meaning. */
int rt_set_instance_materials(rt_ctx* ctx, const uint32_t* remaps, uint32_t n_remaps, const uint32_t* remap_of_instance,
                              uint32_t n_instances);

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
/* How the traversal kernels of the next frame stage the BVH into shared memory, for the current scene and options: *mode =
 * 0 nothing, 1 the whole structure, 2 the first RT_OPT_TOP_SMEM records, 3 the whole structure plus the octant-ordered record
 * tables (RT_OPT_OCTANT_BVH); *bytes = dynamic shared memory per CTA.  Either pointer may be NULL.  (The one-kernel frame
 * of RT_OPT_FRAME_KERNEL runs mode 1 where this says 3; RT_OPT_COUNT_TRAVERSAL runs unstaged kernels whatever this says.) */
int rt_bvh_staging(rt_ctx* ctx, uint32_t* mode, uint64_t* bytes);
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
