/*
 * rt_kernel_types.cuh — device-side state of the wavefront path tracer: per-bounce counters, queue planes, per-frame constants, warp helpers.
 * Part of the single translation unit rt_kernels.cu (included there, inside its anonymous namespace).
 */
#pragma once

// ------------------------------------------------------------------------------------ device state
struct DevCounters
{
    uint32_t n_primary;                          // rays entering bounce 0
    uint32_t pad0;
    // rays spawned by the shading pass of bounce b: shadow rays and continuation rays (= the rays entering bounce b+1).
    // Adjacent + 8-byte aligned so that ONE 64-bit atomic reserves slots in both output queues.
    struct alignas(8) Emit { uint32_t shadow, next; };
    Emit emit[RT_MAX_BOUNCES + 1];
    struct alignas(8) HitMiss { uint32_t hit, miss; };   // adjacent + 8-byte aligned: one 64-bit atomic advances both
    HitMiss hm[RT_MAX_BOUNCES + 1];              // hit-queue entries / misses of bounce b
    uint32_t n_emissive[RT_MAX_BOUNCES + 1];
    uint32_t n_unoccluded[RT_MAX_BOUNCES + 1];
    uint32_t work_ext[RT_MAX_BOUNCES + 1];       // persistent-kernel work cursors
    uint32_t work_shade[RT_MAX_BOUNCES + 1];
    uint32_t work_shadow[RT_MAX_BOUNCES + 1];
    unsigned long long nodes_ext[RT_MAX_BOUNCES + 1], tris_ext[RT_MAX_BOUNCES + 1];
    unsigned long long nodes_shadow[RT_MAX_BOUNCES + 1], tris_shadow[RT_MAX_BOUNCES + 1];
};

__host__ __device__ __forceinline__ const uint32_t* in_count_ptr(const DevCounters* c, uint32_t bounce)
{
    return bounce == 0 ? &c->n_primary : &c->emit[bounce - 1].next;
}

// The two buffers of one plane of the extension-ray queue, by bounce parity.  Read through a select, not an array index: a kernel
// parameter indexed by a run-time value is first copied to the thread's stack, which every thread of every launch then writes.
struct PlanePair
{
    float4* p[2];
    __host__ __device__ __forceinline__ float4* operator[](int i) const { return i ? p[1] : p[0]; }
};

struct Queues
{
    PlanePair A, B, C;
    float4* sA; float4* sB; float4* sC;
    float4* hits;
    uint32_t* shadow_flags;
    float4* hitq;
    uint32_t* missq;
};

// Per-frame constants that change from frame to frame (sample index, camera): kept in a small device buffer that a
// 1-thread kernel refreshes at the start of every frame, so that the rest of the frame's launches have frame-invariant
// arguments and the whole frame can be replayed as ONE CUDA graph (rt_integrate) with a single node-parameter update.
struct FrameDyn;

struct FrameParams
{
    uint32_t width, height, rank, world, n_local;
    int white_furnace;
    const int* bn;                 // blue-noise sampler tables (kBlueNoise) or nullptr (kRandom)
    const FrameDyn* dyn;
    float4* gather;                // k_frame only: this rank's slab of the gathered radiance on the presenting device (peer memory,
                                   // rt_set_gather_target) — a pixel's radiance is pushed there the moment its path ends; else nullptr
    // adaptive sampling (rt_set_adaptive_sampling), else nullptr: primary rays are traced for the local pixels active[0 .. *n_active)
    // (ascending) instead of every local pixel
    const uint32_t* active;
    const uint32_t* n_active;
};

// Adaptive sampling, device-resident control block of k_adaptive_update (one per context while the feature is on)
struct AdaptiveCtl
{
    uint32_t n_active;             // entries of the active list: pixels that trace the next sample
    uint32_t n_next;               // the compaction's new count, moved to n_active by the update's last CTA
    uint32_t frames;               // samples since rt_reset = the sample count of every active pixel
    uint32_t ticket, done;         // the update's CTA order (decoupled look-back) and completion count, back to 0 after every update
    uint32_t epoch;                // tags the update's tile states: 1 .. 2^30 - 1, advanced by every update
};

// AOV outputs of bounce 0 (kernels/cl/aov.cl:44-110), written by the bounce-0 shading pass when enabled
struct AovCam { f3 position, front, up, right; float angle, aspect_ratio; };
struct AovParams
{
    int enabled;
    float4* albedo; float* depth; float4* normal; float2* velocity;
    const float4* prev_pos;        // RT_OPT_OBJECT_MOTION: the previous positions, 3 float4 per triangle (tris_ref layout); else nullptr
};

struct FrameDyn
{
    uint32_t sample_idx;
    uint32_t max_bounces;          // emitter sampling: the frame's last bounce, which samples analytic lights only
    uint32_t pad[2];
    RayGenConsts raygen;
    AovCam cam, prev;
};

__global__ void k_set_frame(FrameDyn* dst, FrameDyn value) { *dst = value; }

// kernels/cl/aov.cl:30-42
__device__ __forceinline__ f2 project_screen(f3 position, const AovCam& c)
{
    f3 d = normalize(position - c.position);
    f3 ipd = d / dot(c.front, d);
    float u = dot(c.right, ipd) / (c.angle * c.aspect_ratio);
    float v = dot(c.up, ipd) / (c.angle);
    f2 r; r.x = u * 0.5f + 0.5f; r.y = v * 0.5f + 0.5f;
    return r;
}

__device__ __forceinline__ uint32_t pack_pixel(uint32_t px, uint32_t py) { return px | (py << 16); }
__device__ __forceinline__ uint32_t local_index(const FrameParams& p, uint32_t pxy)
{
    uint32_t px = pxy & 0xFFFFu, py = pxy >> 16;
    return (p.world == 1 ? py : py / p.world) * p.width + px;
}

// Persistent warps drain a queue 32 entries at a time: lane 0 advances the work cursor, every lane gets the group's first entry.
// Measured alternatives that were slower: 64 entries per grab (-4 %), and issuing the next round's grab before the current
// round's work to hide the atomic's latency (-5 %): both make a warp own more work at a time, and the coarser tail costs more
// than the hidden latency saves.
__device__ __forceinline__ uint32_t warp_grab(uint32_t* cursor)
{
    uint32_t at = 0;
    if ((threadIdx.x & 31) == 0) at = atomicAdd(cursor, 32u);
    return __shfl_sync(0xffffffffu, at, 0);
}

// Shadow-ray records.  sA = (origin.xyz, word), sC = (light sample.xyz, 0), and sB = (dir.xyz, t_max) only where the
// light does not fix them: for a directional light they are its record light_rec[2 * l] (light_sample), which the shadow pass
// reads in place of sB.  The word is the local pixel index (low 24 bits) and the light byte l (high 8 bits); RT_SHADOW_3PLANE
// marks every other ray (point lights, emitter and environment samples, lights from index 255 on), whose sB is stored.  Partitions
// of 2^24 local pixels or more store every ray with three planes and the whole local index in the word.
#define RT_SHADOW_3PLANE 0xFFu
__device__ __forceinline__ bool shadow_two_plane(const FrameParams& p) { return p.n_local <= (1u << 24); }
__device__ __forceinline__ uint32_t shadow_word(const FrameParams& p, uint32_t li, uint32_t light)
{
    return shadow_two_plane(p) ? li | (light << 24) : li;
}
// Writes the shadow ray of local pixel li in slot si; sB only for a three-plane record
__device__ __forceinline__ void put_shadow(const FrameParams& p, const Queues& q, uint32_t si, uint32_t li, uint32_t light, f3 o, f3 d, float t_max,
                                           f3 sample)
{
    q.sA[si] = make_float4(o.x, o.y, o.z, __uint_as_float(shadow_word(p, li, light)));
    if (!shadow_two_plane(p) || light == RT_SHADOW_3PLANE) q.sB[si] = make_float4(d.x, d.y, d.z, t_max);
    q.sC[si] = make_float4(sample.x, sample.y, sample.z, 0.0f);
}
// The (dir.xyz, t_max) plane of the shadow ray in slot si whose sA word is w, and its local pixel li
__device__ __forceinline__ float4 shadow_dir(const FrameParams& p, const DevScene& sc, const Queues& q, uint32_t si, uint32_t w, uint32_t& li)
{
    if (shadow_two_plane(p))
    {
        li = w & 0xFFFFFFu;
        const uint32_t light = w >> 24;
        if (light != RT_SHADOW_3PLANE) return __ldg(sc.light_rec + (size_t)light * 2);
        return q.sB[si];
    }
    li = w;
    return q.sB[si];
}

__device__ __forceinline__ float4 add_radiance(float4* radiance, uint32_t li, f3 v)
{
    float4 r = radiance[li];
    r.x += v.x; r.y += v.y; r.z += v.z;
    radiance[li] = r;
    return r;
}

__device__ __forceinline__ void warp_count(uint32_t* counter, bool pred)
{
    unsigned mask = __ballot_sync(0xffffffffu, pred);
    if (mask != 0 && (threadIdx.x & 31) == __ffs(mask) - 1) atomicAdd(counter, (uint32_t)__popc(mask));
}

__device__ __forceinline__ void warp_sum64(unsigned long long* counter, uint32_t v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(counter, (unsigned long long)v);
}
