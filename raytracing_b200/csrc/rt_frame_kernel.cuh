/*
 * rt_frame_kernel.cuh — the one-kernel frame (k_frame): every CTA an independent wavefront over its own pixels, its phases built from
 * the warp work items that the per-phase kernels use (rt_kernels.cu).
 * Part of the single translation unit rt_kernels.cu (included there, inside its anonymous namespace).
 */
#pragma once

// ---- whole-frame kernel (RT_OPT_FRAME_KERNEL, default) ---------------------------------------------------------
// ONE launch per frame.  Every CTA is an independent wavefront path tracer over its own subset of the partition's pixels
// (groups of 32 consecutive local pixels, dealt round-robin to the resident CTAs), with its own region of every queue:
// a path never leaves the CTA that generated its primary ray.  The per-bounce schedule is the one of rt_extend_shade /
// rt_shadow_accumulate (integrator.cpp:27-59 fused the same way):
//     T(b): closest-hit traversal of bounce b  +  shadow pass of bounce b-1   -> hit queue / miss queue
//     S(b): shading of the hit queue, then of the miss queue                   -> shadow queue, ray queue of bounce b+1
// but the queue cursors and counters live in SHARED memory and the phases are separated by __syncthreads(): no global
// atomics on the ray path, no grid-wide synchronisation, no launch boundary between phases (the ~10-15 us floor that 22
// dependent launches per frame cost a small multi-GPU partition), and the 4 CTAs of an SM are in different phases at any
// time, so a CTA waiting for its slowest warp at a barrier leaves the issue slots to its neighbours.  Primary rays are
// generated inside T(0) (no separate pass over the queue).  Results are bit-identical: every per-pixel quantity is a
// function of (pixel, sample index, bounce) only, and the order of the additions into a pixel's radiance is unchanged.
struct CtaFrame
{
    uint32_t cur_trace, cur_shade;           // work cursors of the current T / S phase
    uint32_t ext_n[2], shadow_n[2];          // rays entering bounce b (parity b & 1), shadow rays spawned by S(b) (parity b & 1)
    unsigned long long hm[2];                // hits (low word) and misses (high word) of T(b), parity b & 1
    unsigned long long emit[2];              // shadow rays (low word) and continuation rays (high word) spawned by S(b): slot reservation
    uint32_t n_emissive, n_unoccluded;
    uint32_t ended_n[2];                     // fused gather: pixels whose path ended at a hit in S(b) (no continuation), parity b & 1
    uint32_t n_src;                          // entries of the primary-ray source: local pixels, or active pixels (adaptive sampling)
};

template <int SMEM, bool EMIT = false>
__global__ void __launch_bounds__(RT_FRAME_MAX_THREADS, 1) k_frame(FrameParams p, DevScene sc, int mode, Queues q, DevCounters* ctr, float4* radiance,
                                                              AovParams aov, uint32_t max_bounces, uint32_t slots_per_cta,
                                                              const __grid_constant__ FrameDyn dyn)
{
    extern __shared__ __align__(128) float4 s_bvh[];
    __shared__ uint64_t s_mbar;
    __shared__ CtaFrame s;
    p.dyn = &dyn;                                  // per-frame constants (sample index, camera) arrive as a kernel parameter
    stage_bvh<SMEM>(s_bvh, sc, &s_mbar);
    const int lane = threadIdx.x & 31;
    const uint32_t base = blockIdx.x * slots_per_cta;          // this CTA's region of every queue: slots [base, base + slots_per_cta)
    // (queue pointers are re-read from the kernel parameters where they are used: nothing but `base` stays live across the
    // traversal and shading loops)
    if (threadIdx.x == 0)
    {   // groups of 32 consecutive entries of the primary-ray source (local pixels, or the ascending active list) are dealt
        // round-robin; with adaptive sampling the grid stays sized by the partition and the active count is read here
        const uint32_t n_src = p.active ? *p.n_active : p.n_local;
        const uint32_t n_groups = (n_src + 31u) / 32u;
        const uint32_t cta = blockIdx.x, n_cta = gridDim.x;
        const uint32_t my_groups = cta < n_groups ? (n_groups - cta + n_cta - 1u) / n_cta : 0u;
        s.cur_trace = 0; s.cur_shade = 0; s.ext_n[0] = my_groups * 32u; s.ext_n[1] = 0; s.shadow_n[0] = s.shadow_n[1] = 0;
        s.hm[0] = s.hm[1] = 0ull; s.emit[0] = s.emit[1] = 0ull; s.n_emissive = 0; s.n_unoccluded = 0; s.ended_n[0] = s.ended_n[1] = 0;
        s.n_src = n_src;
        // n_primary adds up over the frames of a multi-sample call (the counters are not cleared between them) once it varies
        if (blockIdx.x == 0) ctr->n_primary = p.active ? ctr->n_primary + n_src : p.n_local;
    }
    __syncthreads();
    uint32_t nv = 0, nt = 0;     // (not counted here: RT_OPT_COUNT_TRAVERSAL uses the per-phase kernels)

    for (uint32_t b = 0; b <= max_bounces + 1u; ++b)
    {
        // ---------------------------------------------------------------- T(b): extension rays of bounce b, then shadow rays of bounce b-1
        {
            const int in = b & 1;
            const uint32_t n_ext = b <= max_bounces ? s.ext_n[in] : 0u;          // the last round is the shadow pass of the last bounce only
            const uint32_t ext_span = (n_ext + 31u) & ~31u;
            const uint32_t n_sh = b == 0 ? 0u : s.shadow_n[(b - 1u) & 1];
            const uint32_t total = ext_span + n_sh;
            if (threadIdx.x == 0)
            {   // state of the NEXT phases that nobody reads during this one
                s.cur_shade = 0; s.ext_n[(b + 1u) & 1] = 0; s.shadow_n[in] = 0; s.emit[in] = 0ull; s.ended_n[in] = 0;
            }
            for (uint32_t at; (at = warp_grab(&s.cur_trace)) < total;)
            {
                if (at < ext_span)
                {
                    const uint32_t i = at + lane;
                    bool live = i < n_ext;
                    float4 a, bb;
                    if (b == 0)
                    {   // primary rays generated in the first traversal pass; slot i <-> source entry j: local pixel j, or active[j]
                        const uint32_t j = (blockIdx.x + (i >> 5) * gridDim.x) * 32u + (uint32_t)lane;
                        live = j < s.n_src;
                        if (live) primary_ray(p, q, aov, base + i, p.active ? p.active[j] : j, a, bb);
                    }
                    else if (live) { a = q.A[in][base + i]; bb = q.B[in][base + i]; }
                    closest_group<false, SMEM, true>(sc, mode, s_bvh, q, base, i, live, a, bb, &s.hm[in], nv, nt);
                }
                else shadow_group<false, SMEM, true>(p, sc, mode, s_bvh, q, base, at - ext_span + lane, n_sh, radiance, &s.n_unoccluded, nv, nt);
            }
            __syncthreads();
            if (p.gather && b > 0)
            {   // fused gather: the shadow rays of bounce b-1 are accumulated, so the pixels whose path ended at a hit of S(b-1) are
                // final; after the last round so are the paths that were still alive (their rays sit in the queue S(max) filled)
                const int pin = (b - 1u) & 1;
                const uint32_t n_end = s.ended_n[pin];
                const uint32_t* list = pin ? (const uint32_t*)q.hits + base : q.shadow_flags + base;
                for (uint32_t k = threadIdx.x; k < n_end; k += blockDim.x) { const uint32_t li = list[k]; p.gather[li] = radiance[li]; }
                if (b > max_bounces)
                {
                    const uint32_t n_alive = s.ext_n[in];
                    for (uint32_t k = threadIdx.x; k < n_alive; k += blockDim.x)
                    {
                        const uint32_t li = local_index(p, __float_as_uint(q.B[in][base + k].w));
                        p.gather[li] = radiance[li];
                    }
                }
            }
            if (threadIdx.x == 0)
            {   // per-bounce statistics (rt_read_frame_stats): one fire-and-forget global add per CTA and counter
                const unsigned long long hm = s.hm[in];
                if (b <= max_bounces && hm) atomicAdd((unsigned long long*)&ctr->hm[b], hm);
                if (b > 0 && s.n_unoccluded) atomicAdd(&ctr->n_unoccluded[b - 1u], s.n_unoccluded);
                s.n_unoccluded = 0;
            }
        }
        if (b > max_bounces) break;
        // ---------------------------------------------------------------- S(b): ShadeSurfaceHits over the hit queue, ShadeMissedRays over the miss queue
        {
            const int in = b & 1, out = (b + 1u) & 1;
            const unsigned long long hm = s.hm[in];
            const uint32_t n_hit = (uint32_t)hm, n_miss = (uint32_t)(hm >> 32);
            const uint32_t hit_span = (n_hit + 31u) & ~31u;            // warps never mix hits and misses
            const uint32_t total = hit_span + n_miss;
            if (threadIdx.x == 0) { s.cur_trace = 0; s.hm[out] = 0ull; }
            for (uint32_t at; (at = warp_grab(&s.cur_shade)) < total;)
            {
                if (at < hit_span)
                {
                    const uint32_t k = at + lane;
                    const bool hit = k < n_hit;
                    float4 h = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
                    if (hit) h = q.hitq[base + k];
                    uint32_t pixel;
                    const bool ends = shade_hit_group<false, EMIT, false, EMIT>(p, sc, aov, q, base, b, hit, h, __float_as_uint(h.w), radiance, &s.emit[in], &s.n_emissive, pixel);
                    if (p.gather)
                    {   // paths that end at this hit (no continuation ray): final once their shadow ray is accumulated in T(b+1)
                        const unsigned dmask = __ballot_sync(0xffffffffu, ends);
                        if (dmask)
                        {
                            uint32_t at0 = 0;
                            if (lane == 0) at0 = atomicAdd(&s.ended_n[in], (uint32_t)__popc(dmask));
                            at0 = __shfl_sync(0xffffffffu, at0, 0);
                            uint32_t* list = in ? (uint32_t*)q.hits + base : q.shadow_flags + base;
                            if (ends) list[at0 + __popc(dmask & ((1u << lane) - 1u))] = local_index(p, pixel);
                        }
                    }
                }
                else if (at - hit_span + lane < n_miss) shade_miss<EMIT>(sc, p, q, b, base + q.missq[base + at - hit_span + lane], radiance);
            }
            __syncthreads();
            if (threadIdx.x == 0)
            {
                const unsigned long long em = s.emit[in];
                s.shadow_n[in] = (uint32_t)em; s.ext_n[out] = (uint32_t)(em >> 32);
                if (em) atomicAdd((unsigned long long*)&ctr->emit[b], em);
                if (s.n_emissive) atomicAdd(&ctr->n_emissive[b], s.n_emissive);
                s.n_emissive = 0;
            }
            __syncthreads();
        }
    }
}
