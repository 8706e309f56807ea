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
                        if (live) primary_ray(p, q, aov, 0, base + i, p.active ? p.active[j] : j, p.dyn->sample_idx, 0u, a, bb);
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

// ---- regenerating one-kernel frame (rt_integrate_samples) -----------------------------------------------------
// n_samples consecutive frames in ONE launch.  It keeps k_frame's structure (CTA-private pixels and queue regions, shared-memory
// cursors, T and S phases separated by __syncthreads()), but a round is no longer a bounce: every queue entry carries its own path
// state, and when a pixel's path ends the CTA starts that pixel's next sample in the next traversal round (path regeneration).
// Rounds stay full instead of draining towards the longest path of a sample, and the CTA runs about n_samples x the mean path
// length rounds instead of n_samples x (max_bounces + 2).
//   Path state: C.w of the extension-ray planes and sC.w of the shadow queue hold the path's bounce (low 8 bits) and its sample
//   offset k (absolute sample index dyn.sample_idx + k, the upper 24 bits: a launch renders at most RT_MAX_REGEN_SAMPLES samples).
//   Bit-exactness: every per-pixel quantity is a function of (pixel, sample index, bounce), and the per-pixel order of the additions
//   into the radiance is that of n_samples frames in sequence, because sample k+1 of a pixel starts only after the last addition of
//   sample k.  A path that misses in S(r) is finished in S(r); a path that ends at a hit in S(r) (no continuation ray, or bounce ==
//   max_bounces) is finished when its shadow ray is accumulated in T(r+1).  In both cases the pixel's next primary ray is traced in
//   T(r+1), and its first addition comes in S(r+1), after the barrier.  At most one path per pixel is alive, so the queue regions
//   of k_frame suffice.
struct CtaRegen
{
    uint32_t cur_trace, cur_shade;           // work cursors of the current T / S phase
    uint32_t ext_n[2], shadow_n[2];          // continuation rays entering round r (parity r & 1), shadow rays spawned by S(r) (parity r & 1)
    unsigned long long hm[2];                // slots of the hit (low word) and miss (high word) queues taken by T(r), parity r & 1
    unsigned long long emit[2];              // slots of the shadow (low) and ray (high) queues taken by S(r), parity r & 1
    uint32_t regen_n[2], last_n[2];          // paths that ended in S(r), parity r & 1: with a next sample / of the last sample (fused gather)
    // per-bounce statistics of the whole call, added to the DevCounters once per CTA
    uint32_t n_hit[RT_MAX_BOUNCES + 1], n_miss[RT_MAX_BOUNCES + 1], n_emissive[RT_MAX_BOUNCES + 1];
    uint32_t n_shadow[RT_MAX_BOUNCES + 1], n_cont[RT_MAX_BOUNCES + 1], n_unoccluded[RT_MAX_BOUNCES + 1];
};

// counters[key] += the lanes of the warp with `pred` whose key is the lane's; same_key = __match_any_sync over the key
__device__ __forceinline__ void count_keyed(uint32_t* counters, uint32_t key, unsigned same_key, bool pred)
{
    const unsigned m = __ballot_sync(0xffffffffu, pred) & same_key;
    if (pred && (threadIdx.x & 31) == __ffs(m) - 1) atomicAdd(counters + key, (uint32_t)__popc(m));
}

// The paths that end in S(r) go into the CTA's list of parity r & 1 (`cap` uint2 entries): from the front (local pixel, k + 1) when the
// pixel has a next sample — T(r+1) generates it — and, when `keep_last`, from the back (local pixel, -) for the last sample's paths
// that ended at a hit: the fused gather pushes those pixels after T(r+1) has accumulated their shadow rays.
__device__ __forceinline__ void record_ended(CtaRegen& s, uint2* list, uint32_t cap, int par, bool ends, uint32_t li, uint32_t k,
                                             uint32_t n_samples, bool keep_last)
{
    const bool again = ends && k + 1u < n_samples, last = ends && !again && keep_last;
    const unsigned am = __ballot_sync(0xffffffffu, again), lm = __ballot_sync(0xffffffffu, last);
    if ((am | lm) == 0u) return;
    const int lane = threadIdx.x & 31;
    uint32_t a0 = 0, l0 = 0;
    if (lane == 0)
    {
        if (am) a0 = atomicAdd(&s.regen_n[par], (uint32_t)__popc(am));
        if (lm) l0 = atomicAdd(&s.last_n[par], (uint32_t)__popc(lm));
    }
    a0 = __shfl_sync(0xffffffffu, a0, 0); l0 = __shfl_sync(0xffffffffu, l0, 0);
    const unsigned lt_mask = (1u << lane) - 1u;
    if (again) list[a0 + __popc(am & lt_mask)] = make_uint2(li, k + 1u);
    if (last) list[cap - 1u - (l0 + __popc(lm & lt_mask))] = make_uint2(li, 0u);
}

// shadow_group with the path state: the unoccluded rays are counted by the bounce that spawned them
template <int SMEM>
__device__ __forceinline__ void shadow_group_regen(const FrameParams& p, const DevScene& sc, int mode, const float4* s_bvh, const Queues& q, uint32_t base,
                                                   uint32_t i, uint32_t n, float4* radiance, CtaRegen& s, uint32_t& nv, uint32_t& nt)
{
    bool un = false;
    uint32_t bounce = 0;
    if (i < n)
    {
        const float4 a = q.sA[base + i];
        uint32_t li;
        const float4 b = shadow_dir(p, sc, q, base + i, __float_as_uint(a.w), li);
        float bu, bv, bt;
        un = trace_staged<true, false, SMEM, true>(sc, mode, s_bvh, a, b, bu, bv, bt, nv, nt) == RT_INVALID_ID;
        if (un)
        {
            const float4 c = q.sC[base + i];
            add_radiance(radiance, li, mk3(c));
            bounce = __float_as_uint(c.w) & 0xFFu;
        }
    }
    count_keyed(s.n_unoccluded, bounce, __match_any_sync(0xffffffffu, bounce), un);
}

// shade_hit_group with the path state: the lane's own bounce and sample index, statistics by bounce, no continuation ray past
// max_bounces (it is still counted in n_cont, as in a frame), the state carried into the spawned rays.  Returns whether the path ends
// at this hit; li and state are the path's local pixel and state.
__device__ __forceinline__ bool shade_hit_regen(const FrameParams& p, const DevScene& sc, const AovParams& aov, const Queues& q, uint32_t base, int in,
                                                uint32_t max_bounces, bool hit, float4 h, uint32_t i, float4* radiance, CtaRegen& s,
                                                uint32_t& li, uint32_t& state)
{
    ShadeOut so;
    so.emissive = so.spawn_next = so.spawn_shadow = false;
    uint32_t pixel = 0, bounce = 0;
    li = 0; state = 0;
    if (hit)
    {
        const float4 a = q.A[in][base + i], b = q.B[in][base + i], c = q.C[in][base + i];
        pixel = __float_as_uint(b.w); state = __float_as_uint(c.w); bounce = state & 0xFFu;
        shade_hit(sc, p, aov, bounce, pixel, mk3(a), mk3(b), mk3(c), 0.0f, __float_as_uint(h.z), h.x, h.y, state >> 8, so);
        li = local_index(p, pixel);
        if (so.emissive) add_radiance(radiance, li, so.emission_add);
    }
    const bool ss = hit && so.spawn_shadow, sn = hit && so.spawn_next, cont = sn && bounce < max_bounces;
    const unsigned same = __match_any_sync(0xffffffffu, bounce);
    count_keyed(s.n_hit, bounce, same, hit);
    count_keyed(s.n_emissive, bounce, same, hit && so.emissive);
    count_keyed(s.n_shadow, bounce, same, ss);
    count_keyed(s.n_cont, bounce, same, sn);
    const unsigned smask = __ballot_sync(0xffffffffu, ss), nmask = __ballot_sync(0xffffffffu, cont);
    const int lane = threadIdx.x & 31;
    const unsigned lt_mask = (1u << lane) - 1u;
    unsigned long long slot = 0ull;
    if ((smask | nmask) != 0u)
    {
        if (lane == 0) slot = atomicAdd(&s.emit[in], (unsigned long long)__popc(smask) | ((unsigned long long)__popc(nmask) << 32));
        slot = __shfl_sync(0xffffffffu, slot, 0);
    }
    if (ss)
    {
        const uint32_t si = base + (uint32_t)slot + __popc(smask & lt_mask);
        put_shadow(p, q, si, li, so.s_light, so.s_origin, so.s_dir, so.s_tmax, so.s_sample, state);
    }
    if (cont)
    {
        const int out = in ^ 1;
        const uint32_t ni = base + (uint32_t)(slot >> 32) + __popc(nmask & lt_mask);
        q.A[out][ni] = make_float4(so.n_origin.x, so.n_origin.y, so.n_origin.z, 0.0f);
        q.B[out][ni] = make_float4(so.n_dir.x, so.n_dir.y, so.n_dir.z, __uint_as_float(pixel));
        q.C[out][ni] = make_float4(so.n_throughput.x, so.n_throughput.y, so.n_throughput.z, __uint_as_float(state + 1u));
    }
    return hit && !cont;
}

template <int SMEM>
__global__ void __launch_bounds__(RT_FRAME_MAX_THREADS, 1) k_frame_regen(FrameParams p, DevScene sc, int mode, Queues q, DevCounters* ctr, float4* radiance,
                                                                    AovParams aov, uint32_t max_bounces, uint32_t n_samples, uint32_t slots_per_cta,
                                                                    const __grid_constant__ FrameDyn dyn)
{
    extern __shared__ __align__(128) float4 s_bvh[];
    __shared__ uint64_t s_mbar;
    __shared__ CtaRegen s;
    p.dyn = &dyn;
    stage_bvh<SMEM>(s_bvh, sc, &s_mbar);
    const int lane = threadIdx.x & 31;
    const uint32_t base = blockIdx.x * slots_per_cta;          // this CTA's region of every queue, as in k_frame
    uint32_t n_first;                                          // the CTA's groups of 32 pixels: the primary rays of sample 0, in T(0)
    {
        const uint32_t n_groups = (p.n_local + 31u) / 32u;
        const uint32_t cta = blockIdx.x, n_cta = gridDim.x;
        n_first = (cta < n_groups ? (n_groups - cta + n_cta - 1u) / n_cta : 0u) * 32u;
    }
    for (uint32_t b = threadIdx.x; b <= RT_MAX_BOUNCES; b += blockDim.x)
    {
        s.n_hit[b] = 0; s.n_miss[b] = 0; s.n_emissive[b] = 0; s.n_shadow[b] = 0; s.n_cont[b] = 0; s.n_unoccluded[b] = 0;
    }
    if (threadIdx.x == 0)
    {
        s.cur_trace = 0; s.cur_shade = 0; s.ext_n[0] = s.ext_n[1] = 0; s.shadow_n[0] = s.shadow_n[1] = 0;
        s.hm[0] = s.hm[1] = 0ull; s.emit[0] = s.emit[1] = 0ull; s.regen_n[0] = s.regen_n[1] = 0; s.last_n[0] = s.last_n[1] = 0;
        if (blockIdx.x == 0) ctr->n_primary = p.n_local * n_samples;
    }
    __syncthreads();
    uint32_t nv = 0, nt = 0;

    for (uint32_t r = 0;; ++r)
    {
        const int in = r & 1, prev = in ^ 1;
        // the lists of ended paths live in the CTA's region of q.hits (2 x slots_per_cta uint2), one per parity
        uint2* const lists = (uint2*)(q.hits + base);
        // ---------------------------------------------------------------- T(r): continuation rays, then the regenerated primary rays
        // (slots n_ext.. of the same queue), then the shadow rays of S(r-1)
        const uint32_t n_ext = s.ext_n[in];
        const uint32_t n_new = r == 0 ? n_first : s.regen_n[prev];
        const uint32_t ext_span = (n_ext + n_new + 31u) & ~31u;
        const uint32_t n_sh = r == 0 ? 0u : s.shadow_n[prev];
        const uint32_t total = ext_span + n_sh;
        {
            const uint2* ended = lists + prev * slots_per_cta;
            if (threadIdx.x == 0) { s.cur_shade = 0; s.emit[in] = 0ull; s.regen_n[in] = 0; s.last_n[in] = 0; }
            for (uint32_t at; (at = warp_grab(&s.cur_trace)) < total;)
            {
                if (at < ext_span)
                {
                    const uint32_t i = at + lane;
                    bool live = i < n_ext;
                    float4 a, bb;
                    if (live) { a = q.A[in][base + i]; bb = q.B[in][base + i]; }
                    else if (i < n_ext + n_new)
                    {   // a pixel's next sample
                        const uint32_t j = i - n_ext;
                        uint32_t li, k = 0;
                        if (r == 0) li = (blockIdx.x + (j >> 5) * gridDim.x) * 32u + (j & 31u);
                        else { const uint2 e = ended[j]; li = e.x; k = e.y; }
                        live = li < p.n_local;
                        if (live) primary_ray(p, q, aov, in, base + i, li, p.dyn->sample_idx + k, k << 8, a, bb);
                    }
                    closest_group<false, SMEM, true>(sc, mode, s_bvh, q, base, i, live, a, bb, &s.hm[in], nv, nt);
                }
                else shadow_group_regen<SMEM>(p, sc, mode, s_bvh, q, base, at - ext_span + lane, n_sh, radiance, s, nv, nt);
            }
            __syncthreads();
            if (p.gather && r > 0)
            {   // fused gather: the last samples' paths that ended at a hit of S(r-1) have had their shadow rays accumulated
                const uint32_t n_last = s.last_n[prev];
                for (uint32_t k = threadIdx.x; k < n_last; k += blockDim.x)
                {
                    const uint32_t li = ended[slots_per_cta - 1u - k].x;
                    p.gather[li] = radiance[li];
                }
            }
        }
        if (total == 0u) break;            // no path alive and no sample left to start
        // ---------------------------------------------------------------- S(r): the hit queue, then the miss queue
        {
            const unsigned long long hm = s.hm[in];
            const uint32_t n_hit = (uint32_t)hm, n_miss = (uint32_t)(hm >> 32);
            const uint32_t hit_span = (n_hit + 31u) & ~31u;            // warps never mix hits and misses
            const uint32_t total_s = hit_span + n_miss;
            uint2* const list = lists + in * slots_per_cta;
            if (threadIdx.x == 0) { s.cur_trace = 0; s.hm[prev] = 0ull; }
            for (uint32_t at; (at = warp_grab(&s.cur_shade)) < total_s;)
            {
                uint32_t li = 0, state = 0;
                if (at < hit_span)
                {
                    const uint32_t k = at + lane;
                    const bool hit = k < n_hit;
                    float4 h = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
                    if (hit) h = q.hitq[base + k];
                    const bool ends = shade_hit_regen(p, sc, aov, q, base, in, max_bounces, hit, h, __float_as_uint(h.w), radiance, s, li, state);
                    record_ended(s, list, slots_per_cta, in, ends, li, state >> 8, n_samples, p.gather != nullptr);
                }
                else
                {   // ShadeMissedRays (shade_miss) with the path state; the last sample's pixel is final here
                    const uint32_t k = at - hit_span + lane;
                    const bool miss = k < n_miss;
                    if (miss)
                    {
                        const uint32_t slot = base + q.missq[base + k];
                        const float4 b = q.B[in][slot], c = q.C[in][slot];
                        const f3 sky = p.white_furnace ? splat(0.5f) : sample_sky(sc, mk3(b));
                        li = local_index(p, __float_as_uint(b.w)); state = __float_as_uint(c.w);
                        const float4 rr = add_radiance(radiance, li, sky * mk3(c));
                        if (p.gather && (state >> 8) + 1u == n_samples) p.gather[li] = rr;
                    }
                    count_keyed(s.n_miss, state & 0xFFu, __match_any_sync(0xffffffffu, state & 0xFFu), miss);
                    record_ended(s, list, slots_per_cta, in, miss, li, state >> 8, n_samples, false);
                }
            }
            __syncthreads();
            if (threadIdx.x == 0)
            {
                const unsigned long long em = s.emit[in];
                s.shadow_n[in] = (uint32_t)em; s.ext_n[prev] = (uint32_t)(em >> 32);
            }
            __syncthreads();
        }
    }
    // per-bounce statistics (rt_read_frame_stats): one global add per CTA and non-zero counter
    for (uint32_t b = threadIdx.x; b <= max_bounces; b += blockDim.x)
    {
        if (s.n_hit[b]) atomicAdd(&ctr->hm[b].hit, s.n_hit[b]);
        if (s.n_miss[b]) atomicAdd(&ctr->hm[b].miss, s.n_miss[b]);
        if (s.n_emissive[b]) atomicAdd(&ctr->n_emissive[b], s.n_emissive[b]);
        if (s.n_shadow[b]) atomicAdd(&ctr->emit[b].shadow, s.n_shadow[b]);
        if (s.n_cont[b]) atomicAdd(&ctr->emit[b].next, s.n_cont[b]);
        if (s.n_unoccluded[b]) atomicAdd(&ctr->n_unoccluded[b], s.n_unoccluded[b]);
    }
}
