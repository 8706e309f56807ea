/*
 * rt_traverse.cuh — BVH staging (TMA bulk copies), the traversal steps, and the traversal functions built from them: literal
 * reference-order traversal, the child-box layout traversal, the two-level instanced traversal, and trace_staged, the traversal call
 * of every kernel.
 * Part of the single translation unit rt_kernels.cu (included there, inside its anonymous namespace).
 */
#pragma once

#include "rt_octant.h"

// ------------------------------------------------------------------------------------ TMA staging of a small BVH
// When the whole traversal structure (interior records + triangle records) is small enough, every CTA of a
// traversal kernel copies it ONCE into shared memory with two TMA bulk copies (cp.async.bulk, completion signalled
// through an mbarrier transaction count) issued by one elected thread, and all node / triangle fetches of the
// kernel become shared-memory loads: the L1 data pipe is the second-busiest unit of the traversal kernels (ncu:
// l1tex data-pipe wavefronts ~58 % of peak, a divergent LDG.128 touches one 128-byte line per active lane), while a
// 16-byte LDS from 32 different records needs 4 conflict-free wavefronts.  The kernels are persistent, so the copy
// is amortised over every ray the CTA traces.
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// SMEM 1 stages the whole structure (records, then triangles: two bulk copies), SMEM 2 the first sc.top_k interior records —
// breadth-first, the top of the tree (rt_bvh_layout.h) — with one bulk copy, deeper records and all triangles staying behind
// L1/L2 (RT_OPT_TOP_SMEM); SMEM 0 stages nothing.  SMEM 3 stages what SMEM 1 does and then builds, behind the triangles, the
// eight octant-ordered copies of the interior records (rt_octant.h; table s at dst + wnodes_f4 + wtris_f4 + s * wnodes_f4) and
// one flag word behind them: 1 when every record passed rt_oct_record_ok and the tables exist, 0 when the CTA must not use them.
// The staging mode of the traversal kernels of instanced scenes (rt_upload_instanced_scene): nothing is staged and the two-level
// traversal (trace_instanced) runs.  Those kernels take a DevInstScene: DevScene describes the concatenated meshes (nodes_ref,
// tris_ref, wnodes, wtris, tri_shade) and the fields below the instances.  The flat kernels keep DevScene, so their parameters
// and code are unchanged.
#define RT_SMEM_INST 4
struct DevInstScene : DevScene
{
    const float4* inst_hdr;        // 3 float4: (top root box min xyz, root ref), (root box max xyz, instance count) as int bits,
                                   // (slack a, slack b, -, -) of rt_instances.h
    const float4* top;             // top-level records (rt_bvh_layout.h layout, leaf ref = ~instance), rt_instances.h
    const float4* irec;            // 8 float4 per instance: W rows, M rows, (mesh root ref, mesh record base in float4, first
                                   // triangle, base) as int bits, (det sign, first node bits, material row offset, -): the row
                                   // offset r * n_materials of rt_set_instance_materials as uint bits, RT_INVALID_ID for none
    const uint32_t* ibase;         // base (first virtual triangle id) per instance, ascending
    const float4* prev_tri;        // RT_OPT_OBJECT_MOTION: the previous positions of every mesh triangle (tris_ref layout); else nullptr
    const uint32_t* mtl_map;       // rt_set_instance_materials: the remap rows, row offset + scene material id -> material id;
                                   // nullptr before the first assignment (every row offset is then RT_INVALID_ID)
};
template <bool INST> using SceneOf = typename std::conditional<INST, DevInstScene, DevScene>::type;

template <int SMEM>
__device__ __forceinline__ void stage_bvh(float4* dst, const DevScene& sc, uint64_t* mbar)
{
    if (SMEM == 0 || SMEM == RT_SMEM_INST) return;
    const uint32_t bar = smem_u32(mbar);
    constexpr bool WHOLE = SMEM == 1 || SMEM == 3;
    const uint32_t nodes_bytes = (WHOLE ? sc.wnodes_f4 : sc.top_k * 4u) * 16u, tris_bytes = WHOLE ? sc.wtris_f4 * 16u : 0u;
    if (threadIdx.x == 0)
    {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(1));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0)
    {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(nodes_bytes + tris_bytes) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(smem_u32(dst)), "l"(sc.wnodes), "r"(nodes_bytes), "r"(bar) : "memory");
        if (WHOLE)
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(smem_u32(dst + sc.wnodes_f4)), "l"(sc.wtris), "r"(tris_bytes), "r"(bar) : "memory");
    }
    uint32_t done = 0;
    while (!done)
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                     : "=r"(done) : "r"(bar), "r"(0) : "memory");
    if (SMEM == 3)
    {   // every thread has seen the copies complete: build the 4-wide octant tables (rt_octant.h) from the staged records
        const uint32_t n = sc.root_ref < 0 ? 0u : sc.wnodes_f4 / 4u;      // a root-leaf tree has no interior record to visit
        float* recs = (float*)dst;
        float4* oct = dst + sc.wnodes_f4 + sc.wtris_f4;
        uint32_t* flag = (uint32_t*)(oct + 8u * sc.wnodes_f4);
        // Which records are wide nodes (even depth): parent links, then pointer jumping over the depth parity.  Scratch in the
        // table area, which is written only after the numbering: word = (ancestor + 1) << 1 | parity of the distance to it.
        uint32_t *link = (uint32_t*)oct, *next = link + n;
        for (uint32_t r = threadIdx.x; r < n; r += blockDim.x) link[r] = 0u;
        __syncthreads();
        bool ok = true;
        for (uint32_t r = threadIdx.x; r < n; r += blockDim.x)
            for (int c = 0; c < 2; ++c)
            {
                const int ref = __float_as_int(recs[16u * r + 12u + c]);
                if (ref >= 0) { if ((uint32_t)ref < n) link[ref] = ((r + 1u) << 1) | 1u; else ok = false; }
            }
        __syncthreads();
        for (int round = 0; round < 6; ++round)                          // 2^6 levels: trees are at most 64 deep (build_layout)
        {
            bool more = false;
            for (uint32_t r = threadIdx.x; r < n; r += blockDim.x)
            {
                const uint32_t w = link[r];
                const uint32_t up = (w >> 1) ? link[(w >> 1) - 1u] : 0u;
                next[r] = (w >> 1) ? ((up & ~1u) | ((w ^ up) & 1u)) : w;
                more = more || (up >> 1) != 0u;
            }
            uint32_t* t = link; link = next; next = t;
            if (!__syncthreads_or(more)) break;                           // every record has reached the root
        }
        // first slots: a prefix sum over the wide records in record order, by the first warp; kept in word 15 of each record
        if (threadIdx.x < 32u)
        {
            uint32_t base = 0;
            for (uint32_t r0 = 0; r0 < n; r0 += 32u)
            {
                const uint32_t r = r0 + threadIdx.x;
                const uint32_t w = r < n ? link[r] : 1u;
                const uint32_t cnt = (w & 1u) ? 0u : rt_wide_count(recs + 16u * r);
                uint32_t incl = cnt;
                for (int d = 1; d < 32; d <<= 1) { const uint32_t v = __shfl_up_sync(0xFFFFFFFFu, incl, d); if ((int)threadIdx.x >= d) incl += v; }
                if (r < n) recs[16u * r + 15u] = __uint_as_float(cnt ? base + incl - cnt : 0xFFFFFFFFu);
                ok = ok && !(w >> 1);                                    // every record reached the root (no cycle, not too deep)
                base += __shfl_sync(0xFFFFFFFFu, incl, 31);
            }
            ok = ok && base <= 2u * n;                                   // the tables' room (a tree takes at most 2n slots)
        }
        ok = __syncthreads_and(ok) != 0;
        if (ok)
            for (uint32_t i = threadIdx.x; i < 8u * n; i += blockDim.x)
            {
                const uint32_t r = i % n, s = i / n, slot = __float_as_uint(recs[16u * r + 15u]);
                if (s == 0u) ok = ok && rt_oct_record_ok(recs + 16u * r);
                if (slot == 0xFFFFFFFFu) continue;
                if (s == 0u) ok = ok && rt_wide_nests(recs + 16u * r, recs, n);
                rt_wide_node(recs, r, s, (float*)(oct + s * sc.wnodes_f4) + 8u * slot);
            }
        ok = __syncthreads_and(ok) != 0;
        if (threadIdx.x == 0) *flag = ok ? 1u : 0u;
        __syncthreads();
    }
}

// Programmatic dependent launch (RT_OPT_PDL): a kernel launched with the programmatic-stream-serialization attribute may
// start (launch its CTAs, stage the BVH) while the previous kernel of the stream is still draining; pdl_wait() blocks
// until that kernel has completed and its memory is visible, and is a no-op for a normal launch.  Every persistent
// kernel lets ITS dependent start as early as possible: its CTAs are all resident by then (persistent_grid), so
// the dependent's CTAs only take the slots that exiting CTAs free.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// SMEM: 0 records behind L1/L2 (ld.global.nc), 1 all records in shared memory, 2 the first sc.top_k interior records in shared
// memory and the rest in global memory (one generic load serves both)
template <int SMEM>
__device__ __forceinline__ float4 ld_bvh(const float4* p) { return SMEM ? *p : __ldg(p); }

// ------------------------------------------------------------------------------------ traversal steps
// The steps every traversal loop below is made of: the slab test of a box, the binary child-pair step, the pop of a deferred far
// child and the ray-triangle test.  One expression order each, shared by the literal, child-box and instanced traversals, which
// is what keeps them bit-identical.
// RT_FMA_TRAVERSAL (an experiment build, tools/build_variant.py; NOT bit-exact): contracted slab, cross and dot products.
#ifdef RT_FMA_TRAVERSAL
#define RT_CROSS(a, b) mk3(__fmaf_rn((a).y, (b).z, -((a).z * (b).y)), __fmaf_rn((a).z, (b).x, -((a).x * (b).z)), __fmaf_rn((a).x, (b).y, -((a).y * (b).x)))
#define RT_DOT(a, b) __fmaf_rn((a).x, (b).x, __fmaf_rn((a).y, (b).y, (a).z * (b).z))
#else
#define RT_CROSS(a, b) cross(a, b)
#define RT_DOT(a, b) dot(a, b)
#endif

// Slab interval [lo, hi] of the ray (o, inv = 1 / d) in the box (bmin, bmax), lo clamped below by t_min; the box is hit when
// fminf(hi, t_max) >= lo (inclusive).
__device__ __forceinline__ void slab(f3 bmin, f3 bmax, f3 o, f3 inv, float t_min, float& lo, float& hi)
{
#ifdef RT_FMA_TRAVERSAL
    // plane * inv - origin * inv in one FFMA per plane
    const f3 noi = mk3(-(o.x * inv.x), -(o.y * inv.y), -(o.z * inv.z));
    const f3 t0 = mk3(__fmaf_rn(bmin.x, inv.x, noi.x), __fmaf_rn(bmin.y, inv.y, noi.y), __fmaf_rn(bmin.z, inv.z, noi.z));
    const f3 t1 = mk3(__fmaf_rn(bmax.x, inv.x, noi.x), __fmaf_rn(bmax.y, inv.y, noi.y), __fmaf_rn(bmax.z, inv.z, noi.z));
#else
    const f3 t0 = (bmin - o) * inv, t1 = (bmax - o) * inv;
#endif
    lo = fmaxf(fmaxf(fmaxf(fminf(t0.x, t1.x), fminf(t0.y, t1.y)), fminf(t0.z, t1.z)), t_min);
    hi = fminf(fminf(fmaxf(t0.x, t1.x), fmaxf(t0.y, t1.y)), fmaxf(t0.z, t1.z));
}

// Does the ray hit the box (bmin, bmax) within [t_min, t_max]?
__device__ __forceinline__ bool box_hit(f3 bmin, f3 bmax, f3 o, f3 inv, float t_min, float t_max)
{
    float lo, hi;
    slab(bmin, bmax, o, inv, t_min, lo, hi);
    return fminf(hi, t_max) >= lo;
}

// Binary child-pair step on a child-box record (a, b, c, m) (rt_bvh_layout.h): both children's boxes tested, near and far
// child chosen by the ray's sign on the record's split axis (the second child is near iff inv[axis] < 0), and the far child's
// entry distance.  PACKED: the sign-bit form (sign_bits bit k: inv[k] < 0), for records in shared memory; otherwise predicate
// selects on the signs of inv (sign_bits unused), for records behind L1/L2 (trace_fast says why).
struct ChildPair { int near_ref, far_ref; bool near_hit, far_hit; float far_lo; };
template <bool PACKED>
__device__ __forceinline__ ChildPair child_pair(float4 a, float4 b, float4 c, float4 m, f3 o, f3 inv, uint32_t sign_bits, float t_min, float t_max)
{
    // child 0 box: min (a.x,a.y,a.z) max (a.w,b.x,b.y); child 1 box: min (b.z,b.w,c.x) max (c.y,c.z,c.w)
    float lo0, hi0, lo1, hi1;
    slab(mk3(a.x, a.y, a.z), mk3(a.w, b.x, b.y), o, inv, t_min, lo0, hi0);
    slab(mk3(b.z, b.w, c.x), mk3(c.y, c.z, c.w), o, inv, t_min, lo1, hi1);
    const bool h0 = fminf(hi0, t_max) >= lo0, h1 = fminf(hi1, t_max) >= lo1;
    const int r0 = __float_as_int(m.x), r1 = __float_as_int(m.y);
    const uint32_t axis = __float_as_uint(m.z);
    const bool swap = PACKED ? ((sign_bits >> axis) & 1u) != 0u : (axis == 0 ? inv.x < 0 : (axis == 1 ? inv.y < 0 : inv.z < 0));
    ChildPair s;
    s.near_ref = swap ? r1 : r0; s.far_ref = swap ? r0 : r1;
    s.near_hit = swap ? h1 : h0; s.far_hit = swap ? h0 : h1;
    s.far_lo = swap ? lo0 : lo1;
    return s;
}

// Pop: the deferred far child on top of the stack, as (reference, entry distance).  A pushed child is re-tested against the
// (possibly shrunk) t_max, as the reference does when it pops it; its slab interval was already valid at push time.  Entries
// that fail are dropped.  Returns false when the stack runs empty.  Two stack shapes: packed 64-bit entries, or two arrays.
__device__ __forceinline__ bool pop(const int2* stack, int& sp, float t_max, int& cur)
{
    while (sp > 0)
    {
        --sp;
        const int2 e = stack[sp];
        if (t_max >= __int_as_float(e.y)) { cur = e.x; return true; }
    }
    return false;
}
__device__ __forceinline__ bool pop(const int* stack_ref, const float* stack_t, int& sp, float t_max, int& cur)
{
    while (sp > 0) { --sp; if (t_max >= stack_t[sp]) { cur = stack_ref[sp]; return true; } }
    return false;
}

// Ray-triangle test (Möller-Trumbore) of the triangle (p1, e1 = p2 - p1, e2 = p3 - p1), inclusive, with back-face culling:
// det < 1e-8 rejects.  SIGNED (instanced scenes): the culling test reads det * cull (cull = sign(det M) of a mirrored instance:
// -1), so that a mirrored instance culls the faces its flattened triangles would; u, v and t still divide by det.  A hit with t
// in [t_min, t_max] calls hit(u, v, t) and returns true.  PIN: see trace_fast.
// The hit is handed to a callable rather than returned through references: a returned (u, v, t) joins the miss paths before
// the caller's branch, and ptxas then spills the closest-hit kernels at their 48 registers.
template <bool SIGNED, bool PIN = false, class Hit>
__device__ __forceinline__ bool tri_hit(f3 p1, f3 e1, f3 e2, f3 o, f3 d, float cull, float t_min, float t_max, Hit&& hit)
{
    const f3 pvec = RT_CROSS(d, e2);
    float det = RT_DOT(e1, pvec);
    if (PIN) asm volatile("" : "+f"(det));
    const float cdet = SIGNED ? det * cull : det;
    if (cdet < 1e-8f || -cdet > 1e-8f) return false;
    const float inv_det = 1.0f / det;
    const f3 tvec = o - p1;
    const float u = RT_DOT(tvec, pvec) * inv_det;
    if (u < 0.0f || u > 1.0f) return false;
    const f3 qvec = RT_CROSS(tvec, e1);
    const float v = RT_DOT(d, qvec) * inv_det;
    if (v < 0.0f || u + v > 1.0f) return false;
    const float t = RT_DOT(e2, qvec) * inv_det;
    if (t < t_min || t > t_max) return false;
    hit(u, v, t);
    return true;
}
#undef RT_CROSS
#undef RT_DOT

// ------------------------------------------------------------------------------------ traversal
// Literal restatement of kernels/cl/trace_bvh.cl:99-211 on the reference node layout: per-ray
// DFS, 64-entry private stack, far child pushed unconditionally and box-tested when popped,
// near child chosen by ray_sign[axis], inclusive tests, later equal-t hit overwrites, back-face
// culling (det < 1e-8 rejects, tri_hit).  ANY = the -D SHADOW_RAYS variant (returns 0 on first hit).
template <bool ANY, bool COUNT, bool SIGNED = false>
__device__ __forceinline__ uint32_t trace_literal(const DevScene& sc, f3 o, f3 d, float t_min, float t_max,
                                                  float& bu, float& bv, float& bt, uint32_t& nv, uint32_t& nt, float cull = 1.0f)
{
    f3 inv = splat(1.0f) / d;
    int sx = inv.x < 0, sy = inv.y < 0, sz = inv.z < 0;
    uint32_t prim = RT_INVALID_ID;
    int to_visit = 0, cur = 0;
    int stack[64];
    for (;;)
    {
        float4 n0 = __ldg(sc.nodes_ref + (size_t)cur * 3), n1 = __ldg(sc.nodes_ref + (size_t)cur * 3 + 1), n2 = __ldg(sc.nodes_ref + (size_t)cur * 3 + 2);
        if (COUNT) ++nv;
        bool box = box_hit(mk3(n0), mk3(n1), o, inv, t_min, t_max);
        uint32_t offset = __float_as_uint(n2.x), npa = __float_as_uint(n2.y);
        if (box)
        {
            int nprims = (int)(npa >> 16);
            if (nprims > 0)
            {
                for (int i = 0; i < nprims; ++i)
                {
                    const float4* tp = sc.tris_ref + (size_t)(offset + i) * 3;
                    f3 p1 = mk3(__ldg(tp)), p2 = mk3(__ldg(tp + 1)), p3 = mk3(__ldg(tp + 2));
                    if (COUNT) ++nt;
                    const bool hit = tri_hit<SIGNED>(p1, p2 - p1, p3 - p1, o, d, cull, t_min, t_max, [&](float u, float v, float t) {
                        bu = u; bv = v; bt = t;
                        prim = offset + i;
                        t_max = t;
                    });
                    if (ANY && hit) return 0u;
                }
                if (to_visit == 0) break;
                cur = stack[--to_visit];
            }
            else
            {
                uint32_t axis = npa & 0xFFFFu;
                int s = axis == 0 ? sx : (axis == 1 ? sy : sz);
                if (s) { stack[to_visit++] = cur + 1; cur = (int)offset; }
                else   { stack[to_visit++] = (int)offset; cur = cur + 1; }
            }
        }
        else
        {
            if (to_visit == 0) break;
            cur = stack[--to_visit];
        }
    }
    return prim;
}

// Optimised traversal on the child-box node layout (rt_bvh_layout.h).  Same visiting order and
// the same arithmetic per box / triangle test as trace_literal, so results are bit-identical
// for finite rays; non-finite rays (NaN/inf components; their traversal is garbage-in but must
// still match) take the literal path.
// PIN: the whole-frame kernel shares its register budget with the shading code and ptxas then re-derives the sign bits on
// every step and recomputes the determinant after its branch; an empty asm makes both values opaque (kept in registers).
// SMEM 3: `wnodes` and `wtris` are those of SMEM 1 and the 4-wide octant tables follow the triangles (stage_bvh).  The interior
// step reads the wide node from the table of the ray's octant, slab-tests its 2..4 children in the order the binary traversal
// visits them, continues into the first that hits and defers the others with their entry distances: the visits, hits and
// results of the binary traversal in about half the steps (tools/wide_bvh_model.cpp).  The ordered slab test takes the same
// decisions as the pairwise one for a ray that passes rt_oct_ray_ok on records that passed rt_oct_record_ok (rt_octant.h has
// the argument), and skipping a collapsed child's own box test is exact where rt_wide_nests holds.  Any other ray, and every
// ray of a CTA whose records failed, is traced by the SMEM 1 traversal on the canonical staged records (a loop of its own: a
// branch inside the ordered loop was measured and cost half the gain):
// exactly what RT_OPT_OCTANT_BVH 0 computes, also where that differs from the literal traversal (a NaN t_max from a triangle
// with an infinite vertex ends the staged traversal and not the literal one).
template <bool ANY, bool COUNT, int SMEM, bool PIN = false, bool SIGNED = false>
__device__ __forceinline__ uint32_t trace_fast(const DevScene& sc, const float4* wnodes, const float4* wtris, f3 o, f3 d, float t_min, float t_max,
                                               float& bu, float& bv, float& bt, uint32_t& nv, uint32_t& nt, float cull = 1.0f)
{
    constexpr bool OCT = SMEM == 3, PACKED = SMEM == 1 || OCT;
    float fin = ((o.x + o.y) + o.z) + ((d.x + d.y) + d.z);
    if (!(fabsf(fin) <= 3.0e38f) || COUNT)
        return trace_literal<ANY, COUNT, SIGNED>(sc, o, d, t_min, t_max, bu, bv, bt, nv, nt, cull);

    f3 inv = splat(1.0f) / d;
    if (OCT && !(rt_oct_ray_ok(inv.x, inv.y, inv.z) && (!ANY || t_max == t_max) && *(const uint32_t*)(wtris + sc.wtris_f4 + 8u * sc.wnodes_f4) != 0u))
        return trace_fast<ANY, COUNT, OCT ? 1 : SMEM, PIN, SIGNED>(sc, wnodes, wtris, o, d, t_min, t_max, bu, bv, bt, nv, nt, cull);
    const bool sx = inv.x < 0, sy = inv.y < 0, sz = inv.z < 0;
    uint32_t sign_bits = (sx ? 1u : 0u) | (sy ? 2u : 0u) | (sz ? 4u : 0u);
    if (PIN) asm volatile("" : "+r"(sign_bits));
    uint32_t prim = RT_INVALID_ID;
    int sp = 0;
    int cur = sc.root_ref;
    // Deferred far children: (node reference, entry distance).  Two code shapes, chosen by where the BVH records live
    // (measured, same results): with the records in shared memory the kernel is purely issue-bound and the packed
    // 64-bit stack entry + the sign-bit axis test win (CornellBox frame -2.7 %); with the records behind L1/L2 the two
    // 32-bit arrays (a discarded pop costs one load) and predicate selects are faster (ShaderBalls +1 %, Dragon +3.5 %).
    // A wide step can defer up to three children where the binary one defers one, so SMEM 3 has twice the 64 binary entries.
    int2 stack[OCT && !ANY ? 128 : PACKED && !OCT ? 64 : 1];
    // An any-hit ray returns at its first hit, so its t_max never shrinks and every deferred child passes the pop test (its entry
    // distance was at most t_max when it was pushed): SMEM 3 keeps only the references.  A NaN t_max, which the pop test would
    // reject, takes the SMEM 1 loop (the guard above).
    int any_stack[OCT && ANY ? 128 : 1];
    int stack_ref[PACKED ? 1 : 64];
    float stack_t[PACKED ? 1 : 64];
    // the records of this ray's octant, as an offset from the canonical ones; opaque, so that it stays in a register instead of
    // being re-derived from the sign bits and the two sizes on every step
    uint32_t oct_at = OCT ? sc.wnodes_f4 + sc.wtris_f4 + sign_bits * sc.wnodes_f4 : 0u;
    if (OCT) asm volatile("" : "+r"(oct_at));
    // root box (the reference tests every node it visits, including the root; a single-leaf tree has nothing else to test)
    if (!box_hit(mk3(__ldg(sc.nodes_ref)), mk3(__ldg(sc.nodes_ref + 1)), o, inv, t_min, t_max)) return prim;
    for (;;)
    {
        while (cur >= 0)
        {
            if (OCT)
            {   // the wide node at slot `cur` of this ray's table: 2..4 slots of (entry xyz, exit | exit yz, ref, count), in visiting order
                // The children are tested last to first: each hit defers the one found before it, so the first child that hits
                // is continued into and the other hit children are deferred in reverse order, with no per-child state kept.
                // An any-hit ray tests them first to last instead and so walks the tree far to near: its t_max never changes,
                // so every box test has the same outcome in any order and the ray reaches the same leaves, but a shadow ray
                // that starts on a surface is usually stopped by what lies far from its origin (a wall, the ceiling), and
                // the near subtrees, which hold the surface it leaves, are then never walked.
                const float4* np = wnodes + (oct_at + (uint32_t)cur * 2u);
                const uint32_t cnt = __float_as_uint(np[1].w);
                bool found = false;
                int next_ref = 0;
                float next_lo = 0.0f;
#pragma unroll
                for (int k = 0; k < 4; ++k)
                {
                    const int j = ANY ? k : 3 - k;
                    if (j >= 2 && (uint32_t)j >= cnt) continue;
                    const float4 p = np[2 * j], q = np[2 * j + 1];
                    float lo, hi;
                    rt_slab_ordered(p.x, p.y, p.z, p.w, q.x, q.y, o.x, o.y, o.z, inv.x, inv.y, inv.z, t_min, lo, hi);
                    if (fminf(hi, t_max) >= lo)
                    {
                        if (found)
                        {
                            if (ANY) any_stack[sp] = next_ref; else stack[sp] = make_int2(next_ref, __float_as_int(next_lo));
                            ++sp;
                        }
                        next_ref = __float_as_int(q.z); next_lo = lo; found = true;
                    }
                }
                if (found) { cur = next_ref; continue; }
                if (ANY) { if (sp == 0) return prim; cur = any_stack[--sp]; continue; }
                if (!pop(stack, sp, t_max, cur)) return prim;
                continue;
            }
            // SMEM == 2: `wnodes` is the staged top of the tree (records [0, sc.top_k)), deeper records come from sc.wnodes
            const float4* np = (SMEM == 2 && (uint32_t)cur >= sc.top_k) ? sc.wnodes + (size_t)cur * 4 : wnodes + (size_t)cur * 4;
            const ChildPair s = child_pair<PACKED>(ld_bvh<SMEM>(np), ld_bvh<SMEM>(np + 1), ld_bvh<SMEM>(np + 2), ld_bvh<SMEM>(np + 3),
                                                   o, inv, sign_bits, t_min, t_max);
            if (s.near_hit)
            {
                if (s.far_hit)
                {
                    if (PACKED) stack[sp] = make_int2(s.far_ref, __float_as_int(s.far_lo));
                    else { stack_ref[sp] = s.far_ref; stack_t[sp] = s.far_lo; }
                    ++sp;
                }
                cur = s.near_ref;
            }
            else if (s.far_hit) cur = s.far_ref;
            else if (!(PACKED ? pop(stack, sp, t_max, cur) : pop(stack_ref, stack_t, sp, t_max, cur))) return prim;
        }
        // leaf: triangles [~cur ...] until the end-of-leaf flag
        uint32_t ti = (uint32_t)(~cur);
        for (;;)
        {
            const float4* tp = wtris + (size_t)ti * 3;
            float4 q0 = ld_bvh<PACKED>(tp), q1 = ld_bvh<PACKED>(tp + 1), q2 = ld_bvh<PACKED>(tp + 2);
            bool last = __float_as_uint(q2.y) != 0u;
            const bool hit = tri_hit<SIGNED, PIN>(mk3(q0.x, q0.y, q0.z), mk3(q0.w, q1.x, q1.y), mk3(q1.z, q1.w, q2.x), o, d, cull, t_min, t_max,
                                                  [&](float u, float v, float t) { bu = u; bv = v; bt = t; prim = ti; t_max = t; });
            if (ANY && hit) return 0u;
            if (last) break;
            ++ti;
        }
        if (OCT && ANY) { if (sp == 0) return prim; cur = any_stack[--sp]; continue; }
        if (!(PACKED ? pop(stack, sp, t_max, cur) : pop(stack_ref, stack_t, sp, t_max, cur))) return prim;
    }
}

// Two-level traversal of an instanced scene (rt_b200.h, instanced scenes).  The top-level tree is walked as trace_fast walks a
// flat one from L1 (same slab test, near/far order, pop rule and 64-entry stack), on every box widened by the ray's slack
// e = max|o| * a + b (rt_instances.h: no box culls a hit the mesh's tree finds); at an instance leaf the ray is moved into
// object space by W and the mesh's tree is traced by trace_fast itself, on a view of DevScene whose arrays start at the mesh's,
// with the shared t_max and a stack of its own.  A hit stores the instance's virtual id, base + the mesh's triangle index.
// COUNT counts every node whose box is tested once: the top-level root (the header box) and the two children of each top-level
// record visited, then the mesh nodes of trace_literal (trace_fast's counting path; it tests the mesh's root box again).
template <bool ANY, bool COUNT>
__device__ __forceinline__ uint32_t trace_instanced(const DevInstScene& sc, f3 o, f3 d, float t_min, float t_max,
                                                    float& bu, float& bv, float& bt, uint32_t& nv, uint32_t& nt)
{
    uint32_t prim = RT_INVALID_ID;
    const float4 h0 = __ldg(sc.inst_hdr), h1 = __ldg(sc.inst_hdr + 1), h2 = __ldg(sc.inst_hdr + 2);
    if (__float_as_uint(h1.w) == 0u) return prim;                  // no instances: every ray misses
    const f3 inv = splat(1.0f) / d;
    const float e = fmaxf(fmaxf(fabsf(o.x), fabsf(o.y)), fabsf(o.z)) * h2.x + h2.y;
    if (COUNT) ++nv;
    if (!box_hit(mk3(h0.x - e, h0.y - e, h0.z - e), mk3(h1.x + e, h1.y + e, h1.z + e), o, inv, t_min, t_max)) return prim;   // root box
    int cur = __float_as_int(h0.w);
    int sp = 0;
    int stack_ref[64];
    float stack_t[64];
    for (;;)
    {
        while (cur >= 0)
        {
            const float4* np = sc.top + (size_t)cur * 4;
            if (COUNT) nv += 2;
            const float4 a = __ldg(np), b = __ldg(np + 1), c = __ldg(np + 2);
            // child 0: min (a.x, a.y, a.z) max (a.w, b.x, b.y); child 1: min (b.z, b.w, c.x) max (c.y, c.z, c.w)
            const ChildPair s = child_pair<false>(make_float4(a.x - e, a.y - e, a.z - e, a.w + e), make_float4(b.x + e, b.y + e, b.z - e, b.w - e),
                                                  make_float4(c.x - e, c.y + e, c.z + e, c.w + e), __ldg(np + 3), o, inv, 0u, t_min, t_max);
            if (s.near_hit)
            {
                if (s.far_hit) { stack_ref[sp] = s.far_ref; stack_t[sp] = s.far_lo; ++sp; }
                cur = s.near_ref;
            }
            else if (s.far_hit) cur = s.far_ref;
            else if (!pop(stack_ref, stack_t, sp, t_max, cur)) return prim;
        }
        {   // instance leaf: the ray in object space, then the mesh's tree
            const float4* ir = sc.irec + (size_t)(~cur) * 8;
            const float4 w0 = __ldg(ir), w1 = __ldg(ir + 1), w2 = __ldg(ir + 2), mi = __ldg(ir + 6), mj = __ldg(ir + 7);
            const f3 oo = mk3(((w0.x * o.x + w0.y * o.y) + w0.z * o.z) + w0.w, ((w1.x * o.x + w1.y * o.y) + w1.z * o.z) + w1.w,
                              ((w2.x * o.x + w2.y * o.y) + w2.z * o.z) + w2.w);
            const f3 od = mk3((w0.x * d.x + w0.y * d.y) + w0.z * d.z, (w1.x * d.x + w1.y * d.y) + w1.z * d.z, (w2.x * d.x + w2.y * d.y) + w2.z * d.z);
            const uint32_t rec = __float_as_uint(mi.y), first = __float_as_uint(mi.z);
            DevScene ms = sc;
            ms.root_ref = __float_as_int(mi.x);
            ms.wnodes = sc.wnodes + rec; ms.wtris = sc.wtris + (size_t)first * 3;
            ms.tris_ref = sc.tris_ref + (size_t)first * 3; ms.nodes_ref = sc.nodes_ref + (size_t)__float_as_uint(mj.y) * 3;
            float u, v, t;
            const uint32_t p = trace_fast<ANY, COUNT, 0, false, true>(ms, ms.wnodes, ms.wtris, oo, od, t_min, t_max, u, v, t, nv, nt, mj.x);
            if (p != RT_INVALID_ID)
            {
                if (ANY) return 0u;
                prim = __float_as_uint(mi.w) + p; bu = u; bv = v; bt = t; t_max = t;
            }
        }
        if (!pop(stack_ref, stack_t, sp, t_max, cur)) return prim;
    }
}

// The traversal call of every persistent kernel, for the kernel's staging mode (stage_bvh): ray (a, b) = (origin, -), (dir, w).
// A shadow ray (ANY) carries its t_max in b.w; an extension ray carries its pixel there, and its t_max is RT_MAX_RENDER_DIST.
// SMEM 0: mode 0 (RT_OPT_TRAVERSAL 0) is the literal traversal, otherwise trace_fast from L1/L2; s_bvh is not read.  PIN
// (trace_fast) is applied to the staged modes only.  RT_SMEM_INST: sc is a DevInstScene, and mode and s_bvh are not read.
template <bool ANY, bool COUNT, int SMEM, bool PIN, class Scene>
__device__ __forceinline__ uint32_t trace_staged(const Scene& sc, int mode, const float4* s_bvh, float4 a, float4 b,
                                                 float& bu, float& bv, float& bt, uint32_t& nv, uint32_t& nt)
{
    const float t_max = ANY ? b.w : RT_MAX_RENDER_DIST;
    if constexpr (SMEM == RT_SMEM_INST) return trace_instanced<ANY, COUNT>(sc, mk3(a), mk3(b), 0.0f, t_max, bu, bv, bt, nv, nt);
    else {
    if (SMEM == 1 || SMEM == 3) return trace_fast<ANY, COUNT, SMEM, PIN>(sc, s_bvh, s_bvh + sc.wnodes_f4, mk3(a), mk3(b), 0.0f, t_max, bu, bv, bt, nv, nt);
    if (SMEM == 2) return trace_fast<ANY, COUNT, 2, PIN>(sc, s_bvh, sc.wtris, mk3(a), mk3(b), 0.0f, t_max, bu, bv, bt, nv, nt);
    if (mode == 0) return trace_literal<ANY, COUNT>(sc, mk3(a), mk3(b), 0.0f, t_max, bu, bv, bt, nv, nt);
    return trace_fast<ANY, COUNT, 0>(sc, sc.wnodes, sc.wtris, mk3(a), mk3(b), 0.0f, t_max, bu, bv, bt, nv, nt);
    }
}
