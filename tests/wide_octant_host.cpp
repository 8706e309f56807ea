/* tests/wide_octant_host.cpp — TEST INFRASTRUCTURE: the 4-wide octant tables of raytracing_b200/csrc/rt_octant.h (the code the
 * traversal kernels compile) behind C entry points for tests/test_wide_octant_cpu.py: the tables a CTA builds in stage_bvh<3>,
 * and trace_fast's walk of them. */
#include <cstdint>
#include <cstring>
#include <vector>
#include "rt_octant.h"

static uint32_t bits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

/* The tables of the n canonical records recs_in (16 floats each): recs_out = the records with word 15 set as stage_bvh<3> sets
 * it (first slot of a wide node, else 0xFFFFFFFF), tables = 8 tables of 2n slots (8 floats each; slots past *n_slots are left
 * as they are).  The wide nodes are found here by walking parent links (stage_bvh<3> jumps pointers).  Returns 1 when the tables
 * may be used: references in range, a tree at most 64 deep, every record passes rt_oct_record_ok and every wide node
 * rt_wide_nests; 0 otherwise (the tables are then not written). */
extern "C" int wide_tables(const float* recs_in, uint32_t n, float* recs_out, float* tables, uint32_t* n_slots)
{
    memcpy(recs_out, recs_in, (size_t)n * 64);
    std::vector<int64_t> parent(n, -1);
    for (uint32_t r = 0; r < n; ++r)
        for (int c = 0; c < 2; ++c)
        {
            const int ref = (int)bits(recs_in[16 * r + 12 + c]);
            if (ref < 0) continue;
            if ((uint32_t)ref >= n) return 0;
            parent[ref] = r;
        }
    uint32_t slot = 0;
    for (uint32_t r = 0; r < n; ++r)
    {
        uint32_t depth = 0;
        for (int64_t p = parent[r]; p >= 0; p = parent[p])
            if (++depth > 64) return 0;
        const uint32_t first = (depth & 1u) ? 0xFFFFFFFFu : slot;
        if (!(depth & 1u)) slot += rt_wide_count(recs_in + 16 * r);
        memcpy(recs_out + 16 * r + 15, &first, 4);
    }
    *n_slots = slot;
    if (slot > 2 * n) return 0;
    bool ok = true;
    for (uint32_t r = 0; r < n; ++r)
    {
        ok = ok && rt_oct_record_ok(recs_out + 16 * r);
        if (bits(recs_out[16 * r + 15]) != 0xFFFFFFFFu) ok = ok && rt_wide_nests(recs_out + 16 * r, recs_out, n);
    }
    if (!ok) return 0;
    for (uint32_t s = 0; s < 8; ++s)
        for (uint32_t r = 0; r < n; ++r)
        {
            const uint32_t first = bits(recs_out[16 * r + 15]);
            if (first != 0xFFFFFFFFu) rt_wide_node(recs_out, r, s, tables + ((size_t)s * 2 * n + first) * 8);
        }
    return 1;
}

/* trace_fast<ANY, false, 3>'s walk on the host: tables of n records (wide_tables), the triangle records of rt_bvh_layout.h (12
 * floats each), root_box = the root's min xyz, max xyz (tested pairwise first), rays (origin 3, direction 3, t_max).  Rays that
 * fail rt_oct_ray_ok are not walked, nor any-hit rays with a NaN t_max: status 0.  prim = 0xFFFFFFFF for a miss; any_hit: prim = 0 on the first hit, as the
 * device's ANY returns.  counts[0] += wide nodes visited, counts[1] += child boxes tested, counts[2] += deepest stack. */
extern "C" void wide_walk(const float* tables, uint32_t n, const float* tris, int root_ref, const float* root_box, uint64_t n_rays,
                          const float* o, const float* d, const float* t_max_in, int any_hit, uint32_t* prim_out, float* uvt_out,
                          uint8_t* status, uint64_t* counts)
{
    for (uint64_t i = 0; i < n_rays; ++i)
    {
        const float *oi = o + 3 * i, *di = d + 3 * i;
        const float inv[3] = { 1.0f / di[0], 1.0f / di[1], 1.0f / di[2] };
        uint32_t prim = 0xFFFFFFFFu; float bu = 0, bv = 0, bt = 0;
        prim_out[i] = prim; uvt_out[3 * i] = uvt_out[3 * i + 1] = uvt_out[3 * i + 2] = 0.0f;
        status[i] = rt_oct_ray_ok(inv[0], inv[1], inv[2]) && (!any_hit || t_max_in[i] == t_max_in[i]);
        if (!status[i]) continue;
        const float* base = tables + (size_t)rt_oct_octant(inv[0], inv[1], inv[2]) * 2 * n * 8;
        float t_max = t_max_in[i];
        int cur = root_ref, sp = 0, stack_ref[128]; float stack_t[128];
        float rlo, rhi;
        rt_slab_pairwise(root_box, oi[0], oi[1], oi[2], inv[0], inv[1], inv[2], 0.0f, rlo, rhi);
        bool done = !(rt_oct_min(rhi, t_max) >= rlo);
        while (!done)
        {
            while (cur >= 0)
            {   // children last to first: each hit defers the one found before it
                const float* np = base + (size_t)cur * 8;
                const uint32_t cnt = bits(np[7]);
                ++counts[0]; counts[1] += cnt;
                bool found = false; int next_ref = 0; float next_lo = 0.0f;
                for (int j = (int)cnt - 1; j >= 0; --j)
                {
                    const float* q = np + 8 * j;
                    float lo, hi;
                    rt_slab_ordered(q[0], q[1], q[2], q[3], q[4], q[5], oi[0], oi[1], oi[2], inv[0], inv[1], inv[2], 0.0f, lo, hi);
                    if (rt_oct_min(hi, t_max) >= lo)
                    {
                        if (found) { stack_ref[sp] = next_ref; stack_t[sp] = next_lo; ++sp; if ((uint64_t)sp > counts[2]) counts[2] = sp; }
                        next_ref = (int)bits(q[6]); next_lo = lo; found = true;
                    }
                }
                if (found) { cur = next_ref; continue; }
                if (any_hit) { if (sp == 0) { done = true; break; } cur = stack_ref[--sp]; continue; }   // t_max never shrank: no pop test
                while (sp > 0) { --sp; if (t_max >= stack_t[sp]) { cur = stack_ref[sp]; found = true; break; } }
                if (!found) { done = true; break; }
            }
            if (done) break;
            for (uint32_t ti = (uint32_t)~cur;; ++ti)
            {   // the triangle test of trace_fast on (p1, e1, e2, end-of-leaf flag)
                const float* q = tris + 12 * (size_t)ti;
                const float p1[3] = { q[0], q[1], q[2] }, e1[3] = { q[3], q[4], q[5] }, e2[3] = { q[6], q[7], q[8] };
                const float pv[3] = { di[1] * e2[2] - di[2] * e2[1], di[2] * e2[0] - di[0] * e2[2], di[0] * e2[1] - di[1] * e2[0] };
                const float det = e1[0] * pv[0] + e1[1] * pv[1] + e1[2] * pv[2];
                if (!(det < 1e-8f || -det > 1e-8f))
                {
                    const float inv_det = 1.0f / det;
                    const float tv[3] = { oi[0] - p1[0], oi[1] - p1[1], oi[2] - p1[2] };
                    const float u = (tv[0] * pv[0] + tv[1] * pv[1] + tv[2] * pv[2]) * inv_det;
                    if (!(u < 0.0f || u > 1.0f))
                    {
                        const float qv[3] = { tv[1] * e1[2] - tv[2] * e1[1], tv[2] * e1[0] - tv[0] * e1[2], tv[0] * e1[1] - tv[1] * e1[0] };
                        const float v = (di[0] * qv[0] + di[1] * qv[1] + di[2] * qv[2]) * inv_det;
                        if (!(v < 0.0f || u + v > 1.0f))
                        {
                            const float t = (e2[0] * qv[0] + e2[1] * qv[1] + e2[2] * qv[2]) * inv_det;
                            if (!(t < 0.0f || t > t_max))
                            {
                                bu = u; bv = v; bt = t; prim = ti; t_max = t;
                                if (any_hit) { prim = 0; done = true; break; }
                            }
                        }
                    }
                }
                if (bits(q[9]) != 0u) break;
            }
            if (done) break;
            if (any_hit) { if (sp == 0) break; cur = stack_ref[--sp]; continue; }
            bool found = false;
            while (sp > 0) { --sp; if (t_max >= stack_t[sp]) { cur = stack_ref[sp]; found = true; break; } }
            if (!found) done = true;
        }
        prim_out[i] = prim; uvt_out[3 * i] = bu; uvt_out[3 * i + 1] = bv; uvt_out[3 * i + 2] = bt;
    }
}
