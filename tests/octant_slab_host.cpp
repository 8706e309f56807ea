/* tests/octant_slab_host.cpp — TEST INFRASTRUCTURE: raytracing_b200/csrc/rt_octant.h (the octant-ordered interior records and
 * both slab tests, the code the traversal kernels compile) behind C entry points for tests/test_octant_slab_cpu.py. */
#include <cstdint>
#include <cstring>
#include <vector>
#include "rt_octant.h"

static uint32_t bits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static bool same_number(float a, float b) { return (a != a && b != b) || a == b; }      // +0 == -0: rt_octant.h says why

// One node step both ways.  Pairwise: the canonical record and trace_fast's near/far selection by the split axis' sign;
// ordered: the record of the ray's octant.  out[0..5] = near_hit, far_hit, near_ref, far_ref, lo_n bits, lo_f bits, hi_n, hi_f
static void step_pairwise(const float* rec, const float* o, const float* inv, float t_min, float t_max, uint32_t* out)
{
    float lo[2], hi[2];
    for (int c = 0; c < 2; ++c) rt_slab_pairwise(rec + 6 * c, o[0], o[1], o[2], inv[0], inv[1], inv[2], t_min, lo[c], hi[c]);
    uint32_t axis; memcpy(&axis, rec + 14, 4);
    const uint32_t swap = (rt_oct_octant(inv[0], inv[1], inv[2]) >> axis) & 1u;
    const uint32_t n = swap, f = swap ^ 1u;
    out[0] = rt_oct_min(hi[n], t_max) >= lo[n]; out[1] = rt_oct_min(hi[f], t_max) >= lo[f];
    out[2] = bits(rec[12 + n]); out[3] = bits(rec[12 + f]);
    out[4] = bits(lo[n]); out[5] = bits(lo[f]); out[6] = bits(hi[n]); out[7] = bits(hi[f]);
}

static void step_ordered(const float* r, const float* o, const float* inv, float t_min, float t_max, uint32_t* out)
{
    float lo[2], hi[2];
    for (int c = 0; c < 2; ++c)
        rt_slab_ordered(r[6 * c], r[6 * c + 1], r[6 * c + 2], r[6 * c + 3], r[6 * c + 4], r[6 * c + 5], o[0], o[1], o[2], inv[0], inv[1], inv[2], t_min, lo[c], hi[c]);
    out[0] = rt_oct_min(hi[0], t_max) >= lo[0]; out[1] = rt_oct_min(hi[1], t_max) >= lo[1];
    out[2] = bits(r[12]); out[3] = bits(r[13]);
    out[4] = bits(lo[0]); out[5] = bits(lo[1]); out[6] = bits(hi[0]); out[7] = bits(hi[1]);
}

/* n cases: canonical record (16 floats), origin (3), reciprocal direction (3), t_max.  Per case: ray_ok, rec_ok (the two guards)
 * and differs: bit 0 a hit decision or a child reference differs, bit 1 an interval bound is a different number, bit 2 an
 * interval bound has different bits (a superset of bit 1: it also sees the sign of a zero). */
extern "C" void octant_compare(uint64_t n, const float* recs, const float* o, const float* inv, const float* t_max,
                               uint8_t* ray_ok, uint8_t* rec_ok, uint8_t* differs)
{
    for (uint64_t i = 0; i < n; ++i)
    {
        const float *rec = recs + 16 * i, *oi = o + 3 * i, *ii = inv + 3 * i;
        ray_ok[i] = rt_oct_ray_ok(ii[0], ii[1], ii[2]); rec_ok[i] = rt_oct_record_ok(rec);
        uint32_t axis; memcpy(&axis, rec + 14, 4);
        if (axis > 2u) { differs[i] = 0; continue; }          // no table is built from such a record
        float ord[16];
        rt_oct_order(rec, rt_oct_octant(ii[0], ii[1], ii[2]), ord);
        uint32_t a[8], b[8];
        step_pairwise(rec, oi, ii, 0.0f, t_max[i], a); step_ordered(ord, oi, ii, 0.0f, t_max[i], b);
        uint8_t d = 0;
        for (int k = 0; k < 4; ++k) if (a[k] != b[k]) d |= 1;
        for (int k = 4; k < 8; ++k)
        {
            float x, y; memcpy(&x, &a[k], 4); memcpy(&y, &b[k], 4);
            if (!same_number(x, y)) d |= 2;
            if (a[k] != b[k] && !(x != x && y != y)) d |= 4;
        }
        differs[i] = d;
    }
}

/* The traversal of trace_fast on the host: n_rec canonical records, the triangle records of rt_bvh_layout.h (12 floats each),
 * root_box = the root's min xyz, max xyz (tested pairwise first, as trace_fast does), closest hit of n rays (origin 3, direction 3, t_max).  use_tables: rays that pass the guard walk the eight ordered tables
 * (built here with rt_oct_order, as a CTA does after staging), the others — and every ray when a record fails its guard — the
 * canonical records pairwise.  prim = 0xFFFFFFFF for a miss.  Returns the number of rays that walked the tables. */
extern "C" uint64_t octant_walk(const float* recs, uint32_t n_rec, const float* tris, int root_ref, const float* root_box, uint64_t n, const float* o, const float* d,
                                const float* t_max_in, int use_tables, uint32_t* prim_out, float* uvt_out)
{
    std::vector<float> tables((size_t)8 * n_rec * 16);
    bool tables_ok = use_tables != 0;
    for (uint32_t r = 0; r < n_rec; ++r) tables_ok = tables_ok && rt_oct_record_ok(recs + 16 * r);
    if (tables_ok)
        for (uint32_t i = 0; i < 8 * n_rec; ++i) rt_oct_order(recs + 16 * (i % n_rec), i / n_rec, &tables[(size_t)i * 16]);
    uint64_t walked = 0;
    for (uint64_t i = 0; i < n; ++i)
    {
        const float *oi = o + 3 * i, *di = d + 3 * i;
        const float inv[3] = { 1.0f / di[0], 1.0f / di[1], 1.0f / di[2] };
        float t_max = t_max_in[i];
        const bool oct = tables_ok && rt_oct_ray_ok(inv[0], inv[1], inv[2]);
        walked += oct;
        const float* base = oct ? &tables[(size_t)rt_oct_octant(inv[0], inv[1], inv[2]) * n_rec * 16] : recs;
        uint32_t prim = 0xFFFFFFFFu; float bu = 0, bv = 0, bt = 0;
        int cur = root_ref, sp = 0, stack_ref[64]; float stack_t[64];
        float rlo, rhi;
        rt_slab_pairwise(root_box, oi[0], oi[1], oi[2], inv[0], inv[1], inv[2], 0.0f, rlo, rhi);
        bool done = !(rt_oct_min(rhi, t_max) >= rlo);
        while (!done)
        {
            while (cur >= 0)
            {
                uint32_t s[8];
                if (oct) step_ordered(base + 16 * cur, oi, inv, 0.0f, t_max, s); else step_pairwise(base + 16 * cur, oi, inv, 0.0f, t_max, s);
                float far_lo; memcpy(&far_lo, &s[5], 4);
                if (s[0]) { if (s[1]) { stack_ref[sp] = (int)s[3]; stack_t[sp] = far_lo; ++sp; } cur = (int)s[2]; }
                else if (s[1]) cur = (int)s[3];
                else
                {
                    bool found = false;
                    while (sp > 0) { --sp; if (t_max >= stack_t[sp]) { cur = stack_ref[sp]; found = true; break; } }
                    if (!found) { done = true; break; }
                }
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
                            if (!(t < 0.0f || t > t_max)) { bu = u; bv = v; bt = t; prim = ti; t_max = t; }
                        }
                    }
                }
                if (bits(q[9]) != 0u) break;
            }
            bool found = false;
            while (sp > 0) { --sp; if (t_max >= stack_t[sp]) { cur = stack_ref[sp]; found = true; break; } }
            if (!found) done = true;
        }
        prim_out[i] = prim; uvt_out[3 * i] = bu; uvt_out[3 * i + 1] = bv; uvt_out[3 * i + 2] = bt;
    }
    return walked;
}

extern "C" void octant_order(const float* rec, uint32_t s, float* out) { rt_oct_order(rec, s, out); }
