/*
 * rt_octant.h — octant-ordered interior records: the slab test of a shared-memory-resident BVH without the pairwise min/max
 * and without the near/far selects.  Compiles for the host (tests/octant_slab_host.cpp) and the device (rt_traverse.cuh).
 *
 * A canonical interior record (rt_bvh_layout.h, 16 floats) holds the boxes of both children as (min, max) and the split axis:
 *   [0..2] child 0 min   [3..5] child 0 max   [6..8] child 1 min   [9..11] child 1 max   [12] ref 0   [13] ref 1   [14] axis
 * trace_fast sorts every plane pair into (entry, exit) with fminf/fmaxf and picks the near child by the sign of the ray's
 * reciprocal direction on the split axis.  Both answers depend on the ray only through its direction octant
 *   s = (inv.x < 0) | (inv.y < 0) << 1 | (inv.z < 0) << 2,
 * so for each of the 8 octants the record is rewritten once, in the same 64 bytes:
 *   [0..2] near entry   [3..5] near exit   [6..8] far entry   [9..11] far exit   [12] near ref   [13] far ref   [14] axis
 * with entry plane on axis k = box max if bit k of s is set, else box min, and near child = child 1 iff bit `axis` of s is set.
 *
 * WHEN THE ORDERED TEST EQUALS THE PAIRWISE ONE.  Let min <= max, both finite, o finite, inv finite and non-zero, and
 * t0 = (min - o) * inv, t1 = (max - o) * inv (one rounding per operation, no contraction).  Rounding is monotone, so
 * min - o <= max - o; neither is NaN (finite operands; an overflow gives a signed infinity), and a product with a finite
 * non-zero factor is never NaN (inf * x and 0 * x are only NaN for x = 0 resp. inf) and keeps the order for inv > 0 and
 * reverses it for inv < 0.  Hence inv > 0 => t0 <= t1 and inv < 0 => t1 <= t0: fminf(t0, t1) and the entry plane selected by
 * the sign of inv are the same number, likewise fmaxf and the exit plane.  "The same number" is the same bits except when
 * t0 == t1 == 0 with different signs, where fminf/fmaxf order -0 < +0 and the selection may return the other zero; every
 * later use of these values is an fmaxf/fminf chain that ends in the comparisons `min(hi, t_max) >= lo` and
 * `t_max >= far_lo`, and a comparison does not see the sign of a zero.  So the hit decisions, hence the visiting order and
 * every result, are identical.  The two tests can only differ when a NaN appears, which fminf/fmaxf drop and a selection
 * keeps: 0 * inf (a direction component that is zero, or so small that its reciprocal overflows, with the origin on a plane)
 * or a non-finite or inverted box.  rt_oct_ray_ok and rt_oct_record_ok are the guards: a ray or a tree that fails them is
 * traced by a path that evaluates the pairwise test.
 */
#pragma once

#include <cstdint>
#include <cstring>

#ifdef __CUDACC__
#define RT_OCT_FN __host__ __device__ __forceinline__
#else
#define RT_OCT_FN inline
#endif

#define RT_OCT_FLT_MAX 3.402823466e+38f

#ifdef __CUDA_ARCH__
RT_OCT_FN float rt_oct_min(float a, float b) { return fminf(a, b); }
RT_OCT_FN float rt_oct_max(float a, float b) { return fmaxf(a, b); }
RT_OCT_FN float rt_oct_abs(float a) { return fabsf(a); }
#else
// the device's fminf/fmaxf: a NaN operand is dropped, -0 < +0
RT_OCT_FN uint32_t rt_oct_bits(float a) { uint32_t u; memcpy(&u, &a, 4); return u; }
RT_OCT_FN float rt_oct_min(float a, float b) { if (a != a) return b; if (b != b) return a; if (a == b) return (rt_oct_bits(a) >> 31) ? a : b; return a < b ? a : b; }
RT_OCT_FN float rt_oct_max(float a, float b) { if (a != a) return b; if (b != b) return a; if (a == b) return (rt_oct_bits(a) >> 31) ? b : a; return a > b ? a : b; }
RT_OCT_FN float rt_oct_abs(float a) { return a < 0.0f ? -a : (a == 0.0f ? 0.0f : a); }
#endif

// The ray guard: every reciprocal direction component finite and non-zero (false for a NaN component).
RT_OCT_FN bool rt_oct_ray_ok(float ix, float iy, float iz)
{
    const float hi = rt_oct_max(rt_oct_max(rt_oct_abs(ix), rt_oct_abs(iy)), rt_oct_abs(iz));
    const float lo = rt_oct_min(rt_oct_min(rt_oct_abs(ix), rt_oct_abs(iy)), rt_oct_abs(iz));
    return ix == ix && iy == iy && iz == iz && hi <= RT_OCT_FLT_MAX && lo > 0.0f;
}

RT_OCT_FN uint32_t rt_oct_octant(float ix, float iy, float iz) { return (ix < 0 ? 1u : 0u) | (iy < 0 ? 2u : 0u) | (iz < 0 ? 4u : 0u); }

// The record guard: all twelve planes finite, min <= max on every axis of both boxes, split axis 0..2.
RT_OCT_FN bool rt_oct_record_ok(const float* rec)
{
    bool ok = true;
    for (int c = 0; c < 2; ++c)
        for (int k = 0; k < 3; ++k)
        {
            const float lo = rec[6 * c + k], hi = rec[6 * c + 3 + k];
            ok = ok && lo <= hi && rt_oct_abs(lo) <= RT_OCT_FLT_MAX && rt_oct_abs(hi) <= RT_OCT_FLT_MAX;
        }
    uint32_t axis; memcpy(&axis, rec + 14, 4);
    return ok && axis <= 2u;
}

// The record of octant s from the canonical record (which passed rt_oct_record_ok).
RT_OCT_FN void rt_oct_order(const float* rec, uint32_t s, float* out)
{
    uint32_t axis; memcpy(&axis, rec + 14, 4);
    const uint32_t swap = (s >> axis) & 1u;
    for (uint32_t c = 0; c < 2; ++c)
    {
        const float* box = rec + 6 * (c ^ swap);
        for (uint32_t k = 0; k < 3; ++k)
        {
            const bool neg = ((s >> k) & 1u) != 0u;
            out[6 * c + k] = neg ? box[3 + k] : box[k];
            out[6 * c + 3 + k] = neg ? box[k] : box[3 + k];
        }
    }
    out[12] = rec[12 + swap]; out[13] = rec[13 - swap]; out[14] = rec[14]; out[15] = rec[15];
}

/*
 * 4-WIDE OCTANT TABLES.  The binary tree is collapsed as tools/wide_bvh_model.cpp does: the wide nodes are the interior records
 * at even depth (the root is depth 0), and each takes its children, except that an interior child is replaced by that child's
 * two children — 2..4 children per wide node.  In the table of octant s a wide node is a run of consecutive 32-byte slots in
 * the order the binary traversal visits them for a ray of that octant: near child (or, when it is interior, its near and far
 * child), then far child (likewise).  A slot is
 *   [0..2] entry planes   [3..5] exit planes   [6] child ref   [7] the node's child count (2..4), in every slot of the node
 * with the planes ordered as rt_oct_order orders them, child ref < 0 a leaf (first triangle ~ref) and >= 0 the first slot of
 * a wide node.  The slot numbering is the same in every octant: wide nodes in record order, each taking rt_wide_count slots,
 * so every octant's table holds at most twice as many slots as there are records (every binary node but the root takes at
 * most one slot) — the 64 bytes per record of a binary ordered table.  The builder keeps, in word 15 of each record (which no
 * traversal reads), the record's first slot, or 0xFFFFFFFF for a record that is not a wide node.
 *
 * Testing the children of a collapsed child without testing that child's box takes the same decisions as the binary
 * traversal only when the child's box contains both boxes of its own children (then, under monotone rounding, its slab
 * interval contains theirs): rt_wide_nests is that guard.
 */
RT_OCT_FN uint32_t rt_oct_u(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
RT_OCT_FN float rt_oct_f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }

// Slots of the wide node at a record: 1 per leaf child, 2 per interior child.
RT_OCT_FN uint32_t rt_wide_count(const float* rec) { return ((int)rt_oct_u(rec[12]) < 0 ? 1u : 2u) + ((int)rt_oct_u(rec[13]) < 0 ? 1u : 2u); }

// The nesting guard of the wide node at record `rec` of the n records `recs`: every interior child's box contains both
// boxes of that child's own record on every axis (false for a reference out of range and for a NaN plane).
RT_OCT_FN bool rt_wide_nests(const float* rec, const float* recs, uint32_t n)
{
    bool ok = true;
    for (int c = 0; c < 2; ++c)
    {
        const int ref = (int)rt_oct_u(rec[12 + c]);
        if (ref < 0) continue;
        if ((uint32_t)ref >= n) return false;
        const float* box = rec + 6 * c;
        const float* kid = recs + 16 * (uint32_t)ref;
        for (int g = 0; g < 2; ++g)
            for (int k = 0; k < 3; ++k)
                ok = ok && kid[6 * g + k] >= box[k] && kid[6 * g + 3 + k] <= box[3 + k];
    }
    return ok;
}

// The slots of the wide node at record r for octant s, written to out (8 floats per slot).  Every record passed
// rt_oct_record_ok, every child reference is in range and word 15 of every record holds its first slot.
RT_OCT_FN void rt_wide_node(const float* recs, uint32_t r, uint32_t s, float* out)
{
    const float cnt = rt_oct_f(rt_wide_count(recs + 16 * r));
    float ord[16];
    rt_oct_order(recs + 16 * r, s, ord);
    uint32_t k = 0;
    for (int c = 0; c < 2; ++c)
    {
        const int ref = (int)rt_oct_u(ord[12 + c]);
        if (ref < 0)
        {
            for (int j = 0; j < 6; ++j) out[8 * k + j] = ord[6 * c + j];
            out[8 * k + 6] = ord[12 + c]; out[8 * k + 7] = cnt; ++k;
            continue;
        }
        float kid[16];
        rt_oct_order(recs + 16 * (uint32_t)ref, s, kid);
        for (int g = 0; g < 2; ++g)
        {
            const int gref = (int)rt_oct_u(kid[12 + g]);
            for (int j = 0; j < 6; ++j) out[8 * k + j] = kid[6 * g + j];
            out[8 * k + 6] = gref < 0 ? kid[12 + g] : recs[16 * (uint32_t)gref + 15];
            out[8 * k + 7] = cnt; ++k;
        }
    }
}

// One child's slab interval, pairwise (trace_fast on canonical records): box = min xyz, max xyz.
RT_OCT_FN void rt_slab_pairwise(const float* box, float ox, float oy, float oz, float ix, float iy, float iz, float t_min, float& lo, float& hi)
{
    const float t0x = (box[0] - ox) * ix, t0y = (box[1] - oy) * iy, t0z = (box[2] - oz) * iz;
    const float t1x = (box[3] - ox) * ix, t1y = (box[4] - oy) * iy, t1z = (box[5] - oz) * iz;
    lo = rt_oct_max(rt_oct_max(rt_oct_max(rt_oct_min(t0x, t1x), rt_oct_min(t0y, t1y)), rt_oct_min(t0z, t1z)), t_min);
    hi = rt_oct_min(rt_oct_min(rt_oct_max(t0x, t1x), rt_oct_max(t0y, t1y)), rt_oct_max(t0z, t1z));
}

// One child's slab interval on an ordered record: (ex, ey, ez) entry planes, (xx, xy, xz) exit planes.
RT_OCT_FN void rt_slab_ordered(float ex, float ey, float ez, float xx, float xy, float xz, float ox, float oy, float oz,
                               float ix, float iy, float iz, float t_min, float& lo, float& hi)
{
    lo = rt_oct_max(rt_oct_max(rt_oct_max((ex - ox) * ix, (ey - oy) * iy), (ez - oz) * iz), t_min);
    hi = rt_oct_min(rt_oct_min((xx - ox) * ix, (xy - oy) * iy), (xz - oz) * iz);
}
