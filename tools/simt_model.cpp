/*
 * tools/simt_model.cpp — ANALYSIS ONLY (CPU).  Issue-slot model of the traversal kernels' warp schedules.
 *
 * For every ray of a dumped bounce the exact operation sequence of trace_fast (rt_kernels.cu) on the child-box layout
 * (rt_bvh_layout.h) is recorded: interior-record steps, triangle tests with their exit stage, leaf boundaries.  A warp
 * is then simulated under several schedules; a warp-instruction costs one issue slot whatever the number of active lanes,
 * so   cost per ray = issue slots / rays   and   lane utilisation = thread work / (32 * issue slots).
 *
 *   schedule 0  one ray per lane per batch of 32 (the round-1 kernels): the warp waits for its slowest ray
 *   schedule 1  K rays per lane, statically assigned: a lane starts its next ray as soon as its current one ends
 *   schedule 2  ideal dynamic refill: a lane takes the next ray of the warp's global stream at once (upper bound)
 * Both run the while-while loop shape of the kernels: all lanes with an interior record step iterate until none is left,
 * then all lanes with a leaf iterate over its triangles.
 */
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "rt_types.h"
#include "../raytracing_b200/csrc/rt_bvh_layout.h"
#include "../raytracing_b200/csrc/rt_octant.h"

namespace
{
struct V3 { float x, y, z; };
inline V3 operator-(V3 a, V3 b) { return V3{ a.x - b.x, a.y - b.y, a.z - b.z }; }
inline V3 operator*(V3 a, V3 b) { return V3{ a.x * b.x, a.y * b.y, a.z * b.z }; }
inline V3 cross(V3 a, V3 b) { return V3{ a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x }; }
inline float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

enum : uint8_t { OP_NODE = 0, OP_TRI1 = 1, OP_TRI2 = 2, OP_TRI3 = 3, OP_TRI4 = 4, OP_LEAF_END = 5 };

// the operation sequence of trace_fast for one finite ray (non-finite rays: empty sequence)
void record(const rtbvh::WideLayout& wl, const RtLinearBVHNode* nodes, V3 o, V3 d, float t_max, bool any, std::vector<uint8_t>& ops)
{
    ops.clear();
    float fin = ((o.x + o.y) + o.z) + ((d.x + d.y) + d.z);
    if (!(std::fabs(fin) <= 3.0e38f)) return;
    V3 inv{ 1.0f / d.x, 1.0f / d.y, 1.0f / d.z };
    const bool s[3] = { inv.x < 0, inv.y < 0, inv.z < 0 };
    const float t_min = 0.0f;
    {
        V3 t0 = (V3{ nodes[0].bounds_min.x, nodes[0].bounds_min.y, nodes[0].bounds_min.z } - o) * inv;
        V3 t1 = (V3{ nodes[0].bounds_max.x, nodes[0].bounds_max.y, nodes[0].bounds_max.z } - o) * inv;
        float lo = std::fmax(std::fmax(std::fmin(t0.x, t1.x), std::fmin(t0.y, t1.y)), std::fmin(t0.z, t1.z));
        float hi = std::fmin(std::fmin(std::fmax(t0.x, t1.x), std::fmax(t0.y, t1.y)), std::fmax(t0.z, t1.z));
        if (!(std::fmin(hi, t_max) >= std::fmax(lo, t_min))) return;
    }
    int stack_ref[64]; float stack_t[64]; int sp = 0;
    int cur = wl.root_ref;
    const rtbvh::F4* W = wl.nodes.data(); const rtbvh::F4* T = wl.tris.data();
    for (;;)
    {
        while (cur >= 0)
        {
            ops.push_back(OP_NODE);
            const rtbvh::F4 a = W[cur * 4], b = W[cur * 4 + 1], c = W[cur * 4 + 2], m = W[cur * 4 + 3];
            V3 t00 = (V3{ a.x, a.y, a.z } - o) * inv, t01 = (V3{ a.w, b.x, b.y } - o) * inv;
            V3 t10 = (V3{ b.z, b.w, c.x } - o) * inv, t11 = (V3{ c.y, c.z, c.w } - o) * inv;
            float lo0 = std::fmax(std::fmax(std::fmax(std::fmin(t00.x, t01.x), std::fmin(t00.y, t01.y)), std::fmin(t00.z, t01.z)), t_min);
            float hi0 = std::fmin(std::fmin(std::fmax(t00.x, t01.x), std::fmax(t00.y, t01.y)), std::fmax(t00.z, t01.z));
            float lo1 = std::fmax(std::fmax(std::fmax(std::fmin(t10.x, t11.x), std::fmin(t10.y, t11.y)), std::fmin(t10.z, t11.z)), t_min);
            float hi1 = std::fmin(std::fmin(std::fmax(t10.x, t11.x), std::fmax(t10.y, t11.y)), std::fmax(t10.z, t11.z));
            bool h0 = std::fmin(hi0, t_max) >= lo0, h1 = std::fmin(hi1, t_max) >= lo1;
            int r0, r1; uint32_t axis; memcpy(&r0, &m.x, 4); memcpy(&r1, &m.y, 4); memcpy(&axis, &m.z, 4);
            bool swap = s[axis];
            int near_ref = swap ? r1 : r0, far_ref = swap ? r0 : r1;
            bool near_hit = swap ? h1 : h0, far_hit = swap ? h0 : h1;
            float far_lo = swap ? lo0 : lo1;
            if (near_hit) { if (far_hit) { stack_ref[sp] = far_ref; stack_t[sp] = far_lo; ++sp; } cur = near_ref; }
            else if (far_hit) cur = far_ref;
            else
            {
                bool found = false;
                while (sp > 0) { --sp; if (t_max >= stack_t[sp]) { cur = stack_ref[sp]; found = true; break; } }
                if (!found) return;
            }
        }
        uint32_t ti = (uint32_t)(~cur);
        for (;;)
        {
            const rtbvh::F4 q0 = T[ti * 3], q1 = T[ti * 3 + 1], q2 = T[ti * 3 + 2];
            V3 p1{ q0.x, q0.y, q0.z }, e1{ q0.w, q1.x, q1.y }, e2{ q1.z, q1.w, q2.x };
            uint32_t lastb; memcpy(&lastb, &q2.y, 4);
            uint8_t stage = OP_TRI1;
            V3 pvec = cross(d, e2);
            float det = dot(e1, pvec);
            if (!(det < 1e-8f || -det > 1e-8f))
            {
                stage = OP_TRI2;
                float inv_det = 1.0f / det;
                V3 tvec = o - p1;
                float u = dot(tvec, pvec) * inv_det;
                if (!(u < 0.0f || u > 1.0f))
                {
                    stage = OP_TRI3;
                    V3 qvec = cross(tvec, e1);
                    float v = dot(d, qvec) * inv_det;
                    if (!(v < 0.0f || u + v > 1.0f))
                    {
                        stage = OP_TRI4;
                        float t = dot(e2, qvec) * inv_det;
                        if (!(t < t_min || t > t_max)) { t_max = t; if (any) { ops.push_back(stage); return; } }
                    }
                }
            }
            ops.push_back(stage);
            if (lastb) break;
            ++ti;
        }
        ops.push_back(OP_LEAF_END);
        bool found = false;
        while (sp > 0) { --sp; if (t_max >= stack_t[sp]) { cur = stack_ref[sp]; found = true; break; } }
        if (!found) return;
    }
}

struct Costs { double node, tri[5], fetch; };

struct Result { double slots = 0, thread_work = 0; uint64_t rays = 0; };

// One warp drains `count` rays starting at `first` of the op lists.  schedule: 0 batch of 32, 1 static K per lane, 2 dynamic.
Result simulate_warp(const std::vector<std::vector<uint8_t>>& ops, size_t first, size_t count, int schedule, int K, const Costs& c)
{
    Result r; r.rays = count;
    struct Lane { size_t ray = SIZE_MAX; size_t pos = 0; int left = 0; size_t next = 0, stride = 0, end = 0; };
    Lane lane[32];
    size_t pool = first, pool_end = first + count;       // schedules 0 and 2 draw from the pool
    auto has = [&](const Lane& l) { return l.ray != SIZE_MAX; };
    auto skip_empty = [&](Lane& l) { };
    (void)skip_empty;
    auto start_batch = [&]() -> bool {       // schedule 0: 32 consecutive rays, one per lane
        bool any_ray = false;
        for (int i = 0; i < 32; ++i)
        {
            lane[i].ray = SIZE_MAX;
            if (pool < pool_end) { lane[i].ray = pool++; lane[i].pos = 0; any_ray = true; }
        }
        if (any_ray) r.slots += c.fetch;
        for (int i = 0; i < 32; ++i) if (has(lane[i])) r.thread_work += c.fetch;
        return any_ray;
    };
    auto next_ray = [&](Lane& l) -> bool {   // returns true when the lane got a ray
        if (schedule == 2)
        {
            if (pool < pool_end) { l.ray = pool++; l.pos = 0; return true; }
            l.ray = SIZE_MAX; return false;
        }
        // static: rays l.next, l.next + stride, ... < l.end
        if (l.next < l.end) { l.ray = l.next; l.next += l.stride; l.pos = 0; return true; }
        l.ray = SIZE_MAX; return false;
    };
    if (schedule == 1)
    {   // chunks of 32 * K consecutive rays; lane i takes rays i, i + 32, ... of the chunk
        // (the whole count is one sequence of chunks handled by this warp)
    }
    size_t chunk_first = first;
    auto start_chunk = [&]() -> bool {
        if (chunk_first >= pool_end) return false;
        size_t chunk_end = std::min(pool_end, chunk_first + (size_t)32 * K);
        bool any_ray = false;
        for (int i = 0; i < 32; ++i)
        {
            lane[i].next = chunk_first + i; lane[i].stride = 32; lane[i].end = chunk_end;
            if (next_ray(lane[i])) { any_ray = true; r.thread_work += c.fetch; }
        }
        chunk_first = chunk_end;
        if (any_ray) r.slots += c.fetch;
        return any_ray;
    };
    for (;;)
    {
        bool any_ray = false;
        if (schedule == 0) any_ray = start_batch();
        else if (schedule == 1) any_ray = start_chunk();
        else
        {
            for (int i = 0; i < 32; ++i) if (next_ray(lane[i])) { any_ray = true; r.thread_work += c.fetch; }
            if (any_ray) r.slots += c.fetch;
        }
        if (!any_ray) break;
        // run until every lane is out of rays
        for (;;)
        {
            // rays with an empty / exhausted sequence end at once
            bool refill = false, live = false;
            for (int i = 0; i < 32; ++i)
                while (has(lane[i]) && lane[i].pos >= ops[lane[i].ray].size())
                {
                    if (schedule == 0) { lane[i].ray = SIZE_MAX; break; }
                    if (next_ray(lane[i])) { refill = true; r.thread_work += c.fetch; }
                }
            if (refill) r.slots += c.fetch;
            for (int i = 0; i < 32; ++i) live |= has(lane[i]);
            if (!live) break;
            // interior phase
            for (;;)
            {
                int n = 0;
                for (int i = 0; i < 32; ++i)
                    if (has(lane[i]) && lane[i].pos < ops[lane[i].ray].size() && ops[lane[i].ray][lane[i].pos] == OP_NODE) { ++n; ++lane[i].pos; }
                if (!n) break;
                r.slots += c.node; r.thread_work += c.node * n;
            }
            // leaf phase
            for (;;)
            {
                int n = 0; double worst = 0, sum = 0;
                for (int i = 0; i < 32; ++i)
                {
                    if (!has(lane[i]) || lane[i].pos >= ops[lane[i].ray].size()) continue;
                    uint8_t op = ops[lane[i].ray][lane[i].pos];
                    if (op >= OP_TRI1 && op <= OP_TRI4) { ++n; worst = std::max(worst, c.tri[op]); sum += c.tri[op]; ++lane[i].pos; }
                }
                if (!n) break;
                r.slots += worst; r.thread_work += sum;
            }
            for (int i = 0; i < 32; ++i)
                if (has(lane[i]) && lane[i].pos < ops[lane[i].ray].size() && ops[lane[i].ray][lane[i].pos] == OP_LEAF_END) ++lane[i].pos;
        }
        if (schedule == 2) break;
    }
    return r;
}
} // namespace

extern "C" int simt_model(const RtLinearBVHNode* nodes, uint32_t n_nodes, const RtTriangle* tris, uint32_t n_tris,
                          const RtRay* rays, uint32_t n_rays, int any_hit, int schedule, int K, uint32_t rays_per_warp,
                          const double* costs /* node, tri1..tri4, fetch */, double* out /* slots, thread_work, node ops, tri ops */)
{
    rtbvh::WideLayout wl; std::string err;
    if (!rtbvh::build_layout(nodes, n_nodes, tris, n_tris, wl, err)) return 1;
    std::vector<std::vector<uint8_t>> ops(n_rays);
#pragma omp parallel for schedule(dynamic, 1024)
    for (long long i = 0; i < (long long)n_rays; ++i)
    {
        V3 o{ rays[i].origin.x, rays[i].origin.y, rays[i].origin.z }, d{ rays[i].direction.x, rays[i].direction.y, rays[i].direction.z };
        record(wl, nodes, o, d, rays[i].direction.w, any_hit != 0, ops[i]);
    }
    Costs c; c.node = costs[0]; c.tri[0] = 0; for (int k = 1; k <= 4; ++k) c.tri[k] = costs[k]; c.fetch = costs[5];
    double slots = 0, work = 0;
    const size_t per = rays_per_warp ? rays_per_warp : 32;
    const long long n_warps = (long long)((n_rays + per - 1) / per);
#pragma omp parallel for schedule(dynamic, 64) reduction(+ : slots, work)
    for (long long w = 0; w < n_warps; ++w)
    {
        size_t first = (size_t)w * per, count = std::min(per, (size_t)n_rays - first);
        Result r = simulate_warp(ops, first, count, schedule, K, c);
        slots += r.slots; work += r.thread_work;
    }
    double n_node = 0, n_tri = 0;
    for (auto& v : ops) for (uint8_t op : v) { if (op == OP_NODE) ++n_node; else if (op != OP_LEAF_END) ++n_tri; }
    out[0] = slots; out[1] = work; out[2] = n_node; out[3] = n_tri;
    return 0;
}

// ------------------------------------------------------------------ any-hit rays on the 4-wide octant tables (SMEM 3)
// trace_fast<true, false, 3> walks the tables of its ray's octant (rt_octant.h: wide nodes of 2..4 slots, children tested last
// to first, the first hit child continued into, the others kept as references on a 4-byte stack that is popped without a test).
// A lane's walk is a state machine here because the postponed loop changes which step a lane takes next depending on the warp:
//   variant 0  the while-while loop walking near to far: interior steps while any lane has an interior record, then the leaves of every lane
//              that reached one, one triangle per slot, then the pop
//   variant 1  postponed leaves: a lane that reaches a leaf with its pending slot empty keeps the leaf there and pops its next
//              entry; with the slot full it stops.  The interior loop ends when no lane has an interior record, or when the vote of
//              the lanes still in it finds at least `trigger` of them (0: all; -1: no vote) holding a leaf.  The leaf loop then runs every
//              pending leaf; a lane whose leaf ends while it stands on another leaf takes that one in the same loop.
//   variant 2  the while-while loop of variant 0 with the wide step walking far to near: the children are tested first to last
//              and the last that hits is continued into (the order trace_fast<true, false, 3> uses)
// Only rays that take the table walk are modelled (rt_oct_ray_ok, finite t_max); the others run the SMEM 1 loop in both builds.
namespace
{
const int EMPTY = INT32_MIN;                                   // no interior or leaf reference left
struct AnyLane
{
    const float* base; float o[3], d[3], inv[3], t_max;
    int cur = EMPTY, pending = 0, sp = 0, stack[128];
    bool live = false;
};

uint32_t fbits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

void pop(AnyLane& l) { l.cur = l.sp ? l.stack[--l.sp] : EMPTY; }

void wide_step(AnyLane& l, bool far_first)
{
    const float* np = l.base + (size_t)l.cur * 8;
    const uint32_t cnt = fbits(np[7]);
    bool found = false; int next_ref = 0;
    for (int k = 0; k < (int)cnt; ++k)
    {
        const int j = far_first ? k : (int)cnt - 1 - k;
        const float* q = np + 8 * j;
        float lo, hi;
        rt_slab_ordered(q[0], q[1], q[2], q[3], q[4], q[5], l.o[0], l.o[1], l.o[2], l.inv[0], l.inv[1], l.inv[2], 0.0f, lo, hi);
        if (rt_oct_min(hi, l.t_max) >= lo)
        {
            if (found) l.stack[l.sp++] = next_ref;
            next_ref = (int)fbits(q[6]); found = true;
        }
    }
    if (found) l.cur = next_ref; else pop(l);
}

// one triangle test of trace_fast: the exit stage (OP_TRI1..4), *hit and *last
uint8_t tri_step(const float* tris, const AnyLane& l, uint32_t ti, bool* hit, bool* last)
{
    const float* q = tris + 12 * (size_t)ti;
    *last = fbits(q[9]) != 0u; *hit = false;
    V3 p1{ q[0], q[1], q[2] }, e1{ q[3], q[4], q[5] }, e2{ q[6], q[7], q[8] }, d{ l.d[0], l.d[1], l.d[2] }, o{ l.o[0], l.o[1], l.o[2] };
    V3 pvec = cross(d, e2);
    float det = dot(e1, pvec);
    if (det < 1e-8f || -det > 1e-8f) return OP_TRI1;
    float inv_det = 1.0f / det;
    V3 tvec = o - p1;
    float u = dot(tvec, pvec) * inv_det;
    if (u < 0.0f || u > 1.0f) return OP_TRI2;
    V3 qvec = cross(tvec, e1);
    float v = dot(d, qvec) * inv_det;
    if (v < 0.0f || u + v > 1.0f) return OP_TRI3;
    float t = dot(e2, qvec) * inv_det;
    *hit = !(t < 0.0f || t > l.t_max);
    return OP_TRI4;
}

// costs: wide step, tri1..tri4, ray fetch, postponing overhead per interior step (postpone test + vote)
Result simulate_any_warp(const float* tables, uint32_t n, const float* tris, int root_ref, const float* root_box, const float* rays,
                         size_t first, size_t count, int variant, int trigger, const double* c, uint64_t* unoccluded)
{
    Result r; r.rays = count;
    for (size_t b = first; b < first + count; b += 32)
    {
        AnyLane lane[32];
        int m = (int)std::min<size_t>(32, first + count - b);
        r.slots += c[5]; r.thread_work += c[5] * m;
        for (int i = 0; i < m; ++i)
        {
            AnyLane& l = lane[i];
            const float* ray = rays + 7 * (b + i);
            for (int k = 0; k < 3; ++k) { l.o[k] = ray[k]; l.d[k] = ray[3 + k]; l.inv[k] = 1.0f / ray[3 + k]; }
            l.t_max = ray[6];
            if (!rt_oct_ray_ok(l.inv[0], l.inv[1], l.inv[2]) || l.t_max != l.t_max) continue;
            l.base = tables + (size_t)rt_oct_octant(l.inv[0], l.inv[1], l.inv[2]) * 2 * n * 8;
            float lo, hi;
            rt_slab_pairwise(root_box, l.o[0], l.o[1], l.o[2], l.inv[0], l.inv[1], l.inv[2], 0.0f, lo, hi);
            if (!(rt_oct_min(hi, l.t_max) >= lo)) continue;
            l.live = true; l.cur = root_ref;
            if (variant == 1 && l.cur < 0) { l.pending = l.cur; l.cur = EMPTY; }
        }
        auto is_leaf = [](int ref) { return ref < 0 && ref != EMPTY; };
        for (;;)
        {
            bool any_live = false;
            for (int i = 0; i < m; ++i) any_live |= lane[i].live;
            if (!any_live) break;
            for (;;)
            {   // interior loop
                int n_in = 0, n_pend = 0;
                for (int i = 0; i < m; ++i)
                {
                    AnyLane& l = lane[i];
                    if (!l.live || l.cur < 0) continue;
                    ++n_in;
                    wide_step(l, variant == 2);
                    if (variant == 1 && is_leaf(l.cur) && l.pending == 0) { l.pending = l.cur; pop(l); }
                    if (variant == 1 && l.pending != 0) ++n_pend;
                    if (variant != 1 && l.cur == EMPTY) { l.live = false; ++*unoccluded; }
                }
                if (!n_in) break;
                const double step = c[0] + (variant == 1 ? c[6] : 0.0);
                r.slots += step; r.thread_work += step * n_in;
                if (variant == 1 && trigger >= 0 && n_pend >= (trigger ? std::min(trigger, n_in) : n_in)) break;
            }
            for (;;)
            {   // leaf loop: lane state ti = ~leaf
                int n_in = 0; double worst = 0, sum = 0;
                for (int i = 0; i < m; ++i)
                {
                    AnyLane& l = lane[i];
                    int* leaf = variant == 1 ? &l.pending : &l.cur;
                    if (!l.live || !is_leaf(*leaf)) continue;
                    ++n_in;
                    bool hit, last;
                    const uint8_t st = tri_step(tris, l, (uint32_t)~*leaf, &hit, &last);
                    worst = std::max(worst, c[st]); sum += c[st];
                    if (hit) { l.live = false; continue; }
                    if (!last) { --*leaf; continue; }
                    if (variant != 1) { l.cur = EMPTY; l.pending = 1; continue; }   // pops after the loop
                    if (is_leaf(l.cur)) { l.pending = l.cur; pop(l); } else l.pending = 0;
                }
                if (!n_in) break;
                r.slots += worst; r.thread_work += sum;
            }
            for (int i = 0; i < m; ++i)
            {
                AnyLane& l = lane[i];
                if (!l.live) continue;
                if (variant != 1 && l.pending == 1) { l.pending = 0; pop(l); }
                if (l.cur == EMPTY && l.pending == 0) { l.live = false; ++*unoccluded; }
            }
        }
    }
    return r;
}
} // namespace

// The SMEM 3 any-hit loop over rays (7 floats: origin, direction, t_max): tables of n records (tests/wide_octant_host.cpp,
// wide_tables), triangle records of rt_bvh_layout.h.  costs: wide step, tri1..tri4, fetch, postponing overhead.
// out: slots, thread work, rays walked to the end without a hit.
extern "C" int simt_any_model(const float* tables, uint32_t n, const float* tris, int root_ref, const float* root_box, const float* rays,
                              uint32_t n_rays, int variant, int trigger, const double* costs, double* out)
{
    double slots = 0, work = 0; uint64_t unocc = 0;
    const uint32_t per = 32 * 64;
    const long long n_chunks = (long long)((n_rays + per - 1) / per);
#pragma omp parallel for schedule(dynamic, 16) reduction(+ : slots, work, unocc)
    for (long long w = 0; w < n_chunks; ++w)
    {
        size_t first = (size_t)w * per, count = std::min<size_t>(per, (size_t)n_rays - first);
        uint64_t u = 0;
        Result r = simulate_any_warp(tables, n, tris, root_ref, root_box, rays, first, count, variant, trigger, costs, &u);
        slots += r.slots; work += r.thread_work; unocc += u;
    }
    out[0] = slots; out[1] = work; out[2] = (double)unocc;
    return 0;
}
