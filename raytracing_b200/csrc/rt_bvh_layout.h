/*
 * rt_bvh_layout.h — host-side conversion (done once in rt_upload_scene) of the reference's
 * LinearBVHNode[] / Triangle[] into the device layout the optimised traversal kernel reads.
 * Analogous to the RTTriangle[] array the reference derives at upload
 * (/root/reference/src/integrator/cl_pt_integrator.cpp:392-402).
 *
 * Reference layout (acceleration input, bvh.cpp:223-245): depth-first array of 48-byte nodes;
 * an interior node's first child is the next node, its second child is `offset`; leaves hold
 * [offset, offset + count) into the leaf-ordered triangle array.
 *
 * Device layout:
 *   wnodes: one 64-byte record (4 x float4) per INTERIOR node holding BOTH children's boxes, so
 *           one record fetch decides both children (the reference fetches a 48-byte node per
 *           visited child, 8 bytes of which are padding):
 *             [0] c0.min.xyz, c0.max.x   [1] c0.max.yz, c1.min.xy   [2] c1.min.z, c1.max.xyz
 *             [3] (ref0, ref1, split axis, 0) as int bits;  ref >= 0: interior record index,
 *                 ref < 0: leaf, first triangle = ~ref
 *   wtris:  48 bytes (3 x float4) per triangle in the same (leaf) order, i.e. index == primitive_id:
 *             p1.xyz, e1.x | e1.yz, e2.xy | e2.z, end_of_leaf flag, 0, 0     (e1 = p2-p1, e2 = p3-p1,
 *           the two subtractions trace_bvh.cl:30-31 performs per test, done once here in the same
 *           IEEE arithmetic)
 * Record ORDER: the first `top_n` interior records are the top of the tree in breadth-first order (root = record 0), the rest follow
 * in the reference's depth-first order.  Any prefix of the array is therefore a connected top part of the tree, which is what
 * lets a traversal kernel stage "the first k records" into shared memory with one TMA bulk copy (RT_OPT_TOP_SMEM) when the whole
 * structure does not fit.  Record indices are internal (child references); primitive ids are untouched.
 * The visiting order of the traversal is unchanged (near child by ray sign of the split axis,
 * far child deferred), so hit results are identical to the reference order; see trace_fast().
 */
#pragma once

#include <cmath>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "rt_types.h"

namespace rtbvh
{

struct F4 { float x, y, z, w; };

struct WideLayout
{
    std::vector<F4> nodes;   // 4 per interior node
    std::vector<F4> tris;    // 3 per triangle
    int root_ref = 0;
    int max_depth = 0;
    uint32_t top_n = 0;      // records [0, top_n) are the top of the tree in breadth-first order
};

#ifndef RT_BVH_TOP_RECORDS
#define RT_BVH_TOP_RECORDS 1024u     // 64 KB of records: upper bound of what a kernel may stage (it stages a prefix)
#endif

inline float int_bits(int v) { float f; memcpy(&f, &v, 4); return f; }

// Record numbering of the interior nodes (interior_order: the depth-first order of build_layout's walk): breadth-first for the
// first top_n, depth-first for the others.  Returns top_n.
inline uint32_t number_records(const RtLinearBVHNode* nodes, uint64_t n_nodes, const std::vector<uint32_t>& interior_order,
                               std::vector<int>& wide_index)
{
    const uint32_t n_interior = (uint32_t)interior_order.size();
    const uint32_t top_n = n_interior < RT_BVH_TOP_RECORDS ? n_interior : RT_BVH_TOP_RECORDS;
    std::vector<uint32_t> bfs;                     // binary node indices of interior nodes in BFS order (prefix only)
    bfs.reserve(top_n);
    if (n_interior > 0) bfs.push_back(0u);
    for (size_t head = 0; head < bfs.size() && bfs.size() < top_n; ++head)
    {
        const RtLinearBVHNode& n = nodes[bfs[head]];
        const uint32_t kids[2] = { bfs[head] + 1u, n.offset };
        for (uint32_t k : kids)
            if ((nodes[k].num_primitives_axis >> 16) == 0 && bfs.size() < top_n) bfs.push_back(k);
    }
    std::vector<uint8_t> in_top(n_nodes, 0);
    for (uint32_t b : bfs) in_top[b] = 1;
    int next = 0;
    for (uint32_t b : bfs) wide_index[b] = next++;
    for (uint32_t node : interior_order) if (!in_top[node]) wide_index[node] = next++;
    return (uint32_t)bfs.size();
}

inline bool build_layout(const RtLinearBVHNode* nodes, uint64_t n_nodes, const RtTriangle* tris, uint64_t n_tris,
                         WideLayout& out, std::string& err)
{
    if (n_nodes == 0 || n_tris == 0) { err = "empty BVH"; return false; }
    std::vector<int> wide_index(n_nodes, -1);
    std::vector<uint8_t> seen(n_nodes, 0), covered(n_tris, 0), last_flag(n_tris, 0);
    // iterative DFS from the root: validates indices, acyclicity, leaf coverage, depth
    struct Item { uint32_t node; int depth; };
    std::vector<Item> stack;
    stack.push_back({ 0u, 1 });
    int n_interior = 0, max_depth = 0;
    std::vector<uint32_t> interior_order;
    while (!stack.empty())
    {
        Item it = stack.back(); stack.pop_back();
        if (it.node >= n_nodes) { err = "child index out of range"; return false; }
        if (seen[it.node]) { err = "node reachable twice (not a tree)"; return false; }
        seen[it.node] = 1;
        if (it.depth > max_depth) max_depth = it.depth;
        const RtLinearBVHNode& n = nodes[it.node];
        uint32_t count = n.num_primitives_axis >> 16;
        if (count > 0)
        {
            if ((uint64_t)n.offset + count > n_tris) { err = "leaf range outside the triangle array"; return false; }
            for (uint32_t i = 0; i < count; ++i)
            {
                if (covered[n.offset + i]) { err = "triangle referenced by two leaves"; return false; }
                covered[n.offset + i] = 1;
            }
            last_flag[n.offset + count - 1] = 1;
        }
        else
        {
            if ((n.num_primitives_axis & 0xFFFFu) > 2) { err = "split axis out of range"; return false; }
            wide_index[it.node] = n_interior++;
            interior_order.push_back(it.node);
            // push second child first so the first child (node+1) is numbered next: DFS order is kept
            stack.push_back({ n.offset, it.depth + 1 });
            stack.push_back({ it.node + 1, it.depth + 1 });
        }
    }
    // the reference kernel's private stack holds 64 entries (trace_bvh.cl:142)
    if (max_depth > 64) { err = "BVH deeper than the 64-entry traversal stack of trace_bvh.cl:142"; return false; }
    out.max_depth = max_depth;
    out.top_n = number_records(nodes, n_nodes, interior_order, wide_index);

    auto ref_of = [&](uint32_t child) -> int {
        const RtLinearBVHNode& c = nodes[child];
        if ((c.num_primitives_axis >> 16) > 0) return ~(int)c.offset;
        return wide_index[child];
    };
    out.nodes.assign((size_t)(n_interior ? n_interior : 1) * 4, F4{ 0, 0, 0, 0 });
    for (uint32_t node : interior_order)
    {
        const RtLinearBVHNode& n = nodes[node];
        const RtLinearBVHNode& c0 = nodes[node + 1];
        const RtLinearBVHNode& c1 = nodes[n.offset];
        F4* w = &out.nodes[(size_t)wide_index[node] * 4];
        w[0] = F4{ c0.bounds_min.x, c0.bounds_min.y, c0.bounds_min.z, c0.bounds_max.x };
        w[1] = F4{ c0.bounds_max.y, c0.bounds_max.z, c1.bounds_min.x, c1.bounds_min.y };
        w[2] = F4{ c1.bounds_min.z, c1.bounds_max.x, c1.bounds_max.y, c1.bounds_max.z };
        w[3] = F4{ int_bits(ref_of(node + 1)), int_bits(ref_of(n.offset)), int_bits((int)(n.num_primitives_axis & 0xFFFFu)), 0.0f };
    }
    const RtLinearBVHNode& root = nodes[0];
    out.root_ref = ((root.num_primitives_axis >> 16) > 0) ? ~(int)root.offset : 0;

    out.tris.resize((size_t)n_tris * 3);
    for (uint64_t i = 0; i < n_tris; ++i)
    {
        const RtFloat3 &p1 = tris[i].v1.position, &p2 = tris[i].v2.position, &p3 = tris[i].v3.position;
        // volatile-free plain float subtractions; x86-64 (no FMA in the baseline ISA) rounds each once
        float e1x = p2.x - p1.x, e1y = p2.y - p1.y, e1z = p2.z - p1.z;
        float e2x = p3.x - p1.x, e2y = p3.y - p1.y, e2z = p3.z - p1.z;
        // triangles not referenced by any reachable leaf can never be visited; flag them as leaf ends too
        uint32_t flag = (last_flag[i] || !covered[i]) ? 1u : 0u;
        out.tris[i * 3 + 0] = F4{ p1.x, p1.y, p1.z, e1x };
        out.tris[i * 3 + 1] = F4{ e1y, e1z, e2x, e2y };
        float fl; memcpy(&fl, &flag, 4);
        out.tris[i * 3 + 2] = F4{ e2z, fl, 0.0f, 0.0f };
    }
    return true;
}

// Refit map of rt_update_triangles, from a node array build_layout has accepted.  For every node reachable from the root:
// link[n] = (parent node, parent's record * 2 + 0 for its first child / + 1 for its second), RT_REFIT_NONE twice for the root;
// leaves: the reachable leaves.  Unreachable nodes keep RT_REFIT_NONE and are never refit.
#define RT_REFIT_NONE 0xFFFFFFFFu
struct RefitMap { std::vector<uint32_t> link, leaves; };

inline void build_refit_map(const RtLinearBVHNode* nodes, uint64_t n_nodes, RefitMap& m)
{
    m.link.assign((size_t)n_nodes * 2, RT_REFIT_NONE);
    m.leaves.clear();
    std::vector<uint32_t> interior_order, stack{ 0u };
    while (!stack.empty())
    {   // build_layout's walk: the first child is visited first
        const uint32_t node = stack.back(); stack.pop_back();
        const RtLinearBVHNode& n = nodes[node];
        if ((n.num_primitives_axis >> 16) > 0) { m.leaves.push_back(node); continue; }
        interior_order.push_back(node);
        stack.push_back(n.offset);
        stack.push_back(node + 1);
    }
    std::vector<int> wide_index(n_nodes, -1);
    number_records(nodes, n_nodes, interior_order, wide_index);
    for (uint32_t p : interior_order)
    {
        const uint32_t r = (uint32_t)wide_index[p] * 2u;
        m.link[(size_t)(p + 1) * 2] = p;            m.link[(size_t)(p + 1) * 2 + 1] = r;
        m.link[(size_t)nodes[p].offset * 2] = p;    m.link[(size_t)nodes[p].offset * 2 + 1] = r + 1u;
    }
}

// ---------------------------------------------------------------------------------------------------
// Shading records.  Everything below is a pure function of the uploaded scene evaluated ONCE on the host
// with the same IEEE binary32 operations, in the same order, that the reference performs per hit on the
// device (x86-64 baseline ISA has no FMA; the file is compiled with -ffp-contract=off), so the kernels
// load a few float4 instead of recomputing them per path vertex.  Results are bit-identical.
//
//   tri_shade: 7 x float4 per triangle (112 B instead of the reference's 160-byte Triangle):
//      [0] p1.xyz, mtlIndex bits   [1] p2.xyz, gn.x   [2] p3.xyz, gn.y   [3] n1.xyz, gn.z
//      [4] n2.xyz, uv1.x           [5] n3.xyz, uv1.y  [6] uv2.xy, uv3.xy
//      gn = normalize(cross(p2 - p1, p3 - p1)), hit_surface.cl:91
//   mat_rec: 4 x float4 per material: [0] diffuse.rgb, roughness  [1] specular.rgb, metalness
//      [2] emission.rgb, ior  [3] transparency, has_texture flag   (utils.h:133-190, material.h:251-264)
//   light_rec: 2 x float4 per light: [0] point: origin.xyz | directional: normalize(origin*MAX_RENDER_DIST),
//      w = |origin*MAX_RENDER_DIST|   [1] radiance.xyz, type bits   (light.h:30-65, hit_surface.cl:122-123)

inline float bits_float(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }

inline void normalize3(float x, float y, float z, float* out)
{
    float inv = 1.0f / sqrtf(x * x + y * y + z * z);        // same association as rt::dot / rt::normalize
    out[0] = x * inv; out[1] = y * inv; out[2] = z * inv;
}

inline void build_tri_shade(const RtTriangle* tris, uint64_t n, std::vector<F4>& out)
{
    out.resize((size_t)n * 7);
    for (uint64_t i = 0; i < n; ++i)
    {
        const RtTriangle& t = tris[i];
        const RtFloat3 &p1 = t.v1.position, &p2 = t.v2.position, &p3 = t.v3.position;
        float e1x = p2.x - p1.x, e1y = p2.y - p1.y, e1z = p2.z - p1.z;
        float e2x = p3.x - p1.x, e2y = p3.y - p1.y, e2z = p3.z - p1.z;
        float cx = e1y * e2z - e1z * e2y, cy = e1z * e2x - e1x * e2z, cz = e1x * e2y - e1y * e2x;
        float gn[3];
        normalize3(cx, cy, cz, gn);
        F4* r = &out[(size_t)i * 7];
        r[0] = F4{ p1.x, p1.y, p1.z, bits_float(t.mtlIndex) };
        r[1] = F4{ p2.x, p2.y, p2.z, gn[0] };
        r[2] = F4{ p3.x, p3.y, p3.z, gn[1] };
        r[3] = F4{ t.v1.normal.x, t.v1.normal.y, t.v1.normal.z, gn[2] };
        r[4] = F4{ t.v2.normal.x, t.v2.normal.y, t.v2.normal.z, t.v1.texcoord.x };
        r[5] = F4{ t.v3.normal.x, t.v3.normal.y, t.v3.normal.z, t.v1.texcoord.y };
        r[6] = F4{ t.v2.texcoord.x, t.v2.texcoord.y, t.v3.texcoord.x, t.v3.texcoord.y };
    }
}

inline void build_mat_rec(const RtPackedMaterial* mats, uint64_t n, std::vector<F4>& out)
{
    out.resize((size_t)n * 4);
    for (uint64_t i = 0; i < n; ++i)
    {
        const RtPackedMaterial& m = mats[i];
        auto rgb = [](uint32_t d, float* o) { o[0] = (float)(d & 0xFF) / 255.0f; o[1] = (float)((d >> 8) & 0xFF) / 255.0f; o[2] = (float)((d >> 16) & 0xFF) / 255.0f; };
        float dif[3], spec[3];
        rgb(m.diffuse_albedo, dif); rgb(m.specular_albedo, spec);
        float f = ldexpf(1.0f, (int)(m.emission >> 24) - (128 + 8));
        float em[3] = { (float)(int)(m.emission & 0xFF) * f, (float)(int)((m.emission >> 8) & 0xFF) * f, (float)(int)((m.emission >> 16) & 0xFF) * f };
        uint32_t rm = m.roughness_metalness, it = m.ior_emission_idx_transparency;
        bool textured = (m.diffuse_albedo >> 24) != 0xFF || (m.specular_albedo >> 24) != 0xFF || ((rm >> 8) & 0xFF) != 0xFF ||
                        (rm >> 24) != 0xFF || ((it >> 8) & 0xFF) != 0xFF || (it >> 24) != 0xFF;
        F4* r = &out[(size_t)i * 4];
        r[0] = F4{ dif[0], dif[1], dif[2], (float)(rm & 0xFF) / 255.0f };
        r[1] = F4{ spec[0], spec[1], spec[2], (float)((rm >> 16) & 0xFF) / 255.0f };
        r[2] = F4{ em[0], em[1], em[2], (float)(it & 0xFF) / 25.5f };
        r[3] = F4{ (float)((it >> 16) & 0xFF) / 255.0f, bits_float(textured ? 1u : 0u), 0.0f, 0.0f };
    }
}

inline void build_light_rec(const RtLight* lights, uint64_t n, std::vector<F4>& out)
{
    out.resize((size_t)n * 2);
    for (uint64_t i = 0; i < n; ++i)
    {
        const RtLight& l = lights[i];
        F4* r = &out[(size_t)i * 2];
        if (l.type == RT_LIGHT_TYPE_POINT) r[0] = F4{ l.origin.x, l.origin.y, l.origin.z, 0.0f };
        else
        {
            float vx = l.origin.x * RT_MAX_RENDER_DIST, vy = l.origin.y * RT_MAX_RENDER_DIST, vz = l.origin.z * RT_MAX_RENDER_DIST;
            float d2 = vx * vx + vy * vy + vz * vz;
            float len = sqrtf(d2), inv = 1.0f / sqrtf(d2);
            r[0] = F4{ vx * inv, vy * inv, vz * inv, len };
        }
        r[1] = F4{ l.radiance.x, l.radiance.y, l.radiance.z, bits_float(l.type) };
    }
}

} // namespace rtbvh
