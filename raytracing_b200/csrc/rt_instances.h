/*
 * rt_instances.h — the host half of instanced scenes (rt_upload_instanced_scene / rt_set_instances, include/rt_b200.h): the check
 * and inversion of each instance's matrix, the virtual triangle ids, and the top-level tree over the instances.  Shared by the
 * library and the host harness the tests compare with an independent restatement (tests/instance_tree_model.py).
 * Compile with -ffp-contract=off.
 *
 * Per instance i with object-to-world M (row-major 3x4, rows r0 r1 r2) and mesh m:
 *   det    of the 3x3 part in double; rejected unless every entry of M is finite and det != 0.
 *   W      world-to-object: the 3x3 inverse adj(A) / det and the translation -(inverse * t), both in double, rounded to float.
 *   base   the prefix sum of n_triangles(mesh) in instance order; the sum must stay below RT_INVALID_ID (0xFFFFFFFF).
 *   box    the 8 corners of the mesh's root box (node first_node of the mesh) transformed by M in double
 *          (x = ((m00*cx + m01*cy) + m02*cz) + m03), min / max per component, widened by pad = RT_INST_BOX_PAD * s on each side,
 *          s = the largest |value| of the six, and rounded outward to float.  The box only culls; the pad covers the rounding of
 *          the ray transform.
 * Top-level tree (one instance per leaf), built recursively over a list of instances, starting with all of them in index order:
 *   one instance: a leaf.  Otherwise centroid c = (lo + hi) * 0.5f (float) per instance; the centroid bounds' extent per axis
 *   (float max - min); axis = 0, then 1 if ext1 > ext_axis, then 2 if ext2 > ext_axis; the list is sorted stably by (c[axis],
 *   instance id); the first child gets the first n / 2 (rounded down), the second the rest.  An interior node's box is the
 *   union of its children's boxes (min(a, b) = b < a ? b : a, max(a, b) = a < b ? b : a, as the refit rule).
 * Records: rt_bvh_layout.h's child-box layout, interior nodes numbered in depth-first preorder (root = record 0, first child
 * before second); a child reference >= 0 is a record, < 0 is the leaf of instance ~ref; the split axis is the node's axis.
 * The depth is at most ceil(log2 n) + 1, well inside the 64-entry stack of the traversal.
 */
#pragma once

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "rt_b200.h"

#define RT_INST_BOX_PAD 0x1p-20

namespace rtinst
{

struct Box { float lo[3], hi[3]; };

// The instance's world-to-object matrix (12 floats, row-major 3x4) and the sign of det (+1 / -1); false for a matrix that is not
// finite or is singular.
inline bool invert(const float* m, float* w, float* det_sign)
{
    for (int k = 0; k < 12; ++k) if (!std::isfinite(m[k])) return false;
    const double a = m[0], b = m[1], c = m[2], d = m[4], e = m[5], f = m[6], g = m[8], h = m[9], k = m[10];
    const double det = a * (e * k - f * h) - b * (d * k - f * g) + c * (d * h - e * g);
    if (!(det != 0.0) || !std::isfinite(det)) return false;
    const double inv[9] = { (e * k - f * h) / det, (c * h - b * k) / det, (b * f - c * e) / det,
                            (f * g - d * k) / det, (a * k - c * g) / det, (c * d - a * f) / det,
                            (d * h - e * g) / det, (b * g - a * h) / det, (a * e - b * d) / det };
    const double t[3] = { m[3], m[7], m[11] };
    for (int r = 0; r < 3; ++r)
    {
        for (int col = 0; col < 3; ++col) w[4 * r + col] = (float)inv[3 * r + col];
        w[4 * r + 3] = (float)(-(inv[3 * r] * t[0] + inv[3 * r + 1] * t[1] + inv[3 * r + 2] * t[2]));
    }
    *det_sign = det < 0.0 ? -1.0f : 1.0f;
    return true;
}

inline float round_down(double v) { float f = (float)v; return (double)f > v ? std::nextafter(f, -INFINITY) : f; }
inline float round_up(double v) { float f = (float)v; return (double)f < v ? std::nextafter(f, INFINITY) : f; }

// World box of a mesh root box (lo, hi) placed by M.
inline Box world_box(const float* m, const float* lo, const float* hi)
{
    double mn[3] = { INFINITY, INFINITY, INFINITY }, mx[3] = { -INFINITY, -INFINITY, -INFINITY };
    for (int corner = 0; corner < 8; ++corner)
    {
        const double p[3] = { (corner & 1) ? hi[0] : lo[0], (corner & 2) ? hi[1] : lo[1], (corner & 4) ? hi[2] : lo[2] };
        for (int r = 0; r < 3; ++r)
        {
            const double v = (((double)m[4 * r] * p[0] + (double)m[4 * r + 1] * p[1]) + (double)m[4 * r + 2] * p[2]) + (double)m[4 * r + 3];
            mn[r] = std::min(mn[r], v); mx[r] = std::max(mx[r], v);
        }
    }
    double s = 0.0;
    for (int r = 0; r < 3; ++r) s = std::max(s, std::max(std::fabs(mn[r]), std::fabs(mx[r])));
    const double pad = RT_INST_BOX_PAD * s;
    Box b;
    for (int r = 0; r < 3; ++r) { b.lo[r] = round_down(mn[r] - pad); b.hi[r] = round_up(mx[r] + pad); }
    return b;
}

inline float fmin_(float a, float b) { return b < a ? b : a; }
inline float fmax_(float a, float b) { return a < b ? b : a; }
inline Box unite(const Box& a, const Box& b)
{
    Box u;
    for (int r = 0; r < 3; ++r) { u.lo[r] = fmin_(a.lo[r], b.lo[r]); u.hi[r] = fmax_(a.hi[r], b.hi[r]); }
    return u;
}

struct Tree
{
    std::vector<float> records;   // 16 floats per interior node (rt_bvh_layout.h's layout)
    Box root = {};                // union of every instance box
    int root_ref = 0;             // 0, or ~0 for a single instance
};

inline float int_bits(int v) { float f; memcpy(&f, &v, 4); return f; }

// Builds records for the instances in ids (n >= 2) at record `at` and returns the subtree's box.
inline Box build_node(const std::vector<Box>& boxes, std::vector<uint32_t> ids, Tree& t, int& ref)
{
    if (ids.size() == 1) { ref = ~(int)ids[0]; return boxes[ids[0]]; }
    const int at = (int)(t.records.size() / 16);
    ref = at;
    t.records.resize(t.records.size() + 16);
    float cmin[3] = { INFINITY, INFINITY, INFINITY }, cmax[3] = { -INFINITY, -INFINITY, -INFINITY };
    std::vector<float> cen(ids.size() * 3);
    for (size_t i = 0; i < ids.size(); ++i)
        for (int r = 0; r < 3; ++r)
        {
            const float c = (boxes[ids[i]].lo[r] + boxes[ids[i]].hi[r]) * 0.5f;
            cen[3 * i + r] = c; cmin[r] = fmin_(cmin[r], c); cmax[r] = fmax_(cmax[r], c);
        }
    int axis = 0;
    const float ext[3] = { cmax[0] - cmin[0], cmax[1] - cmin[1], cmax[2] - cmin[2] };
    if (ext[1] > ext[axis]) axis = 1;
    if (ext[2] > ext[axis]) axis = 2;
    std::vector<size_t> order(ids.size());
    for (size_t i = 0; i < order.size(); ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](size_t x, size_t y) {
        const float cx = cen[3 * x + axis], cy = cen[3 * y + axis];
        return cx < cy || (cx == cy && ids[x] < ids[y]);
    });
    const size_t half = ids.size() / 2;
    std::vector<uint32_t> lo_ids, hi_ids;
    for (size_t i = 0; i < order.size(); ++i) (i < half ? lo_ids : hi_ids).push_back(ids[order[i]]);
    int r0 = 0, r1 = 0;
    const Box b0 = build_node(boxes, std::move(lo_ids), t, r0);
    const Box b1 = build_node(boxes, std::move(hi_ids), t, r1);
    float* rec = t.records.data() + 16 * (size_t)at;
    const float v[16] = { b0.lo[0], b0.lo[1], b0.lo[2], b0.hi[0], b0.hi[1], b0.hi[2], b1.lo[0], b1.lo[1],
                          b1.lo[2], b1.hi[0], b1.hi[1], b1.hi[2], int_bits(r0), int_bits(r1), int_bits(axis), 0.0f };
    memcpy(rec, v, sizeof(v));
    return unite(b0, b1);
}

// The top-level tree over n >= 1 instance boxes.
inline void build_tree(const std::vector<Box>& boxes, Tree& t)
{
    t.records.clear();
    std::vector<uint32_t> ids(boxes.size());
    for (size_t i = 0; i < ids.size(); ++i) ids[i] = (uint32_t)i;
    t.root = build_node(boxes, std::move(ids), t, t.root_ref);
}

// Device record of one instance: 8 float4 = W rows (3), M rows (3), (mesh root ref, mesh's first record in float4, first
// triangle, base) as int bits, (det sign, first node as int bits, -, -).
struct Prepared
{
    std::vector<float> rec;       // 32 floats per instance
    std::vector<uint32_t> base;   // one per instance
    std::vector<Box> boxes;
    Tree tree;
};

struct MeshInfo { int root_ref; uint32_t rec_f4, first_tri, n_tris, first_node; float lo[3], hi[3]; };

inline bool prepare(const RtInstance* inst, uint32_t n, const std::vector<MeshInfo>& meshes, Prepared& out, std::string& err)
{
    out.rec.assign((size_t)n * 32, 0.0f); out.base.assign(n, 0u); out.boxes.resize(n);
    uint64_t next = 0;
    for (uint32_t i = 0; i < n; ++i)
    {
        const RtInstance& in = inst[i];
        if (in.mesh >= meshes.size()) { err = "instance " + std::to_string(i) + " names mesh " + std::to_string(in.mesh) + " of " + std::to_string(meshes.size()); return false; }
        float* r = out.rec.data() + (size_t)i * 32;
        float sign = 1.0f;
        if (!invert(in.object_to_world, r, &sign)) { err = "instance " + std::to_string(i) + " has a matrix that is not finite or is singular"; return false; }
        const MeshInfo& m = meshes[in.mesh];
        memcpy(r + 12, in.object_to_world, 48);
        out.base[i] = (uint32_t)next;
        const int w[4] = { m.root_ref, (int)m.rec_f4, (int)m.first_tri, (int)next };
        memcpy(r + 24, w, 16);
        r[28] = sign; r[29] = int_bits((int)m.first_node);
        next += m.n_tris;
        if (next >= 0xFFFFFFFFull) { err = "the instances cover 2^32 - 1 or more triangle ids"; return false; }
        out.boxes[i] = world_box(in.object_to_world, m.lo, m.hi);
    }
    if (n) build_tree(out.boxes, out.tree);
    else out.tree = Tree();
    return true;
}

} // namespace rtinst
