/*
 * rt_refit.cuh — the device side of rt_update_triangles (include/rt_b200.h): new triangle positions, normals and texcoords are
 * turned into the traversal and shading records in place, and the BVH boxes are refit bottom-up with the topology kept.
 * Compiled with -fmad=false like the rest of rt_kernels.cu: every record is the same IEEE binary32 value rt_bvh_layout.h
 * derives on the host at upload.
 */
#pragma once

#include <cfloat>
#include <cstdint>

#include "rt_bvh_layout.h"

// std::min / std::max as the reference's Bounds3 uses them (mathlib.hpp Min / Max): the second operand wins only if strictly
// smaller / larger, so a NaN in either position and the sign of equal zeros resolve the same way on both sides.
__device__ __forceinline__ float refit_min(float a, float b) { return (b < a) ? b : a; }
__device__ __forceinline__ float refit_max(float a, float b) { return (a < b) ? b : a; }

// Triangle first + i from src[i] (RtTriangle: 10 float4 = v1 {position, texcoord, normal}, v2, v3, mtlIndex + padding) into the
// tris_ref, wtris and tri_shade records (build_layout / build_tri_shade).  Kept: the end-of-leaf flag word of wtris and the
// material word of tri_shade (materials stay those of the upload; mtlIndex is never read).
// MOTION (RT_OPT_OBJECT_MOTION): the triangle's tris_ref entry is copied to prev_pos before it is overwritten, so prev_pos holds
// the positions of the call before; the instance without it is the code of the option off (prev_pos is not read).
template <bool MOTION = false>
__global__ void __launch_bounds__(256) k_refit_records(const float4* __restrict__ src, uint32_t first, uint32_t n, float4* tris_ref,
                                                       float4* wtris, float4* tri_shade, float4* prev_pos)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4* t = src + (size_t)i * 10;
    const float4 p1 = t[0], uv1 = t[1], n1 = t[2], p2 = t[3], uv2 = t[4], n2 = t[5], p3 = t[6], uv3 = t[7], n3 = t[8];
    const size_t g = (size_t)first + i;
    if (MOTION)
    {
        const float4 q1 = tris_ref[g * 3 + 0], q2 = tris_ref[g * 3 + 1], q3 = tris_ref[g * 3 + 2];
        prev_pos[g * 3 + 0] = q1; prev_pos[g * 3 + 1] = q2; prev_pos[g * 3 + 2] = q3;
    }
    tris_ref[g * 3 + 0] = p1; tris_ref[g * 3 + 1] = p2; tris_ref[g * 3 + 2] = p3;   // RtRTTriangle, the .w words included
    const float e1x = p2.x - p1.x, e1y = p2.y - p1.y, e1z = p2.z - p1.z;
    const float e2x = p3.x - p1.x, e2y = p3.y - p1.y, e2z = p3.z - p1.z;
    wtris[g * 3 + 0] = make_float4(p1.x, p1.y, p1.z, e1x);
    wtris[g * 3 + 1] = make_float4(e1y, e1z, e2x, e2y);
    reinterpret_cast<float*>(wtris + g * 3 + 2)[0] = e2z;
    const float cx = e1y * e2z - e1z * e2y, cy = e1z * e2x - e1x * e2z, cz = e1x * e2y - e1y * e2x;
    const float inv = 1.0f / sqrtf(cx * cx + cy * cy + cz * cz);          // rtbvh::normalize3
    float4* r = tri_shade + g * 7;
    float* r0 = reinterpret_cast<float*>(r);
    r0[0] = p1.x; r0[1] = p1.y; r0[2] = p1.z;
    r[1] = make_float4(p2.x, p2.y, p2.z, cx * inv);
    r[2] = make_float4(p3.x, p3.y, p3.z, cy * inv);
    r[3] = make_float4(n1.x, n1.y, n1.z, cz * inv);
    r[4] = make_float4(n2.x, n2.y, n2.z, uv1.x);
    r[5] = make_float4(n3.x, n3.y, n3.z, uv1.y);
    r[6] = make_float4(uv2.x, uv2.y, uv3.x, uv3.y);
}

// *bad = 1 if a position coordinate (xyz of v1, v2, v3) of src[0 .. n) (RtTriangle layout) is not finite; the caller clears it
// (rt_update_mesh_triangles_device checks before it writes anything)
__global__ void __launch_bounds__(256) k_check_positions(const float4* __restrict__ src, uint32_t n, uint32_t* bad)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4* t = src + (size_t)i * 10;
    const float4 p1 = t[0], p2 = t[3], p3 = t[6];
    const float s[9] = { p1.x, p1.y, p1.z, p2.x, p2.y, p2.z, p3.x, p3.y, p3.z };
    bool ok = true;
    for (int k = 0; k < 9; ++k) ok = ok && isfinite(s[k]);
    if (!ok) *bad = 1u;
}

// Positions of the listed triangles from tris_ref (the emitter table's areas after an update): 3 float4 per entry.
__global__ void __launch_bounds__(256) k_gather_positions(const float4* __restrict__ tris_ref, const uint32_t* __restrict__ idx, uint32_t n,
                                                          float4* out)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const size_t t = idx[i];
    out[(size_t)i * 3 + 0] = tris_ref[t * 3 + 0]; out[(size_t)i * 3 + 1] = tris_ref[t * 3 + 1]; out[(size_t)i * 3 + 2] = tris_ref[t * 3 + 2];
}

// Box of `node` into nodes_ref (xyz of bounds_min / bounds_max; the .w words are kept) and into its child slot of the parent's
// wide record (rt_bvh_layout.h: slot 0 = floats 0..5, slot 1 = floats 6..11 of the 16-float record).
__device__ __forceinline__ void refit_store(float* nodes_ref, float* wnodes, uint32_t node, uint32_t slot, const float* lo, const float* hi)
{
    float* b = nodes_ref + (size_t)node * 12;
    b[0] = lo[0]; b[1] = lo[1]; b[2] = lo[2]; b[4] = hi[0]; b[5] = hi[1]; b[6] = hi[2];
    if (slot == RT_REFIT_NONE) return;
    float* w = wnodes + (size_t)(slot >> 1) * 16 + (slot & 1u) * 6;
    w[0] = lo[0]; w[1] = lo[1]; w[2] = lo[2]; w[3] = hi[0]; w[4] = hi[1]; w[5] = hi[2];
}

// Leaf box of triangles off .. off + count - 1: start at (FLT_MAX, -FLT_MAX) and fold Union(Bounds3(p1, p2), p3) of every
// triangle in leaf order (Triangle::GetBounds).
__device__ __forceinline__ void refit_leaf_box(const float4* __restrict__ tris_ref, uint32_t off, uint32_t count, float* lo, float* hi)
{
    lo[0] = FLT_MAX; lo[1] = FLT_MAX; lo[2] = FLT_MAX; hi[0] = -FLT_MAX; hi[1] = -FLT_MAX; hi[2] = -FLT_MAX;
    for (uint32_t k = 0; k < count; ++k)
    {
        const float4* t = tris_ref + (size_t)(off + k) * 3;
        const float4 p1 = t[0], p2 = t[1], p3 = t[2];
        lo[0] = refit_min(lo[0], refit_min(refit_min(p1.x, p2.x), p3.x));
        lo[1] = refit_min(lo[1], refit_min(refit_min(p1.y, p2.y), p3.y));
        lo[2] = refit_min(lo[2], refit_min(refit_min(p1.z, p2.z), p3.z));
        hi[0] = refit_max(hi[0], refit_max(refit_max(p1.x, p2.x), p3.x));
        hi[1] = refit_max(hi[1], refit_max(refit_max(p1.y, p2.y), p3.y));
        hi[2] = refit_max(hi[2], refit_max(refit_max(p1.z, p2.z), p3.z));
    }
}

// Bottom-up refit, one thread per leaf, from its refit_leaf_box.  The thread then publishes the box (__threadfence, then one
// atomicAdd on the parent's arrival counter); the second thread to arrive reads both children back from L2 and writes
// Union(first, second), and climbs.  Every box is a fixed function of its children, so the result does not depend on the arrival order.  The depth is at
// most 64 (build_layout checks it), which bounds the climb.  tris_ref holds the new positions (k_refit_records ran before).
__global__ void __launch_bounds__(256) k_refit(const uint32_t* __restrict__ leaves, uint32_t n_leaves, const uint2* __restrict__ link,
                                               uint32_t* arrivals, float* nodes_ref, const float4* __restrict__ tris_ref, float* wnodes)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_leaves) return;
    uint32_t node = leaves[i];
    const float4* nodes4 = reinterpret_cast<const float4*>(nodes_ref);
    const float4 meta = __ldcg(nodes4 + (size_t)node * 3 + 2);
    const uint32_t off = __float_as_uint(meta.x), count = __float_as_uint(meta.y) >> 16;
    float lo[3], hi[3];
    refit_leaf_box(tris_ref, off, count, lo, hi);
    for (;;)
    {
        const uint2 l = link[node];
        refit_store(nodes_ref, wnodes, node, l.y, lo, hi);
        if (l.x == RT_REFIT_NONE) return;
        __threadfence();
        if (atomicAdd(arrivals + l.x, 1u) == 0u) return;     // the sibling is not done yet: it climbs
        __threadfence();
        node = l.x;
        const uint32_t second = __float_as_uint(__ldcg(nodes4 + (size_t)node * 3 + 2).x);
        const float4 amin = __ldcg(nodes4 + (size_t)(node + 1) * 3), amax = __ldcg(nodes4 + (size_t)(node + 1) * 3 + 1);
        const float4 bmin = __ldcg(nodes4 + (size_t)second * 3), bmax = __ldcg(nodes4 + (size_t)second * 3 + 1);
        lo[0] = refit_min(amin.x, bmin.x); lo[1] = refit_min(amin.y, bmin.y); lo[2] = refit_min(amin.z, bmin.z);
        hi[0] = refit_max(amax.x, bmax.x); hi[1] = refit_max(amax.y, bmax.y); hi[2] = refit_max(amax.z, bmax.z);
    }
}
