/*
 * rt_lbvh.cuh — the device side of rt_rebuild_bvh (include/rt_b200.h): a linear BVH (one triangle per leaf, Morton order) built
 * from the device copy of the positions, written straight into the reference-layout nodes, the traversal records and the refit
 * map, without a host round trip.  Steps: the key-point bounds, one key per triangle, a radix sort (CUB, the toolkit's), the
 * Karras (2012) internal nodes, preorder numbering, the breadth-first top records (one CTA), the node / record / map writes; the
 * boxes then come from k_refit (rt_refit.cuh), so the box rule lives in one place.  Compiled with -fmad=false like the rest of
 * rt_kernels.cu: the key arithmetic is the rule's float arithmetic, uncontracted.
 */
#pragma once

#include <cstdint>

#include <cub/device/device_radix_sort.cuh>

#include "rt_bvh_layout.h"
#include "rt_refit.cuh"

#define RT_LBVH_NONE 0xFFFFFFFFu

// Order-preserving float -> uint32 map (finite values only, never 0), so that 0 is the identity of an atomicMax reduction:
// bounds[a] holds ~lbvh_ord(min) and bounds[3 + a] lbvh_ord(max) of the finite key points of axis a.
__device__ __forceinline__ uint32_t lbvh_ord(float f)
{
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float lbvh_unord(uint32_t o) { return __uint_as_float((o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o); }

// s = (p1 + p2) + p3 per component (the rule's key point)
__device__ __forceinline__ float3 lbvh_key_point(const float4* __restrict__ tris_ref, uint32_t i)
{
    const float4 p1 = tris_ref[(size_t)i * 3], p2 = tris_ref[(size_t)i * 3 + 1], p3 = tris_ref[(size_t)i * 3 + 2];
    return make_float3((p1.x + p2.x) + p3.x, (p1.y + p2.y) + p3.y, (p1.z + p2.z) + p3.z);
}

// Per-axis min / max over the finite key points; `bounds` (6 words) is zero before the launch.
__global__ void __launch_bounds__(256) k_lbvh_bounds(const float4* __restrict__ tris_ref, uint32_t n, uint32_t* bounds)
{
    uint32_t lo[3] = { 0u, 0u, 0u }, hi[3] = { 0u, 0u, 0u };       // ~ord(min), ord(max); 0 = no finite value yet
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    {
        const float3 s = lbvh_key_point(tris_ref, i);
        const float v[3] = { s.x, s.y, s.z };
        for (int a = 0; a < 3; ++a)
            if (isfinite(v[a]))
            {
                const uint32_t o = lbvh_ord(v[a]);
                lo[a] = max(lo[a], ~o); hi[a] = max(hi[a], o);
            }
    }
    for (int a = 0; a < 3; ++a)
    {
        const uint32_t l = __reduce_max_sync(0xFFFFFFFFu, lo[a]), h = __reduce_max_sync(0xFFFFFFFFu, hi[a]);
        if ((threadIdx.x & 31u) == 0u)
        {
            if (l) atomicMax(bounds + a, l);
            if (h) atomicMax(bounds + 3 + a, h);
        }
    }
}

// bit j of q -> bit 3j (the caller shifts by the axis' offset)
__device__ __forceinline__ uint32_t lbvh_spread(uint32_t q)
{
    q = (q | (q << 16)) & 0x030000FFu;
    q = (q | (q << 8)) & 0x0300F00Fu;
    q = (q | (q << 4)) & 0x030C30C3u;
    q = (q | (q << 2)) & 0x09249249u;
    return q;
}

// One 30-bit Morton code per triangle (ids = the identity, the sort's values), and the end-of-leaf flag of every wtris record
// (one triangle per leaf).
__global__ void __launch_bounds__(256) k_lbvh_keys(const float4* __restrict__ tris_ref, uint32_t n, const uint32_t* __restrict__ bounds,
                                                   uint32_t* codes, uint32_t* ids, float4* wtris)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float3 s = lbvh_key_point(tris_ref, i);
    const float v[3] = { s.x, s.y, s.z };
    uint32_t code = 0;
    for (int a = 0; a < 3; ++a)
    {
        uint32_t q = 0;
        const uint32_t bl = bounds[a], bh = bounds[3 + a];
        if (isfinite(v[a]) && bl && bh)
        {
            const float lo = lbvh_unord(~bl), hi = lbvh_unord(bh);
            const float k = (hi > lo) ? 1024.0f / (hi - lo) : 0.0f;
            const float x = (v[a] - lo) * k;
            q = (x >= 1023.0f) ? 1023u : (x > 0.0f ? (uint32_t)x : 0u);     // NaN: 0
        }
        code |= lbvh_spread(q) << (2 - a);
    }
    codes[i] = code; ids[i] = i;
    reinterpret_cast<uint32_t*>(wtris + (size_t)i * 3 + 2)[1] = 1u;
}

__device__ __forceinline__ uint64_t lbvh_key(const uint32_t* __restrict__ codes, const uint32_t* __restrict__ ids, int64_t j)
{
    return ((uint64_t)codes[j] << 32) | ids[j];
}
// length of the common prefix of key i (ki) and key j; -1 outside [0, n)
__device__ __forceinline__ int lbvh_delta(const uint32_t* __restrict__ codes, const uint32_t* __restrict__ ids, int64_t n, uint64_t ki, int64_t j)
{
    return (j < 0 || j >= n) ? -1 : __clzll(ki ^ lbvh_key(codes, ids, j));
}

// Internal node i of the radix tree over the sorted keys (Karras 2012, "Maximizing parallelism in the construction of BVHs,
// octrees, and k-d trees"): inner[i] = (first leaf a, last leaf b, split g, axis); the first child covers [a, g], the second
// [g + 1, b]; a child range of one key is a leaf, otherwise it is internal node g (first) or g + 1 (second).
// parent[x] = (parent internal node << 1) | (x is its second child), RT_LBVH_NONE for the root (node 0).
__global__ void __launch_bounds__(256) k_lbvh_karras(const uint32_t* __restrict__ codes, const uint32_t* __restrict__ ids, uint32_t n,
                                                     uint4* inner, uint32_t* parent)
{
    const int64_t i = blockIdx.x * blockDim.x + threadIdx.x, nn = n;
    if (i >= nn - 1) return;
    const uint64_t ki = lbvh_key(codes, ids, i);
    const int d = (lbvh_delta(codes, ids, nn, ki, i + 1) - lbvh_delta(codes, ids, nn, ki, i - 1)) > 0 ? 1 : -1;
    const int dmin = lbvh_delta(codes, ids, nn, ki, i - d);
    int64_t lmax = 2;
    while (lbvh_delta(codes, ids, nn, ki, i + lmax * d) > dmin) lmax *= 2;
    int64_t l = 0;
    for (int64_t t = lmax >> 1; t >= 1; t >>= 1)
        if (lbvh_delta(codes, ids, nn, ki, i + (l + t) * d) > dmin) l += t;
    const int64_t j = i + l * d;
    const int dnode = lbvh_delta(codes, ids, nn, ki, j);
    int64_t s = 0, t = l;
    do
    {
        t = (t + 1) >> 1;
        if (lbvh_delta(codes, ids, nn, ki, i + (s + t) * d) > dnode) s += t;
    } while (t > 1);
    const uint32_t g = (uint32_t)(i + s * d + (d < 0 ? -1 : 0));
    const uint32_t a = (uint32_t)min(i, j), b = (uint32_t)max(i, j);
    const int h = 63 - dnode;                                  // highest bit in which key[a] and key[b] differ
    const uint32_t axis = h >= 32 ? 2u - (uint32_t)((h - 32) % 3) : 0u;
    inner[i] = make_uint4(a, b, g, axis);
    if (a != g) parent[g] = (uint32_t)i << 1;
    if (b != g + 1u) parent[g + 1] = ((uint32_t)i << 1) | 1u;
    if (i == 0) parent[0] = RT_LBVH_NONE;
}

// Interior preorder index of internal node i: a + d - r (d ancestors, r of which it lies in the second branch of): the nodes
// before it in preorder are its d ancestors and the r complete subtrees left of its path, which hold leaves [0, a).
__global__ void __launch_bounds__(256) k_lbvh_number(const uint4* __restrict__ inner, const uint32_t* __restrict__ parent, uint32_t n_inner,
                                                     uint32_t* ipre)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_inner) return;
    uint32_t d = 0, r = 0;
    for (uint32_t p = parent[i]; p != RT_LBVH_NONE; p = parent[p >> 1]) { ++d; r += p & 1u; }
    ipre[i] = inner[i].x + d - r;
}

// One CTA of 1024 threads: the first top_n (<= 1024) interior nodes in breadth-first order (first child before second), one
// level per step, then sorted by interior preorder index: top[k] = (interior preorder index, breadth-first record), ascending.
__global__ void __launch_bounds__(1024) k_lbvh_top(const uint4* __restrict__ inner, const uint32_t* __restrict__ ipre, uint32_t top_n,
                                                   uint2* top)
{
    __shared__ uint32_t bfs[RT_BVH_TOP_RECORDS];
    __shared__ uint32_t warp_sum[32];
    __shared__ uint32_t s_total;
    const uint32_t t = threadIdx.x, lane = t & 31u, warp = t >> 5;
    uint32_t head = 0, count = 1;
    if (t == 0) bfs[0] = 0;
    __syncthreads();
    while (count < top_n && head < count)
    {
        const uint32_t f = count - head;
        uint4 u = make_uint4(0, 0, 0, 0);
        bool c0 = false, c1 = false;
        if (t < f)
        {
            u = inner[bfs[head + t]];
            c0 = u.x != u.z; c1 = u.y != u.z + 1u;               // interior children
        }
        const uint32_t k = (uint32_t)c0 + (uint32_t)c1;
        // block exclusive scan of k
        uint32_t incl = k;
        for (int o = 1; o < 32; o <<= 1)
        {
            const uint32_t v = __shfl_up_sync(0xFFFFFFFFu, incl, o);
            if (lane >= (uint32_t)o) incl += v;
        }
        if (lane == 31) warp_sum[warp] = incl;
        __syncthreads();
        if (warp == 0)
        {
            uint32_t w = warp_sum[lane], wi = w;
            for (int o = 1; o < 32; o <<= 1)
            {
                const uint32_t v = __shfl_up_sync(0xFFFFFFFFu, wi, o);
                if (lane >= (uint32_t)o) wi += v;
            }
            warp_sum[lane] = wi - w;
            if (lane == 31) s_total = wi;
        }
        __syncthreads();
        uint32_t pos = count + warp_sum[warp] + incl - k;
        if (c0 && pos < top_n) bfs[pos++] = u.z;
        if (c1 && pos < top_n) bfs[pos] = u.z + 1u;
        head = count;
        count = min(count + s_total, top_n);
        __syncthreads();
    }
    const uint32_t mine = t < top_n ? ipre[bfs[t]] : 0u;
    __syncthreads();
    if (t < top_n) bfs[t] = mine;
    __syncthreads();
    if (t < top_n)
    {   // rank among the top_n (the indices are distinct)
        uint32_t rank = 0;
        for (uint32_t j = 0; j < top_n; ++j) rank += bfs[j] < mine ? 1u : 0u;
        top[rank] = make_uint2(mine, t);
    }
}

// Record of the interior node with interior preorder index x: its breadth-first slot if it is one of the top_n, otherwise
// top_n + x - (top records before it in preorder).
__device__ __forceinline__ uint32_t lbvh_record(const uint2* __restrict__ top, uint32_t top_n, uint32_t x)
{
    uint32_t lo = 0, hi = top_n;                                // first entry >= x
    while (lo < hi)
    {
        const uint32_t m = (lo + hi) >> 1;
        if (top[m].x < x) lo = m + 1; else hi = m;
    }
    return (lo < top_n && top[lo].x == x) ? top[lo].y : top_n + x - lo;
}

__device__ __forceinline__ void lbvh_store_node(float4* nodes_ref, uint32_t node, uint32_t offset, uint32_t prims_axis)
{
    float4* p = nodes_ref + (size_t)node * 3;
    p[0] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);                 // boxes: k_refit; the .w words and the padding stay 0
    p[1] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    p[2] = make_float4(__uint_as_float(offset), __uint_as_float(prims_axis), 0.0f, 0.0f);
}

// Internal node i: its node, its children's leaf nodes, its record's child references and axis, and the refit map entries of
// its children (link = (parent node, record * 2 + slot); leaves[j] = node of sorted leaf j).  Preorder: the first child is
// node + 1, the second node + 2 * (leaves of the first child).
__global__ void __launch_bounds__(256) k_lbvh_write(const uint4* __restrict__ inner, const uint32_t* __restrict__ ipre,
                                                    const uint32_t* __restrict__ ids, const uint2* __restrict__ top, uint32_t top_n,
                                                    uint32_t n_inner, float4* nodes_ref, float4* wnodes, uint2* link, uint32_t* leaves)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_inner) return;
    const uint4 u = inner[i];
    const uint32_t a = u.x, b = u.y, g = u.z, axis = u.w;
    const uint32_t x = ipre[i], node = x + a, rec = lbvh_record(top, top_n, x);
    const uint32_t n0 = node + 1u, n1 = node + 2u * (g - a + 1u);
    int r0, r1;
    if (a == g) { r0 = ~(int)ids[g]; lbvh_store_node(nodes_ref, n0, ids[g], 1u << 16); leaves[g] = n0; }
    else r0 = (int)lbvh_record(top, top_n, ipre[g]);
    if (b == g + 1u) { r1 = ~(int)ids[g + 1]; lbvh_store_node(nodes_ref, n1, ids[g + 1], 1u << 16); leaves[g + 1] = n1; }
    else r1 = (int)lbvh_record(top, top_n, ipre[g + 1]);
    lbvh_store_node(nodes_ref, node, n1, axis);
    wnodes[(size_t)rec * 4 + 3] = make_float4(__int_as_float(r0), __int_as_float(r1), __uint_as_float(axis), 0.0f);
    link[n0] = make_uint2(node, rec * 2u);
    link[n1] = make_uint2(node, rec * 2u + 1u);
    if (i == 0) link[0] = make_uint2(RT_REFIT_NONE, RT_REFIT_NONE);
}

// n = 1: the root is the single leaf; one zero record; the triangle's flag.
__global__ void k_lbvh_single(float4* nodes_ref, float4* wnodes, float4* wtris, uint2* link, uint32_t* leaves)
{
    lbvh_store_node(nodes_ref, 0, 0, 1u << 16);
    for (int k = 0; k < 4; ++k) wnodes[k] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    reinterpret_cast<uint32_t*>(wtris + 2)[1] = 1u;
    link[0] = make_uint2(RT_REFIT_NONE, RT_REFIT_NONE);
    leaves[0] = 0;
}
