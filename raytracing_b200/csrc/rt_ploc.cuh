/*
 * rt_ploc.cuh — the device side of rt_rebuild_bvh_ploc (include/rt_b200.h): parallel locally-ordered clustering (Meister & Bittner
 * 2018, "Parallel Locally-Ordered Clustering for Bounding Volume Hierarchy Construction") over the triangles in the key order of
 * rt_rebuild_bvh, one triangle per leaf.  The keys, their sort and every write of the tree are rt_lbvh.cuh's: the clustered tree
 * is turned into the radix-tree form k_lbvh_top and k_lbvh_write read, and k_refit computes the boxes.  Compiled with -fmad=false
 * like the rest of rt_kernels.cu: the distances are the rule's float arithmetic, uncontracted.
 *
 * Any binary tree whose leaves are numbered in its own in-order (0 .. n-1) has the form of a Karras radix tree: an internal node
 * covering leaves [a, b] with split g (its first child covers [a, g]) is indexed b if it is a first child, a if it is a second
 * child or the root (index 0).  Every index in [0, n-2] is used once: index i can only be the first child of the node split at i
 * or the second child of the node split at i - 1, and of these two nodes (both ancestors of leaf i) the lower one has leaf i
 * as the child on that side.  k_ploc_number derives a, b and g from the subtree sizes.
 */
#pragma once

#include <cfloat>
#include <cstdint>

#include <cub/device/device_select.cuh>

#include "rt_b200.h"
#include "rt_lbvh.cuh"
#include "rt_refit.cuh"

#define RT_PLOC_TILE 256
#define RT_PLOC_MAX_DEPTH 64                                  // build_layout's limit: the 64-entry traversal stack

// A cluster: its box, lo.w = its node reference (a leaf is its triangle id, interior node k is n + k), hi.w = leaves under it.
struct PlocCluster { float4 lo, hi; };

// A(lo, hi) of the rule: +inf unless >= 0 and finite
__device__ __forceinline__ float ploc_area(float lx, float ly, float lz, float hx, float hy, float hz)
{
    const float ex = hx - lx, ey = hy - ly, ez = hz - lz;
    const float a = (ex * ey + ey * ez) + ez * ex;
    return (a >= 0.0f && a <= FLT_MAX) ? a : __int_as_float(0x7F800000);
}

// Position i of the initial list: the leaf box of the triangle of sorted key i.
__global__ void __launch_bounds__(256) k_ploc_init(const uint32_t* __restrict__ ids, uint32_t n, const float4* __restrict__ tris_ref,
                                                   PlocCluster* out)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t t = ids[i];
    float lo[3], hi[3];
    refit_leaf_box(tris_ref, t, 1u, lo, hi);
    out[i] = { make_float4(lo[0], lo[1], lo[2], __uint_as_float(t)), make_float4(hi[0], hi[1], hi[2], __uint_as_float(1u)) };
}

// nn[i] = the position j != i within RT_PLOC_RADIUS of i with the smallest A(Union(lower, higher)); at equal distance the
// smaller gap |j - i|, then the pair whose lower position is even, then the smaller j (tk below orders i's candidates so).  Each
// CTA stages its tile and a halo of RT_PLOC_RADIUS clusters on each side.
__global__ void __launch_bounds__(RT_PLOC_TILE) k_ploc_nearest(const PlocCluster* __restrict__ cl, uint32_t count, uint32_t* nn)
{
    constexpr int R = RT_PLOC_RADIUS, S = RT_PLOC_TILE + 2 * RT_PLOC_RADIUS;
    __shared__ float s[6][S];
    const int base = (int)(blockIdx.x * RT_PLOC_TILE) - R;
    for (int k = threadIdx.x; k < S; k += RT_PLOC_TILE)
    {
        const int p = base + k;
        if (p >= 0 && p < (int)count)
        {
            const float4 lo = cl[p].lo, hi = cl[p].hi;
            s[0][k] = lo.x; s[1][k] = lo.y; s[2][k] = lo.z; s[3][k] = hi.x; s[4][k] = hi.y; s[5][k] = hi.z;
        }
    }
    __syncthreads();
    const int i = (int)(blockIdx.x * RT_PLOC_TILE + threadIdx.x);
    if (i >= (int)count) return;
    const int m = threadIdx.x + R;
    const float lx = s[0][m], ly = s[1][m], lz = s[2][m], hx = s[3][m], hy = s[4][m], hz = s[5][m];
    float best = 0.0f;
    int bj = -1;
    uint32_t bt = 0;
#pragma unroll
    for (int o = -R; o <= R; ++o)
    {
        const int j = i + o, q = m + o;
        if (o == 0 || j < 0 || j >= (int)count) continue;
        float d;
        if (o < 0)      // Union(box_j, box_i): the lower position first
            d = ploc_area(refit_min(s[0][q], lx), refit_min(s[1][q], ly), refit_min(s[2][q], lz),
                          refit_max(s[3][q], hx), refit_max(s[4][q], hy), refit_max(s[5][q], hz));
        else
            d = ploc_area(refit_min(lx, s[0][q]), refit_min(ly, s[1][q]), refit_min(lz, s[2][q]),
                          refit_max(hx, s[3][q]), refit_max(hy, s[4][q]), refit_max(hz, s[5][q]));
        const uint32_t tk = ((uint32_t)(o < 0 ? -o : o) * 2u + ((uint32_t)(o < 0 ? j : i) & 1u)) * 2u + (o > 0 ? 1u : 0u);
        if (bj < 0 || d < best || (d == best && tk < bt)) { best = d; bj = j; bt = tk; }
    }
    nn[i] = (uint32_t)bj;
}

// The mutual pairs merge: the lower position i of a pair allocates interior node k (any order: the topology does not depend on
// it), stores its children in the rule's order, its axis and sizes, the children's parent links, and replaces cluster i by the
// merged one; keep[p] = 0 for the higher position of every pair.  inner[k] = (first child, second child, leaves of the first,
// axis), size[k] = leaves under k, parent[node reference] = (k << 1) | (second child).
__global__ void __launch_bounds__(256) k_ploc_merge(PlocCluster* cl, uint32_t count, const uint32_t* __restrict__ nn, uint8_t* keep,
                                                    uint32_t n, uint32_t* made, uint4* inner, uint32_t* size, uint32_t* parent)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const uint32_t j = nn[i];
    const bool mutual = nn[j] == i;
    keep[i] = (mutual && j < i) ? 0 : 1;
    if (!mutual || j < i) return;
    const PlocCluster L = cl[i], H = cl[j];
    const float cl3[3] = { L.lo.x + L.hi.x, L.lo.y + L.hi.y, L.lo.z + L.hi.z };
    const float ch3[3] = { H.lo.x + H.hi.x, H.lo.y + H.hi.y, H.lo.z + H.hi.z };
    const float d[3] = { fabsf(ch3[0] - cl3[0]), fabsf(ch3[1] - cl3[1]), fabsf(ch3[2] - cl3[2]) };
    uint32_t axis = 0;
    if (d[1] > d[axis]) axis = 1;
    if (d[2] > d[axis]) axis = 2;
    const bool h_first = ch3[axis] < cl3[axis];
    const uint32_t rl = __float_as_uint(L.lo.w), rh = __float_as_uint(H.lo.w);
    const uint32_t sl = __float_as_uint(L.hi.w), sh = __float_as_uint(H.hi.w);
    const uint32_t k = atomicAdd(made, 1u);
    const uint32_t first = h_first ? rh : rl, second = h_first ? rl : rh;
    inner[k] = make_uint4(first, second, h_first ? sh : sl, axis);
    size[k] = sl + sh;
    parent[first] = k << 1;
    parent[second] = (k << 1) | 1u;
    cl[i] = { make_float4(refit_min(L.lo.x, H.lo.x), refit_min(L.lo.y, H.lo.y), refit_min(L.lo.z, H.lo.z), __uint_as_float(n + k)),
              make_float4(refit_max(L.hi.x, H.hi.x), refit_max(L.hi.y, H.hi.y), refit_max(L.hi.z, H.hi.z), __uint_as_float(sl + sh)) };
}

// One thread per node reference x: a climb to the root (at most RT_PLOC_MAX_DEPTH levels; a deeper node sets *deep and stops)
// gives its level, its preorder node index and a = the leaves before it in preorder.  A leaf is leaf a of the in-order:
// ids[a] = its triangle.  Interior node x is written in the radix-tree form of k_lbvh_top / k_lbvh_write (see the top of the
// file): inner_k[idx] = (a, b, g, axis) and ipre[idx] = its interior preorder index (node index - a), what k_lbvh_karras and
// k_lbvh_number give the linear BVH.  The subtree sizes come from the clusters (hi.w), so no bottom-up pass is needed.
__global__ void __launch_bounds__(256) k_ploc_number(uint32_t n, const uint4* __restrict__ inner, const uint32_t* __restrict__ size,
                                                     const uint32_t* __restrict__ parent, uint32_t* ids, uint4* inner_k, uint32_t* ipre,
                                                     uint32_t* deep)
{
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= 2 * n - 1) return;
    const uint32_t own = parent[x];
    uint32_t a = 0, pre = 0, level = 1;
    for (uint32_t p = own; p != RT_LBVH_NONE; p = parent[n + (p >> 1)])
    {
        if (++level > RT_PLOC_MAX_DEPTH) { *deep = 1u; return; }
        if (p & 1u)
        {
            const uint32_t first = inner[p >> 1].z;
            a += first; pre += 2u * first;
        }
        else
            pre += 1u;
    }
    if (x < n) { ids[a] = x; return; }
    const uint4 u = inner[x - n];
    const uint32_t b = a + size[x - n] - 1u, g = a + u.z - 1u;
    const uint32_t idx = (own == RT_LBVH_NONE || (own & 1u)) ? a : b;
    inner_k[idx] = make_uint4(a, b, g, u.w);
    ipre[idx] = pre - a;
}

// The end-of-leaf flag of every wtris record (one triangle per leaf), written once the tree is known to fit.
__global__ void __launch_bounds__(256) k_ploc_flags(uint32_t n, float4* wtris)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) reinterpret_cast<uint32_t*>(wtris + (size_t)i * 3 + 2)[1] = 1u;
}
