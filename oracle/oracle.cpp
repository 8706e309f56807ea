/*
 * oracle.cpp — TEST INFRASTRUCTURE.  Scalar CPU restatement of the reference's
 * wavefront path-tracing hot path, one function per reference kernel/helper, each
 * citing the file:line it follows (paths relative to /root/reference/src).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may load
 * this library; the product (raytracing_b200/csrc) never does.
 *
 * PARITY PIN: the reference ships no golden vectors (SURVEY 4, 8c).  This
 * restatement is pinned against the reference's own kernels compiled for the CPU
 * (oracle/_ref, built by oracle/build_ref.py where /root/reference exists):
 * tests/test_oracle_vs_ref.py requires bit-identical primary hits, per-bounce
 * counters and radiance, and tests/golden/ holds outputs of oracle/_ref.
 *
 * Arithmetic policy (shared with the CUDA kernels): IEEE binary32, no FMA
 * contraction (-ffp-contract=off), left-to-right sums, transcendental functions
 * from include/rt_math.h, min/max with fmin/fmax semantics, the one fp64
 * sub-expression of GGX_Sample (bxdf.h:160) evaluated in double.
 */
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "rt_math.h"
#include "rt_types.h"

namespace
{

struct V3 { float x, y, z; };
struct V2 { float x, y; };

inline V3 v3(float x, float y, float z) { return V3{ x, y, z }; }
inline V3 v3(const RtFloat3& f) { return V3{ f.x, f.y, f.z }; }
inline V3 operator+(V3 a, V3 b) { return v3(a.x + b.x, a.y + b.y, a.z + b.z); }
inline V3 operator-(V3 a, V3 b) { return v3(a.x - b.x, a.y - b.y, a.z - b.z); }
inline V3 operator*(V3 a, V3 b) { return v3(a.x * b.x, a.y * b.y, a.z * b.z); }
inline V3 operator/(V3 a, V3 b) { return v3(a.x / b.x, a.y / b.y, a.z / b.z); }
inline V3 operator*(V3 a, float b) { return v3(a.x * b, a.y * b, a.z * b); }
inline V3 operator*(float a, V3 b) { return v3(a * b.x, a * b.y, a * b.z); }
inline V3 operator/(V3 a, float b) { return v3(a.x / b, a.y / b, a.z / b); }
inline V3 operator-(float a, V3 b) { return v3(a - b.x, a - b.y, a - b.z); }
inline V3 operator-(V3 a) { return v3(-a.x, -a.y, -a.z); }
inline float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
inline V3 cross(V3 a, V3 b) { return v3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
inline float length(V3 a) { return sqrtf(dot(a, a)); }
inline V3 normalize(V3 a) { float inv = 1.0f / sqrtf(dot(a, a)); return a * inv; }
inline V3 splat(float a) { return v3(a, a, a); }
inline V3 mix(V3 a, V3 b, float t) { return a + (b - a) * t; }

// ------------------------------------------------------------------ RNG
// kernels/common/utils.h:113-121
inline uint32_t WangHash(uint32_t x)
{
    x = (x ^ 61u) ^ (x >> 16);
    x = x + (x << 3);
    x = x ^ (x >> 4);
    x = x * 0x27d4eb2du;
    x = x ^ (x >> 15);
    return x;
}

// kernels/cl/raygeneration.cl:28-38 — Wang-hash rounds, then one LCG step
inline float GetRandomFloat(uint32_t* seed)
{
    uint32_t s = WangHash(*seed);
    s = 1103515245u * s + 12345u;
    *seed = s;
    return (float)s * 2.3283064365386963e-10f;
}

// kernels/common/sampling.h:40-61 (kBlueNoise sampler).  The tables are the caller's (the reference ships them in
// utils/blue_noise_sampler.hpp); orc_set_sampler_tables selects the sampler for the renders that follow.
// sampling.h:50 indexes rankingTile with the un-wrapped dimension, which runs past the table's end for the last
// tile pixels once the dimension exceeds 7 (undefined in the reference): such reads return 0 (include/rt_b200.h).
static const int32_t* g_bn_sobol = nullptr;
static const int32_t* g_bn_scrambling = nullptr;
static const int32_t* g_bn_ranking = nullptr;
inline float SampleBlueNoise(int pixel_i, int pixel_j, int sample_index, int sample_dimension)
{
    pixel_i = pixel_i & 127;
    pixel_j = pixel_j & 127;
    sample_index = sample_index & 255;
    sample_dimension = sample_dimension & 255;
    int tile = (pixel_i + pixel_j * 128) * 8;
    int ranking_index = sample_dimension + tile;
    int ranked_sample_index = sample_index ^ (ranking_index < RT_BN_TILE_COUNT ? g_bn_ranking[ranking_index] : 0);
    int value = g_bn_sobol[sample_dimension + ranked_sample_index * 256];
    value = value ^ g_bn_scrambling[(sample_dimension % 8) + tile];
    return (0.5f + (float)value) / 256.0f;
}

// kernels/common/sampling.h:64-82.  kRandom results are in [0,1] INCLUSIVE.
inline float SampleRandom(uint32_t px, uint32_t py, uint32_t sample_index, uint32_t bounce, uint32_t type)
{
    uint32_t dim = bounce * 5u + type;
    if (g_bn_sobol) return SampleBlueNoise((int)px, (int)py, (int)sample_index, (int)dim);
    uint32_t seed = WangHash(px);
    seed = WangHash(seed + WangHash(py));
    seed = WangHash(seed + WangHash(sample_index));
    seed = WangHash(seed + WangHash(dim));
    return (float)seed * 2.3283064365386963e-10f;
}
enum { SAMPLE_LAYER = 1, SAMPLE_U = 2, SAMPLE_V = 3, SAMPLE_LIGHT = 4 };

// ------------------------------------------------------------------ scene view
struct Scene
{
    const RtTriangle* triangles; uint32_t n_triangles;
    const RtLinearBVHNode* nodes; uint32_t n_nodes;
    const RtPackedMaterial* materials; uint32_t n_materials;
    const RtLight* lights; uint32_t n_lights;
    const RtTexture* textures; uint32_t n_textures;
    const uint32_t* texels; uint32_t n_texels;
    const float* env; uint32_t env_w, env_h;
    RtSceneInfo info;
};

struct Ray { V3 o; float tmin; V3 d; float tmax; };

// ------------------------------------------------------------------ ray generation
// kernels/cl/raygeneration.cl:40-49.  x can be 3 when the random float is exactly
// 1.0f (p ~ 3e-8): the reference then reads past hexPoints[]; here the index is
// clamped to 2 (documented deviation; the result is scaled by aperture anyway).
inline V2 PointInHexagon(uint32_t* seed)
{
    const V2 hex[3] = { { -1.0f, 0.0f }, { 0.5f, 0.866f }, { 0.5f, -0.866f } };
    int x = (int)floorf(GetRandomFloat(seed) * 3.0f);
    if (x > 2) x = 2;
    V2 v1 = hex[x], v2 = hex[(x + 1) % 3];
    float p1 = GetRandomFloat(seed), p2 = GetRandomFloat(seed);
    return V2{ p1 * v1.x + p2 * v2.x, p1 * v1.y + p2 * v2.y };
}

// kernels/cl/raygeneration.cl:65-139
inline Ray RayGeneration(uint32_t pixel_idx, uint32_t width, uint32_t height, const RtCamera& cam, uint32_t sample_idx)
{
    uint32_t px = pixel_idx % width, py = pixel_idx / width;
    float inv_w = 1.0f / (float)width, inv_h = 1.0f / (float)height;
    uint32_t seed = pixel_idx + (1103515245u * sample_idx + 12345u);          // :98, HashUInt32 :61
    float x = ((float)px + GetRandomFloat(&seed)) * inv_w;
    float y = ((float)py + GetRandomFloat(&seed)) * inv_h;
    float angle = rt_tanf(0.5f * cam.fov);
    x = (x * 2.0f - 1.0f) * angle * cam.aspect_ratio;
    y = (y * 2.0f - 1.0f) * angle;
    V3 front = v3(cam.front), up = v3(cam.up), pos = v3(cam.position);
    V3 right = cross(front, up);
    V3 dir = normalize(x * right + y * up + front);
    V3 aimed = pos + cam.focus_distance * dir;
    V2 dof = PointInHexagon(&seed);
    float r = cam.aperture;
    V3 new_pos = pos + dof.x * r * right + dof.y * r * up;
    Ray ray;
    ray.o = new_pos; ray.tmin = 0.0f;
    ray.d = normalize(aimed - new_pos); ray.tmax = RT_MAX_RENDER_DIST;
    return ray;
}

// ------------------------------------------------------------------ traversal
struct TraceCounters { uint64_t nodes_visited, tris_tested; };

#ifdef ORACLE_FMA_TRAVERSAL
// Build variant liboracle_fma.so (make fma): a CPU MODEL of the CUDA kernels' -DRT_FMA_TRAVERSAL experiment build
// (raytracing_b200/csrc/rt_traverse.cuh: slab planes as fma(plane, inv, -(o * inv)), cross and dot products of the triangle test
// contracted the same way).  It is not part of any parity test and nothing ships with it: tools/fma_sensitivity.py uses it to
// report how far a contracted traversal moves the image (profiles/r02_fma_sensitivity.txt).
inline float fdot(V3 a, V3 b) { return fmaf(a.x, b.x, fmaf(a.y, b.y, a.z * b.z)); }
inline V3 fcross(V3 a, V3 b) { return v3(fmaf(a.y, b.z, -(a.z * b.y)), fmaf(a.z, b.x, -(a.x * b.z)), fmaf(a.x, b.y, -(a.y * b.x))); }
inline bool RayTriangleFma(const Ray& ray, V3 p1, V3 p2, V3 p3, float* u_out, float* v_out, float* t_out)
{
    V3 e1 = p2 - p1, e2 = p3 - p1;
    V3 pvec = fcross(ray.d, e2);
    float det = fdot(e1, pvec);
    if (det < 1e-8f || -det > 1e-8f) return false;
    float inv_det = 1.0f / det;
    V3 tvec = ray.o - p1;
    float u = fdot(tvec, pvec) * inv_det;
    if (u < 0.0f || u > 1.0f) return false;
    V3 qvec = fcross(tvec, e1);
    float v = fdot(ray.d, qvec) * inv_det;
    if (v < 0.0f || u + v > 1.0f) return false;
    float t = fdot(e2, qvec) * inv_det;
    if (t < ray.tmin || t > ray.tmax) return false;
    *u_out = u; *v_out = v; *t_out = t;
    return true;
}
#endif

// kernels/cl/trace_bvh.cl:28-73 — back-face culling (det < 1e-8 rejects), inclusive edges
inline bool RayTriangle(const Ray& ray, V3 p1, V3 p2, V3 p3, float* u_out, float* v_out, float* t_out)
{
    V3 e1 = p2 - p1, e2 = p3 - p1;
    V3 pvec = cross(ray.d, e2);
    float det = dot(e1, pvec);
    if (det < 1e-8f || -det > 1e-8f) return false;
    float inv_det = 1.0f / det;
    V3 tvec = ray.o - p1;
    float u = dot(tvec, pvec) * inv_det;
    if (u < 0.0f || u > 1.0f) return false;
    V3 qvec = cross(tvec, e1);
    float v = dot(ray.d, qvec) * inv_det;
    if (v < 0.0f || u + v > 1.0f) return false;
    float t = dot(e2, qvec) * inv_det;
    if (t < ray.tmin || t > ray.tmax) return false;
    *u_out = u; *v_out = v; *t_out = t;
    return true;
}

// kernels/cl/trace_bvh.cl:75-97
inline bool RayBounds(const RtLinearBVHNode& n, V3 o, V3 inv_dir, float t_min, float t_max)
{
    V3 t0 = (v3(n.bounds_min) - o) * inv_dir;
    V3 t1 = (v3(n.bounds_max) - o) * inv_dir;
    float lo = rt_fmaxf(rt_fmaxf(rt_fminf(t0.x, t1.x), rt_fminf(t0.y, t1.y)), rt_fminf(t0.z, t1.z));
    float hi = rt_fminf(rt_fminf(rt_fmaxf(t0.x, t1.x), rt_fmaxf(t0.y, t1.y)), rt_fmaxf(t0.z, t1.z));
    float tmin = rt_fmaxf(lo, t_min);
    float tmax = rt_fminf(hi, t_max);
    return tmax >= tmin;
}

#ifdef ORACLE_FMA_TRAVERSAL
inline bool RayBoundsFma(const RtLinearBVHNode& n, V3 o, V3 inv_dir, float t_min, float t_max)
{
    V3 noi = v3(-(o.x * inv_dir.x), -(o.y * inv_dir.y), -(o.z * inv_dir.z));
    V3 t0 = v3(fmaf(n.bounds_min.x, inv_dir.x, noi.x), fmaf(n.bounds_min.y, inv_dir.y, noi.y), fmaf(n.bounds_min.z, inv_dir.z, noi.z));
    V3 t1 = v3(fmaf(n.bounds_max.x, inv_dir.x, noi.x), fmaf(n.bounds_max.y, inv_dir.y, noi.y), fmaf(n.bounds_max.z, inv_dir.z, noi.z));
    float lo = rt_fmaxf(rt_fmaxf(rt_fminf(t0.x, t1.x), rt_fminf(t0.y, t1.y)), rt_fminf(t0.z, t1.z));
    float hi = rt_fminf(rt_fminf(rt_fmaxf(t0.x, t1.x), rt_fmaxf(t0.y, t1.y)), rt_fmaxf(t0.z, t1.z));
    return rt_fminf(hi, t_max) >= rt_fmaxf(lo, t_min);
}
#endif

// kernels/cl/trace_bvh.cl:99-211.  any_hit == the -D SHADOW_RAYS variant.
// Returns primitive id (closest) or 0 (any hit) / RT_INVALID_ID.
inline uint32_t TraceBvh(const Scene& sc, Ray ray, bool any_hit, RtHit* hit_out, TraceCounters* ctr)
{
    V3 inv_dir = splat(1.0f) / ray.d;                                      // :125, unguarded
    int sign[3] = { inv_dir.x < 0, inv_dir.y < 0, inv_dir.z < 0 };
    uint32_t prim = RT_INVALID_ID;
    float bu = 0.0f, bv = 0.0f, bt = 0.0f;
    int to_visit = 0, cur = 0;
    int stack[64];
    uint64_t nv = 0, nt = 0;
#ifdef ORACLE_FMA_TRAVERSAL
    // as the experiment build: rays with a non-finite component and the root box keep the exact arithmetic
    const float fin = ((ray.o.x + ray.o.y) + ray.o.z) + ((ray.d.x + ray.d.y) + ray.d.z);
    const bool contracted = std::fabs(fin) <= 3.0e38f;
#define ORC_BOUNDS(node, index) ((contracted && (index) != 0) ? RayBoundsFma(node, ray.o, inv_dir, ray.tmin, ray.tmax) : RayBounds(node, ray.o, inv_dir, ray.tmin, ray.tmax))
#define ORC_TRIANGLE(...) (contracted ? RayTriangleFma(__VA_ARGS__) : RayTriangle(__VA_ARGS__))
#else
#define ORC_BOUNDS(node, index) RayBounds(node, ray.o, inv_dir, ray.tmin, ray.tmax)
#define ORC_TRIANGLE(...) RayTriangle(__VA_ARGS__)
#endif
    for (;;)
    {
        const RtLinearBVHNode& node = sc.nodes[cur];
        ++nv;
        if (ORC_BOUNDS(node, cur))
        {
            int nprims = (int)(node.num_primitives_axis >> 16);
            if (nprims > 0)
            {
                for (int i = 0; i < nprims; ++i)
                {
                    const RtTriangle& t = sc.triangles[node.offset + i];
                    ++nt;
                    if (ORC_TRIANGLE(ray, v3(t.v1.position), v3(t.v2.position), v3(t.v3.position), &bu, &bv, &bt))
                    {
                        prim = node.offset + i;
                        ray.tmax = bt;                                         // :157-162, later equal-t hit overwrites
                        if (any_hit) { prim = 0; goto done; }                  // :164-167
                    }
                }
                if (to_visit == 0) break;
                cur = stack[--to_visit];
            }
            else if (sign[node.num_primitives_axis & 0xFFFF])                  // :181-190 near child first
            {
                stack[to_visit++] = cur + 1;
                cur = (int)node.offset;
            }
            else
            {
                stack[to_visit++] = (int)node.offset;
                cur = cur + 1;
            }
        }
        else
        {
            if (to_visit == 0) break;
            cur = stack[--to_visit];
        }
    }
done:
    if (ctr) { ctr->nodes_visited += nv; ctr->tris_tested += nt; }
    if (hit_out) { hit_out->bc.x = bu; hit_out->bc.y = bv; hit_out->primitive_id = prim; hit_out->t = bt; }
    return prim;
}

// ------------------------------------------------------------------ environment
// OpenCL 1.2 spec 8.2 (normalized coords, CLK_ADDRESS_REPEAT, CLK_FILTER_LINEAR) as
// used by kernels/cl/miss.cl:28-39
inline V3 SampleSky(const Scene& sc, V3 dir)
{
    float cx = rt_atan2f(dir.x, dir.y) + RT_PI;
    float cy = rt_acosf(dir.z);
    cx = cx < 0.0f ? cx + RT_TWO_PI : cx;
    cx *= RT_INV_TWO_PI;
    cy *= RT_INV_PI;
    int w = (int)sc.env_w, h = (int)sc.env_h;
    float wt = (float)w, ht = (float)h;
    float u = (cx - floorf(cx)) * wt, v = (cy - floorf(cy)) * ht;
    float fu = floorf(u - 0.5f), fv = floorf(v - 0.5f);
    int i0 = (fu >= -1.0f && fu <= wt) ? (int)fu : 0;        // NaN guard: texel 0
    int j0 = (fv >= -1.0f && fv <= ht) ? (int)fv : 0;
    int i1 = i0 + 1, j1 = j0 + 1;
    if (i0 < 0) i0 += w;
    if (i1 > w - 1) i1 -= w;
    if (j0 < 0) j0 += h;
    if (j1 > h - 1) j1 -= h;
    float a = (u - 0.5f) - fu, b = (v - 0.5f) - fv;
    const float* e = sc.env;
    auto texel = [&](int i, int j) { const float* p = e + ((size_t)j * w + i) * 4; return v3(p[0], p[1], p[2]); };
    return texel(i0, j0) * ((1.0f - a) * (1.0f - b)) + texel(i1, j0) * (a * (1.0f - b))
         + texel(i0, j1) * ((1.0f - a) * b) + texel(i1, j1) * (a * b);
}

// ------------------------------------------------------------------ materials
struct Material
{
    V3 diffuse_albedo; float roughness;
    V3 specular_albedo; float metalness;
    V3 emission; float ior;
    float transparency;
};

// kernels/common/material.h:319-369 (nearest texel, flat RGBA8 array)
inline V3 SampleTexture(const Scene& sc, const RtTexture& tex, V2 uv)
{
    uv.x -= floorf(uv.x); uv.y -= floorf(uv.y);
    uv.y = 1.f - uv.y;
    float fx = uv.x * (float)tex.width, fy = uv.y * (float)tex.height;
    int tx = (fx == fx) ? (int)fx : 0, ty = (fy == fy) ? (int)fy : 0;          // NaN guard
    tx = tx < 0 ? 0 : (tx > tex.width - 1 ? tex.width - 1 : tx);
    ty = ty < 0 ? 0 : (ty > tex.height - 1 ? tex.height - 1 : ty);
    uint32_t d = sc.texels[tex.data_start + ty * tex.width + tx];
    V3 c = v3((float)(d & 0xFF), (float)((d >> 8) & 0xFF), (float)((d >> 16) & 0xFF)) / 255.0f;   // utils.h:123-131
    return v3(rt_fminf(rt_fmaxf(c.x, 0.0f), 1.0f), rt_fminf(rt_fmaxf(c.y, 0.0f), 1.0f), rt_fminf(rt_fmaxf(c.z, 0.0f), 1.0f));
}
inline V3 pow3(V3 a, float e) { return v3(rt_powf(a.x, e), rt_powf(a.y, e), rt_powf(a.z, e)); }

// kernels/common/material.h:251-264 (OpenCL branch) + utils.h:133-190 unpackers
inline Material ApplyTextures(const Scene& sc, const RtPackedMaterial& pm, V2 uv)
{
    Material m;
    auto rgb = [](uint32_t d) { return v3((float)(d & 0xFF), (float)((d >> 8) & 0xFF), (float)((d >> 16) & 0xFF)) / 255.0f; };
    m.diffuse_albedo = rgb(pm.diffuse_albedo);
    uint32_t idx = pm.diffuse_albedo >> 24;
    if (idx != RT_INVALID_TEXTURE_IDX) m.diffuse_albedo = pow3(SampleTexture(sc, sc.textures[idx], uv), 2.2f);
    m.specular_albedo = rgb(pm.specular_albedo);
    idx = pm.specular_albedo >> 24;
    if (idx != RT_INVALID_TEXTURE_IDX) m.specular_albedo = pow3(SampleTexture(sc, sc.textures[idx], uv), 2.2f);
    {   // UnpackRGBE utils.h:149-158
        uint32_t e = pm.emission;
        float f = ldexpf(1.0f, (int)(e >> 24) - (128 + 8));
        m.emission = v3((float)(int)(e & 0xFF), (float)(int)((e >> 8) & 0xFF), (float)(int)((e >> 16) & 0xFF)) * f;
    }
    uint32_t rm = pm.roughness_metalness;
    m.roughness = (float)(rm & 0xFF) / 255.0f;
    m.metalness = (float)((rm >> 16) & 0xFF) / 255.0f;
    idx = (rm >> 8) & 0xFF;
    if (idx != RT_INVALID_TEXTURE_IDX) m.roughness = SampleTexture(sc, sc.textures[idx], uv).x;
    idx = (rm >> 24) & 0xFF;
    if (idx != RT_INVALID_TEXTURE_IDX) m.metalness = SampleTexture(sc, sc.textures[idx], uv).x;
    uint32_t it = pm.ior_emission_idx_transparency;
    m.ior = (float)(it & 0xFF) / 25.5f;
    m.transparency = (float)((it >> 16) & 0xFF) / 255.0f;
    idx = (it >> 8) & 0xFF;
    if (idx != RT_INVALID_TEXTURE_IDX) m.emission = m.emission * pow3(SampleTexture(sc, sc.textures[idx], uv), 2.2f);
    idx = (it >> 24) & 0xFF;
    if (idx != RT_INVALID_TEXTURE_IDX) m.transparency *= SampleTexture(sc, sc.textures[idx], uv).x;
    return m;
}

// kernels/common/bxdf.h:57-61, 71-74, 90-95, 104-119
inline float IorToF0(float a, float b) { float r = (b - a) / (b + a); return r * r; }
inline V3 FresnelSchlick(V3 f0, float h_dot_o) { return f0 + (1.0f - f0) * rt_powf(1.0f - h_dot_o, 5.0f); }
inline float GGX_D(float alpha, float n_dot_h)
{
    float a2 = alpha * alpha;
    float denom = n_dot_h * n_dot_h * (a2 - 1.0f) + 1.0f;
    return a2 * RT_INV_PI / (denom * denom);
}
inline float V_SmithGGXCorrelated(float n_dot_i, float n_dot_o, float alphaG)
{
    float a2 = alphaG * alphaG;
    float lv = n_dot_o * sqrtf((-n_dot_i * a2 + n_dot_i) * n_dot_i + a2);
    float ll = n_dot_i * sqrtf((-n_dot_o * a2 + n_dot_o) * n_dot_o + a2);
    return 0.5f / (lv + ll);
}
inline float Luma(V3 c) { return dot(c, v3(0.299f, 0.587f, 0.114f)); }                 // utils.h:108-111
inline V3 reflect(V3 v, V3 n) { return v - 2.0f * dot(v, n) * n; }                     // utils.h:83-86

// kernels/common/utils.h:99-106
inline V3 TangentToWorld(V3 dir, V3 n)
{
    V3 axis = fabsf(n.x) > 0.001f ? v3(0.0f, 1.0f, 0.0f) : v3(1.0f, 0.0f, 0.0f);
    V3 t = normalize(cross(axis, n));
    V3 b = cross(n, t);
    return normalize(b * dir.x + t * dir.y + n * dir.z);
}

// kernels/common/bxdf.h:157-168 — cos_theta has an fp64 sub-expression (literals 1.0)
inline V3 GGX_Sample(V2 s, V3 n, float alpha)
{
    float phi = RT_TWO_PI * s.x;
    float cos_theta = (float)(1.0f / sqrt(1.0 + (double)(alpha * alpha * s.y) / (1.0 - (double)s.y)));
    float sin_theta = sqrtf(rt_fmaxf(0.0f, 1.0f - cos_theta * cos_theta));
    V3 axis = fabsf(n.x) > 0.001f ? v3(0.0f, 1.0f, 0.0f) : v3(1.0f, 0.0f, 0.0f);
    V3 t = normalize(cross(axis, n));
    V3 b = cross(n, t);
    return normalize(b * rt_cosf(phi) * sin_theta + t * rt_sinf(phi) * sin_theta + n * cos_theta);
}

// kernels/common/material.h:132-169
inline V3 EvaluateMaterial(const Material& m, V3 normal, V3 incoming, V3 outgoing)
{
    if (m.transparency < 0.5f) return v3(0.0f, 0.0f, 0.0f);
    V3 half_vec = normalize(incoming + outgoing);
    float n_dot_i = rt_fmaxf(dot(normal, incoming), RT_EPS);
    float n_dot_o = rt_fmaxf(dot(normal, outgoing), RT_EPS);
    float n_dot_h = rt_fmaxf(dot(normal, half_vec), RT_EPS);
    float h_dot_o = rt_fmaxf(dot(half_vec, outgoing), RT_EPS);
    float alpha = m.roughness * m.roughness;
    float f0_dielectric = IorToF0(1.0f, m.ior);
    V3 f0 = mix(splat(f0_dielectric), m.specular_albedo, m.metalness);
    V3 diffuse_color = (1.0f - m.metalness) * m.diffuse_albedo;
    V3 fresnel = FresnelSchlick(f0, h_dot_o);
    float specular = GGX_D(alpha, n_dot_h) * V_SmithGGXCorrelated(n_dot_i, n_dot_o, alpha);
    V3 diffuse = diffuse_color * RT_INV_PI;
    return fresnel * specular + (1.0f - fresnel) * diffuse;
}

// kernels/common/material.h:171-241 (+ :51-117).  Operand order note for :230/:236:
// `fresnel * SampleSpecular(.., outgoing, pdf) * max(dot(*outgoing, normal), 0)` —
// the sampler is evaluated before the cosine factor that reads its output.
inline V3 SampleBxdf(float s1, V2 s, Material m, V3 normal, V3 incoming, bool white_furnace, V3* outgoing, float* pdf, float* offset)
{
    if (white_furnace) { m.diffuse_albedo = splat(1.0f); m.specular_albedo = splat(1.0f); }
    float alpha = m.roughness * m.roughness;
    float f0_dielectric = IorToF0(1.0f, m.ior);
    V3 f0 = mix(splat(f0_dielectric), m.specular_albedo, m.metalness);
    V3 diffuse_albedo = (1.0f - m.metalness) * m.diffuse_albedo;
    V3 specular_albedo = mix(m.specular_albedo, splat(1.0f), m.metalness);
    V3 fresnel = FresnelSchlick(f0, dot(normal, incoming)) * specular_albedo;
    float specular_weight = Luma(specular_albedo * fresnel);
    float diffuse_weight = Luma(diffuse_albedo * (1.0f - fresnel));
    float weight_sum = diffuse_weight + specular_weight;
    float specular_pdf = specular_weight / weight_sum;
    float diffuse_pdf = diffuse_weight / weight_sum;
    *offset = 1.0f;
    if (m.transparency < 0.5f)
    {   // SampleTransparency :105-117
        *pdf = 1.0f; *outgoing = -incoming; *offset = -1.0f;
        return splat(1.0f);
    }
    V3 bxdf;
    if (s1 <= specular_pdf)
    {   // SampleSpecular :66-103
        V3 spec;
        if (alpha <= 1e-4f)
        {
            *outgoing = reflect(-incoming, normal);
            *pdf = 1.0f;
            float n_dot_o = dot(*outgoing, normal);
            spec = splat(1.0f / n_dot_o);
        }
        else
        {
            V3 wh = GGX_Sample(s, normal, alpha);
            *outgoing = reflect(-incoming, wh);
            float n_dot_o = dot(normal, *outgoing);
            float n_dot_h = dot(normal, wh);
            float n_dot_i = dot(normal, incoming);
            float D = GGX_D(alpha, n_dot_h);
            float G = V_SmithGGXCorrelated(n_dot_i, n_dot_o, alpha);
            *pdf = D * n_dot_h / (4.0f * dot(wh, *outgoing));
            spec = splat(D * G);
        }
        bxdf = fresnel * spec * rt_fmaxf(dot(*outgoing, normal), 0.0f);
        *pdf *= specular_pdf;
    }
    else
    {   // SampleDiffuse :51-64, SampleHemisphereCosine bxdf.h:33-54
        float phi = RT_TWO_PI * s.x;
        float sin_theta = sqrtf(s.y);
        float cos_theta = sqrtf(1.0f - s.y);
        *pdf = cos_theta * RT_INV_PI;
        V3 tbn = v3(rt_cosf(phi) * sin_theta, rt_sinf(phi) * sin_theta, cos_theta);
        *outgoing = TangentToWorld(tbn, normal);
        bxdf = (1.0f - fresnel) * (diffuse_albedo * RT_INV_PI) * rt_fmaxf(dot(*outgoing, normal), 0.0f);
        *pdf *= diffuse_pdf;
    }
    return bxdf;
}

// kernels/common/light.h:30-65
inline V3 Light_Sample(const Scene& sc, V3 position, float s, V3* outgoing, float* pdf)
{
    int n = (int)sc.info.analytic_light_count;
    int idx = (int)(s * (float)sc.info.analytic_light_count);
    idx = idx < 0 ? 0 : (idx > n - 1 ? n - 1 : idx);
    const RtLight& light = sc.lights[idx];
    *pdf = 1.0f / (float)sc.info.analytic_light_count;
    V3 radiance = v3(light.radiance);
    if (light.type == RT_LIGHT_TYPE_POINT)
    {
        V3 to_light = v3(light.origin) - position;
        radiance = radiance / dot(to_light, to_light);
        *outgoing = to_light;
    }
    else
    {
        *outgoing = v3(light.origin) * RT_MAX_RENDER_DIST;
    }
    return radiance;
}

inline V3 Interp(V3 a, V3 b, V3 c, float u, float v) { return a * (1.0f - u - v) + b * u + c * v; }       // utils.h:93-96

} // namespace

// ====================================================================== C API
extern "C" {

typedef struct OrcScene
{
    const RtTriangle* triangles; uint32_t n_triangles;
    const RtLinearBVHNode* nodes; uint32_t n_nodes;
    const RtPackedMaterial* materials; uint32_t n_materials;
    const RtLight* lights; uint32_t n_lights;
    const RtTexture* textures; uint32_t n_textures;
    const uint32_t* texels; uint32_t n_texels;
    const float* env; uint32_t env_width, env_height;
    RtSceneInfo info;
} OrcScene;

#define ORC_MAX_BOUNCES 256     /* per-bounce counters for bounces 0..RT_MAX_BOUNCES */
typedef struct OrcStats
{
    uint32_t n_ext[ORC_MAX_BOUNCES], n_miss[ORC_MAX_BOUNCES], n_hit[ORC_MAX_BOUNCES];
    uint32_t n_shadow[ORC_MAX_BOUNCES], n_cont[ORC_MAX_BOUNCES], n_unoccluded[ORC_MAX_BOUNCES];
    uint32_t n_emissive_hits[ORC_MAX_BOUNCES];
    uint64_t nodes_ext[ORC_MAX_BOUNCES], tris_ext[ORC_MAX_BOUNCES];      /* closest-hit traversal work */
    uint64_t nodes_shadow[ORC_MAX_BOUNCES], tris_shadow[ORC_MAX_BOUNCES]; /* any-hit traversal work */
} OrcStats;

static Scene to_scene(const OrcScene* s)
{
    Scene sc;
    sc.triangles = s->triangles; sc.n_triangles = s->n_triangles;
    sc.nodes = s->nodes; sc.n_nodes = s->n_nodes;
    sc.materials = s->materials; sc.n_materials = s->n_materials;
    sc.lights = s->lights; sc.n_lights = s->n_lights;
    sc.textures = s->textures; sc.n_textures = s->n_textures;
    sc.texels = s->texels; sc.n_texels = s->n_texels;
    sc.env = s->env; sc.env_w = s->env_width; sc.env_h = s->env_height;
    sc.info = s->info;
    return sc;
}

uint32_t orc_wang_hash(uint32_t x) { return WangHash(x); }
/* kBlueNoise when all three tables are given (sobol[65536], scrambling[131072], ranking[131072]; not copied — they
 * must outlive the renders), kRandom when any is NULL. */
void orc_set_sampler_tables(const int32_t* sobol, const int32_t* scrambling, const int32_t* ranking)
{
    bool on = sobol && scrambling && ranking;
    g_bn_sobol = on ? sobol : nullptr; g_bn_scrambling = on ? scrambling : nullptr; g_bn_ranking = on ? ranking : nullptr;
}
float orc_sample_random(uint32_t px, uint32_t py, uint32_t sample, uint32_t bounce, uint32_t type) { return SampleRandom(px, py, sample, bounce, type); }

/* Primary rays for pixels [first, first+count): kernels/cl/raygeneration.cl:65-139 */
void orc_generate_rays(const RtCamera* cam, uint32_t width, uint32_t height, uint32_t sample_idx,
                       uint32_t first, uint32_t count, RtRay* rays)
{
#pragma omp parallel for schedule(static)
    for (long long i = 0; i < (long long)count; ++i)
    {
        Ray r = RayGeneration(first + (uint32_t)i, width, height, *cam, sample_idx);
        rays[i].origin = RtFloat3{ r.o.x, r.o.y, r.o.z, r.tmin };
        rays[i].direction = RtFloat3{ r.d.x, r.d.y, r.d.z, r.tmax };
    }
}

/* Closest-hit (any_hit = 0) or any-hit trace of n rays: kernels/cl/trace_bvh.cl:99-211.
 * hits (closest) or flags (any: 0 / 0xFFFFFFFF) may be NULL.  counters[2] += {nodes, tris}. */
void orc_trace(const OrcScene* scene, const RtRay* rays, uint32_t n, int any_hit, RtHit* hits, uint32_t* flags, uint64_t* counters)
{
    Scene sc = to_scene(scene);
    uint64_t nv = 0, nt = 0;
#pragma omp parallel for schedule(dynamic, 256) reduction(+ : nv, nt)
    for (long long i = 0; i < (long long)n; ++i)
    {
        Ray r; r.o = v3(rays[i].origin); r.tmin = rays[i].origin.w; r.d = v3(rays[i].direction); r.tmax = rays[i].direction.w;
        TraceCounters c = { 0, 0 };
        RtHit h;
        uint32_t p = TraceBvh(sc, r, any_hit != 0, &h, &c);
        if (hits) hits[i] = h;
        if (flags) flags[i] = p;
        nv += c.nodes_visited; nt += c.tris_tested;
    }
    if (counters) { counters[0] += nv; counters[1] += nt; }
}

/* Environment lookup for n unit directions (xyz, stride 3 floats) -> rgb: kernels/cl/miss.cl:28-39 */
void orc_sample_sky(const OrcScene* scene, const float* dirs, uint32_t n, float* rgb)
{
    Scene sc = to_scene(scene);
    for (uint32_t i = 0; i < n; ++i)
    {
        V3 c = SampleSky(sc, v3(dirs[3 * i], dirs[3 * i + 1], dirs[3 * i + 2]));
        rgb[3 * i] = c.x; rgb[3 * i + 1] = c.y; rgb[3 * i + 2] = c.z;
    }
}

/*
 * One Integrator::Integrate() worth of work (integrator/integrator.cpp:27-59) for one
 * sample: GenerateRays, then for bounce 0..max_bounces INCLUSIVE: IntersectRays,
 * ShadeMissedRays, ShadeSurfaceHits, IntersectShadowRays, AccumulateDirectSamples.
 * radiance (float4 per pixel) is ACCUMULATED INTO (caller zeroes it = Reset()).
 * Only pixels of rows y with (y % row_step) == row_first are traced (row_step = 1:
 * whole image) — the scanline partition used for multi-GPU runs.
 * primary_hits (per pixel, optional) receives the bounce-0 Hit of each traced pixel.
 * Compaction is a deterministic in-order scan (the reference uses atomic appends; the
 * per-pixel results do not depend on ray order, SURVEY A.4-2).
 */
/* Analysis hook (profiling studies only): when set, orc_render copies the rays entering bounce g_dump_bounce and their
 * per-ray traversal work (nodes visited, triangles tested) into the caller's arrays. */
static int g_dump_bounce = -1;
static RtRay* g_dump_rays = nullptr;
static uint32_t* g_dump_work = nullptr;   /* 2 per ray */
static uint32_t* g_dump_count = nullptr;
void orc_set_dump(int bounce, RtRay* rays, uint32_t* work, uint32_t* count) { g_dump_bounce = bounce; g_dump_rays = rays; g_dump_work = work; g_dump_count = count; }

void orc_render(const OrcScene* scene, const RtCamera* cam, uint32_t width, uint32_t height,
                uint32_t max_bounces, uint32_t sample_idx, int white_furnace,
                uint32_t row_first, uint32_t row_step,
                float* radiance, RtHit* primary_hits, OrcStats* stats)
{
    Scene sc = to_scene(scene);
    if (row_step == 0) row_step = 1;
    std::vector<uint32_t> pix;
    for (uint32_t y = row_first; y < height; y += row_step)
        for (uint32_t x = 0; x < width; ++x) pix.push_back(y * width + x);
    size_t n_live = pix.size();
    std::vector<Ray> rays(n_live), next_rays(n_live);
    std::vector<uint32_t> next_pix(n_live);
    std::vector<V3> throughputs((size_t)width * height);
    std::vector<RtHit> hits(n_live);
    struct Shadow { Ray ray; uint32_t pixel; V3 sample; bool valid; };
    std::vector<Shadow> shadow(n_live);
    std::vector<uint8_t> cont(n_live);
    if (stats) memset(stats, 0, sizeof(*stats));

#pragma omp parallel for schedule(static)
    for (long long i = 0; i < (long long)n_live; ++i)
    {
        rays[i] = RayGeneration(pix[i], width, height, *cam, sample_idx);
        throughputs[pix[i]] = splat(1.0f);
    }

    for (uint32_t bounce = 0; bounce <= max_bounces; ++bounce)
    {
        uint64_t nv = 0, nt = 0, nvs = 0, nts = 0;
        uint32_t n_miss = 0, n_emis = 0;
        // IntersectRays + ShadeMissedRays + ShadeSurfaceHits, per ray
#pragma omp parallel for schedule(dynamic, 256) reduction(+ : nv, nt, n_miss, n_emis)
        for (long long i = 0; i < (long long)n_live; ++i)
        {
            TraceCounters c = { 0, 0 };
            RtHit hit;
            const Ray& ray = rays[i];
            TraceBvh(sc, ray, false, &hit, &c);
            nv += c.nodes_visited; nt += c.tris_tested;
            if ((int)bounce == g_dump_bounce && g_dump_rays)
            {
                g_dump_rays[i].origin = RtFloat3{ ray.o.x, ray.o.y, ray.o.z, 0.0f };
                g_dump_rays[i].direction = RtFloat3{ ray.d.x, ray.d.y, ray.d.z, ray.tmax };
                g_dump_work[2 * i] = (uint32_t)c.nodes_visited; g_dump_work[2 * i + 1] = (uint32_t)c.tris_tested;
                if (i == 0) *g_dump_count = (uint32_t)n_live;
            }
            hits[i] = hit;
            uint32_t pixel = pix[i];
            float* rad = radiance + (size_t)pixel * 4;
            shadow[i].valid = false; cont[i] = 0;
            if (hit.primitive_id == RT_INVALID_ID)
            {   // kernels/cl/miss.cl:41-77
                ++n_miss;
                V3 sky = white_furnace ? splat(0.5f) : SampleSky(sc, ray.d);
                V3 add = sky * throughputs[pixel];
                rad[0] += add.x; rad[1] += add.y; rad[2] += add.z;
                continue;
            }
            // kernels/cl/hit_surface.cl:30-186
            V3 incoming = -ray.d;
            uint32_t px = pixel % width, py = pixel / width;
            const RtTriangle& tri = sc.triangles[hit.primitive_id];
            V3 p1 = v3(tri.v1.position), p2 = v3(tri.v2.position), p3 = v3(tri.v3.position);
            float u = hit.bc.x, v = hit.bc.y;
            V3 position = Interp(p1, p2, p3, u, v);
            V3 geometry_normal = normalize(cross(p2 - p1, p3 - p1));
            float w0 = 1.0f - u - v;
            V2 texcoord = { tri.v1.texcoord.x * w0 + tri.v2.texcoord.x * u + tri.v3.texcoord.x * v,
                            tri.v1.texcoord.y * w0 + tri.v2.texcoord.y * u + tri.v3.texcoord.y * v };
            V3 normal = normalize(Interp(v3(tri.v1.normal), v3(tri.v2.normal), v3(tri.v3.normal), u, v));
            Material material = ApplyTextures(sc, sc.materials[tri.mtlIndex], texcoord);
            V3 hit_throughput = throughputs[pixel];
            if (!white_furnace && dot(material.emission, splat(1.0f)) > 0.0f)
            {   // :107-112
                ++n_emis;
                V3 add = hit_throughput * material.emission;
                rad[0] += add.x; rad[1] += add.y; rad[2] += add.z;
            }
            {   // direct lighting :115-145
                float s_light = SampleRandom(px, py, sample_idx, bounce, SAMPLE_LIGHT);
                V3 outgoing; float pdf;
                V3 light_radiance = Light_Sample(sc, position, s_light, &outgoing, &pdf);
                float distance_to_light = length(outgoing);
                outgoing = normalize(outgoing);
                V3 brdf = EvaluateMaterial(material, normal, incoming, outgoing);
                V3 light_sample = light_radiance * hit_throughput * brdf / pdf * rt_fmaxf(dot(outgoing, normal), 0.0f);
                if (pdf > 0.0f && dot(light_sample, light_sample) > 0.0f)
                {
                    Shadow& s = shadow[i];
                    s.valid = true; s.pixel = pixel; s.sample = light_sample;
                    s.ray.o = position + normal * RT_EPS; s.ray.tmin = 0.0f;
                    s.ray.d = outgoing; s.ray.tmax = distance_to_light;
                }
            }
            {   // indirect lighting :148-184
                V2 s = { SampleRandom(px, py, sample_idx, bounce, SAMPLE_U), SampleRandom(px, py, sample_idx, bounce, SAMPLE_V) };
                float s1 = SampleRandom(px, py, sample_idx, bounce, SAMPLE_LAYER);
                float pdf = 0.0f, offset;
                V3 outgoing = v3(0, 0, 0);
                V3 bxdf = SampleBxdf(s1, s, material, normal, incoming, white_furnace != 0, &outgoing, &pdf, &offset);
                V3 throughput = splat(0.0f);
                if (pdf > 0.0f) throughput = bxdf / pdf;
                throughputs[pixel] = throughputs[pixel] * throughput;
                if (pdf > 0.0f)
                {
                    cont[i] = 1;
                    Ray& o = next_rays[i];
                    o.o = position + geometry_normal * RT_EPS * offset; o.tmin = 0.0f;
                    o.d = outgoing; o.tmax = RT_MAX_RENDER_DIST;
                }
            }
        }
        if (bounce == 0 && primary_hits)
            for (size_t i = 0; i < n_live; ++i) primary_hits[pix[i]] = hits[i];

        // IntersectShadowRays + AccumulateDirectSamples (trace_bvh.cl -D SHADOW_RAYS, accumulate_direct_samples.cl:27-53)
        uint32_t n_shadow = 0, n_unocc = 0;
#pragma omp parallel for schedule(dynamic, 256) reduction(+ : nvs, nts, n_shadow, n_unocc)
        for (long long i = 0; i < (long long)n_live; ++i)
        {
            if (!shadow[i].valid) continue;
            ++n_shadow;
            TraceCounters c = { 0, 0 };
            uint32_t f = TraceBvh(sc, shadow[i].ray, true, nullptr, &c);
            nvs += c.nodes_visited; nts += c.tris_tested;
            if (f == RT_INVALID_ID)
            {
                ++n_unocc;
                float* rad = radiance + (size_t)shadow[i].pixel * 4;
                rad[0] += shadow[i].sample.x; rad[1] += shadow[i].sample.y; rad[2] += shadow[i].sample.z;
            }
        }

        // compaction of continuation rays (in order)
        size_t n_next = 0;
        for (size_t i = 0; i < n_live; ++i)
            if (cont[i]) { rays[n_next] = next_rays[i]; next_pix[n_next] = pix[i]; ++n_next; }
        if (stats && bounce < ORC_MAX_BOUNCES)
        {
            stats->n_ext[bounce] = (uint32_t)n_live; stats->n_miss[bounce] = n_miss; stats->n_hit[bounce] = (uint32_t)n_live - n_miss;
            stats->n_shadow[bounce] = n_shadow; stats->n_cont[bounce] = (uint32_t)n_next; stats->n_unoccluded[bounce] = n_unocc;
            stats->n_emissive_hits[bounce] = n_emis;
            stats->nodes_ext[bounce] = nv; stats->tris_ext[bounce] = nt; stats->nodes_shadow[bounce] = nvs; stats->tris_shadow[bounce] = nts;
        }
        pix.swap(next_pix); pix.resize(n_next); next_pix.resize(n_live);
        n_live = n_next;
        if (n_live == 0)
        {
            // later bounces launch over zero live rays in the reference; nothing to do
            break;
        }
    }
}

/* ---- "next" rows (SURVEY 8f): AOVs, temporal denoiser, resolve -------------------------------------------- */

// kernels/cl/aov.cl:30-42
static V2 ProjectScreen(V3 position, const RtCamera& cam)
{
    V3 d = normalize(position - v3(cam.position));
    V3 ipd = d / dot(v3(cam.front), d);
    float angle = rt_tanf(0.5f * cam.fov);
    V3 right = cross(v3(cam.front), v3(cam.up));
    float u = dot(right, ipd) / (angle * cam.aspect_ratio);
    float v = dot(v3(cam.up), ipd) / (angle);
    return V2{ u * 0.5f + 0.5f, v * 0.5f + 0.5f };
}

/* GenerateAOV (kernels/cl/aov.cl:44-110) on top of the initial values RayGeneration writes
 * (raygeneration.cl:129-133): albedo float4/pixel, depth float/pixel, normal float4/pixel, velocity float2/pixel. */
void orc_aovs(const OrcScene* scene, const RtCamera* cam, const RtCamera* prev_cam, uint32_t width, uint32_t height,
              uint32_t sample_idx, float* albedo, float* depth, float* normal, float* velocity)
{
    Scene sc = to_scene(scene);
    size_t n = (size_t)width * height;
#pragma omp parallel for schedule(dynamic, 256)
    for (long long i = 0; i < (long long)n; ++i)
    {
        albedo[4 * i] = albedo[4 * i + 1] = albedo[4 * i + 2] = 0.0f; albedo[4 * i + 3] = 0.0f;
        depth[i] = RT_MAX_RENDER_DIST;
        normal[4 * i] = normal[4 * i + 1] = normal[4 * i + 2] = 0.0f; normal[4 * i + 3] = 0.0f;
        velocity[2 * i] = velocity[2 * i + 1] = 0.0f;
        Ray ray = RayGeneration((uint32_t)i, width, height, *cam, sample_idx);
        RtHit hit;
        TraceBvh(sc, ray, false, &hit, nullptr);
        if (hit.primitive_id == RT_INVALID_ID) continue;
        const RtTriangle& tri = sc.triangles[hit.primitive_id];
        float u = hit.bc.x, v = hit.bc.y, w0 = 1.0f - u - v;
        V3 position = Interp(v3(tri.v1.position), v3(tri.v2.position), v3(tri.v3.position), u, v);
        V2 texcoord = { tri.v1.texcoord.x * w0 + tri.v2.texcoord.x * u + tri.v3.texcoord.x * v,
                        tri.v1.texcoord.y * w0 + tri.v2.texcoord.y * u + tri.v3.texcoord.y * v };
        V3 nrm = normalize(Interp(v3(tri.v1.normal), v3(tri.v2.normal), v3(tri.v3.normal), u, v));
        Material m = ApplyTextures(sc, sc.materials[tri.mtlIndex], texcoord);
        albedo[4 * i] = m.diffuse_albedo.x; albedo[4 * i + 1] = m.diffuse_albedo.y; albedo[4 * i + 2] = m.diffuse_albedo.z;
        depth[i] = length(ray.o - position);
        normal[4 * i] = nrm.x; normal[4 * i + 1] = nrm.y; normal[4 * i + 2] = nrm.z;
        V2 a = ProjectScreen(position, *cam), b = ProjectScreen(position, *prev_cam);
        velocity[2 * i] = a.x - b.x; velocity[2 * i + 1] = a.y - b.y;
    }
}

/* TemporalAccumulation (kernels/cl/denoiser.cl:27-79): radiance.xyz = mix(radiance, prev_radiance[reprojected], 0.9) */
void orc_temporal_accumulation(uint32_t width, uint32_t height, float* radiance, const float* prev_radiance,
                               const float* depth, const float* prev_depth, const float* velocity)
{
    for (uint32_t idx = 0; idx < width * height; ++idx)
    {
        int x = (int)(idx % width), y = (int)(idx / width);
        float dv = depth[idx];
        if (dv == RT_MAX_RENDER_DIST) continue;
        float pu = ((float)x + 0.5f) / (float)width - velocity[2 * idx];
        float pv = ((float)y + 0.5f) / (float)height - velocity[2 * idx + 1];
        float fx = pu * (float)width, fy = pv * (float)height;
        if (!(fx == fx) || !(fy == fy) || fabsf(fx) > 1.0e9f || fabsf(fy) > 1.0e9f) continue;   // NaN/overflow guard: out of range
        int px = (int)fx, py = (int)fy;
        if (px < 0 || px >= (int)width || py < 0 || py >= (int)height) continue;
        int pidx = py * (int)width + px;
        float pd = prev_depth[pidx];
        if (fabsf(dv - pd) / dv > 0.1f) continue;
        for (int c = 0; c < 3; ++c)
        {
            float cur = radiance[4 * idx + c], prev = prev_radiance[4 * pidx + c];
            radiance[4 * idx + c] = cur + (prev - cur) * 0.9f;
        }
    }
}

/* ResolveRadiance (kernels/cl/resolve_radiance.cl:31-86); aov: 0 shaded colour, 1 albedo, 2 depth, 3 normal, 4 motion */
void orc_resolve(uint32_t width, uint32_t height, uint32_t aov, const float* radiance, const float* albedo, const float* depth,
                 const float* normal, const float* velocity, uint32_t sample_count, int denoiser, float* out)
{
    for (uint32_t i = 0; i < width * height; ++i)
    {
        float* o = out + 4 * (size_t)i;
        o[3] = 1.0f;
        if (aov == 1) { o[0] = albedo[4 * i]; o[1] = albedo[4 * i + 1]; o[2] = albedo[4 * i + 2]; }
        else if (aov == 2) { float d = depth[i] * 0.1f; o[0] = o[1] = o[2] = d; }
        else if (aov == 3) { for (int c = 0; c < 3; ++c) o[c] = normal[4 * i + c] * 0.5f + 0.5f; }
        else if (aov == 4) { o[0] = velocity[2 * i]; o[1] = velocity[2 * i + 1]; o[2] = 0.0f; }
        else
        {
            for (int c = 0; c < 3; ++c)
            {
                float hdr = radiance[4 * i + c];
                if (!denoiser) hdr = hdr / (float)sample_count;
                o[c] = hdr / (hdr + 1.0f);
            }
        }
    }
}

} // extern "C"
