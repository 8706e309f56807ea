/*
 * rt_device.cuh — device-side building blocks of the wavefront path tracer:
 * RNG, primary-ray generation, environment lookup, material unpacking, Lambert/GGX
 * evaluation and sampling, light sampling.  Written for sm_90a, compiled with
 * -fmad=false: every float operation is a separately rounded IEEE binary32 op in the
 * order written, transcendental functions come from include/rt_math.h, so results are
 * bit-identical to the reference semantics pinned by oracle/ (see DESIGN.md "Arithmetic
 * policy").  Each function cites the reference code whose behaviour it reproduces
 * (paths relative to /root/reference/src).
 */
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "rt_math.h"
#include "rt_types.h"

namespace rt
{

struct f3 { float x, y, z; };
struct f2 { float x, y; };

__device__ __forceinline__ f3 mk3(float x, float y, float z) { f3 r; r.x = x; r.y = y; r.z = z; return r; }
__device__ __forceinline__ f3 mk3(float4 v) { return mk3(v.x, v.y, v.z); }
__device__ __forceinline__ f3 splat(float a) { return mk3(a, a, a); }
__device__ __forceinline__ f3 operator+(f3 a, f3 b) { return mk3(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ f3 operator-(f3 a, f3 b) { return mk3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ f3 operator*(f3 a, f3 b) { return mk3(a.x * b.x, a.y * b.y, a.z * b.z); }
__device__ __forceinline__ f3 operator/(f3 a, f3 b) { return mk3(a.x / b.x, a.y / b.y, a.z / b.z); }
__device__ __forceinline__ f3 operator*(f3 a, float b) { return mk3(a.x * b, a.y * b, a.z * b); }
__device__ __forceinline__ f3 operator*(float a, f3 b) { return mk3(a * b.x, a * b.y, a * b.z); }
__device__ __forceinline__ f3 operator/(f3 a, float b) { return mk3(a.x / b, a.y / b, a.z / b); }
__device__ __forceinline__ f3 operator-(float a, f3 b) { return mk3(a - b.x, a - b.y, a - b.z); }
__device__ __forceinline__ f3 operator-(f3 a) { return mk3(-a.x, -a.y, -a.z); }
__device__ __forceinline__ float dot(f3 a, f3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ f3 cross(f3 a, f3 b) { return mk3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
__device__ __forceinline__ float length(f3 a) { return sqrtf(dot(a, a)); }
__device__ __forceinline__ f3 normalize(f3 a) { float inv = 1.0f / sqrtf(dot(a, a)); return a * inv; }
__device__ __forceinline__ f3 mix(f3 a, f3 b, float t) { return a + (b - a) * t; }

// ---------------------------------------------------------------------------- RNG
// kernels/common/utils.h:113-121
__device__ __forceinline__ uint32_t wang_hash(uint32_t x)
{
    x = (x ^ 61u) ^ (x >> 16);
    x = x + (x << 3);
    x = x ^ (x >> 4);
    x = x * 0x27d4eb2du;
    x = x ^ (x >> 15);
    return x;
}

// kernels/cl/raygeneration.cl:28-38
__device__ __forceinline__ float lcg_random_float(uint32_t& seed)
{
    uint32_t s = wang_hash(seed);
    s = 1103515245u * s + 12345u;
    seed = s;
    return (float)s * 2.3283064365386963e-10f;
}

// kernels/common/sampling.h:64-82 (kRandom).  The pixel part of the hash chain is shared
// by the four draws of a bounce, so it is computed once per path vertex.
__device__ __forceinline__ uint32_t sample_seed_pixel(uint32_t px, uint32_t py, uint32_t sample_index)
{
    uint32_t seed = wang_hash(px);
    seed = wang_hash(seed + wang_hash(py));
    seed = wang_hash(seed + wang_hash(sample_index));
    return seed;
}
__device__ __forceinline__ float sample_random(uint32_t pixel_seed, uint32_t bounce, uint32_t type)
{
    uint32_t seed = wang_hash(pixel_seed + wang_hash(bounce * 5u + type));
    return (float)seed * 2.3283064365386963e-10f;
}
enum { SAMPLE_LAYER = 1, SAMPLE_U = 2, SAMPLE_V = 3, SAMPLE_LIGHT = 4 };

// kernels/common/sampling.h:40-61 (kBlueNoise).  `bn` is the caller's three tables back to back (rt_upload_sampler_tables):
// sobol_256spp_256d[65536] | scramblingTile[131072] | rankingTile[131072].  The ranking tile is indexed with the
// UN-wrapped dimension (sampling.h:50), which runs past the table for the last tile pixels once the dimension exceeds 7;
// those reads return 0 here (include/rt_b200.h).
__device__ __forceinline__ float sample_blue_noise(const int* __restrict__ bn, uint32_t px, uint32_t py, uint32_t sample_index, uint32_t dim)
{
    int pixel_i = (int)px & 127, pixel_j = (int)py & 127;
    int sample = (int)sample_index & 255, d = (int)dim & 255;
    int tile = (pixel_i + pixel_j * 128) * 8;
    int ri = d + tile;
    int ranked = sample ^ (ri < RT_BN_TILE_COUNT ? __ldg(bn + RT_BN_SOBOL_COUNT + RT_BN_TILE_COUNT + ri) : 0);
    int value = __ldg(bn + d + ranked * 256);
    value = value ^ __ldg(bn + RT_BN_SOBOL_COUNT + (d % 8) + tile);
    return (0.5f + (float)value) / 256.0f;
}

// ---------------------------------------------------------------------------- ray generation
struct RayGenConsts
{
    f3 position, front, up, right;
    float tan_half_fov, aspect_ratio, aperture, focus_distance;
    float inv_width, inv_height;
};

// kernels/cl/raygeneration.cl:65-139 (hexagon index clamped to 2 when the random float is exactly 1,
// where the reference reads past its 3-entry table; see oracle/oracle.cpp PointInHexagon)
__device__ __forceinline__ void generate_primary_ray(const RayGenConsts& c, uint32_t pixel_idx, uint32_t px, uint32_t py,
                                                     uint32_t sample_idx, f3& origin, f3& dir)
{
    uint32_t seed = pixel_idx + (1103515245u * sample_idx + 12345u);
    float x = ((float)px + lcg_random_float(seed)) * c.inv_width;
    float y = ((float)py + lcg_random_float(seed)) * c.inv_height;
    // ((x*2-1) * angle) * aspect: angle*aspect is NOT pre-multiplied (rounding order)
    x = (x * 2.0f - 1.0f) * c.tan_half_fov * c.aspect_ratio;
    y = (y * 2.0f - 1.0f) * c.tan_half_fov;
    f3 d = normalize(x * c.right + y * c.up + c.front);
    f3 aimed = c.position + c.focus_distance * d;
    int hx = (int)floorf(lcg_random_float(seed) * 3.0f);
    hx = hx > 2 ? 2 : hx;
    float v1x = hx == 0 ? -1.0f : 0.5f, v1y = hx == 0 ? 0.0f : (hx == 1 ? 0.866f : -0.866f);
    int h2 = (hx + 1) % 3;
    float v2x = h2 == 0 ? -1.0f : 0.5f, v2y = h2 == 0 ? 0.0f : (h2 == 1 ? 0.866f : -0.866f);
    float p1 = lcg_random_float(seed), p2 = lcg_random_float(seed);
    float dofx = p1 * v1x + p2 * v2x, dofy = p1 * v1y + p2 * v2y;
    float r = c.aperture;
    origin = c.position + dofx * r * c.right + dofy * r * c.up;
    dir = normalize(aimed - origin);
}

// ---------------------------------------------------------------------------- scene view
struct DevScene
{
    const float4* nodes_ref;       // reference LinearBVHNode[]: 3 x float4 per node
    const float4* tris_ref;        // RTTriangle[]: 3 x float4 (positions), cl_pt_integrator.cpp:392-402
    const float4* tri_shade;       // 7 x float4 per triangle: positions, normals, uvs, material, geometric normal (rt_bvh_layout.h)
    const uint32_t* materials;     // PackedMaterial[]: 5 x uint32 (only read for textured materials)
    const float4* mat_rec;         // 4 x float4 per material: unpacked constants (rt_bvh_layout.h)
    const float4* light_rec;       // 2 x float4 per light
    const int4* textures;          // Texture[]
    const uint32_t* texels;
    const float4* env;             // RGBA32F
    int env_w, env_h;
    uint32_t light_count;
    // optimised traversal layout (built at upload, see rt_bvh_layout.h)
    const float4* wnodes;          // 4 x float4 per interior node
    const float4* wtris;           // 3 x float4 per triangle: p1, e1, e2 (+ end-of-leaf flag)
    uint32_t wnodes_f4, wtris_f4;  // sizes of the two arrays in float4 (for the TMA staging of small scenes)
    uint32_t top_n;                // interior records [0, top_n) are the top of the tree in breadth-first order
    uint32_t top_k;                // of those, the records a kernel staged into shared memory (set per launch; 0 = none)
    int root_ref;
    // emitter sampling (RT_OPT_EMITTER_SAMPLING, rt_emitters.h): nullptr / 0 while it is off or inactive (P_e = 0)
    const float* emit_pdfA;        // per triangle
    const float* emit_cdf;         // per emitter
    const uint32_t* emit_list;     // per emitter: triangle id
    uint32_t n_emit;
    float emit_pe;
    // environment sampling (RT_OPT_ENV_SAMPLING, rt_envmap.h): nullptr while it is off or inactive
    const float* env_marg;         // per row
    const float* env_cond;         // per texel
    const float* env_pdf;          // per texel: P_v * p_uv
    // light-kind draw (rt_set_light_selection) while either table exists: P_e + P_v, and whether the analytic kind has weight 0
    float light_pev;
    uint32_t no_analytic;
};

// ---------------------------------------------------------------------------- environment
// kernels/cl/miss.cl:28-39 with the OpenCL 1.2 (spec 8.2) sampler
// CLK_NORMALIZED_COORDS_TRUE | CLK_ADDRESS_REPEAT | CLK_FILTER_LINEAR done in software with
// float weights (hardware texture filtering uses 9-bit fixed-point weights).
__device__ __forceinline__ f3 sample_sky(const DevScene& sc, f3 dir)
{
    float cx = rt_atan2f(dir.x, dir.y) + RT_PI;
    float cy = rt_acosf(dir.z);
    cx = cx < 0.0f ? cx + RT_TWO_PI : cx;
    cx *= RT_INV_TWO_PI;
    cy *= RT_INV_PI;
    int w = sc.env_w, h = sc.env_h;
    float wt = (float)w, ht = (float)h;
    float u = (cx - floorf(cx)) * wt, v = (cy - floorf(cy)) * ht;
    float fu = floorf(u - 0.5f), fv = floorf(v - 0.5f);
    int i0 = (fu >= -1.0f && fu <= wt) ? (int)fu : 0;      // NaN guard
    int j0 = (fv >= -1.0f && fv <= ht) ? (int)fv : 0;
    int i1 = i0 + 1, j1 = j0 + 1;
    if (i0 < 0) i0 += w;
    if (i1 > w - 1) i1 -= w;
    if (j0 < 0) j0 += h;
    if (j1 > h - 1) j1 -= h;
    float a = (u - 0.5f) - fu, b = (v - 0.5f) - fv;
    f3 t00 = mk3(__ldg(sc.env + (size_t)j0 * w + i0)), t10 = mk3(__ldg(sc.env + (size_t)j0 * w + i1));
    f3 t01 = mk3(__ldg(sc.env + (size_t)j1 * w + i0)), t11 = mk3(__ldg(sc.env + (size_t)j1 * w + i1));
    return t00 * ((1.0f - a) * (1.0f - b)) + t10 * (a * (1.0f - b)) + t01 * ((1.0f - a) * b) + t11 * (a * b);
}

// ---------------------------------------------------------------------------- materials
struct Material
{
    f3 diffuse_albedo; float roughness;
    f3 specular_albedo; float metalness;
    f3 emission; float ior;
    float transparency;
};

// The BSDF constants of a material (derive_bsdf): the values evaluate_material, sample_bxdf and bxdf_eval_sampled rebuilt from it
// on every hit, computed once per call by derive_bsdf so that the three cannot drift apart.  They are derived, not loaded from a
// per-material table: the shading pass waits on memory latency, and loading them at any of the call sites measured slower on an
// H100 than the arithmetic it saves (DESIGN.md section 4).
struct Bsdf
{
    f3 f0;                         // mix(ior_to_f0(1, ior), specular_albedo, metalness)
    f3 diffuse_mix;                // (1 - metalness) * diffuse_albedo
    f3 specular_mix;               // mix(specular_albedo, 1, metalness)
    f3 diffuse_lambert;            // diffuse_mix * (1 / pi)
    float diffuse_weight;          // luma(diffuse_mix): sample_bxdf's diffuse lobe weight when the Fresnel term is 0
};

// kernels/common/material.h:319-369
__device__ __forceinline__ f3 sample_texture(const DevScene& sc, uint32_t tex_idx, f2 uv)
{
    int4 tex = __ldg(sc.textures + tex_idx);      // data_start, width, height, pad
    uv.x -= floorf(uv.x); uv.y -= floorf(uv.y);
    uv.y = 1.f - uv.y;
    float fx = uv.x * (float)tex.y, fy = uv.y * (float)tex.z;
    int tx = (fx == fx) ? (int)fx : 0, ty = (fy == fy) ? (int)fy : 0;
    tx = tx < 0 ? 0 : (tx > tex.y - 1 ? tex.y - 1 : tx);
    ty = ty < 0 ? 0 : (ty > tex.z - 1 ? tex.z - 1 : ty);
    uint32_t d = __ldg(sc.texels + tex.x + ty * tex.y + tx);
    f3 c = mk3((float)(d & 0xFF), (float)((d >> 8) & 0xFF), (float)((d >> 16) & 0xFF)) / 255.0f;
    return mk3(fminf(fmaxf(c.x, 0.0f), 1.0f), fminf(fmaxf(c.y, 0.0f), 1.0f), fminf(fmaxf(c.z, 0.0f), 1.0f));
}
__device__ __forceinline__ f3 pow3(f3 a, float e) { return mk3(rt_powf(a.x, e), rt_powf(a.y, e), rt_powf(a.z, e)); }
__device__ __forceinline__ f3 unpack_rgb8(uint32_t d)
{
    return mk3((float)(d & 0xFF), (float)((d >> 8) & 0xFF), (float)((d >> 16) & 0xFF)) / 255.0f;
}

__device__ __forceinline__ float luma(f3 c) { return dot(c, mk3(0.299f, 0.587f, 0.114f)); }
__device__ __forceinline__ float ior_to_f0(float a, float b) { float r = (b - a) / (b + a); return r * r; }

// The per-material values of material.h:132-241 that do not depend on the hit's directions, in the reference's operation order.
__device__ __forceinline__ Bsdf derive_bsdf(const Material& m)
{
    Bsdf d;
    d.f0 = mix(splat(ior_to_f0(1.0f, m.ior)), m.specular_albedo, m.metalness);
    d.diffuse_mix = (1.0f - m.metalness) * m.diffuse_albedo;
    d.specular_mix = mix(m.specular_albedo, splat(1.0f), m.metalness);
    d.diffuse_lambert = d.diffuse_mix * RT_INV_PI;
    d.diffuse_weight = luma(d.diffuse_mix);
    return d;
}

// kernels/common/material.h:251-264 (OpenCL branch), utils.h:123-190
// (inlined on purpose: as a called function it costs the hot path more (call ABI: registers, stack) than its size saves)
__device__ __forceinline__ Material unpack_material(const DevScene& sc, uint32_t mtl_index, f2 uv)
{
    const uint32_t* pm = sc.materials + (size_t)mtl_index * 5;
    uint32_t w0 = __ldg(pm), w1 = __ldg(pm + 1), w2 = __ldg(pm + 2), w3 = __ldg(pm + 3), w4 = __ldg(pm + 4);
    Material m;
    m.diffuse_albedo = unpack_rgb8(w0);
    if ((w0 >> 24) != RT_INVALID_TEXTURE_IDX) m.diffuse_albedo = pow3(sample_texture(sc, w0 >> 24, uv), 2.2f);
    m.specular_albedo = unpack_rgb8(w1);
    if ((w1 >> 24) != RT_INVALID_TEXTURE_IDX) m.specular_albedo = pow3(sample_texture(sc, w1 >> 24, uv), 2.2f);
    {
        float f = ldexpf(1.0f, (int)(w2 >> 24) - (128 + 8));
        m.emission = mk3((float)(int)(w2 & 0xFF), (float)(int)((w2 >> 8) & 0xFF), (float)(int)((w2 >> 16) & 0xFF)) * f;
    }
    m.roughness = (float)(w3 & 0xFF) / 255.0f;
    m.metalness = (float)((w3 >> 16) & 0xFF) / 255.0f;
    if (((w3 >> 8) & 0xFF) != RT_INVALID_TEXTURE_IDX) m.roughness = sample_texture(sc, (w3 >> 8) & 0xFF, uv).x;
    if ((w3 >> 24) != RT_INVALID_TEXTURE_IDX) m.metalness = sample_texture(sc, w3 >> 24, uv).x;
    m.ior = (float)(w4 & 0xFF) / 25.5f;
    m.transparency = (float)((w4 >> 16) & 0xFF) / 255.0f;
    if (((w4 >> 8) & 0xFF) != RT_INVALID_TEXTURE_IDX) m.emission = m.emission * pow3(sample_texture(sc, (w4 >> 8) & 0xFF, uv), 2.2f);
    if ((w4 >> 24) != RT_INVALID_TEXTURE_IDX) m.transparency *= sample_texture(sc, w4 >> 24, uv).x;
    return m;
}

// Untextured materials (every material of the shipped scenes): the unpack of material.h:251-264 /
// utils.h:123-190 is a pure function of the 20 packed bytes, so rt_upload_scene evaluates it once per
// material on the host with the same IEEE operations (rt_bvh_layout.h) and the kernel loads the result.
__device__ __forceinline__ Material load_material(const DevScene& sc, uint32_t mtl_index, f2 uv)
{
    const float4* r = sc.mat_rec + (size_t)mtl_index * 4;
    float4 r3 = __ldg(r + 3);
    if (__float_as_uint(r3.y) != 0u) return unpack_material(sc, mtl_index, uv);     // has a texture: per-hit path
    float4 r0 = __ldg(r), r1 = __ldg(r + 1), r2 = __ldg(r + 2);
    Material m;
    m.diffuse_albedo = mk3(r0); m.roughness = r0.w;
    m.specular_albedo = mk3(r1); m.metalness = r1.w;
    m.emission = mk3(r2); m.ior = r2.w;
    m.transparency = r3.x;
    return m;
}

// kernels/common/bxdf.h:57-61, 71-74, 90-95, 104-119; utils.h:83-86, 99-111
__device__ __forceinline__ f3 fresnel_schlick(f3 f0, float h_dot_o) { return f0 + (1.0f - f0) * rt_powf(1.0f - h_dot_o, 5.0f); }
__device__ __forceinline__ float ggx_d(float alpha, float n_dot_h)
{
    float a2 = alpha * alpha;
    float denom = n_dot_h * n_dot_h * (a2 - 1.0f) + 1.0f;
    return a2 * RT_INV_PI / (denom * denom);
}
__device__ __forceinline__ float v_smith_ggx_correlated(float n_dot_i, float n_dot_o, float alphaG)
{
    float a2 = alphaG * alphaG;
    float lv = n_dot_o * sqrtf((-n_dot_i * a2 + n_dot_i) * n_dot_i + a2);
    float ll = n_dot_i * sqrtf((-n_dot_o * a2 + n_dot_o) * n_dot_o + a2);
    return 0.5f / (lv + ll);
}
__device__ __forceinline__ f3 reflect(f3 v, f3 n) { return v - 2.0f * dot(v, n) * n; }

// tangent frame of utils.h:99-106 / bxdf.h:163-165
__device__ __forceinline__ void tangent_frame(f3 n, f3& t, f3& b)
{
    f3 axis = fabsf(n.x) > 0.001f ? mk3(0.0f, 1.0f, 0.0f) : mk3(1.0f, 0.0f, 0.0f);
    t = normalize(cross(axis, n));
    b = cross(n, t);
}

// kernels/common/material.h:132-169
__device__ __forceinline__ f3 evaluate_material(const Material& m, const Bsdf& d, f3 normal, f3 incoming, f3 outgoing)
{
    if (m.transparency < 0.5f) return mk3(0.0f, 0.0f, 0.0f);
    f3 half_vec = normalize(incoming + outgoing);
    float n_dot_i = fmaxf(dot(normal, incoming), RT_EPS);
    float n_dot_o = fmaxf(dot(normal, outgoing), RT_EPS);
    float n_dot_h = fmaxf(dot(normal, half_vec), RT_EPS);
    float h_dot_o = fmaxf(dot(half_vec, outgoing), RT_EPS);
    float alpha = m.roughness * m.roughness;
    f3 fresnel = fresnel_schlick(d.f0, h_dot_o);
    float specular = ggx_d(alpha, n_dot_h) * v_smith_ggx_correlated(n_dot_i, n_dot_o, alpha);
    f3 diffuse = d.diffuse_lambert;
    return fresnel * specular + (1.0f - fresnel) * diffuse;
}

// kernels/common/material.h:171-241 with SampleDiffuse :51-64, SampleSpecular :66-103,
// SampleTransparency :105-117, SampleHemisphereCosine bxdf.h:33-54, GGX_Sample bxdf.h:157-168
// (cos_theta's fp64 sub-expression kept in double).
__device__ __forceinline__ f3 sample_bxdf(float s1, f2 s, Material m, Bsdf d, f3 normal, f3 incoming, bool white_furnace,
                                          f3& outgoing, float& pdf, float& offset)
{
    if (white_furnace) { m.diffuse_albedo = splat(1.0f); m.specular_albedo = splat(1.0f); d = derive_bsdf(m); }
    float alpha = m.roughness * m.roughness;
    const float n_dot_in = dot(normal, incoming);
    // Lobe weights without specular (every CornellBox material): when specular_mix is exactly (0, 0, 0) the general rule below gives
    // fresnel = +-0, specular_pdf = +-0 and diffuse_pdf = 1, bit for bit, as long as
    //   - fresnel_schlick(f0, n.i) is finite: f0 is in [0, 1] and |n.i| <= 2 keeps (1 - n.i)^5 below 243, so x * 0 is +-0 for it;
    //   - diffuse_weight = luma(diffuse_mix * (1 - +-0)) = luma(diffuse_mix): 1 - +-0 = 1, and x * 1 = x;
    //   - specular_weight = luma(0 * +-0) = +-0, so weight_sum = w + +-0 = w, specular_pdf = +-0 / w = +-0 and diffuse_pdf = w / w = 1
    //     for a finite nonzero w.
    // The fast path takes +0 for fresnel and specular_pdf.  The sign of a zero changes nothing: s1 <= +-0 is the same test for
    // every s1 (s1 = 0 takes the specular lobe in both), and that lobe's pdf is then pdf * +-0, never > 0, so neither its bxdf
    // nor its pdf reaches a continuation ray; in the diffuse lobe 1 - +-0 = 1.  A NaN n.i, or a zero or non-finite diffuse
    // weight, takes the general path.
    const bool no_specular = d.specular_mix.x == 0.0f && d.specular_mix.y == 0.0f && d.specular_mix.z == 0.0f &&
                             fabsf(n_dot_in) <= 2.0f && d.diffuse_weight > 0.0f && d.diffuse_weight <= 3.402823466e38f;
    f3 fresnel;
    float specular_pdf, diffuse_pdf;
    if (no_specular)
    { fresnel = splat(0.0f); specular_pdf = 0.0f; diffuse_pdf = 1.0f; }
    else
    {
        fresnel = fresnel_schlick(d.f0, n_dot_in) * d.specular_mix;
        float specular_weight = luma(d.specular_mix * fresnel);
        float diffuse_weight = luma(d.diffuse_mix * (1.0f - fresnel));
        float weight_sum = diffuse_weight + specular_weight;
        specular_pdf = specular_weight / weight_sum;
        diffuse_pdf = diffuse_weight / weight_sum;
    }
    offset = 1.0f;
    if (m.transparency < 0.5f)
    {
        pdf = 1.0f; outgoing = -incoming; offset = -1.0f;
        return splat(1.0f);
    }
    f3 bxdf;
    float phi = RT_TWO_PI * s.x;
    // sin/cos of phi are needed by the rough-specular and by the diffuse lobe: evaluated once, ahead of the branch (a warp that
    // holds both kinds of hits runs both sides of it)
    double sphi, cphi;
    rt_sincos_d((double)phi, &sphi, &cphi);
    if (s1 <= specular_pdf)
    {
        f3 spec;
        if (alpha <= 1e-4f)
        {
            outgoing = reflect(-incoming, normal);
            pdf = 1.0f;
            float n_dot_o = dot(outgoing, normal);
            spec = splat(1.0f / n_dot_o);
        }
        else
        {
            float cos_theta = (float)(1.0f / sqrt(1.0 + (double)(alpha * alpha * s.y) / (1.0 - (double)s.y)));
            float sin_theta = sqrtf(fmaxf(0.0f, 1.0f - cos_theta * cos_theta));
            f3 t, b;
            tangent_frame(normal, t, b);
            f3 wh = normalize(b * (float)cphi * sin_theta + t * (float)sphi * sin_theta + normal * cos_theta);
            outgoing = reflect(-incoming, wh);
            float n_dot_o = dot(normal, outgoing);
            float n_dot_h = dot(normal, wh);
            float n_dot_i = dot(normal, incoming);
            float D = ggx_d(alpha, n_dot_h);
            float G = v_smith_ggx_correlated(n_dot_i, n_dot_o, alpha);
            pdf = D * n_dot_h / (4.0f * dot(wh, outgoing));
            spec = splat(D * G);
        }
        bxdf = fresnel * spec * fmaxf(dot(outgoing, normal), 0.0f);
        pdf *= specular_pdf;
    }
    else
    {
        float sin_theta = sqrtf(s.y);
        float cos_theta = sqrtf(1.0f - s.y);
        pdf = cos_theta * RT_INV_PI;
        f3 tbn = mk3((float)cphi * sin_theta, (float)sphi * sin_theta, cos_theta);
        f3 t, b;
        tangent_frame(normal, t, b);
        outgoing = normalize(b * tbn.x + t * tbn.y + normal * tbn.z);
        bxdf = (1.0f - fresnel) * d.diffuse_lambert * fmaxf(dot(outgoing, normal), 0.0f);
        pdf *= diffuse_pdf;
    }
    return bxdf;
}

// Emitter sampling (include/rt_b200.h, RT_OPT_EMITTER_SAMPLING): the BSDF that sample_bxdf integrates, evaluated for a given
// direction `o`, and the density p_b(o) of its non-delta lobes.  Same lobe weights as sample_bxdf:
//   spec = alpha > 1e-4 and n.h > 0 and h.o > 0 and n.o > 0 ? (fresnel * (D * G)) * n.o : 0,  h = normalize(i + o), D = ggx_d(alpha, n.h),
//          G = v_smith(n.i, n.o, alpha) (evaluated only above the horizon: below it, with alpha^2 under half an ulp of 1, its
//          denominator is exactly 0, and inf * 0 would make g NaN)
//   diff = ((1 - fresnel) * (diffuse_albedo / pi)) * max(n.o, 0);   g = spec + diff;   0 for pass-through materials
//   p_b  = (n.h > 0 and h.o > 0 ? specular_pdf * (D * n.h / (4 * h.o)) : 0) + diffuse_pdf * (max(n.o, 0) * (1 / pi))
// The specular terms are 0 when alpha <= 1e-4 (a delta lobe, left to BSDF sampling).  `spec_pdf` and `alpha` let the caller tell
// whether the lobe sample_bxdf picked with s1 was a delta.
__device__ __forceinline__ f3 bxdf_eval_sampled(const Material& m, const Bsdf& d, f3 normal, f3 incoming, f3 o, float& p_b, float& spec_pdf, float& alpha)
{
    alpha = m.roughness * m.roughness;
    f3 fresnel = fresnel_schlick(d.f0, dot(normal, incoming)) * d.specular_mix;
    float specular_weight = luma(d.specular_mix * fresnel);
    float diffuse_weight = luma(d.diffuse_mix * (1.0f - fresnel));
    float weight_sum = diffuse_weight + specular_weight;
    spec_pdf = specular_weight / weight_sum;
    float diffuse_pdf = diffuse_weight / weight_sum;
    p_b = 0.0f;
    if (m.transparency < 0.5f) return splat(0.0f);
    const float cos_o = fmaxf(dot(o, normal), 0.0f);
    f3 g = (1.0f - fresnel) * d.diffuse_lambert * cos_o;
    float ps = 0.0f;
    if (alpha > 1e-4f)
    {
        f3 h = normalize(incoming + o);
        float n_dot_h = dot(normal, h), h_dot_o = dot(h, o);
        float D = ggx_d(alpha, n_dot_h);
        if (n_dot_h > 0.0f && h_dot_o > 0.0f)
        {   // the directions the specular sampler reaches with a positive density (it never continues a path elsewhere)
            if (cos_o > 0.0f)
            {
                float G = v_smith_ggx_correlated(dot(normal, incoming), dot(normal, o), alpha);
                g = fresnel * splat(D * G) * cos_o + g;
            }
            ps = spec_pdf * (D * n_dot_h / (4.0f * h_dot_o));
        }
    }
    p_b = ps + diffuse_pdf * (cos_o * RT_INV_PI);
    return g;
}

// MIS weight of a strategy with density `p` against one with density `q` (power heuristic, beta 2): 1 / (1 + (q/p)^2), NaN -> 0
__device__ __forceinline__ float mis_power(float p, float q)
{
    float r = q / p;
    float w = 1.0f / (1.0f + r * r);
    return w == w ? w : 0.0f;
}

// kernels/common/light.h:30-65 followed by hit_surface.cl:122-123 (length + normalize of the direction).
// For directional lights `outgoing = origin * MAX_RENDER_DIST`, its length and its normalisation are constants
// of the light: computed once at upload with the same operations (rt_bvh_layout.h).  `directional` is the index of the
// light's record when the light is directional (its record holds outgoing_n and distance), else -1.
__device__ __forceinline__ f3 light_sample(const DevScene& sc, f3 position, float s, f3& outgoing_n, float& distance, float& pdf, int& directional)
{
    int n = (int)sc.light_count;
    int idx = (int)(s * (float)sc.light_count);
    idx = idx < 0 ? 0 : (idx > n - 1 ? n - 1 : idx);
    float4 l0 = __ldg(sc.light_rec + (size_t)idx * 2), l1 = __ldg(sc.light_rec + (size_t)idx * 2 + 1);
    pdf = 1.0f / (float)sc.light_count;
    f3 radiance = mk3(l1);
    if (__float_as_uint(l1.w) == RT_LIGHT_TYPE_POINT)
    {
        f3 to_light = mk3(l0) - position;
        radiance = radiance / dot(to_light, to_light);
        distance = length(to_light);
        outgoing_n = normalize(to_light);
        directional = -1;
    }
    else
    {
        directional = idx;
        outgoing_n = mk3(l0);
        distance = l0.w;
    }
    return radiance;
}

} // namespace rt
