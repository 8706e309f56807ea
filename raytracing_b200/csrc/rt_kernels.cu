/*
 * rt_kernels.cu — the sm_90a kernels of the wavefront path tracer and the C ABI
 * (include/rt_b200.h) that launches them.  One translation unit so that the shading
 * code and the warp work items (closest hit, shadow rays, shading of 32 queue entries)
 * inline into the stepwise kernels (one per reference kernel), the per-phase kernels
 * and the one-kernel frame (rt_frame_kernel.cuh) alike.  Build: nvcc -gencode arch=compute_90a,code=sm_90a -fmad=false (see
 * __graft_entry__.build()).  There is no CPU fallback anywhere in this file.
 *
 * Data layout in HBM (all SoA streams of float4, indexed by compacted ray slot):
 *   extension-ray queue q[b&1]:  A = (origin.xyz, pixel_idx bits)
 *                                B = (dir.xyz, t_max)
 *                                C = (path throughput.xyz, -)
 *   shadow-ray queue:            A = (origin.xyz, local pixel index | light byte << 24)
 *                                B = (dir.xyz, t_max = distance to light), not stored for a directional light
 *                                C = (light sample.xyz, 0)                        (rt_kernel_types.cuh, put_shadow)
 *   hit queue:                   (bc.x, bc.y, primitive_id bits, ray slot bits)   — rays that hit, compacted
 *   miss queue:                  ray slot (uint32)                                — rays that missed, compacted
 *   hits (stepwise path only):   (bc.x, bc.y, primitive_id bits, t)
 *   radiance:                    float4 per LOCAL pixel (scanline partition, see rt_set_partition)
 * "pixel_idx bits" is the pixel packed as x | y << 16 (the RNG and the radiance index need x and y, never the
 * linear index, and this saves two integer divisions per path vertex); the API converts back.
 * The reference keeps throughput in a per-pixel buffer that every bounce scatters to
 * (hit_surface.cl:105,166); there is at most one live path per pixel, so carrying it in
 * the ray stream is equivalent and turns the scatter into a coalesced stream.
 * Ray counters are per bounce (q_count[b], shadow_count[b]): nothing has to be cleared
 * between kernels (the reference launches two 1-thread clear kernels per bounce,
 * integrator.cpp:45-46) and the per-bounce statistics fall out for free.
 */
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <type_traits>
#include <vector>

#include "rt_b200.h"
#include "rt_bvh_layout.h"
#include "rt_device.cuh"
#include "rt_emitters.h"
#include "rt_envmap.h"
#include "rt_instances.h"
#include "rt_refit.cuh"
#include "rt_lbvh.cuh"
#include "rt_ploc.cuh"
#include "rt_owned.h"

using namespace rt;

// minimum resident CTAs per SM requested from ptxas for the hot kernels (register budget = 65536 / (256 * N)):
// 5 x 256 threads at <= 48 registers fill the 64 K-register file of an SM (the same on H100).  The shading kernel runs 3 x 256 at
// <= 85 registers (80, no spills): on an H100 it is 12 % faster than 4 x 256 at 64 registers, which spills (DESIGN.md section 4)
#ifndef RT_MINB_TRACE
#define RT_MINB_TRACE 5
#endif
#ifndef RT_MINB_SHADE
#define RT_MINB_SHADE 3
#endif
// k_shade_queues<true> (large partitions) shades up to RT_SHADE_BATCH hit-queue entries per CTA at a time and writes their continuation rays out sorted by a
// 6-bit key (RT_SORT_BINS keys): 48 B of shared memory per staged ray, so 1024 rays x 3 resident CTAs take 3 x 52 KB of an SM's 227 KB
#ifndef RT_SHADE_BATCH
#define RT_SHADE_BATCH 1024
#endif
#define RT_SORT_BINS 64
// Probe-only builds (tools/shade_probe.py, through tools/build_variant.py); their results are not the renderer's.
// RT_SHADE_PROBE 1: memory floor, shade_hit makes its table reads and spawns both rays but does no shading arithmetic (every
// schedule); 2: math floor, each warp of k_shade_queues<false> shades its first hit group's entries again for every hit group it takes.
#ifndef RT_SHADE_PROBE
#define RT_SHADE_PROBE 0
#endif
// The whole-frame kernel (k_frame) is compiled for up to 1024 threads per CTA (64 registers): the CTA size is chosen at launch
// (RT_OPT_FRAME_THREADS) — 1024 threads = one CTA per SM, all 32 warps of an SM in the same phase; 256 threads = 4 CTAs per SM
// in different phases
#define RT_FRAME_MAX_THREADS 1024

namespace
{

#include "rt_kernel_types.cuh"
#include "rt_traverse.cuh"

// ------------------------------------------------------------------------------------ shading
// Instanced scenes: a point through the 3x4 rows r (((r.x*p.x + r.y*p.y) + r.z*p.z) + r.w per row) and a normal through the
// transpose of W's 3x3 part (rows w), all float in the order written
__device__ __forceinline__ f3 xform_point(float4 r0, float4 r1, float4 r2, f3 p)
{
    return mk3(((r0.x * p.x + r0.y * p.y) + r0.z * p.z) + r0.w, ((r1.x * p.x + r1.y * p.y) + r1.z * p.z) + r1.w,
               ((r2.x * p.x + r2.y * p.y) + r2.z * p.z) + r2.w);
}
__device__ __forceinline__ f3 xform_normal(float4 w0, float4 w1, float4 w2, f3 n)
{
    return mk3((w0.x * n.x + w1.x * n.y) + w2.x * n.z, (w0.y * n.x + w1.y * n.y) + w2.y * n.z, (w0.z * n.x + w1.z * n.y) + w2.z * n.z);
}

struct ShadeOut
{
    bool spawn_shadow, spawn_next, emissive;
    f3 emission_add;
    f3 s_origin, s_dir, s_sample; float s_tmax;
    uint32_t s_light;              // the shadow ray's light record when s_dir and s_tmax are those of a directional light, else RT_SHADOW_3PLANE
    f3 n_origin, n_dir, n_throughput;
    float n_pdf;                   // C.w of the continuation ray: its p_b with emitter or environment sampling on, else 0
};

// kernels/cl/miss.cl:41-77: radiance += sky * throughput, for the ray in slot `slot` of ray queue `in`.
// EMIT (the sampled-light instance, shade_hit): with an environment table, a BSDF-sampled ray (C.w = p_b > 0) adds
// (sky * throughput) * mis(p_b, p_v(dir)), weighted against the environment strategy that could have drawn its direction.
// Plane A is not read: a miss needs the direction and the pixel (B) and the throughput (C); at bounce 0 the throughput of every
// path is (1, 1, 1) with C.w = 0, so C is not read either.
template <bool EMIT = false>
__device__ __forceinline__ void shade_miss(const DevScene& sc, const FrameParams& p, const Queues& q, uint32_t bounce, uint32_t slot, float4* radiance)
{
    const int in = bounce & 1;
    const float4 b = q.B[in][slot], c = bounce == 0 ? make_float4(1.0f, 1.0f, 1.0f, 0.0f) : q.C[in][slot];
    f3 sky = p.white_furnace ? splat(0.5f) : sample_sky(sc, mk3(b));
    uint32_t li = local_index(p, __float_as_uint(b.w));
    f3 add = sky * mk3(c);
    if (EMIT && c.w > 0.0f && sc.env_pdf)
        add = add * mis_power(c.w, rtenv::pdf_dir(sc.env_pdf, sc.env_w, sc.env_h, b.x, b.y, b.z));
    float4 r = add_radiance(radiance, li, add);
    if (p.gather) p.gather[li] = r;        // the path ends here: its pixel is final (its last shadow ray was accumulated a phase ago)
}

// kernels/cl/hit_surface.cl:30-186, for the path of sample p.dyn->sample_idx.
// prev_pdf: C.w of the ray (sampled lights: p_b of its direction at the previous vertex, 0 for primary rays and after a delta lobe).
// EMIT: the scene has an active emitter table (sc.emit_*, RT_OPT_EMITTER_SAMPLING) or environment table (sc.env_*,
// RT_OPT_ENV_SAMPLING), each read only while it exists; a template flag, so that the kernels without it are the code of both options off.
// INST: an instanced scene (rt_b200.h): prim is a virtual id; the hit is shaded on its mesh triangle and moved to world space by the
// instance's M (position) and W^T (normals); the AOV's previous position places the mesh triangle's previous positions
// (sc.prev_tri) by the instance's previous M (aov.prev_pos, 3 float4 per instance) when object motion is on; an instance with a
// material row (rt_set_instance_materials) shades with sc.mtl_map[row offset + the triangle's material].
template <bool EMIT = false, bool INST = false>
__device__ __forceinline__ void shade_hit(const SceneOf<INST>& sc, const FrameParams& p, const AovParams& aov, uint32_t bounce, uint32_t pxy,
                                          f3 ray_origin, f3 ray_dir, f3 hit_throughput, float prev_pdf, uint32_t prim, float u, float v,
                                          ShadeOut& out)
{
#if RT_SHADE_PROBE == 1
    {   // memory floor: the shading record, material and blue-noise reads of the hit, each value used by a few adds, and a shadow
        // ray and a continuation ray (back along the incoming ray) for every hit
        const float4* tq = sc.tri_shade + (size_t)prim * 7;
        const float4 q0 = __ldg(tq), q1 = __ldg(tq + 1), q2 = __ldg(tq + 2), q3 = __ldg(tq + 3), q4 = __ldg(tq + 4), q5 = __ldg(tq + 5);
        const float4* mr = sc.mat_rec + (size_t)__float_as_uint(q0.w) * 4;
        const float4 m0 = __ldg(mr), m2 = __ldg(mr + 2);
        float s = 0.0f;
        if (p.bn)
            for (uint32_t d = 0; d < 5; ++d)
                s += sample_blue_noise(p.bn, pxy & 0xFFFFu, pxy >> 16, p.dyn->sample_idx, bounce * 5u + d);
        const float w0 = 1.0f - u - v;
        const f3 position = mk3(q0) * w0 + mk3(q1) * u + mk3(q2) * v;
        out.emissive = false;
        out.spawn_shadow = out.spawn_next = true;
        out.s_origin = position; out.s_dir = mk3(q3) + mk3(q4) + mk3(q5) + mk3(q1.w, q2.w, q3.w); out.s_tmax = s + m2.x;
        // a scene whose first light is directional stores two planes, as the renderer does
        out.s_light = __float_as_uint(__ldg(sc.light_rec + 1).w) == RT_LIGHT_TYPE_DIRECTIONAL ? 0u : RT_SHADOW_3PLANE;
        out.s_sample = hit_throughput * mk3(m0);
        out.n_origin = position; out.n_dir = -ray_dir; out.n_throughput = hit_throughput * mk3(m0); out.n_pdf = prev_pdf + q4.w + q5.w;
        (void)ray_origin; (void)aov;
        return;
    }
#endif
    f3 incoming = -ray_dir;
    uint32_t px = pxy & 0xFFFFu, py = pxy >> 16;
    uint32_t tri = prim, inst = 0;
    if constexpr (INST)
    {   // the instance of the virtual id: the last base <= prim
        uint32_t lo = 0, hi = __float_as_uint(__ldg(sc.inst_hdr + 1).w) - 1u;
        while (lo < hi)
        {
            const uint32_t mid = (lo + hi + 1u) >> 1;
            if (__ldg(sc.ibase + mid) <= prim) lo = mid; else hi = mid - 1u;
        }
        inst = lo;
        const float4 mi = __ldg(sc.irec + (size_t)inst * 8 + 6);
        tri = __float_as_uint(mi.z) + (prim - __float_as_uint(mi.w));
    }
    const float4* tp = sc.tri_shade + (size_t)tri * 7;
    float4 r0 = __ldg(tp), r1 = __ldg(tp + 1), r2 = __ldg(tp + 2), r3 = __ldg(tp + 3), r4 = __ldg(tp + 4), r5 = __ldg(tp + 5);
    f3 p1 = mk3(r0), p2 = mk3(r1), p3 = mk3(r2), n1 = mk3(r3), n2 = mk3(r4), n3 = mk3(r5);
    uint32_t mtl = __float_as_uint(r0.w);
    if constexpr (INST)
    {   // per-instance materials (rt_set_instance_materials): the instance's row, read wherever the mesh triangle's material is
        const uint32_t row = __float_as_uint(__ldg(sc.irec + (size_t)inst * 8 + 7).z);
        if (row != RT_INVALID_ID) mtl = __ldg(sc.mtl_map + row + mtl);
    }
    f3 geometry_normal = mk3(r1.w, r2.w, r3.w);       // normalize(cross(p2-p1, p3-p1)), precomputed at upload
    float w0 = 1.0f - u - v;
    f3 position = p1 * w0 + p2 * u + p3 * v;
    f3 normal;
    f3 obj_position = position;
    f3 inst_prev = position;                          // INST: the velocity AOV's previous position (object motion)
    if constexpr (INST)
    {   // world space: position = M * p; normals = normalize(W^T * n), the geometric one from the unnormalised cross product (the
        // upload's normalize of it, when W is the identity) times sign(det M)
        const float4* ir = sc.irec + (size_t)inst * 8;
        const float4 wr0 = __ldg(ir), wr1 = __ldg(ir + 1), wr2 = __ldg(ir + 2);
        position = xform_point(__ldg(ir + 3), __ldg(ir + 4), __ldg(ir + 5), obj_position);
        normal = normalize(xform_normal(wr0, wr1, wr2, n1 * w0 + n2 * u + n3 * v));
        geometry_normal = normalize(xform_normal(wr0, wr1, wr2, cross(p2 - p1, p3 - p1))) * __ldg(ir + 7).x;
        if (bounce == 0 && aov.enabled && aov.prev_pos)
        {   // object motion, for the AOV block below (here, where tri, u and v are live anyway: carrying them to the block costs the
            // shading kernels spills): the mesh triangle's previous positions at the same barycentrics, placed by the instance's
            // previous transform
            const float4* qt = sc.prev_tri + (size_t)tri * 3;
            const f3 q = mk3(__ldg(qt)) * w0 + mk3(__ldg(qt + 1)) * u + mk3(__ldg(qt + 2)) * v;
            const float4* qp = aov.prev_pos + (size_t)inst * 3;
            inst_prev = xform_point(__ldg(qp), __ldg(qp + 1), __ldg(qp + 2), q);
        }
    }
    else normal = normalize(n1 * w0 + n2 * u + n3 * v);
    f2 texcoord; texcoord.x = 0.0f; texcoord.y = 0.0f;
    if (__float_as_uint(__ldg(sc.mat_rec + (size_t)mtl * 4 + 3).y) != 0u)
    {   // texture coordinates are only needed by textured materials (hit_surface.cl:96-97)
        float4 r6 = __ldg(tp + 6);
        texcoord.x = r4.w * w0 + r6.x * u + r6.z * v; texcoord.y = r5.w * w0 + r6.y * u + r6.w * v;
    }
    Material material = load_material(sc, mtl, texcoord);

    if (bounce == 0 && aov.enabled)
    {   // GenerateAOV, aov.cl:106-109
        uint32_t li = local_index(p, pxy);
        aov.albedo[li] = make_float4(material.diffuse_albedo.x, material.diffuse_albedo.y, material.diffuse_albedo.z, 0.0f);
        aov.depth[li] = length(ray_origin - position);
        aov.normal[li] = make_float4(normal.x, normal.y, normal.z, 0.0f);
        f3 prev = position;
        if (aov.prev_pos)
        {   // object motion: the same barycentrics on the triangle's previous positions (INST: computed above)
            if constexpr (INST) prev = inst_prev;
            else
            {
                const float4* qp = aov.prev_pos + (size_t)prim * 3;
                prev = mk3(__ldg(qp)) * w0 + mk3(__ldg(qp + 1)) * u + mk3(__ldg(qp + 2)) * v;
            }
        }
        f2 s0 = project_screen(position, p.dyn->cam), s1 = project_screen(prev, p.dyn->prev);
        aov.velocity[li] = make_float2(s0.x - s1.x, s0.y - s1.y);
    }

    // sampled lights (RT_OPT_EMITTER_SAMPLING, RT_OPT_ENV_SAMPLING): on at this vertex iff the scene has an active emitter or
    // environment table and the frame traces the continuation ray of this bounce
    const bool emit_on = EMIT && bounce < p.dyn->max_bounces;
    out.emissive = false;
    if (!p.white_furnace && dot(material.emission, splat(1.0f)) > 0.0f)
    {
        out.emissive = true;
        out.emission_add = hit_throughput * material.emission;
        if (EMIT && prev_pdf > 0.0f && sc.emit_pdfA)
        {   // BSDF sample of an emitter: weighted against the emitter strategy that could have produced this direction
            const float pdfA = __ldg(sc.emit_pdfA + prim);
            if (pdfA > 0.0f)
            {
                f3 dv = position - ray_origin;
                float cos_e = -dot(ray_dir, geometry_normal);
                float p_l = pdfA * dot(dv, dv) / cos_e;
                out.emission_add = out.emission_add * mis_power(prev_pdf, p_l);
            }
        }
    }
    uint32_t pixel_seed = sample_seed_pixel(px, py, p.dyn->sample_idx);
    out.spawn_shadow = false;
    out.s_light = RT_SHADOW_3PLANE;
    bool pick_emitter = false, pick_env = false;
    if (EMIT && emit_on)
    {   // light kind (rt_set_light_selection): emitter iff P_e >= 1 or c < P_e, else environment iff the analytic weight is 0 or
        // c < P_e + P_v, else analytic (P_e = 0 without an emitter table, P_v = 0 without an environment table)
        const float ck = sample_random(pixel_seed, 0u, 0x10000u + 4u * bounce);
        pick_emitter = sc.emit_pe >= 1.0f || ck < sc.emit_pe;
        pick_env = !pick_emitter && sc.env_pdf && (sc.no_analytic || ck < sc.light_pev);
    }
    if (pick_emitter)
    {   // next-event estimation on an emissive triangle
        float k1 = sample_random(pixel_seed, 0u, 0x10000u + 4u * bounce + 1u);
        const float k2 = sample_random(pixel_seed, 0u, 0x10000u + 4u * bounce + 2u);
        const float k3 = sample_random(pixel_seed, 0u, 0x10000u + 4u * bounce + 3u);
        k1 = fminf(k1, 0.99999994f);
        uint32_t lo = 0, hi = sc.n_emit - 1u;
        while (lo < hi)
        {   // first CDF entry above k1
            const uint32_t mid = (lo + hi) >> 1;
            if (__ldg(sc.emit_cdf + mid) > k1) hi = mid; else lo = mid + 1u;
        }
        const uint32_t t = __ldg(sc.emit_list + lo);
        const float4* ep = sc.tri_shade + (size_t)t * 7;
        float4 e0 = __ldg(ep), e1 = __ldg(ep + 1), e2 = __ldg(ep + 2), e3 = __ldg(ep + 3);
        const float sq = sqrtf(k2);
        const float b0 = 1.0f - sq, b1 = sq * (1.0f - k3), b2 = sq * k3;
        f3 y = mk3(e0) * b0 + mk3(e1) * b1 + mk3(e2) * b2;
        const uint32_t emtl = __float_as_uint(e0.w);
        f2 euv; euv.x = 0.0f; euv.y = 0.0f;
        if (__float_as_uint(__ldg(sc.mat_rec + (size_t)emtl * 4 + 3).y) != 0u)
        {
            float4 e4 = __ldg(ep + 4), e5 = __ldg(ep + 5), e6 = __ldg(ep + 6);
            euv.x = e4.w * b0 + e6.x * b1 + e6.z * b2; euv.y = e5.w * b0 + e6.y * b1 + e6.w * b2;
        }
        const f3 le = load_material(sc, emtl, euv).emission;
        const f3 o = position + geometry_normal * RT_EPS;
        const f3 dv = y - o;
        const float d2 = dot(dv, dv);
        const float d = sqrtf(d2);
        const f3 w = normalize(dv);
        const float cos_e = -dot(w, mk3(e1.w, e2.w, e3.w));
        if (cos_e > 0.0f)
        {
            const float p_l = __ldg(sc.emit_pdfA + t) * d2 / cos_e;
            float p_b, spec_pdf, alpha;
            const f3 g = bxdf_eval_sampled(material, derive_bsdf(material), normal, incoming, w, p_b, spec_pdf, alpha);
            const f3 ls = hit_throughput * g * le * (mis_power(p_l, p_b) / p_l);
            out.spawn_shadow = (p_l > 0.0f) && (dot(ls, ls) > 0.0f);
            out.s_origin = o;
            out.s_dir = w; out.s_tmax = 0.999f * d; out.s_sample = ls;
        }
    }
    else if (pick_env)
    {   // next-event estimation on the environment map: its shadow ray is unoccluded exactly where a continuation ray would miss
        const float k1 = sample_random(pixel_seed, 0u, 0x10000u + 4u * bounce + 1u);
        const float k2 = sample_random(pixel_seed, 0u, 0x10000u + 4u * bounce + 2u);
        const float k3 = sample_random(pixel_seed, 0u, 0x10000u + 4u * bounce + 3u);
        const float k4 = sample_random(pixel_seed, 0u, 0x20000u + bounce);
        f3 w;
        rtenv::sample(sc.env_marg, sc.env_cond, sc.env_w, sc.env_h, k1, k2, k3, k4, w.x, w.y, w.z);
        const float p_v = rtenv::pdf_dir(sc.env_pdf, sc.env_w, sc.env_h, w.x, w.y, w.z);
        const f3 le = sample_sky(sc, w);
        float p_b, spec_pdf, alpha;
        const f3 g = bxdf_eval_sampled(material, derive_bsdf(material), normal, incoming, w, p_b, spec_pdf, alpha);
        const f3 ls = hit_throughput * g * le * (mis_power(p_v, p_b) / p_v);
        out.spawn_shadow = (p_v > 0.0f) && (dot(ls, ls) > 0.0f);
        out.s_origin = position + geometry_normal * RT_EPS;
        out.s_dir = w; out.s_tmax = RT_MAX_RENDER_DIST; out.s_sample = ls;
    }
    else
    {   // direct lighting (next-event estimation on analytic lights)
        float s_light = p.bn ? sample_blue_noise(p.bn, px, py, p.dyn->sample_idx, bounce * 5u + SAMPLE_LIGHT)
                             : sample_random(pixel_seed, bounce, SAMPLE_LIGHT);
        f3 outgoing; float pdf, distance_to_light;
        int directional;
        f3 light_radiance = light_sample(sc, position, s_light, outgoing, distance_to_light, pdf, directional);
        // light_sample = L * throughput * brdf / pdf * max(n.l, 0); a shadow ray is spawned iff pdf > 0 and
        // dot(sample, sample) > 0 (hit_surface.cl:127-129).  When max(n.l, 0) is 0 every component of the sample is
        // +-0 or NaN whatever the BRDF evaluates to, so the ray is never spawned: the BRDF evaluation is skipped then.
        const float cos_l = fmaxf(dot(outgoing, normal), 0.0f);
        if (cos_l > 0.0f)
        {
            f3 brdf = evaluate_material(material, derive_bsdf(material), normal, incoming, outgoing);
            // one light: pdf = 1 / 1 = 1 and x / 1 = x for every x but a NaN, whose quotient may carry other NaN bits; a sample with a
            // NaN component is never stored (dot(ls, ls) > 0 is false), so the division is skipped
            f3 ls = light_radiance * hit_throughput * brdf;
            if (sc.light_count != 1u) ls = ls / pdf;
            ls = ls * cos_l;
            if (EMIT && emit_on) ls = ls / (1.0f - sc.light_pev);
            out.spawn_shadow = (pdf > 0.0f) && (dot(ls, ls) > 0.0f);
            out.s_origin = position + normal * RT_EPS;
            out.s_dir = outgoing; out.s_tmax = distance_to_light; out.s_sample = ls;
            out.s_light = directional >= 0 && directional < (int)RT_SHADOW_3PLANE ? (uint32_t)directional : RT_SHADOW_3PLANE;
        }
    }
    {   // BSDF sampling
        f2 s; float s1;
        if (p.bn)
        {
            const uint32_t sample_idx = p.dyn->sample_idx;
            s.x = sample_blue_noise(p.bn, px, py, sample_idx, bounce * 5u + SAMPLE_U);
            s.y = sample_blue_noise(p.bn, px, py, sample_idx, bounce * 5u + SAMPLE_V);
            s1 = sample_blue_noise(p.bn, px, py, sample_idx, bounce * 5u + SAMPLE_LAYER);
        }
        else
        {
            s.x = sample_random(pixel_seed, bounce, SAMPLE_U); s.y = sample_random(pixel_seed, bounce, SAMPLE_V);
            s1 = sample_random(pixel_seed, bounce, SAMPLE_LAYER);
        }
        float pdf = 0.0f, offset = 1.0f;
        f3 outgoing = mk3(0.0f, 0.0f, 0.0f);
        // (derived here, not loaded: holding loaded constants from here on costs k_shade_queues spills at its 80 registers)
        f3 bxdf = sample_bxdf(s1, s, material, derive_bsdf(material), normal, incoming, p.white_furnace != 0, outgoing, pdf, offset);
        f3 throughput = splat(0.0f);
        if (pdf > 0.0f) throughput = bxdf / pdf;
        out.n_throughput = hit_throughput * throughput;
        out.spawn_next = pdf > 0.0f;
        out.n_origin = position + geometry_normal * RT_EPS * offset;
        out.n_dir = outgoing;
        out.n_pdf = 0.0f;
        if (EMIT && emit_on)
        {   // the continuation's p_b for the MIS weight of an emitter it hits or of the sky it misses into (0 after a delta lobe)
            float p_b, spec_pdf, alpha;
            bxdf_eval_sampled(material, derive_bsdf(material), normal, incoming, outgoing, p_b, spec_pdf, alpha);
            const bool delta = material.transparency < 0.5f || (s1 <= spec_pdf && alpha <= 1e-4f);
            out.n_pdf = delta ? 0.0f : p_b;
        }
    }
}

// ------------------------------------------------------------------------------------ warp work items
// The bodies shared by the per-phase kernels and the one-kernel frame (rt_frame_kernel.cuh); the closest-hit, shadow and shading
// items each handle one group of 32 queue entries.  Entry i of a queue lives in slot base + i: base is 0 for the per-phase
// kernels and the CTA's region of every queue for k_frame.  The slot and statistics counters are global memory (DevCounters)
// for the per-phase kernels and shared memory (CtaFrame) for k_frame.

// RayGeneration (raygeneration.cl:65-139): the primary ray (a, b) of local pixel li for sample `sample_idx` in queue-plane layout
// (a = origin, b = direction + packed pixel); clears the pixel's AOVs
__device__ __forceinline__ void make_primary_ray(const FrameParams& p, const AovParams& aov, uint32_t li, uint32_t sample_idx, float4& a, float4& b)
{
    const uint32_t px = li % p.width, py = (li / p.width) * p.world + p.rank;
    f3 o, d;
    generate_primary_ray(p.dyn->raygen, py * p.width + px, px, py, sample_idx, o, d);
    a = make_float4(o.x, o.y, o.z, 0.0f);
    b = make_float4(d.x, d.y, d.z, __uint_as_float(pack_pixel(px, py)));
    if (aov.enabled)
    {   // raygeneration.cl:129-133
        aov.albedo[li] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        aov.depth[li] = RT_MAX_RENDER_DIST;
        aov.normal[li] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        aov.velocity[li] = make_float2(0.0f, 0.0f);
    }
}

// make_primary_ray of sample p.dyn->sample_idx, stored in slot `slot` of ray queue 0 with throughput 1 and C.w = 0
__device__ __forceinline__ void primary_ray(const FrameParams& p, const Queues& q, const AovParams& aov, uint32_t slot, uint32_t li, float4& a, float4& b)
{
    make_primary_ray(p, aov, li, p.dyn->sample_idx, a, b);
    q.A[0][slot] = a; q.B[0][slot] = b; q.C[0][slot] = make_float4(1.0f, 1.0f, 1.0f, 0.0f);
}

// Closest hit of the ray (a, b) of entry i (live lanes) and hit/miss stream compaction: __ballot + __popc give every lane its
// slot, ONE 64-bit atomic per warp on `hm` reserves the slots of both queues (hits in the low word, misses in the high).
template <bool COUNT, int SMEM, bool PIN, class Scene>
__device__ __forceinline__ void closest_group(const Scene& sc, int mode, const float4* s_bvh, const Queues& q, uint32_t base, uint32_t i, bool live,
                                              float4 a, float4 b, unsigned long long* hm, uint32_t& nv, uint32_t& nt)
{
    const int lane = threadIdx.x & 31;
    bool hit = false;
    float bu = 0.0f, bv = 0.0f, bt = 0.0f;
    uint32_t prim = RT_INVALID_ID;
    if (live)
    {
        prim = trace_staged<false, COUNT, SMEM, PIN>(sc, mode, s_bvh, a, b, bu, bv, bt, nv, nt);
        hit = prim != RT_INVALID_ID;
    }
    const unsigned hmask = __ballot_sync(0xffffffffu, hit);
    const unsigned mmask = __ballot_sync(0xffffffffu, live && !hit);
    unsigned long long slot = 0ull;
    if (lane == 0) slot = atomicAdd(hm, (unsigned long long)__popc(hmask) | ((unsigned long long)__popc(mmask) << 32));
    slot = __shfl_sync(0xffffffffu, slot, 0);
    const unsigned lt_mask = (1u << lane) - 1u;
    if (hit) q.hitq[base + (uint32_t)slot + __popc(hmask & lt_mask)] = make_float4(bu, bv, __uint_as_float(prim), __uint_as_float(i));
    else if (live) q.missq[base + (uint32_t)(slot >> 32) + __popc(mmask & lt_mask)] = i;
}

// IntersectShadowRays + AccumulateDirectSamples (accumulate_direct_samples.cl:27-53) of shadow-queue entry i < n: any-hit trace,
// the light sample of an unoccluded ray added to its pixel, the unoccluded rays counted on `n_unoccluded`
template <bool COUNT, int SMEM, bool PIN, class Scene>
__device__ __forceinline__ void shadow_group(const FrameParams& p, const Scene& sc, int mode, const float4* s_bvh, const Queues& q, uint32_t base,
                                             uint32_t i, uint32_t n, float4* radiance, uint32_t* n_unoccluded, uint32_t& nv, uint32_t& nt)
{
    bool un = false;
    if (i < n)
    {
        const float4 a = q.sA[base + i];
        uint32_t li;
        const float4 b = shadow_dir(p, sc, q, base + i, __float_as_uint(a.w), li);
        float bu, bv, bt;
        un = trace_staged<true, COUNT, SMEM, PIN>(sc, mode, s_bvh, a, b, bu, bv, bt, nv, nt) == RT_INVALID_ID;
        if (un) add_radiance(radiance, li, mk3(q.sC[base + i]));
    }
    warp_count(n_unoccluded, un);
}

// k_shade_queues' dynamic shared memory: one batch of continuation rays, written out in key order by a counting sort
struct ContStage
{
    float4 mid;                                                        // centre of the scene's bounding box (the origin half of the key)
    float4 A[RT_SHADE_BATCH], B[RT_SHADE_BATCH], C[RT_SHADE_BATCH];    // the rays as the warps staged them (queue planes A, B, C)
    uint16_t perm[RT_SHADE_BATCH];                                     // output position -> staged ray
    uint8_t key[RT_SHADE_BATCH];
    uint32_t count[RT_SORT_BINS];                                      // rays per key, then the next output position of each key
    uint32_t n, at, out;                                               // rays staged, the batch's first cursor entry, its first slot in the queue
};

// The key of a continuation ray: direction octant (high 3 bits) and the octant of the origin about the scene's centre.  It only
// orders the queue, so that the warps of the next traversal and shading passes hold rays that start in the same part of the scene
// and head the same way; no result depends on it.
__device__ __forceinline__ uint32_t ray_key(f3 o, f3 d, float4 mid)
{
    return (d.x < 0.0f ? 8u : 0u) | (d.y < 0.0f ? 16u : 0u) | (d.z < 0.0f ? 32u : 0u)
         | (o.x >= mid.x ? 1u : 0u) | (o.y >= mid.y ? 2u : 0u) | (o.z >= mid.z ? 4u : 0u);
}

// ShadeSurfaceHits (hit_surface.cl) of the hit h = (bc.x, bc.y, primitive_id bits, -) of the ray in entry i (hit lanes): shading,
// emission into the radiance, and compaction of the two output streams — ONE 64-bit atomic per warp on `emit` reserves the slots
// of both queues (shadow rays in the low word, continuation rays in the high).  With STAGE the continuation rays go to the CTA's
// staging area `st` instead (flush_continuations writes them out and counts them) and the atomic reserves shadow-ray slots only.
// Returns whether the lane's path ends at this hit (no continuation ray); `pixel` is the packed pixel of the ray.
// ALL_PLANES (the one-kernel frame with EMIT, whose primary rays are stored whole): read planes A and C of every hit; at its 64
// registers the two uniform branches below cost it spills.
template <bool STAGE = false, bool EMIT = false, bool INST = false, bool ALL_PLANES = false>
__device__ __forceinline__ bool shade_hit_group(const FrameParams& p, const SceneOf<INST>& sc, const AovParams& aov, const Queues& q, uint32_t base, uint32_t bounce,
                                                bool hit, float4 h, uint32_t i, float4* radiance, unsigned long long* emit, uint32_t* n_emissive, uint32_t& pixel,
                                                ContStage* st = nullptr)
{
    const int in = bounce & 1, out = (bounce + 1) & 1;
    ShadeOut so;
    so.emissive = so.spawn_next = so.spawn_shadow = false;
    pixel = 0;
    uint32_t li = 0;
    if (hit)
    {   // plane A (the origin) only where shade_hit reads it: the depth AOV of bounce 0 and, with EMIT, the MIS weight of an emitter
        // hit by a BSDF-sampled ray (never at bounce 0: C.w of a primary ray is 0).  Plane C is (1, 1, 1, 0) at bounce 0.
        const bool origin = ALL_PLANES || (bounce == 0 ? aov.enabled != 0 : EMIT);
        const float4 b = q.B[in][base + i];
        const float4 c = bounce == 0 && !ALL_PLANES ? make_float4(1.0f, 1.0f, 1.0f, 0.0f) : q.C[in][base + i];
        const float4 a = origin ? q.A[in][base + i] : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        pixel = __float_as_uint(b.w);
        shade_hit<EMIT, INST>(sc, p, aov, bounce, pixel, mk3(a), mk3(b), mk3(c), c.w, __float_as_uint(h.z), h.x, h.y, so);
        li = local_index(p, pixel);
        if (so.emissive) add_radiance(radiance, li, so.emission_add);
    }
    const bool ss = hit && so.spawn_shadow, sn = hit && so.spawn_next;
    const unsigned smask = __ballot_sync(0xffffffffu, ss), nmask = __ballot_sync(0xffffffffu, sn);
    const unsigned emask = __ballot_sync(0xffffffffu, hit && so.emissive);
    const int lane = threadIdx.x & 31;
    const unsigned lt_mask = (1u << lane) - 1u;
    unsigned long long slot = 0ull;
    if ((smask | nmask | emask) != 0u)
    {
        if (lane == 0)
        {
            if (STAGE) { if (smask) slot = atomicAdd((uint32_t*)emit, (uint32_t)__popc(smask)); }
            else slot = atomicAdd(emit, (unsigned long long)__popc(smask) | ((unsigned long long)__popc(nmask) << 32));
            if (emask) atomicAdd(n_emissive, (uint32_t)__popc(emask));
        }
        slot = __shfl_sync(0xffffffffu, slot, 0);
    }
    if (ss)
    {
        const uint32_t si = base + (uint32_t)slot + __popc(smask & lt_mask);
        put_shadow(p, q, si, li, so.s_light, so.s_origin, so.s_dir, so.s_tmax, so.s_sample);
    }
    if (STAGE)
    {
        uint32_t j = 0;
        if (nmask)
        {
            if (lane == 0) j = atomicAdd(&st->n, (uint32_t)__popc(nmask));
            j = __shfl_sync(0xffffffffu, j, 0) + __popc(nmask & lt_mask);
        }
        if (sn)
        {
            st->A[j] = make_float4(so.n_origin.x, so.n_origin.y, so.n_origin.z, 0.0f);
            st->B[j] = make_float4(so.n_dir.x, so.n_dir.y, so.n_dir.z, __uint_as_float(pixel));
            st->C[j] = make_float4(so.n_throughput.x, so.n_throughput.y, so.n_throughput.z, so.n_pdf);
            const uint32_t key = ray_key(so.n_origin, so.n_dir, st->mid);
            st->key[j] = (uint8_t)key;
            atomicAdd(&st->count[key], 1u);
        }
    }
    else if (sn)
    {
        const uint32_t ni = base + (uint32_t)(slot >> 32) + __popc(nmask & lt_mask);
        q.A[out][ni] = make_float4(so.n_origin.x, so.n_origin.y, so.n_origin.z, 0.0f);
        q.B[out][ni] = make_float4(so.n_dir.x, so.n_dir.y, so.n_dir.z, __uint_as_float(pixel));
        q.C[out][ni] = make_float4(so.n_throughput.x, so.n_throughput.y, so.n_throughput.z, so.n_pdf);
    }
    return hit && !so.spawn_next;
}

// ------------------------------------------------------------------------------------ kernels
__global__ void __launch_bounds__(256) k_reset(float4* radiance, uint32_t n)
{
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) radiance[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
}

// One thread per LOCAL pixel; slot i of queue 0 = local pixel i, or with adaptive sampling the i-th active pixel (the grid stays
// sized by the partition, so that a captured frame graph serves every frame).
__global__ void __launch_bounds__(256) k_raygen(FrameParams p, Queues q, DevCounters* ctr, AovParams aov)
{
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t n = p.active ? *p.n_active : p.n_local;
    if (i == 0) ctr->n_primary = n;
    if (i >= n) return;
    float4 a, b;
    primary_ray(p, q, aov, i, p.active ? p.active[i] : i, a, b);
}

// IntersectRays (stepwise): closest hit of every live ray of bounce b -> hits[]
// INST: an instanced scene (trace_instanced); mode is not read.  Nothing is staged.
template <bool COUNT, bool INST = false>
__global__ void __launch_bounds__(256) k_intersect(FrameParams p, SceneOf<INST> sc, int mode, Queues q, DevCounters* ctr, uint32_t bounce)
{
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t n = *in_count_ptr(ctr, bounce);
    int in = bounce & 1;
    uint32_t nv = 0, nt = 0;
    if (i < n)
    {
        float4 a = q.A[in][i], b = q.B[in][i];
        float bu = 0.0f, bv = 0.0f, bt = 0.0f;
        const uint32_t prim = trace_staged<false, COUNT, INST ? RT_SMEM_INST : 0, false>(sc, mode, nullptr, a, b, bu, bv, bt, nv, nt);
        q.hits[i] = make_float4(bu, bv, __uint_as_float(prim), bt);
    }
    if (COUNT) { warp_sum64(&ctr->nodes_ext[bounce], nv); warp_sum64(&ctr->tris_ext[bounce], nt); }
}

// ShadeMissedRays (stepwise)
template <bool EMIT>
__global__ void __launch_bounds__(256) k_shade_miss(FrameParams p, DevScene sc, Queues q, DevCounters* ctr, float4* radiance, uint32_t bounce)
{
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t n = *in_count_ptr(ctr, bounce);
    bool miss = false;
    if (i < n)
    {
        miss = __float_as_uint(q.hits[i].z) == RT_INVALID_ID;
        if (miss) shade_miss<EMIT>(sc, p, q, bounce, i, radiance);
    }
    warp_count(&ctr->hm[bounce].miss, miss);
}

// ShadeSurfaceHits (stepwise)
template <bool EMIT, bool INST = false>
__global__ void __launch_bounds__(256) k_shade_hits(FrameParams p, SceneOf<INST> sc, Queues q, DevCounters* ctr, float4* radiance, uint32_t bounce, AovParams aov)
{
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t n = *in_count_ptr(ctr, bounce);
    bool hit = false;
    float4 h = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    if (i < n)
    {
        h = q.hits[i];
        hit = __float_as_uint(h.z) != RT_INVALID_ID;
    }
    uint32_t pixel;
    shade_hit_group<false, EMIT, INST>(p, sc, aov, q, 0, bounce, hit, h, i, radiance, (unsigned long long*)&ctr->emit[bounce], &ctr->n_emissive[bounce], pixel);
}

// IntersectShadowRays (stepwise): any-hit -> flags (0 = occluded, INVALID_ID = unoccluded)
template <bool COUNT, bool INST = false>
__global__ void __launch_bounds__(256) k_intersect_shadow(FrameParams p, SceneOf<INST> sc, int mode, Queues q, DevCounters* ctr, uint32_t bounce)
{
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t n = ctr->emit[bounce].shadow;
    uint32_t nv = 0, nt = 0;
    if (i < n)
    {
        const float4 a = q.sA[i];
        uint32_t li;
        const float4 b = shadow_dir(p, sc, q, i, __float_as_uint(a.w), li);
        float bu, bv, bt;
        q.shadow_flags[i] = trace_staged<true, COUNT, INST ? RT_SMEM_INST : 0, false>(sc, mode, nullptr, a, b, bu, bv, bt, nv, nt);
    }
    if (COUNT) { warp_sum64(&ctr->nodes_shadow[bounce], nv); warp_sum64(&ctr->tris_shadow[bounce], nt); }
}

// AccumulateDirectSamples (stepwise): accumulate_direct_samples.cl:27-53
__global__ void __launch_bounds__(256) k_accumulate(FrameParams p, Queues q, DevCounters* ctr, float4* radiance, uint32_t bounce)
{
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t n = ctr->emit[bounce].shadow;
    bool un = false;
    if (i < n)
    {
        un = q.shadow_flags[i] == RT_INVALID_ID;
        if (un) add_radiance(radiance, shadow_two_plane(p) ? __float_as_uint(q.sA[i].w) & 0xFFFFFFu : __float_as_uint(q.sA[i].w), mk3(q.sC[i]));
    }
    warp_count(&ctr->n_unoccluded[bounce], un);
}

// ---- queue-split schedule (default): hit/miss stream compaction between traversal and shading --------------
// Traversal and shading are separate persistent kernels: the traversal kernel stays small in registers
// (more resident warps to hide the dependent node fetches), and it compacts its results into a HIT queue and a
// MISS queue with one warp-aggregated atomic each (__ballot + __popc), so that the shading kernel runs full
// warps of hits (Lambert/GGX + NEE) and full warps of misses (environment lookup) instead of warps that
// mix the two and idle through each other's code.  Every kernel drains its queues through a global atomic
// cursor (warp_grab).
template <bool COUNT, int SMEM>
__device__ __forceinline__ void closest_phase(const SceneOf<SMEM == RT_SMEM_INST>& sc, int mode, const Queues& q, DevCounters* ctr, uint32_t bounce, const float4* s_bvh)
{
    const uint32_t n = *in_count_ptr(ctr, bounce);
    const int in = bounce & 1;
    uint32_t nv = 0, nt = 0;
    for (uint32_t at; (at = warp_grab(&ctr->work_ext[bounce])) < n;)
    {
        const uint32_t i = at + (threadIdx.x & 31);
        const bool live = i < n;
        float4 a, b;
        if (live) { a = q.A[in][i]; b = q.B[in][i]; }
        closest_group<COUNT, SMEM, false>(sc, mode, s_bvh, q, 0, i, live, a, b, (unsigned long long*)&ctr->hm[bounce], nv, nt);
    }
    if (COUNT) { warp_sum64(&ctr->nodes_ext[bounce], nv); warp_sum64(&ctr->tris_ext[bounce], nt); }
}

// Fused IntersectShadowRays + AccumulateDirectSamples over the bounce's shadow-ray queue
template <bool COUNT, int SMEM>
__device__ __forceinline__ void shadow_phase(const FrameParams& p, const SceneOf<SMEM == RT_SMEM_INST>& sc, int mode, const Queues& q, DevCounters* ctr, float4* radiance,
                                             uint32_t bounce, const float4* s_bvh)
{
    const uint32_t n = ctr->emit[bounce].shadow;
    uint32_t nv = 0, nt = 0;
    for (uint32_t at; (at = warp_grab(&ctr->work_shadow[bounce])) < n;)
        shadow_group<COUNT, SMEM, false>(p, sc, mode, s_bvh, q, 0, at + (threadIdx.x & 31), n, radiance, &ctr->n_unoccluded[bounce], nv, nt);
    if (COUNT) { warp_sum64(&ctr->nodes_shadow[bounce], nv); warp_sum64(&ctr->tris_shadow[bounce], nt); }
}

template <bool COUNT, int SMEM>
__global__ void __launch_bounds__(256, RT_MINB_TRACE) k_shadow_accumulate(FrameParams p, SceneOf<SMEM == RT_SMEM_INST> sc, int mode, Queues q, DevCounters* ctr, float4* radiance, uint32_t bounce)
{
    extern __shared__ __align__(128) float4 s_bvh[];
    __shared__ uint64_t s_mbar;
    stage_bvh<SMEM>(s_bvh, sc, &s_mbar);
    pdl_wait(); pdl_launch_dependents();
    shadow_phase<COUNT, SMEM>(p, sc, mode, q, ctr, radiance, bounce, s_bvh);
}

template <bool COUNT, int SMEM>
__global__ void __launch_bounds__(256, RT_MINB_TRACE) k_trace_closest(FrameParams p, SceneOf<SMEM == RT_SMEM_INST> sc, int mode, Queues q, DevCounters* ctr, uint32_t bounce)
{
    extern __shared__ __align__(128) float4 s_bvh[];
    __shared__ uint64_t s_mbar;
    stage_bvh<SMEM>(s_bvh, sc, &s_mbar);
    pdl_wait(); pdl_launch_dependents();
    closest_phase<COUNT, SMEM>(sc, mode, q, ctr, bounce, s_bvh);
}

// Bounce 0 of the per-phase frame: k_raygen and k_trace_closest(0) in one kernel.  Entry i is generated in registers (local pixel
// i, or active[i] with adaptive sampling), traced, and only the planes the bounce-0 shading pass reads are stored: B (direction,
// pixel), and A (origin) when the AOVs are on.  That pass takes C as (1, 1, 1, 0).  Sets n_primary as k_raygen does.
template <bool COUNT, int SMEM>
__global__ void __launch_bounds__(256, RT_MINB_TRACE) k_trace_primary(FrameParams p, SceneOf<SMEM == RT_SMEM_INST> sc, int mode, Queues q, DevCounters* ctr,
                                                                      AovParams aov)
{
    extern __shared__ __align__(128) float4 s_bvh[];
    __shared__ uint64_t s_mbar;
    stage_bvh<SMEM>(s_bvh, sc, &s_mbar);
    pdl_wait(); pdl_launch_dependents();
    const uint32_t n = p.active ? *p.n_active : p.n_local;
    if (blockIdx.x == 0 && threadIdx.x == 0) ctr->n_primary = n;
    uint32_t nv = 0, nt = 0;
    for (uint32_t at; (at = warp_grab(&ctr->work_ext[0])) < n;)
    {
        const uint32_t i = at + (threadIdx.x & 31);
        const bool live = i < n;
        float4 a, b;
        if (live)
        {
            make_primary_ray(p, aov, p.active ? p.active[i] : i, p.dyn->sample_idx, a, b);
            q.B[0][i] = b;
            if (aov.enabled) q.A[0][i] = a;
        }
        closest_group<COUNT, SMEM, false>(sc, mode, s_bvh, q, 0, i, live, a, b, (unsigned long long*)&ctr->hm[0], nv, nt);
    }
    if (COUNT) { warp_sum64(&ctr->nodes_ext[0], nv); warp_sum64(&ctr->tris_ext[0], nt); }
}

// Closest-hit traversal of bounce b and the shadow pass of bounce b-1 in ONE persistent kernel (RT_OPT_OVERLAP = 2, the
// default): the two are independent (the shadow pass only shares the radiance buffer with LATER shading passes), every
// warp drains the extension queue and then the shadow queue, so the short shadow rays fill the tail of the long
// extension rays without a second launch, a second staging of the BVH or cross-stream events.
template <int SMEM>
__global__ void __launch_bounds__(256, RT_MINB_TRACE) k_trace_both(FrameParams p, SceneOf<SMEM == RT_SMEM_INST> sc, int mode, Queues q, DevCounters* ctr, float4* radiance,
                                                                   uint32_t bounce, uint32_t shadow_bounce)
{
    extern __shared__ __align__(128) float4 s_bvh[];
    __shared__ uint64_t s_mbar;
    stage_bvh<SMEM>(s_bvh, sc, &s_mbar);
    pdl_wait(); pdl_launch_dependents();
    closest_phase<false, SMEM>(sc, mode, q, ctr, bounce, s_bvh);
    shadow_phase<false, SMEM>(p, sc, mode, q, ctr, radiance, shadow_bounce, s_bvh);
}

// The staged continuation rays of a batch into ray queue `out`, sorted by key (counting sort in shared memory), at slots that
// ONE atomic per CTA on `n_next` reserves.  The order of a ray queue never changes a result: at most one path per pixel is
// alive, and the additions into a pixel's radiance are ordered by phase, not by queue slot.
__device__ __forceinline__ void flush_continuations(ContStage& st, const Queues& q, int out, uint32_t* n_next)
{
    __syncthreads();                                            // every warp of the batch has staged its rays
    const uint32_t n = st.n;
    if (threadIdx.x < 32)
    {   // exclusive scan of the key counts, two keys per lane
        const int lane = threadIdx.x;
        const uint32_t c0 = st.count[2 * lane], c1 = st.count[2 * lane + 1];
        uint32_t s = c0 + c1;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1)
        {
            const uint32_t t = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += t;
        }
        s -= c0 + c1;
        st.count[2 * lane] = s; st.count[2 * lane + 1] = s + c0;
        if (lane == 0 && n) st.out = atomicAdd(n_next, n);
    }
    __syncthreads();
    for (uint32_t j = threadIdx.x; j < n; j += blockDim.x) st.perm[atomicAdd(&st.count[st.key[j]], 1u)] = (uint16_t)j;
    __syncthreads();
    const uint32_t o = st.out;
    for (uint32_t d = threadIdx.x; d < n; d += blockDim.x)
    {   // coalesced stores in key order
        const uint32_t j = st.perm[d];
        q.A[out][o + d] = st.A[j]; q.B[out][o + d] = st.B[j]; q.C[out][o + d] = st.C[j];
    }
}

// ShadeSurfaceHits over the hit queue, then ShadeMissedRays over the miss queue (independent pixels).
// SORT = false: every warp takes 32 entries at a time and stores its continuation rays as it shades them.
// SORT = true (large partitions, sorted_shading): the hits are taken by the CTA in batches of up to RT_SHADE_BATCH entries, one
// cursor add each, so that their continuation rays leave sorted by ray_key (flush_continuations); the batch shrinks towards 256
// entries when there are fewer than 4 full batches per CTA, so that the CTAs still finish together.  Misses past the last hit
// batch are taken 32 at a time by each warp.
template <bool SORT, bool EMIT = false, bool INST = false>
__global__ void __launch_bounds__(256, RT_MINB_SHADE) k_shade_queues(FrameParams p, SceneOf<INST> sc, Queues q, DevCounters* ctr, float4* radiance, uint32_t bounce,
                                                                     AovParams aov, float4 scene_mid)
{
    extern __shared__ __align__(16) float4 s_dyn[];
    ContStage& st = *reinterpret_cast<ContStage*>(s_dyn);
    if (SORT && threadIdx.x == 0) st.mid = scene_mid;
    pdl_wait(); pdl_launch_dependents();
    const uint32_t n_hit = ctr->hm[bounce].hit, n_miss = ctr->hm[bounce].miss;
    const uint32_t hit_span = (n_hit + 31u) & ~31u;            // warps never mix hits and misses
    const uint32_t total = hit_span + n_miss;
    if (!SORT)
    {
        const int lane = threadIdx.x & 31;
        uint32_t first = ~0u;                                   // RT_SHADE_PROBE 2 only
        for (uint32_t at; (at = warp_grab(&ctr->work_shade[bounce])) < total;)
        {
            if (at < hit_span)
            {
                if (RT_SHADE_PROBE == 2) { if (first == ~0u) first = at; at = first; }
                const uint32_t k = at + lane;
                const bool hit = k < n_hit;
                float4 h = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
                if (hit) h = q.hitq[k];
                uint32_t pixel;
                shade_hit_group<false, EMIT, INST>(p, sc, aov, q, 0, bounce, hit, h, __float_as_uint(h.w), radiance, (unsigned long long*)&ctr->emit[bounce], &ctr->n_emissive[bounce], pixel);
            }
            else if (at - hit_span + lane < n_miss) shade_miss<EMIT>(sc, p, q, bounce, q.missq[at - hit_span + lane], radiance);
        }
        return;
    }
    const uint32_t batch = min((uint32_t)RT_SHADE_BATCH, max(256u, (n_hit / (gridDim.x * 4u) + 31u) & ~31u));
    const int lane = threadIdx.x & 31, in = bounce & 1;
    for (uint32_t at;;)
    {
        __syncthreads();                                        // the previous batch is written out: staging area and counts are free
        if (threadIdx.x < RT_SORT_BINS) st.count[threadIdx.x] = 0;
        if (threadIdx.x == 0) { st.at = atomicAdd(&ctr->work_shade[bounce], batch); st.n = 0; }
        __syncthreads();
        at = st.at;
        const uint32_t end = min(at + batch, total);
        for (uint32_t g = at + (threadIdx.x & ~31u); g < end; g += blockDim.x)
        {
            if (g < hit_span)
            {
                const uint32_t k = g + lane;
                const bool hit = k < n_hit;
                float4 h = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
                if (hit) h = q.hitq[k];
                uint32_t pixel;
                shade_hit_group<true, EMIT, INST>(p, sc, aov, q, 0, bounce, hit, h, __float_as_uint(h.w), radiance, (unsigned long long*)&ctr->emit[bounce], &ctr->n_emissive[bounce], pixel, &st);
            }
            else if (g - hit_span + lane < n_miss) shade_miss<EMIT>(sc, p, q, bounce, q.missq[g - hit_span + lane], radiance);
        }
        if (at < hit_span) flush_continuations(st, q, in ^ 1, &ctr->emit[bounce].next);
        if (at + batch >= hit_span) break;                      // every later entry is a miss
    }
    for (uint32_t at; (at = warp_grab(&ctr->work_shade[bounce])) < total;)
        if (at - hit_span + lane < n_miss) shade_miss<EMIT>(sc, p, q, bounce, q.missq[at - hit_span + lane], radiance);
}

#include "rt_frame_kernel.cuh"


// resolve_radiance.cl:31-86: shaded colour (radiance / sample_count unless the denoiser is on, then Reinhard x/(1+x))
// or one of the AOV views.  counts (adaptive sampling, else nullptr): the shaded colour divides by the pixel's own sample count.
__global__ void __launch_bounds__(256) k_resolve(const float4* radiance, float4* out, uint32_t n, uint32_t sample_count, int denoiser,
                                                 int aov_index, AovParams aov, const uint32_t* counts)
{
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (aov_index == 1) { float4 a = aov.albedo[i]; out[i] = make_float4(a.x, a.y, a.z, 1.0f); }
    else if (aov_index == 2) { float d = aov.depth[i] * 0.1f; out[i] = make_float4(d, d, d, 1.0f); }
    else if (aov_index == 3) { float4 nn = aov.normal[i]; out[i] = make_float4(nn.x * 0.5f + 0.5f, nn.y * 0.5f + 0.5f, nn.z * 0.5f + 0.5f, 1.0f); }
    else if (aov_index == 4) { float2 v = aov.velocity[i]; out[i] = make_float4(v.x, v.y, 0.0f, 1.0f); }
    else
    {
        float4 r = radiance[i];
        f3 hdr = mk3(r);
        if (!denoiser) hdr = hdr / (float)(counts ? counts[i] : sample_count);
        f3 ldr = hdr / (mk3(hdr.x + 1.0f, hdr.y + 1.0f, hdr.z + 1.0f));
        out[i] = make_float4(ldr.x, ldr.y, ldr.z, 1.0f);
    }
}

// ---- spatial denoiser (rt_set_spatial_denoiser) -------------------------------------------------------------------
// The guides of one pixel in one record: shading normal xyz and depth of the last frame's bounce-0 AOVs.
__global__ void __launch_bounds__(256) k_sd_pack(const float4* normal, const float* depth, float4* guide, uint32_t n)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 nn = normal[i];
    guide[i] = make_float4(nn.x, nn.y, nn.z, depth[i]);
}

__device__ __forceinline__ bool sd_finite(float4 c) { return isfinite(c.x) && isfinite(c.y) && isfinite(c.z); }
// a term of the distance: its difference times its factor, added only when both are positive (a sigma of 0 drops the term)
__device__ __forceinline__ float sd_term(float diff, float k) { return (k > 0.0f && diff > 0.0f) ? diff * k : 0.0f; }

// One a-trous pass (the rule is stated with rt_set_spatial_denoiser in rt_b200.h): 5x5 taps at spacing `step` around every pixel,
// B3-spline weights times rt_expf(-(colour + normal + depth distance)), taps outside the image skipped, taps of non-finite colour
// skipped; taps summed row by row, left to right.  One thread per pixel over 32x8 tiles; the taps are read through L1.
__global__ void __launch_bounds__(256) k_sd_pass(const float4* __restrict__ src, float4* __restrict__ dst, const float4* __restrict__ guide,
                                                 uint32_t width, uint32_t height, int step, float kc, float kn, float sigma_depth)
{
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= width || y >= height) return;
    const float h[5] = { 0.0625f, 0.25f, 0.375f, 0.25f, 0.0625f };
    const uint32_t p = y * width + x;
    const float4 cp = __ldg(&src[p]);
    const float4 gp = __ldg(&guide[p]);
    const bool cfin = sd_finite(cp);
    const float c0x = cfin ? cp.x : 0.0f, c0y = cfin ? cp.y : 0.0f, c0z = cfin ? cp.z : 0.0f;
    const float kcp = cfin ? kc : 0.0f;                        // a non-finite centre drops its colour term
    const float kz = sigma_depth > 0.0f ? 1.0f / (sigma_depth * gp.w) : 0.0f;
    float wsum = 0.0f, s0 = 0.0f, s1 = 0.0f, s2 = 0.0f;
#pragma unroll
    for (int ty = -2; ty <= 2; ++ty)
    {
        const int qy = (int)y + ty * step;
        if (qy < 0 || qy >= (int)height) continue;
#pragma unroll
        for (int tx = -2; tx <= 2; ++tx)
        {
            const int qx = (int)x + tx * step;
            if (qx < 0 || qx >= (int)width) continue;
            const uint32_t q = (uint32_t)qy * width + (uint32_t)qx;
            const float4 cq = __ldg(&src[q]);
            if (!sd_finite(cq)) continue;
            const float4 gq = __ldg(&guide[q]);
            const float dr = c0x - cq.x, dg = c0y - cq.y, db = c0z - cq.z;
            const float dc = (dr * dr + dg * dg) + db * db;
            const float nx = gp.x - gq.x, ny = gp.y - gq.y, nz = gp.z - gq.z;
            const float dn = (nx * nx + ny * ny) + nz * nz;
            const float dz = fabsf(gp.w - gq.w);
            float d = sd_term(dc, kcp);
            d = d + sd_term(dn, kn);
            d = d + sd_term(dz, kz);
            const float w = (h[ty + 2] * h[tx + 2]) * rt_expf(-d);
            if (w > 0.0f)
            {
                wsum = wsum + w;
                s0 = s0 + w * cq.x; s1 = s1 + w * cq.y; s2 = s2 + w * cq.z;
            }
        }
    }
    dst[p] = wsum > 0.0f ? make_float4(s0 / wsum, s1 / wsum, s2 / wsum, 1.0f) : make_float4(cp.x, cp.y, cp.z, 1.0f);
}

// ---- adaptive sampling (rt_set_adaptive_sampling) ----------------------------------------------------------------
struct AdaptiveState
{
    uint32_t* count;               // per local pixel: samples taken
    float* y_prev;                 // per local pixel: luma of the radiance sum at the previous update
    double* q;                     // per local pixel: sum of the squared per-sample luma increments
    uint32_t* list;                // the active local pixels, ascending (n_local entries)
    unsigned long long* tile;      // per tile of the update: (epoch << 2 | flag) << 32 | value, flag 1 aggregate, 2 inclusive prefix
    AdaptiveCtl* ctl;
};

#define RT_AD_THREADS 256
#define RT_AD_ITEMS 4
#define RT_AD_TILE (RT_AD_THREADS * RT_AD_ITEMS)

// rt_reset with the feature on: every local pixel active, in order; the per-pixel state is cleared by memsets beside this launch
__global__ void __launch_bounds__(256) k_adaptive_init(AdaptiveState st, uint32_t n_local)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_local) st.list[i] = i;
    if (i == 0) { st.ctl->n_active = n_local; st.ctl->n_next = 0; st.ctl->frames = 0; st.ctl->ticket = 0; st.ctl->done = 0; st.ctl->epoch = 1; }
}

// The convergence update after a sample: for every active pixel (now at n = frames + 1 samples) update the luma statistics and
// decide whether it stops (DESIGN.md section 4):
//     Y = luma(radiance), y = Y - Y_prev, Q += y^2, m = Y / n, v = max(Q / n - m^2, 0), e = sqrt(v / n) / (1 + m)^2,
//     stop iff n >= min_samples and e <= max_error            (double precision; NaN never stops)
// and compact the survivors into the same list, in place and ascending, in one pass.  Tile t = RT_AD_TILE consecutive list entries,
// taken in CTA arrival order (a ticket), so that the decoupled look-back over the tiles before t only waits on CTAs that are running.
// In place is safe: a tile publishes its count only after it has read its entries, and a survivor moves to an index no larger than
// its own.  The grid is sized by the partition (a captured frame graph replays it unchanged); tiles past the active count only take
// part in the completion count, whose last CTA moves the new count into n_active, advances frames and the epoch and re-arms the
// ticket (every CTA has read them by then).
__global__ void __launch_bounds__(RT_AD_THREADS) k_adaptive_update(const float4* radiance, AdaptiveState st, double max_error, uint32_t min_samples)
{
    __shared__ uint32_t s_t, s_n, s_frames, s_epoch, s_prefix;
    __shared__ uint32_t s_warp[RT_AD_THREADS / 32];
    if (threadIdx.x == 0)
    {
        volatile AdaptiveCtl* ctl = st.ctl;
        s_n = ctl->n_active; s_frames = ctl->frames; s_epoch = ctl->epoch;
        s_t = atomicAdd(&st.ctl->ticket, 1u);
    }
    __syncthreads();
    const uint32_t t = s_t, n_act = s_n;
    if ((size_t)t * RT_AD_TILE < n_act)
    {
        const uint32_t n = s_frames + 1u;
        const double dn = (double)n;
        const uint32_t first = t * RT_AD_TILE + threadIdx.x * RT_AD_ITEMS;
        uint32_t li[RT_AD_ITEMS];
        unsigned keep = 0u;
#pragma unroll
        for (int k = 0; k < RT_AD_ITEMS; ++k)
        {
            const uint32_t j = first + k;
            li[k] = 0;
            if (j >= n_act) continue;
            const uint32_t pix = st.list[j];
            li[k] = pix;
            const float Y = luma(mk3(radiance[pix]));
            const double y = (double)Y - (double)st.y_prev[pix];
            const double Q = st.q[pix] + y * y;
            st.q[pix] = Q; st.y_prev[pix] = Y; st.count[pix] = n;
            const double m = (double)Y / dn;
            double v = Q / dn - m * m;
            if (v < 0.0) v = 0.0;
            const double d = 1.0 + m;
            const double e = sqrt(v / dn) / (d * d);
            if (!(n >= min_samples && e <= max_error)) keep |= 1u << k;
        }
        // block-wide exclusive scan of the survivors, in list order
        const uint32_t mine = (uint32_t)__popc(keep);
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        uint32_t incl = mine;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += u; }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        if (warp == 0)
        {
            uint32_t agg = 0;
            if (lane == 0)
                for (int w = 0; w < RT_AD_THREADS / 32; ++w) { const uint32_t c = s_warp[w]; s_warp[w] = agg; agg += c; }
            agg = __shfl_sync(0xffffffffu, agg, 0);
            // decoupled look-back: publish the aggregate, then add up the tiles before this one, 32 at a time (lane k looks at tile
            // end - k), back to the nearest inclusive prefix
            const unsigned long long tag = (unsigned long long)(s_epoch << 2);
            volatile unsigned long long* tile = st.tile;
            if (lane == 0) tile[t] = ((tag | (t == 0 ? 2ull : 1ull)) << 32) | agg;
            uint32_t prefix = 0;
            for (int32_t end = (int32_t)t - 1; end >= 0; end -= 32)
            {
                const int32_t u = end - lane;
                unsigned long long w, flag;
                do
                {   // tiles before the first are an inclusive prefix of 0
                    w = 0ull; flag = 2ull;
                    if (u >= 0) { w = tile[u]; const unsigned long long wt = w >> 32; flag = (wt & ~3ull) == tag ? (wt & 3ull) : 0ull; }
                } while (__any_sync(0xffffffffu, flag == 0ull));                  // a tile has not published for this update yet
                const unsigned inc = __ballot_sync(0xffffffffu, flag == 2ull);
                const int last = inc ? __ffs(inc) - 1 : 31;
                uint32_t v = lane <= last ? (uint32_t)w : 0u;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
                prefix += v;
                if (inc) break;
            }
            if (lane == 0)
            {
                if (t > 0) tile[t] = ((tag | 2ull) << 32) | (prefix + agg);
                s_prefix = prefix;
                if ((size_t)(t + 1u) * RT_AD_TILE >= n_act) { st.ctl->n_next = prefix + agg; __threadfence(); }   // the last active tile
            }
        }
        __syncthreads();
        uint32_t at = s_prefix + s_warp[warp] + incl - mine;
#pragma unroll
        for (int k = 0; k < RT_AD_ITEMS; ++k)
            if (keep & (1u << k)) st.list[at++] = li[k];
    }
    if (threadIdx.x == 0)
    {
        __threadfence();
        if (atomicAdd(&st.ctl->done, 1u) == gridDim.x - 1u)
        {   // every CTA has finished: the next update and the next frame see the new state
            volatile AdaptiveCtl* ctl = st.ctl;
            ctl->n_active = n_act ? ctl->n_next : 0u;
            ctl->frames = s_frames + 1u;
            ctl->epoch = s_epoch % 0x3FFFFFFFu + 1u;
            ctl->ticket = 0; ctl->done = 0;
        }
    }
}

// ResolveRadiance of a gathered multi-GPU frame: pixel (x, y) lives in slab y % world at local row y / world
__global__ void __launch_bounds__(256) k_resolve_gathered(const float4* slabs, size_t stride_f4, float4* out, uint32_t width, uint32_t height,
                                                          uint32_t world, uint32_t sample_count)
{
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= width * height) return;
    uint32_t y = i / width, x = i - y * width;
    float4 r = slabs[(size_t)(y % world) * stride_f4 + (size_t)(y / world) * width + x];
    f3 hdr = mk3(r) / (float)sample_count;
    f3 ldr = hdr / (mk3(hdr.x + 1.0f, hdr.y + 1.0f, hdr.z + 1.0f));
    out[i] = make_float4(ldr.x, ldr.y, ldr.z, 1.0f);
}

// TemporalAccumulation, denoiser.cl:27-79 (single-GPU only: the reprojected pixel may be any pixel of the image)
__global__ void __launch_bounds__(256) k_temporal(uint32_t width, uint32_t height, float4* radiance, const float4* prev_radiance,
                                                  const float* depth, const float* prev_depth, const float2* velocity)
{
    uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= width * height) return;
    int x = (int)(idx % width), y = (int)(idx / width);
    float dv = depth[idx];
    if (dv == RT_MAX_RENDER_DIST) return;
    float2 mv = velocity[idx];
    float pu = ((float)x + 0.5f) / (float)width - mv.x;
    float pv = ((float)y + 0.5f) / (float)height - mv.y;
    float fx = pu * (float)width, fy = pv * (float)height;
    if (!(fx == fx) || !(fy == fy) || fabsf(fx) > 1.0e9f || fabsf(fy) > 1.0e9f) return;      // NaN / overflow: out of range
    int px = (int)fx, py = (int)fy;
    if (px < 0 || px >= (int)width || py < 0 || py >= (int)height) return;
    int pidx = py * (int)width + px;
    float pd = prev_depth[pidx];
    if (fabsf(dv - pd) / dv > 0.1f) return;
    float4 cur = radiance[idx], prev = prev_radiance[pidx];
    cur.x = cur.x + (prev.x - cur.x) * 0.9f; cur.y = cur.y + (prev.y - cur.y) * 0.9f; cur.z = cur.z + (prev.z - cur.z) * 0.9f;
    radiance[idx] = cur;
}

// Completion flags of the fused gather (one uint32 per rank, in the presenting device's memory, behind the slabs): a rank stores its
// frame number after its frame kernel has completed (stream order) — everything it pushed is then visible system-wide — and the
// presenting rank's stream waits until every flag has reached its own frame number.
__global__ void k_gather_signal(uint32_t* flag, uint32_t frame)
{
    __threadfence_system();
    *(volatile uint32_t*)flag = frame;
    __threadfence_system();
}
__global__ void k_gather_wait(const uint32_t* flags, uint32_t world, uint32_t frame)
{
    if (threadIdx.x < world)
        while ((int32_t)(*(volatile const uint32_t*)(flags + threadIdx.x) - frame) < 0) __nanosleep(200);
    __threadfence_system();
}

// rt_math_eval: the functions of include/rt_math.h evaluated on the device (parity tap: tests compare them bitwise with the
// same header compiled for the host)
__global__ void k_math_eval(int fn, const float* a, const float* b, float* out, uint64_t n)
{
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x = a[i], y = b[i];
    float r = 0.0f;
    switch (fn)
    {
    case 0: r = rt_sinf(x); break;
    case 1: r = rt_cosf(x); break;
    case 2: r = rt_tanf(x); break;
    case 3: r = rt_atan2f(x, y); break;
    case 4: r = rt_acosf(x); break;
    case 5: r = rt_powf(x, y); break;
    case 6: r = rt_fminf(x, y); break;
    case 7: r = rt_fmaxf(x, y); break;
    case 8: r = 1.0f / sqrtf(x); break;          // the normalize() building blocks: IEEE sqrt and division
    case 9: r = x / y; break;
    case 10: r = rt_expf(x); break;
    }
    out[i] = r;
}

// rt_integrate_samples on the per-frame path: the statistics of `frames` frames (added up in f by k_frame, or one per-phase frame)
// added into the call's sums (one CTA).  Every frame has f->n_primary primary rays (with adaptive sampling k_frame adds them up
// itself and frames is 1).
__global__ void __launch_bounds__(256) k_add_counters(DevCounters* sum, const DevCounters* f, uint32_t frames)
{
    for (uint32_t b = threadIdx.x; b <= RT_MAX_BOUNCES; b += blockDim.x)
    {
        sum->emit[b].shadow += f->emit[b].shadow; sum->emit[b].next += f->emit[b].next;
        sum->hm[b].hit += f->hm[b].hit; sum->hm[b].miss += f->hm[b].miss;
        sum->n_emissive[b] += f->n_emissive[b]; sum->n_unoccluded[b] += f->n_unoccluded[b];
        sum->nodes_ext[b] += f->nodes_ext[b]; sum->tris_ext[b] += f->tris_ext[b];
        sum->nodes_shadow[b] += f->nodes_shadow[b]; sum->tris_shadow[b] += f->tris_shadow[b];
    }
    if (threadIdx.x == 0) sum->n_primary += f->n_primary * frames;
}

__global__ void k_unpack_rays(const float4* A, const float4* B, const uint32_t* count, uint32_t width, RtRay* rays, uint32_t* pixels)
{
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= *count) return;
    float4 a = A[i], b = B[i];
    rays[i].origin = RtFloat3{ a.x, a.y, a.z, 0.0f };
    rays[i].direction = RtFloat3{ b.x, b.y, b.z, RT_MAX_RENDER_DIST };      // every extension ray's t_max
    uint32_t pxy = __float_as_uint(b.w);
    pixels[i] = (pxy >> 16) * width + (pxy & 0xFFFFu);
}

} // namespace

// ====================================================================================== host side
struct rt_ctx
{
    int device = 0;
    // A multi-device context (rt_create_multi) owns no device memory itself: it holds one child context per device (child i
    // renders rank i of an n-way scanline partition) and every call on it fans out to the children from the caller's thread.
    std::vector<rt_ctx*> children;
    int present = 0;                               // RT_OPT_PRESENT (groups): 0 parallel read-back, 1 gather to device 0 over NVLink
    float4* gather_buf = nullptr; size_t gather_stride_f4 = 0;   // device 0: the gathered radiance slabs (rt_gather_radiance)
    std::vector<Owned<cudaEvent_t>> gather_events;
    uint32_t width = 0, height = 0, rank = 0, world = 1, n_local = 0, local_rows = 0;
    Owned<cudaStream_t> stream;
    int num_sms = 0;
    std::string error;

    // options
    int white_furnace = 0, sampler = 0, aov = 0, denoiser = 0, count_traversal = 0, kernel_timing = 0, traversal = 1, smem_bvh = 1, octant_bvh = 1;
    uint32_t top_smem_records = 0;                 // RT_OPT_TOP_SMEM

    // per-pixel buffers
    Queues q = {};
    float4* radiance = nullptr;
    float4* resolved = nullptr;
    // whole-frame CUDA graph (RT_OPT_GRAPH): rt_integrate replays the captured launch sequence; only k_set_frame's
    // by-value argument (sample index, camera constants) is updated per frame
    int use_graph = 1;
    uint64_t config_gen = 1, graph_gen = 0;     // config_gen changes whenever a launch argument other than FrameDyn may change
    uint32_t graph_max_bounces = 0;
    Owned<cudaGraph_t> graph;                   // kept alive: node handles used for parameter updates belong to it
    Owned<cudaGraphExec_t> graph_exec;
    cudaGraphNode_t graph_set_frame_node = nullptr;
    void* graph_set_frame_func = nullptr;
    uint64_t graph_launches = 0;
    // shadow pass on a second stream (RT_OPT_OVERLAP): k_shadow_accumulate(b) runs concurrently with k_trace_closest(b+1)
    int overlap = 2;               // RT_OPT_OVERLAP
    bool shadow_deferred = false;  // overlap 2: rt_shadow_accumulate(shadow_deferred_bounce) has been requested but not launched yet
    uint32_t shadow_deferred_bounce = 0;
    Owned<cudaStream_t> shadow_stream;
    Owned<cudaEvent_t> ev_shaded, ev_shadowed;
    bool shadow_pending = false;
    // pipelined read-back (rt_resolve_async): second resolve buffer, copy stream, events
    float4* resolved2 = nullptr;
    float4* resolved_full[2] = { nullptr, nullptr };   // whole-frame resolve targets of rt_resolve_gathered
    Owned<cudaStream_t> copy_stream;
    Owned<cudaEvent_t> resolve_done[2], copy_done[2];
    bool copy_pending[2] = { false, false };
    uint32_t async_index = 0;
    // AOV + denoiser buffers (allocated on first use)
    float4* aov_albedo = nullptr; float* aov_depth = nullptr; float4* aov_normal = nullptr; float2* aov_velocity = nullptr;
    float4* prev_radiance = nullptr; float* prev_depth = nullptr;
    int aov_always = 0;
    RtCamera prev_camera = {}, aov_prev_camera = {};
    DevCounters* counters = nullptr;
    DevCounters* counters_sum = nullptr;           // rt_integrate_samples: the statistics summed over the call's samples
    bool stats_summed = false;                     // rt_read_frame_stats reads counters_sum (after rt_integrate_samples) instead of counters
    FrameDyn* d_dyn = nullptr;
    bool pdl = true;               // RT_OPT_PDL
    int frame_kernel = 2;          // RT_OPT_FRAME_KERNEL: 1 rt_integrate launches ONE persistent kernel per frame (k_frame), 0 one kernel per phase, 2 by partition size
    // fused gather (rt_set_gather_target): this rank's slab and flag in the presenting device's memory, frames signalled so far
    float4* gather_slab = nullptr; uint32_t* gather_flag = nullptr; uint32_t gather_frame = 0;
    uint32_t gather_sample = 0xFFFFFFFFu;          // sample_count after the last frame that was pushed
    char* own_gather = nullptr; size_t own_gather_stride = 0;      // the buffer this context allocated (rt_gather_buffer)
    int grid_div = 1;              // contexts that share this device (rt_create_multi lists a device k times): each launches 1/k of the resident CTAs
    int frame_threads = 0;         // RT_OPT_FRAME_THREADS: threads per CTA of k_frame (0 = by partition size)
    size_t n_alloc = 0;            // entries of every per-pixel queue: n_local + one group of 32 per CTA that can be resident (k_frame's regions)
    int* d_bn = nullptr;           // sobol | scrambling | ranking (rt_upload_sampler_tables)
    struct Occupancy { const void* kernel; int threads; size_t smem; int per_sm; };
    std::vector<Occupancy> occupancy;   // resident CTAs per SM of each persistent kernel (resident_per_sm)
    char* scratch = nullptr; size_t scratch_bytes = 0;

    // scene
    bool scene_ready = false, camera_ready = false;
    DevScene scene = {};
    float4 scene_mid = {};                         // centre of the root box: the origin half of k_shade_queues' sort key
    uint64_t n_tris = 0, n_nodes = 0;              // counts of the upload
    // geometry updates (rt_update_triangles): the refit map (built at the first update, freed by the next upload) and the host
    // variant's staging, two halves of pinned and of device memory (allocated at the first host update)
    uint2* refit_link = nullptr; uint32_t* refit_leaves = nullptr; uint32_t* refit_arrivals = nullptr; uint32_t refit_n_leaves = 0;
    struct Staging { DevAllocs mem; char* host = nullptr; char* dev = nullptr; size_t half = 0; Owned<cudaEvent_t> copied[2]; };
    bool emit_moved = false;                       // emit_tris' positions predate an update: refresh_lights reads them from tris_ref
    // object motion (RT_OPT_OBJECT_MOTION): the previous positions, tris_ref's layout, in motion_mem while the option is on and a
    // scene is uploaded
    int object_motion = 0;
    float4* prev_pos = nullptr;
    // rt_rebuild_bvh: the build temporaries of the linear BVH (allocated with its nodes and records at the first rebuild after an
    // upload, in tree_mem; live = scene.nodes_ref / wnodes and the refit map hold a rebuilt tree's 2n - 1 nodes)
    struct Lbvh
    {
        bool live = false;
        uint32_t* bounds = nullptr;                // 6 words: the key-point box of k_lbvh_bounds
        uint32_t* codes[2] = { nullptr, nullptr }; uint32_t* ids[2] = { nullptr, nullptr };   // the sort's double buffers
        uint4* inner = nullptr;                    // per internal node: first leaf, last leaf, split, axis
        uint2* top = nullptr;                      // the breadth-first top records by preorder (k_lbvh_top)
        char* sort_tmp = nullptr; size_t sort_bytes = 0;
        // rt_rebuild_bvh_ploc's clustering temporaries (allocated at its first call, in tree_mem; clusters = null before)
        struct Ploc
        {
            PlocCluster* clusters = nullptr;       // 2 x n: the list and the compaction's output
            uint32_t* nn = nullptr; uint8_t* keep = nullptr;                  // per position
            uint4* inner = nullptr; uint32_t* size = nullptr;                 // per interior node (k_ploc_merge)
            uint32_t* parent = nullptr;            // per node reference
            uint32_t* made = nullptr;              // device word: interior nodes allocated so far
            uint32_t* host = nullptr;              // pinned: [0] the compaction's count, [1] the depth flag of k_ploc_number
            char* select_tmp = nullptr; size_t select_bytes = 0;
        } ploc;
    } lbvh;
    RtCamera camera = {};
    RayGenConsts raygen = {};
    // instanced scene (rt_upload_instanced_scene): the meshes and the instance buffer in inst_mem, sized for inst_cap instances:
    // header (2 float4), top-level records, instance records (8 float4 each), previous M rows (3 float4 each), bases (uint32)
    bool instanced = false;
    std::vector<rtinst::MeshInfo> meshes;
    uint32_t inst_cap = 0, n_inst = 0;
    std::vector<float> inst_last;                  // per instance index ever listed since the upload: its transform in the last
                                                   // list that had it, 12 floats each (the previous transforms of object motion)
    std::vector<float4> inst_host;                 // the image of the instance buffer the last rt_set_instances copied
    float4 *inst_hdr = nullptr, *inst_top = nullptr, *inst_rec = nullptr, *inst_prev = nullptr;
    uint32_t* inst_base = nullptr;
    std::vector<RtInstance> inst_list;             // the list of the last rt_set_instances (rt_update_mesh_triangles rebuilds its tree)
    // rt_update_mesh_triangles: per mesh, its node count and its refit map (built at the mesh's first update, in tree_mem; node
    // and record indices relative to the mesh's own arrays), and the device variant's check flag (one word, in tree_mem)
    struct MeshRefit { uint64_t n_nodes = 0; uint2* link = nullptr; uint32_t* leaves = nullptr; uint32_t* arrivals = nullptr; uint32_t n_leaves = 0; };
    std::vector<MeshRefit> mesh_refit;
    uint32_t* mesh_bad = nullptr;
    // rt_set_instance_materials: the upload's material count, the assignment kept per instance index (row offset r * n_materials,
    // or RT_INVALID_ID), the remap table in mtl_mem (mtl_cap entries; grows to at least twice its size) and its host image
    uint64_t n_materials = 0;
    std::vector<uint32_t> inst_mtl_row;
    uint32_t* mtl_map = nullptr;
    size_t mtl_cap = 0;
    std::vector<uint32_t> mtl_host;

    // adaptive sampling (rt_set_adaptive_sampling): the requested setting, which rt_reset makes the active one; max_error > 0 = on.
    // The per-pixel state exists only while the active setting is on.
    float ad_req_error = 0.0f; uint32_t ad_req_min = 0;
    float ad_error = 0.0f; uint32_t ad_min = 0;
    AdaptiveState ad = {};
    bool ad_fresh = false;                         // no frame has run since the adaptive state was reset (every local pixel traces the next)

    // emitter sampling (RT_OPT_EMITTER_SAMPLING): the upload's emitter list and what the table needs of it (kept so that the option can be
    // turned on after the upload), the device table (scene.emit_*, allocated while the option is on and P_e > 0)
    int emitter_sampling = 0;
    uint32_t emit_max_bounces = RT_MAX_BOUNCES;    // FrameDyn::max_bounces: the max_bounces of the last rt_integrate[_samples] call
    std::vector<uint32_t> emit_idx;
    std::vector<RtTriangle> emit_tris;             // emit_tris[i]: triangle emit_idx[i] (zero where the index is out of range)
    std::vector<RtPackedMaterial> emit_mats;
    std::vector<RtLight> emit_lights;
    uint64_t emit_n_tris = 0;
    // environment sampling (RT_OPT_ENV_SAMPLING, its table scene.env_* built from the device image) and the light-kind weights
    // (rt_set_light_selection; analytic_lit: an analytic light of the upload has non-zero radiance)
    int env_sampling = 0;
    float light_w[3] = { 1.0f, 1.0f, 1.0f };
    bool analytic_lit = false;

    // spatial denoiser (rt_set_spatial_denoiser): passes (0 = off), sigmas, scratch planes (allocated while it is on)
    uint32_t sd_iters = 0;
    float sd_sigma_c = 0.0f, sd_sigma_n = 0.0f, sd_sigma_z = 0.0f;
    float4* sd_col[2] = { nullptr, nullptr };
    float4* sd_guide = nullptr;
    bool aov_ready = false;                        // the AOV buffers hold the last frame's bounce-0 guides for every local pixel

    uint32_t sample_count = 0;
    uint32_t cur_bounce = 0;
    bool frame_started = false;
    bool primary_fused = false;    // the frame was begun without k_raygen: rt_extend_shade(0) generates its primary rays (k_trace_primary)
    uint64_t launches = 0;

    // kernel timing
    struct Timed { Owned<cudaEvent_t> a, b; int cls; };
    std::vector<Timed> timed;
    std::vector<Owned<cudaEvent_t>> event_pool;
    float ms[RT_K_CLASS_COUNT] = {};
    uint32_t nlaunch[RT_K_CLASS_COUNT] = {};

    // The device memory, one group per lifetime.  Declared last, so freed before the streams and events that order work on it.
    DevAllocs ctx_mem;             // counters, counters_sum, d_dyn, d_bn, resolved_full: the context's
    DevAllocs scratch_mem;         // scratch, replaced when it has to grow
    DevAllocs gather_mem;          // own_gather (rt_gather_buffer), or a multi-device context's gather_buf
    DevAllocs frame_mem;           // q, radiance, resolved, resolved2: the partition's
    DevAllocs aov_mem;             // aov_*, prev_radiance, prev_depth: from the first use to the next partition
    DevAllocs sd_mem;              // sd_col, sd_guide: while the spatial denoiser is on
    DevAllocs ad_mem;              // ad: while adaptive sampling is on
    DevAllocs scene_mem;           // the upload's arrays but the tree
    DevAllocs tree_mem;            // scene.nodes_ref, scene.wnodes, the refit map, lbvh's temporaries (the clustering's included)
    Staging stage;                 // rt_update_triangles' staging
    DevAllocs light_mem;           // the emitter and environment tables
    DevAllocs motion_mem;          // prev_pos: while object motion is on and a scene is uploaded
    DevAllocs inst_mem;            // the instance buffer of an instanced scene
    DevAllocs mtl_mem;             // mtl_map (rt_set_instance_materials): from the first assignment that needs it to the next upload
    std::vector<std::unique_ptr<void, IpcClose>> ipc_opened;
};

static std::string g_create_error;

#define RT_FAIL(ctx, code, ...)                                   \
    do {                                                          \
        char rt_buf_[512];                                        \
        snprintf(rt_buf_, sizeof(rt_buf_), __VA_ARGS__);          \
        (ctx)->error = rt_buf_;                                   \
        return (code);                                            \
    } while (0)

#define RT_CUDA(ctx, expr)                                                                         \
    do {                                                                                           \
        cudaError_t rt_e_ = (expr);                                                                \
        if (rt_e_ != cudaSuccess)                                                                  \
            RT_FAIL(ctx, RT_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(rt_e_), __FILE__, __LINE__); \
    } while (0)

#define RT_CHECK_CTX(ctx) do { if (!(ctx)) return RT_ERR_INVALID_ARGUMENT; } while (0)

// Multi-device contexts: forward the call to every child (variable `k`), in rank order, from the caller's thread.  Kernel
// launches and copies are asynchronous, so the devices work concurrently; the first failing child's message is kept.
#define RT_FANOUT(ctx, call)                                                             \
    do {                                                                                 \
        if (!(ctx)->children.empty())                                                    \
        {                                                                                \
            for (rt_ctx* k : (ctx)->children)                                            \
            {                                                                            \
                int rt_frc_ = (call);                                                    \
                if (rt_frc_ != RT_OK) { (ctx)->error = k->error; return rt_frc_; }       \
            }                                                                            \
            return RT_OK;                                                                \
        }                                                                                \
    } while (0)
#define RT_NOT_ON_GROUP(ctx, what)                                                       \
    do { if (!(ctx)->children.empty()) RT_FAIL(ctx, RT_ERR_UNSUPPORTED, what " is a single-device call: use it on a context of rt_create"); } while (0)

struct rt_ctx;
extern "C" {   // defined with rt_shadow_accumulate
static int launch_shadow_pass(rt_ctx* c, uint32_t bounce, cudaStream_t st);
}

namespace
{

struct TimedLaunch
{
    rt_ctx* c; int cls; Owned<cudaEvent_t> a, b; cudaStream_t st;
    TimedLaunch(rt_ctx* ctx, int k, cudaStream_t stream = nullptr) : c(ctx), cls(k), st(stream ? stream : ctx->stream)
    {
        ++c->launches;
        if (!c->kernel_timing) return;
        auto get = [&](Owned<cudaEvent_t>& e) { if (!c->event_pool.empty()) { e = std::move(c->event_pool.back()); c->event_pool.pop_back(); } else make_event(e, cudaEventDefault); };
        get(a); get(b);
        cudaEventRecord(a, st);
    }
    ~TimedLaunch()
    {
        if (!a) return;
        cudaEventRecord(b, st);
        c->timed.push_back({ std::move(a), std::move(b), cls });
    }
};

inline dim3 grid_for(uint32_t n, uint32_t block = 256) { uint32_t g = (n + block - 1) / block; return dim3(g ? g : 1u); }   // n = 0: one idle block

// Work submitted to the shadow stream must be ordered before anything on the render stream that touches the radiance
// buffer, the shadow queue or the counters again.
int join_shadow(rt_ctx* c)
{
    // callers reach this before their own cudaSetDevice; with several devices in one process (rt_create_multi) the current device
    // may be another context's
    if (c->shadow_deferred || c->shadow_pending) RT_CUDA(c, cudaSetDevice(c->device));
    if (c->shadow_deferred)
    {   // nobody merged the deferred shadow pass into a traversal kernel: it runs on its own, in stream order
        c->shadow_deferred = false;
        int rc = launch_shadow_pass(c, c->shadow_deferred_bounce, c->stream); if (rc) return rc;
    }
    if (c->shadow_pending)
    {
        RT_CUDA(c, cudaStreamWaitEvent(c->stream, c->ev_shadowed, 0));
        c->shadow_pending = false;
    }
    return RT_OK;
}

int post_launch(rt_ctx* c, const char* what)
{
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) RT_FAIL(c, RT_ERR_CUDA, "launch of %s failed: %s", what, cudaGetErrorString(e));
    return RT_OK;
}

bool adaptive_on(const rt_ctx* c);

FrameParams frame_params(const rt_ctx* c)
{
    FrameParams p;
    p.width = c->width; p.height = c->height; p.rank = c->rank; p.world = c->world; p.n_local = c->n_local;
    p.white_furnace = c->white_furnace; p.bn = c->sampler ? c->d_bn : nullptr; p.dyn = c->d_dyn;
    p.gather = nullptr;            // set by the one-kernel frame's launch only
    p.active = adaptive_on(c) ? c->ad.list : nullptr;
    p.n_active = adaptive_on(c) ? &c->ad.ctl->n_active : nullptr;
    return p;
}

// The frame group exists unless the last rt_set_partition could not allocate it.
int frame_buffers_ready(rt_ctx* c)
{
    if (!c->radiance) RT_FAIL(c, RT_ERR_NOT_READY, "frame buffers could not be allocated: call rt_set_partition again");
    return RT_OK;
}

int require_ready(rt_ctx* c)
{
    if (!c->scene_ready) RT_FAIL(c, RT_ERR_NOT_READY, "rt_upload_scene has not been called");
    if (!c->camera_ready) RT_FAIL(c, RT_ERR_NOT_READY, "rt_set_camera has not been called");
    return frame_buffers_ready(c);
}

bool aov_wanted(const rt_ctx* c);
int ensure_aov_buffers(rt_ctx* c);

// ---- adaptive sampling: the active setting is on / either setting is on (what the refused combinations check)
bool adaptive_on(const rt_ctx* c) { return c->ad_error > 0.0f; }
bool adaptive_wanted(const rt_ctx* c) { return c->ad_error > 0.0f || c->ad_req_error > 0.0f; }
uint32_t adaptive_tiles(const rt_ctx* c) { return std::max((c->n_local + RT_AD_TILE - 1u) / RT_AD_TILE, 1u); }

// The per-pixel state for the current partition (allocated on first use) reset to: every local pixel active, counts and
// estimators zero.
int reset_adaptive(rt_ctx* c)
{
    const size_t n = std::max(c->n_local, 1u), tiles = adaptive_tiles(c);
    if (!c->ad.count)
    {
        ++c->config_gen;
        DevAllocs g;
        AdaptiveState a = {};
        cudaError_t e;
        if ((e = g.alloc(a.count, n)) || (e = g.alloc(a.y_prev, n)) || (e = g.alloc(a.q, n)) || (e = g.alloc(a.list, n)) ||
            (e = g.alloc(a.tile, tiles)) || (e = g.alloc(a.ctl, 1)))
        {   // the frames run with the feature off until a later rt_reset succeeds (the requested setting stays)
            c->ad_error = 0.0f; c->ad_min = 0;
            RT_FAIL(c, RT_ERR_CUDA, "allocating the adaptive-sampling state failed: %s", cudaGetErrorString(e));
        }
        c->ad_mem = std::move(g); c->ad = a;
    }
    RT_CUDA(c, cudaMemsetAsync(c->ad.count, 0, n * 4, c->stream)); RT_CUDA(c, cudaMemsetAsync(c->ad.y_prev, 0, n * 4, c->stream));
    RT_CUDA(c, cudaMemsetAsync(c->ad.q, 0, n * 8, c->stream)); RT_CUDA(c, cudaMemsetAsync(c->ad.tile, 0, tiles * 8, c->stream));
    c->ad_fresh = true;
    TimedLaunch t(c, RT_K_MISC);
    k_adaptive_init<<<grid_for(c->n_local), 256, 0, c->stream>>>(c->ad, c->n_local);
    return post_launch(c, "k_adaptive_init");
}

// the convergence update that closes a sample (rt_advance_sample_count, after k_frame, and a node of the per-phase frame graph)
int launch_adaptive_update(rt_ctx* c)
{
    TimedLaunch t(c, RT_K_MISC);
    k_adaptive_update<<<adaptive_tiles(c), RT_AD_THREADS, 0, c->stream>>>(c->radiance, c->ad, (double)c->ad_error, c->ad_min);
    return post_launch(c, "k_adaptive_update");
}

int alloc_frame_buffers(rt_ctx* c)
{
    if (c->stream) cudaStreamSynchronize(c->stream);
    if (c->shadow_stream) cudaStreamSynchronize(c->shadow_stream);
    if (c->copy_stream) cudaStreamSynchronize(c->copy_stream); // a pipelined read-back may still be reading the resolve buffers
    c->shadow_pending = false; c->shadow_deferred = false;     // the frame in flight (if any) is abandoned with its buffers
    ++c->config_gen;
    // the per-pixel buffers go before the new ones are allocated, so that the peak does not hold both
    c->frame_mem.clear(); c->sd_mem.clear(); c->aov_mem.clear(); c->ad_mem.clear();
    c->q = {}; c->radiance = c->resolved = c->resolved2 = nullptr; c->sd_col[0] = c->sd_col[1] = c->sd_guide = nullptr;
    c->aov_albedo = c->aov_normal = c->prev_radiance = nullptr; c->aov_depth = c->prev_depth = nullptr; c->aov_velocity = nullptr;
    c->ad = {}; c->aov_ready = false;
    c->local_rows = (c->height > c->rank) ? (c->height - c->rank + c->world - 1) / c->world : 0;
    c->n_local = c->local_rows * c->width;
    // k_frame gives every resident CTA its own region of each queue, rounded up to whole groups of 32 slots
    size_t n = (size_t)c->n_local + 32u + (size_t)c->num_sms * 32u * 32u;       // up to 32 resident CTAs per SM
    c->n_alloc = n;
    DevAllocs g;
    Queues q = {};
    float4 *radiance = nullptr, *resolved = nullptr;
    cudaError_t e = cudaSuccess;
    auto get = [&](auto*& view) { if (e == cudaSuccess) e = g.alloc(view, n); };
    for (int i = 0; i < 2; ++i) { get(q.A.p[i]); get(q.B.p[i]); get(q.C.p[i]); }
    get(q.sA); get(q.sB); get(q.sC); get(q.hits); get(q.shadow_flags); get(q.hitq); get(q.missq); get(radiance); get(resolved);
    if (e != cudaSuccess) RT_FAIL(c, RT_ERR_CUDA, "allocating the frame buffers failed: %s", cudaGetErrorString(e));
    c->frame_mem = std::move(g); c->q = q; c->radiance = radiance; c->resolved = resolved;
    RT_CUDA(c, cudaMemsetAsync(c->radiance, 0, n * 16, c->stream));
    c->copy_pending[0] = c->copy_pending[1] = false;          // both streams were drained above
    if (adaptive_on(c)) { int rc = reset_adaptive(c); if (rc) return rc; }   // every pixel of the new partition active again
    if (aov_wanted(c)) return ensure_aov_buffers(c);           // a selected view / the denoiser keeps its buffers across a re-partition
    return RT_OK;
}

// Grid of a persistent kernel: exactly the CTAs that are resident at once (occupancy x SMs) — CTAs of a second wave
// would only start, find the cursor exhausted and exit — and no more CTAs than there can be work for (a rank of a
// multi-GPU partition owns few pixels).  Measured: -1.4 % frame time on one GPU, -5 % on a 1/8 partition.
// resident CTAs per SM of a kernel at a launch shape, looked up once per context
int resident_per_sm(rt_ctx* c, const void* kernel, int threads, size_t smem)
{
    for (auto& e : c->occupancy) if (e.kernel == kernel && e.threads == threads && e.smem == smem) return e.per_sm;
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
    c->occupancy.push_back({ kernel, threads, smem, per_sm });
    return per_sm;
}

int persistent_grid(rt_ctx* c, const void* kernel, size_t dyn_smem)
{
    int g = c->num_sms * resident_per_sm(c, kernel, 256, dyn_smem) / c->grid_div;
    if (g < c->num_sms) g = c->num_sms;
    int need = (int)((c->n_local + 255u) / 256u);
    if (need < 1) need = 1;
    return g < need ? g : need;
}
#define RT_PGRID(c, kern, smem) persistent_grid(c, (const void*)(kern), smem)

// Does k_shade_queues write its continuation rays sorted by ray_key?  Measured on an H100 (DESIGN.md section 4): the sorted order
// makes the next traversal 2-12 % faster, but the staging costs the shading pass more than that on a 1080p frame per GPU (15.7 K
// pixels per SM on 132 SMs) and wins on a 4K frame (62.8 K): sorted above 32 K pixels per SM (a variant built with
// -DRT_SORT_MIN_PIXELS_PER_SM=0 sorts at every size, tools/coherence_probe.py).
#ifndef RT_SORT_MIN_PIXELS_PER_SM
#define RT_SORT_MIN_PIXELS_PER_SM 32768u
#endif
bool sorted_shading(const rt_ctx* c) { return (uint64_t)c->n_local > (uint64_t)RT_SORT_MIN_PIXELS_PER_SM * (uint32_t)c->num_sms; }

// Can the traversal kernel of the next bounce also run a deferred shadow pass (k_trace_both)?
bool merged_trace_available(const rt_ctx* c) { return !c->count_traversal && !c->kernel_timing; }

// <<<grid, 256, smem, stream>>> with the programmatic-dependent-launch attribute when RT_OPT_PDL is on
template <class... KArgs, class... Args>
cudaError_t launch_chain(rt_ctx* c, void (*kernel)(KArgs...), int grid, size_t smem, cudaStream_t stream, Args... args)
{
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)grid); cfg.blockDim = dim3(256); cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr.val.programmaticStreamSerializationAllowed = 1;
    if (c->pdl && !c->kernel_timing) { cfg.attrs = &attr; cfg.numAttrs = 1; }
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// How a traversal kernel stages the BVH (TMA bulk copies into dynamic shared memory), decided per launch:
//   mode 1  the whole structure (interior records + triangle records) when it fits 40 KB (5 resident CTAs x 40 KB stay under
//           the 227 KB of an SM);
//   mode 3  mode 1 plus the eight 4-wide octant tables that every CTA builds from the staged records (rt_octant.h; each at
//           most the 64 bytes per record reserved here) and a flag word, when all of it fits the same 40 KB
//           (RT_OPT_OCTANT_BVH, default on): CornellBox, 2.6 KB + 8.7 KB;
//   mode 2  only the top of the tree — the first top_k interior records in breadth-first order (RT_OPT_TOP_SMEM records,
//           default 0 = off, DESIGN.md section 4 says why) — when the structure does not fit;
//   mode 0  nothing staged: literal traversal (RT_OPT_TRAVERSAL 0), RT_OPT_SMEM_BVH off.
struct Stage { int mode; size_t bytes; uint32_t top_k; };
// octant = false: the one-kernel frame (k_frame) stays on mode 1 — at its 64 registers the second traversal loop
// that mode 3 needs for the guarded rays spills inside the frame loop (measured: CornellBox on rank 0 of 4, 0.761 -> 0.811 ms).
Stage bvh_stage(const rt_ctx* c, bool octant = true)
{
    Stage st = { 0, 0, 0 };
    if (!c->smem_bvh || c->traversal != 1 || c->instanced) return st;
    size_t bytes = ((size_t)c->scene.wnodes_f4 + c->scene.wtris_f4) * 16;
    const size_t oct_bytes = bytes + 8 * (size_t)c->scene.wnodes_f4 * 16 + 16;
    if (octant && c->octant_bvh && oct_bytes <= 40 * 1024) { st.mode = 3; st.bytes = oct_bytes; return st; }
    if (bytes <= 40 * 1024) { st.mode = 1; st.bytes = bytes; return st; }
    uint32_t k = c->top_smem_records < c->scene.top_n ? c->top_smem_records : c->scene.top_n;
    if (k >= 8) { st.mode = 2; st.bytes = (size_t)k * 64; st.top_k = k; }
    return st;
}

// The kernel argument of an instanced scene's kernels
DevInstScene inst_scene(const rt_ctx* c)
{
    DevInstScene s;
    static_cast<DevScene&>(s) = c->scene;
    s.inst_hdr = c->inst_hdr; s.top = c->inst_top; s.irec = c->inst_rec; s.ibase = c->inst_base;
    s.prev_tri = c->prev_pos;
    s.mtl_map = c->mtl_map;
    return s;
}

// Calls f(INST, scene) with the context's scene as a kernel argument: (std::true_type, inst_scene(c)) or (std::false_type,
// c->scene), the latter always when the caller's kernels have no instanced variant (HAS_INST false).
template <bool HAS_INST = true, class F>
auto with_scene(const rt_ctx* c, F&& f)
{
    if constexpr (HAS_INST) if (c->instanced) return f(std::true_type(), inst_scene(c));
    return f(std::false_type(), c->scene);
}

// The traversal kernel families and the variants each is instantiated for (COUNT: RT_OPT_COUNT_TRAVERSAL, which stages nothing):
//   PER_PHASE  k_trace_closest, k_trace_primary, k_shadow_accumulate: staging modes 0-3 and RT_SMEM_INST, COUNT on 0 and INST;
//   MERGED     k_trace_both: modes 0-3 and RT_SMEM_INST, no COUNT (merged_trace_available);
//   STEPWISE   k_intersect, k_intersect_shadow: 0 and RT_SMEM_INST, COUNT on both;
//   FRAME      k_frame: modes 0-2 (bvh_stage without the octant tables) on flat scenes, no COUNT.
enum Family { PER_PHASE, MERGED, STEPWISE, FRAME };

// Launches a traversal kernel of family F: calls launch(COUNT, SMEM, scene, dynamic shared-memory bytes) once with this launch's
// COUNT (std::bool_constant) and staging mode SMEM (std::integral_constant), and the DevScene with its top_k or the DevInstScene;
// returns launch's result.  At most 40 KB are staged, under the 48 KB that every kernel may take without raising its limit.
template <Family F, class L>
auto launch_traversal(const rt_ctx* c, L&& launch)
{
    return with_scene<F != FRAME>(c, [&](auto inst, auto sc) {
        using Unstaged = std::integral_constant<int, inst.value ? RT_SMEM_INST : 0>;
        if constexpr (F == PER_PHASE || F == STEPWISE) if (c->count_traversal) return launch(std::true_type(), Unstaged(), sc, (size_t)0);
        constexpr int MAX_MODE = inst.value || F == STEPWISE ? 0 : F == FRAME ? 2 : 3;
        const Stage sg = MAX_MODE ? bvh_stage(c, MAX_MODE == 3) : Stage{ 0, 0, 0 };
        sc.top_k = sg.top_k;
        if constexpr (MAX_MODE >= 1) if (sg.mode == 1) return launch(std::false_type(), std::integral_constant<int, 1>(), sc, sg.bytes);
        if constexpr (MAX_MODE >= 2) if (sg.mode == 2) return launch(std::false_type(), std::integral_constant<int, 2>(), sc, sg.bytes);
        if constexpr (MAX_MODE >= 3) if (sg.mode == 3) return launch(std::false_type(), std::integral_constant<int, 3>(), sc, sg.bytes);
        return launch(std::false_type(), Unstaged(), sc, (size_t)0);
    });
}

AovCam aov_cam(const RtCamera& cam);

FrameDyn frame_dyn(const rt_ctx* c)
{
    FrameDyn dyn;
    memset(&dyn, 0, sizeof(dyn));
    dyn.sample_idx = c->sample_count; dyn.max_bounces = c->emit_max_bounces; dyn.raygen = c->raygen;
    dyn.cam = aov_cam(c->camera); dyn.prev = aov_cam(c->aov_prev_camera);
    return dyn;
}

bool aov_wanted(const rt_ctx* c) { return c->aov != 0 || c->denoiser != 0 || c->aov_always != 0 || c->sd_iters != 0; }

// A frame starts: its bounce-0 pass writes the AOVs of the pixels it traces.  They hold a complete set of guides (aov_ready) after a
// frame with AOVs on in which every local pixel traced — with adaptive sampling, the first frame after a reset; later frames keep
// them complete, since a stopped pixel keeps its AOVs — until a frame runs with them off.
void note_frame_aovs(rt_ctx* c)
{
    if (!(aov_wanted(c) && c->aov_albedo)) c->aov_ready = false;
    else if (!adaptive_on(c) || c->ad_fresh) c->aov_ready = true;
    c->ad_fresh = false;
}

AovCam aov_cam(const RtCamera& cam)
{
    AovCam a;
    a.position = f3{ cam.position.x, cam.position.y, cam.position.z };
    a.front = f3{ cam.front.x, cam.front.y, cam.front.z };
    a.up = f3{ cam.up.x, cam.up.y, cam.up.z };
    a.right = f3{ a.front.y * a.up.z - a.front.z * a.up.y, a.front.z * a.up.x - a.front.x * a.up.z, a.front.x * a.up.y - a.front.y * a.up.x };
    a.angle = rt_tanf(0.5f * cam.fov);          // aov.cl:35
    a.aspect_ratio = cam.aspect_ratio;
    return a;
}

AovParams aov_params(const rt_ctx* c)
{
    AovParams a;
    memset(&a, 0, sizeof(a));
    a.enabled = (aov_wanted(c) && c->aov_albedo) ? 1 : 0;
    a.albedo = c->aov_albedo; a.depth = c->aov_depth; a.normal = c->aov_normal; a.velocity = c->aov_velocity;
    a.prev_pos = c->instanced ? (c->object_motion ? c->inst_prev : nullptr) : c->prev_pos;
    return a;
}

int ensure_aov_buffers(rt_ctx* c)
{
    if (c->aov_albedo) return RT_OK;
    ++c->config_gen;
    c->aov_ready = false;
    size_t n = c->n_local ? c->n_local : 1;
    DevAllocs g;
    float4 *albedo = nullptr, *normal = nullptr, *prev_radiance = nullptr; float *depth = nullptr, *prev_depth = nullptr; float2* velocity = nullptr;
    cudaError_t e;
    if ((e = g.alloc(albedo, n)) || (e = g.alloc(depth, n)) || (e = g.alloc(normal, n)) || (e = g.alloc(velocity, n)) ||
        (e = g.alloc(prev_radiance, n)) || (e = g.alloc(prev_depth, n)))
        RT_FAIL(c, RT_ERR_CUDA, "allocating the AOV buffers failed: %s", cudaGetErrorString(e));
    c->aov_mem = std::move(g); c->aov_albedo = albedo; c->aov_depth = depth; c->aov_normal = normal; c->aov_velocity = velocity;
    c->prev_radiance = prev_radiance; c->prev_depth = prev_depth;
    RT_CUDA(c, cudaMemsetAsync(c->aov_albedo, 0, n * 16, c->stream)); RT_CUDA(c, cudaMemsetAsync(c->aov_depth, 0, n * 4, c->stream));
    RT_CUDA(c, cudaMemsetAsync(c->aov_normal, 0, n * 16, c->stream)); RT_CUDA(c, cudaMemsetAsync(c->aov_velocity, 0, n * 8, c->stream));
    RT_CUDA(c, cudaMemsetAsync(c->prev_radiance, 0, n * 16, c->stream)); RT_CUDA(c, cudaMemsetAsync(c->prev_depth, 0, n * 4, c->stream));
    return RT_OK;
}

int ensure_scratch(rt_ctx* c, size_t bytes)
{
    if (c->scratch_bytes >= bytes) return RT_OK;
    c->scratch_mem.clear(); c->scratch = nullptr; c->scratch_bytes = 0;
    RT_CUDA(c, c->scratch_mem.alloc(c->scratch, bytes));
    c->scratch_bytes = bytes;
    return RT_OK;
}

} // namespace

extern "C" {

const char* rt_last_error(const rt_ctx* ctx) { return ctx ? ctx->error.c_str() : g_create_error.c_str(); }

int rt_create(uint32_t width, uint32_t height, int device, rt_ctx** out_ctx)
{
    if (!out_ctx || width == 0 || height == 0 || width > 65535u || height > 65535u)
    {
        g_create_error = "rt_create: bad arguments (need 1 <= width, height <= 65535)"; return RT_ERR_INVALID_ARGUMENT;
    }
    *out_ctx = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
    {
        g_create_error = std::string("rt_create: no CUDA device (") + cudaGetErrorString(e) + "); this backend has no CPU fallback";
        return RT_ERR_NO_DEVICE;
    }
    if (device < 0 || device >= ndev) { g_create_error = "rt_create: device index out of range"; return RT_ERR_INVALID_ARGUMENT; }
    std::unique_ptr<rt_ctx> c(new rt_ctx);
    c->device = device; c->width = width; c->height = height;
    auto fail = [&](const char* what, cudaError_t err) { g_create_error = std::string("rt_create: ") + what + ": " + cudaGetErrorString(err); return RT_ERR_CUDA; };
    if ((e = cudaSetDevice(device)) != cudaSuccess) return fail("cudaSetDevice", e);
    cudaDeviceProp prop;
    if ((e = cudaGetDeviceProperties(&prop, device)) != cudaSuccess) return fail("cudaGetDeviceProperties", e);
    c->num_sms = prop.multiProcessorCount;
    if ((e = cudaFuncSetAttribute(k_shade_queues<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ContStage))) != cudaSuccess ||
        (e = cudaFuncSetAttribute(k_shade_queues<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ContStage))) != cudaSuccess ||
        (e = cudaFuncSetAttribute(k_shade_queues<true, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ContStage))) != cudaSuccess ||
        (e = cudaFuncSetAttribute(k_shade_queues<true, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ContStage))) != cudaSuccess)
        return fail("cudaFuncSetAttribute(k_shade_queues)", e);
    if ((e = make_stream(c->stream)) != cudaSuccess) return fail("cudaStreamCreate", e);
    if ((e = c->ctx_mem.alloc(c->counters, 1)) != cudaSuccess) return fail("cudaMalloc(counters)", e);
    if ((e = c->ctx_mem.alloc(c->d_dyn, 1)) != cudaSuccess) return fail("cudaMalloc(frame constants)", e);
    cudaMemsetAsync(c->d_dyn, 0, sizeof(FrameDyn), c->stream);
    cudaMemsetAsync(c->counters, 0, sizeof(DevCounters), c->stream);
    int rc = alloc_frame_buffers(c.get());
    if (rc != RT_OK) { g_create_error = c->error; return rc; }
    *out_ctx = c.release();
    return RT_OK;
}

int rt_destroy(rt_ctx* c)
{
    if (!c) return RT_ERR_INVALID_ARGUMENT;
    for (rt_ctx* k : c->children) rt_destroy(k);
    cudaSetDevice(c->device);            // a multi-device context's is its first child's, where the gather buffer lives
    for (cudaStream_t s : { c->stream.get(), c->shadow_stream.get(), c->copy_stream.get() })
        if (s) cudaStreamSynchronize(s);
    delete c;                            // the owners free the buffers, then destroy the events and streams
    return RT_OK;
}

int rt_set_partition(rt_ctx* c, uint32_t rank, uint32_t world)
{
    RT_CHECK_CTX(c); RT_NOT_ON_GROUP(c, "rt_set_partition");
    if (world == 0 || rank >= world) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_set_partition: need rank < world, world >= 1");
    if (world > 1 && c->denoiser)
        RT_FAIL(c, RT_ERR_UNSUPPORTED, "the temporal denoiser reprojects across the whole image and is not available with a multi-GPU partition");
    if (world > 1 && c->sd_iters)
        RT_FAIL(c, RT_ERR_UNSUPPORTED, "the spatial denoiser is not available with a multi-GPU partition (neighbouring rows live on other ranks)");
    RT_CUDA(c, cudaSetDevice(c->device));
    c->rank = rank; c->world = world;
    c->gather_slab = nullptr; c->gather_flag = nullptr;       // a gather target belongs to the partition it was set for
    return alloc_frame_buffers(c);
}

// Copies `bytes` from the host into a new block of g (16 bytes for an empty array) and points *dst at it.
static int upload_to(rt_ctx* c, DevAllocs& g, const void* src, size_t bytes, const void** dst)
{
    char* d = nullptr;
    RT_CUDA(c, g.alloc(d, bytes ? bytes : 16));
    if (bytes) RT_CUDA(c, cudaMemcpy(d, src, bytes, cudaMemcpyHostToDevice));
    *dst = d;
    return RT_OK;
}

static void clear_light_tables(rt_ctx* c)
{
    c->light_mem.clear();
    DevScene& ds = c->scene;
    ds.emit_pdfA = nullptr; ds.emit_cdf = nullptr; ds.emit_list = nullptr; ds.n_emit = 0; ds.emit_pe = 0.0f;
    ds.env_marg = nullptr; ds.env_cond = nullptr; ds.env_pdf = nullptr; ds.light_pev = 0.0f; ds.no_analytic = 0;
}

// (Re)builds the device emitter table (rt_emitters.h) from the kept upload data and the environment table (rt_envmap.h) from the
// device's environment image, with the light-kind probabilities of the current weights.  A table is inactive (not allocated, its
// scene.* pointers null) while its option is off, before an upload, in white-furnace mode and when it has nothing to select; with
// both inactive the frames are those of both options off.  The caller has validated the emitter indices.
static int refresh_lights(rt_ctx* c)
{
    RT_CUDA(c, cudaSetDevice(c->device));
    { int rc = join_shadow(c); if (rc) return rc; }
    RT_CUDA(c, cudaStreamSynchronize(c->stream));     // a frame in flight may still read the old tables
    clear_light_tables(c);
    ++c->config_gen;
    if ((!c->emitter_sampling && !c->env_sampling) || !c->scene_ready) return RT_OK;
    DevScene& ds = c->scene;
    if (c->emitter_sampling && c->emit_moved && !c->emit_idx.empty())
    {   // rt_update_triangles moved the geometry: the emitters' positions (their areas) are read back from tris_ref; their
        // materials stay those of the upload
        const size_t n = c->emit_idx.size(), pos_at = (n * 4 + 15) / 16 * 16;
        std::vector<float4> pos(n * 3);
        { int rc = ensure_scratch(c, pos_at + n * 48); if (rc) return rc; }
        char* d = c->scratch;
        RT_CUDA(c, cudaMemcpyAsync(d, c->emit_idx.data(), n * 4, cudaMemcpyHostToDevice, c->stream));
        {
            TimedLaunch t(c, RT_K_MISC);
            k_gather_positions<<<grid_for((uint32_t)n), 256, 0, c->stream>>>(ds.tris_ref, (const uint32_t*)d, (uint32_t)n, (float4*)(d + pos_at));
            int rc = post_launch(c, "k_gather_positions"); if (rc) return rc;
        }
        RT_CUDA(c, cudaMemcpyAsync(pos.data(), d + pos_at, n * 48, cudaMemcpyDeviceToHost, c->stream));
        RT_CUDA(c, cudaStreamSynchronize(c->stream));
        for (size_t i = 0; i < n; ++i)
        {
            memcpy(&c->emit_tris[i].v1.position, &pos[i * 3 + 0], 16);
            memcpy(&c->emit_tris[i].v2.position, &pos[i * 3 + 1], 16);
            memcpy(&c->emit_tris[i].v3.position, &pos[i * 3 + 2], 16);
        }
        c->emit_moved = false;
    }
    auto tri_of = [&](uint64_t i) -> const RtTriangle& { return c->emit_tris[i]; };
    rtemit::Table et;
    if (c->emitter_sampling)
        rtemit::build(tri_of, c->emit_idx.data(), c->emit_idx.size(), c->emit_n_tris, c->emit_mats.data(), c->emit_lights.data(),
                      ds.light_count, c->white_furnace != 0, et);
    const bool emit_active = et.p_e > 0.0f;
    rtenv::Table vt;
    bool env_active = false;
    if (c->env_sampling && !c->white_furnace)
    {   // the image is read back from the device: the context keeps no host copy of it
        std::vector<float> img((size_t)ds.env_w * ds.env_h * 4);
        RT_CUDA(c, cudaMemcpy(img.data(), ds.env, img.size() * 4, cudaMemcpyDeviceToHost));
        env_active = rtenv::build(img.data(), (uint32_t)ds.env_w, (uint32_t)ds.env_h, vt);
    }
    if (!emit_active && !env_active) return RT_OK;
    const rtenv::Selection sel = rtenv::select(c->analytic_lit, emit_active, env_active, c->light_w[0], c->light_w[1], c->light_w[2]);
    DevAllocs g;
    DevScene lt = ds;                                  // the tables take effect together, once every upload has succeeded
    int rc;
    if (emit_active)
    {
        rtemit::build(tri_of, c->emit_idx.data(), c->emit_idx.size(), c->emit_n_tris, c->emit_mats.data(), c->emit_lights.data(),
                      ds.light_count, c->white_furnace != 0, et, sel.p_e);
        if ((rc = upload_to(c, g, et.pdfA.data(), et.pdfA.size() * 4, (const void**)&lt.emit_pdfA))) return rc;
        if ((rc = upload_to(c, g, et.cdf.data(), et.cdf.size() * 4, (const void**)&lt.emit_cdf))) return rc;
        if ((rc = upload_to(c, g, et.list.data(), et.list.size() * 4, (const void**)&lt.emit_list))) return rc;
        lt.n_emit = (uint32_t)et.list.size(); lt.emit_pe = et.p_e;
    }
    if (env_active)
    {
        rtenv::scale(vt, sel.p_v);
        if ((rc = upload_to(c, g, vt.marg.data(), vt.marg.size() * 4, (const void**)&lt.env_marg))) return rc;
        if ((rc = upload_to(c, g, vt.cond.data(), vt.cond.size() * 4, (const void**)&lt.env_cond))) return rc;
        if ((rc = upload_to(c, g, vt.pdf.data(), vt.pdf.size() * 4, (const void**)&lt.env_pdf))) return rc;
    }
    lt.light_pev = sel.p_ev; lt.no_analytic = sel.no_analytic ? 1u : 0u;
    c->light_mem = std::move(g); ds = lt;
    return RT_OK;
}

// Either table exists: the sampled-light instances of the shading kernels run
static bool lights_sampled(const rt_ctx* c) { return c->scene.emit_pdfA || c->scene.env_pdf; }

// Object motion (RT_OPT_OBJECT_MOTION): the previous positions become the current ones, a device-to-device copy of tris_ref on the
// render stream (after every update submitted before).  The buffer is allocated all-or-nothing at the first call after an upload;
// if that fails the option is turned off.
static int set_prev_positions(rt_ctx* c)
{
    const size_t n = (size_t)c->n_tris * 3;
    if (!c->prev_pos)
    {
        DevAllocs g;
        float4* q = nullptr;
        const cudaError_t e = g.alloc(q, n);
        if (e != cudaSuccess)
        {
            c->object_motion = 0;
            RT_FAIL(c, RT_ERR_CUDA, "object motion: allocating the previous positions (%llu bytes) failed: %s", (unsigned long long)n * 16,
                    cudaGetErrorString(e));
        }
        c->motion_mem = std::move(g); c->prev_pos = q;
    }
    RT_CUDA(c, cudaMemcpyAsync(c->prev_pos, c->scene.tris_ref, n * 16, cudaMemcpyDeviceToDevice, c->stream));
    return RT_OK;
}

// The instance buffer for `cap` instances (allocated before the old one is freed; the caller has drained the stream)
static int alloc_instances(rt_ctx* c, uint32_t cap)
{
    DevAllocs g;
    char* base = nullptr;
    const size_t top = (size_t)std::max(cap, 2u) - 1u;
    const size_t f4 = 3 + top * 4 + (size_t)cap * 8 + (size_t)cap * 3 + ((size_t)cap + 3) / 4;
    RT_CUDA(c, g.alloc(base, f4 * 16));
    RT_CUDA(c, cudaMemset(base, 0, f4 * 16));
    float4* p = (float4*)base;
    c->inst_hdr = p; c->inst_top = p + 3; c->inst_rec = c->inst_top + top * 4; c->inst_prev = c->inst_rec + (size_t)cap * 8;
    c->inst_base = (uint32_t*)(c->inst_prev + (size_t)cap * 3);
    c->inst_mem = std::move(g); c->inst_cap = cap;
    ++c->config_gen;
    return RT_OK;
}

// rt_upload_scene (meshes == nullptr) and rt_upload_instanced_scene
static int upload_scene(rt_ctx* c, const RtSceneDesc* s, const RtMeshDesc* meshes, uint32_t n_meshes)
{
    const char* fn = meshes ? "rt_upload_instanced_scene" : "rt_upload_scene";
    if (!s) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: null scene", fn);
    // cl_pt_integrator.cpp:385,404 assert non-empty triangles/materials; light.h:46 divides by the light count
    if (!s->triangles || s->n_triangles == 0) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: scene has no triangles", fn);
    if (!s->materials || s->n_materials == 0) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: scene has no materials", fn);
    if (!s->nodes || s->n_nodes == 0) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: scene has no BVH nodes", fn);
    if (!s->lights || s->n_lights == 0 || s->scene_info.analytic_light_count == 0)
        RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: at least one analytic light is required (light.h:46 divides by the count)", fn);
    if (s->scene_info.analytic_light_count > s->n_lights) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: analytic_light_count exceeds n_lights", fn);
    if (!s->env_image || s->env_width == 0 || s->env_height == 0) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: environment image required", fn);
    if (s->n_triangles >= 0x7FFFFFFFull || s->n_nodes >= 0x7FFFFFFFull) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: scene too large", fn);
    for (uint64_t i = 0; i < s->n_triangles; ++i)
        if (s->triangles[i].mtlIndex >= s->n_materials) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: triangle %llu has material index out of range", fn, (unsigned long long)i);

    for (uint64_t i = 0; i < s->n_materials; ++i)
    {   // texture indices of the packed materials must exist (0xFF = none)
        const RtPackedMaterial& m = s->materials[i];
        uint32_t idx[6] = { m.diffuse_albedo >> 24, m.specular_albedo >> 24, (m.roughness_metalness >> 8) & 0xFF, m.roughness_metalness >> 24,
                            (m.ior_emission_idx_transparency >> 8) & 0xFF, m.ior_emission_idx_transparency >> 24 };
        for (uint32_t t : idx)
            if (t != RT_INVALID_TEXTURE_IDX && t >= s->n_textures) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: material %llu references texture %u of %llu", fn, (unsigned long long)i, t, (unsigned long long)s->n_textures);
    }
    for (uint64_t i = 0; i < s->n_textures; ++i)
    {
        const RtTexture& t = s->textures[i];
        if (t.width <= 0 || t.height <= 0 || t.data_start < 0 || (uint64_t)t.data_start + (uint64_t)t.width * t.height > s->n_texture_data)
            RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: texture %llu lies outside the texel array", fn, (unsigned long long)i);
        // sample_texture (rt_device.cuh) and material.h:259 index texels in int: the last texel must lie below 2^31
        if ((uint64_t)t.data_start + (uint64_t)t.width * t.height > 0x80000000ull)
            RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: texture %llu ends beyond texel 2^31 - 1", fn, (unsigned long long)i);
    }
    if (c->emitter_sampling)
    {
        if (s->n_emissive && !s->emissive_indices)
            RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: emitter sampling is on and n_emissive > 0 with no emissive_indices", fn);
        std::string err;
        if (!rtemit::check_indices(s->emissive_indices, s->n_emissive, s->n_triangles, err))
            RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: emitter sampling is on and %s", fn, err.c_str());
    }

    RT_CUDA(c, cudaSetDevice(c->device));
    { int rc = join_shadow(c); if (rc) return rc; }     // a shadow pass of an unfinished frame may still read the old scene
    RT_CUDA(c, cudaStreamSynchronize(c->stream));
    c->scene_mem.clear(); c->tree_mem.clear(); c->stage = {};
    c->motion_mem.clear(); c->prev_pos = nullptr;
    c->refit_link = nullptr; c->refit_leaves = nullptr; c->refit_arrivals = nullptr; c->refit_n_leaves = 0;
    c->lbvh = rt_ctx::Lbvh();
    c->scene_ready = false;
    clear_light_tables(c);

    auto upload = [&](const void* src, size_t bytes, const void** dst) { return upload_to(c, c->scene_mem, src, bytes, dst); };
    int rc;
    DevScene& ds = c->scene;
    if ((rc = upload_to(c, c->tree_mem, s->nodes, s->n_nodes * sizeof(RtLinearBVHNode), (const void**)&ds.nodes_ref))) return rc;
    {
        std::vector<rtbvh::F4> rec;
        rtbvh::build_tri_shade(s->triangles, s->n_triangles, rec);
        if ((rc = upload(rec.data(), rec.size() * 16, (const void**)&ds.tri_shade))) return rc;
        rtbvh::build_mat_rec(s->materials, s->n_materials, rec);
        if ((rc = upload(rec.data(), rec.size() * 16, (const void**)&ds.mat_rec))) return rc;
        rtbvh::build_light_rec(s->lights, s->n_lights, rec);
        if ((rc = upload(rec.data(), rec.size() * 16, (const void**)&ds.light_rec))) return rc;
    }
    {   // RTTriangle[] derived at upload, cl_pt_integrator.cpp:392-402
        std::vector<RtRTTriangle> rt(s->n_triangles);
        for (uint64_t i = 0; i < s->n_triangles; ++i)
        {
            rt[i].position1 = s->triangles[i].v1.position; rt[i].position2 = s->triangles[i].v2.position; rt[i].position3 = s->triangles[i].v3.position;
        }
        if ((rc = upload(rt.data(), rt.size() * sizeof(RtRTTriangle), (const void**)&ds.tris_ref))) return rc;
    }
    if ((rc = upload(s->materials, s->n_materials * sizeof(RtPackedMaterial), (const void**)&ds.materials))) return rc;
    if ((rc = upload(s->textures, s->n_textures * sizeof(RtTexture), (const void**)&ds.textures))) return rc;
    if ((rc = upload(s->texture_data, s->n_texture_data * 4, (const void**)&ds.texels))) return rc;
    if ((rc = upload(s->env_image, (size_t)s->env_width * s->env_height * 16, (const void**)&ds.env))) return rc;
    ds.env_w = (int)s->env_width; ds.env_h = (int)s->env_height;
    ds.light_count = s->scene_info.analytic_light_count;
    c->meshes.clear();
    if (meshes)
    {   // every mesh's records as rt_upload_scene derives them from that mesh alone, concatenated; references stay mesh-relative
        std::vector<rtbvh::F4> nodes, tris;
        for (uint32_t k = 0; k < n_meshes; ++k)
        {
            const RtMeshDesc& m = meshes[k];
            rtbvh::WideLayout wl;
            std::string err;
            if (!rtbvh::build_layout(s->nodes + m.first_node, m.n_nodes, s->triangles + m.first_triangle, m.n_triangles, wl, err))
                RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: malformed BVH of mesh %u: %s", fn, k, err.c_str());
            const RtLinearBVHNode& r = s->nodes[m.first_node];
            rtinst::MeshInfo mi = { wl.root_ref, (uint32_t)nodes.size(), (uint32_t)m.first_triangle, (uint32_t)m.n_triangles, (uint32_t)m.first_node,
                                    { r.bounds_min.x, r.bounds_min.y, r.bounds_min.z }, { r.bounds_max.x, r.bounds_max.y, r.bounds_max.z } };
            c->meshes.push_back(mi);
            nodes.insert(nodes.end(), wl.nodes.begin(), wl.nodes.end());
            tris.resize(std::max<size_t>(tris.size(), (size_t)(m.first_triangle + m.n_triangles) * 3));
            std::copy(wl.tris.begin(), wl.tris.end(), tris.begin() + (size_t)m.first_triangle * 3);
        }
        if (nodes.size() >= 0x7FFFFFFFull) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: scene too large", fn);
        if ((rc = upload_to(c, c->tree_mem, nodes.data(), nodes.size() * 16, (const void**)&ds.wnodes))) return rc;
        if ((rc = upload(tris.data(), tris.size() * 16, (const void**)&ds.wtris))) return rc;
        ds.root_ref = 0; ds.top_n = 0; ds.top_k = 0;
        ds.wnodes_f4 = (uint32_t)nodes.size(); ds.wtris_f4 = (uint32_t)tris.size();
    }
    else
    {   // optimised traversal layout
        rtbvh::WideLayout wl;
        std::string err;
        if (!rtbvh::build_layout(s->nodes, s->n_nodes, s->triangles, s->n_triangles, wl, err))
            RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: malformed BVH: %s", fn, err.c_str());
        if ((rc = upload_to(c, c->tree_mem, wl.nodes.data(), wl.nodes.size() * 16, (const void**)&ds.wnodes))) return rc;
        if ((rc = upload(wl.tris.data(), wl.tris.size() * 16, (const void**)&ds.wtris))) return rc;
        ds.root_ref = wl.root_ref;
        ds.wnodes_f4 = (uint32_t)wl.nodes.size(); ds.wtris_f4 = (uint32_t)wl.tris.size();
        ds.top_n = wl.top_n; ds.top_k = 0;
    }
    const RtLinearBVHNode& root = s->nodes[0];
    c->scene_mid = make_float4((root.bounds_min.x + root.bounds_max.x) * 0.5f, (root.bounds_min.y + root.bounds_max.y) * 0.5f,
                               (root.bounds_min.z + root.bounds_max.z) * 0.5f, 0.0f);
    // what the emitter table needs is kept only for a scene that lists emitters (a list with a null pointer counts as empty: with
    // the option off the array was never read, and such uploads stay accepted)
    const uint64_t n_emit = (s->emissive_indices && !meshes) ? s->n_emissive : 0;
    c->emit_idx.assign(s->emissive_indices, s->emissive_indices + n_emit);
    c->emit_tris.assign(n_emit, RtTriangle{});
    for (uint64_t i = 0; i < n_emit; ++i)
        if (s->emissive_indices[i] < s->n_triangles) c->emit_tris[i] = s->triangles[s->emissive_indices[i]];
    if (n_emit) { c->emit_mats.assign(s->materials, s->materials + s->n_materials); c->emit_lights.assign(s->lights, s->lights + s->n_lights); }
    else { c->emit_mats.clear(); c->emit_lights.clear(); }
    c->emit_n_tris = s->n_triangles;
    c->emit_moved = false;
    c->n_tris = s->n_triangles; c->n_nodes = s->n_nodes;
    c->analytic_lit = rtenv::analytic_lit(s->lights, s->scene_info.analytic_light_count);
    c->instanced = meshes != nullptr;
    c->inst_mem.clear(); c->inst_hdr = c->inst_top = c->inst_rec = c->inst_prev = nullptr; c->inst_base = nullptr;
    c->inst_cap = c->n_inst = 0; c->inst_last.clear(); c->inst_list.clear();
    c->mesh_refit.clear(); c->mesh_bad = nullptr;
    c->mtl_mem.clear(); c->mtl_map = nullptr; c->mtl_cap = 0; c->inst_mtl_row.clear();
    c->n_materials = s->n_materials;
    for (uint32_t k = 0; k < (meshes ? n_meshes : 0u); ++k) { rt_ctx::MeshRefit r; r.n_nodes = meshes[k].n_nodes; c->mesh_refit.push_back(r); }
    if (c->instanced && (rc = alloc_instances(c, 1))) return rc;          // no instances yet: every ray misses
    if (c->object_motion && (rc = set_prev_positions(c))) return rc;
    c->scene_ready = true;
    ++c->config_gen;
    return refresh_lights(c);
}

int rt_upload_scene(rt_ctx* c, const RtSceneDesc* s)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_upload_scene(k, s));
    return upload_scene(c, s, nullptr, 0);
}

int rt_upload_instanced_scene(rt_ctx* c, const RtSceneDesc* s, const RtMeshDesc* meshes, uint32_t n_meshes)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_upload_instanced_scene(k, s, meshes, n_meshes));
    if (c->emitter_sampling)
        RT_FAIL(c, RT_ERR_UNSUPPORTED, "rt_upload_instanced_scene: emitter sampling (RT_OPT_EMITTER_SAMPLING 1) is not available on instanced scenes");
    if (!s) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_upload_instanced_scene: null scene");
    if (!meshes || n_meshes == 0) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_upload_instanced_scene: no meshes");
    for (uint32_t k = 0; k < n_meshes; ++k)
    {
        const RtMeshDesc& m = meshes[k];
        if (m.n_triangles == 0 || m.n_nodes == 0 || m.first_triangle > s->n_triangles || m.n_triangles > s->n_triangles - m.first_triangle ||
            m.first_node > s->n_nodes || m.n_nodes > s->n_nodes - m.first_node)
            RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_upload_instanced_scene: mesh %u is empty or lies outside the scene's arrays", k);
        if (!s->nodes) break;                      // upload_scene reports the missing nodes
        const RtLinearBVHNode& r = s->nodes[m.first_node];
        const float b[6] = { r.bounds_min.x, r.bounds_min.y, r.bounds_min.z, r.bounds_max.x, r.bounds_max.y, r.bounds_max.z };
        for (float v : b) if (!std::isfinite(v)) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_upload_instanced_scene: mesh %u has a root box that is not finite", k);
    }
    return upload_scene(c, s, meshes, n_meshes);
}

// The head of the instance buffer's image: the header (top-level root box, root reference, instance count, the slack (a, b) of
// rt_instances.h) and the top-level records, 3 + 4 (n - 1) float4 (3 for n <= 1).  rt_set_instances writes them with the rest of the image,
// rt_update_mesh_triangles alone.
static size_t top_level_image(const rtinst::Prepared& pr, uint32_t n, float4* h)
{
    const rtinst::Box& rb = pr.tree.root;
    h[0] = make_float4(rb.lo[0], rb.lo[1], rb.lo[2], rtinst::int_bits(pr.tree.root_ref));
    h[1] = make_float4(rb.hi[0], rb.hi[1], rb.hi[2], rtinst::int_bits((int)n));
    h[2] = make_float4(pr.tree.slack[0], pr.tree.slack[1], 0.0f, 0.0f);
    memcpy(&h[3], pr.tree.records.data(), pr.tree.records.size() * 4);
    return 3 + pr.tree.records.size() / 4;
}

int rt_set_instances(rt_ctx* c, const RtInstance* instances, uint32_t n)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_set_instances(k, instances, n));
    if (!c->scene_ready || !c->instanced) RT_FAIL(c, RT_ERR_NOT_READY, "rt_set_instances: no instanced scene (rt_upload_instanced_scene)");
    if (n && !instances) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_set_instances: null instances");
    rtinst::Prepared pr;
    std::string err;
    if (!rtinst::prepare(instances, n, c->meshes, pr, err)) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_set_instances: %s", err.c_str());
    RT_CUDA(c, cudaSetDevice(c->device));
    { int rc = join_shadow(c); if (rc) return rc; }     // a deferred shadow pass reads the instances this call rewrites
    if (n > c->inst_cap)
    {   // a larger buffer (at least twice the old, so that a list growing one by one re-captures the frame graph log n times):
        // frames in flight read the old one.  The launch arguments change, so the sort-key origin of the shading pass moves to the
        // centre of the new top-level root box here (it orders rays only; between growths it stays).
        RT_CUDA(c, cudaStreamSynchronize(c->stream));
        int rc = alloc_instances(c, std::max(n, 2u * c->inst_cap)); if (rc) return rc;
        const rtinst::Box& b = pr.tree.root;
        c->scene_mid = make_float4((b.lo[0] + b.hi[0]) * 0.5f, (b.lo[1] + b.hi[1]) * 0.5f, (b.lo[2] + b.hi[2]) * 0.5f, 0.0f);
    }
    const size_t top = (size_t)std::max(c->inst_cap, 2u) - 1u;
    const size_t f4 = 3 + top * 4 + (size_t)c->inst_cap * 11 + ((size_t)c->inst_cap + 3) / 4;
    std::vector<float4>& h = c->inst_host;
    h.assign(f4, make_float4(0.0f, 0.0f, 0.0f, 0.0f));
    top_level_image(pr, n, h.data());
    float4* rec = &h[3 + top * 4];
    memcpy(rec, pr.rec.data(), pr.rec.size() * 4);
    for (uint32_t i = 0; i < n; ++i)              // the material row of index i in the kept assignment (rt_set_instance_materials)
        rec[(size_t)i * 8 + 7].z = rtinst::int_bits((int)(i < c->inst_mtl_row.size() ? c->inst_mtl_row[i] : RT_INVALID_ID));
    float4* prev = rec + (size_t)c->inst_cap * 8;
    // previous transforms: index i's transform in the last earlier list that had index i, else its new one
    const size_t known = c->inst_last.size() / 12;
    for (uint32_t i = 0; i < n; ++i)
        memcpy(prev + (size_t)i * 3, i < known ? &c->inst_last[(size_t)i * 12] : instances[i].object_to_world, 48);
    memcpy(prev + (size_t)c->inst_cap * 3, pr.base.data(), pr.base.size() * 4);
    // one copy of the whole image, in render-stream order after the work submitted before (pageable: the call returns once it is staged)
    RT_CUDA(c, cudaMemcpyAsync(c->inst_hdr, h.data(), f4 * 16, cudaMemcpyHostToDevice, c->stream));
    if (n > known) c->inst_last.resize((size_t)n * 12);
    for (uint32_t i = 0; i < n; ++i) memcpy(&c->inst_last[(size_t)i * 12], instances[i].object_to_world, 48);
    c->inst_list.assign(instances, instances + n);
    c->n_inst = n;
    return RT_OK;
}

// ---- per-instance materials: rt_set_instance_materials (include/rt_b200.h)

int rt_set_instance_materials(rt_ctx* c, const uint32_t* remaps, uint32_t n_remaps, const uint32_t* remap_of_instance, uint32_t n_instances)
{
    const char* what = "rt_set_instance_materials";
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_set_instance_materials(k, remaps, n_remaps, remap_of_instance, n_instances));
    if (!c->scene_ready || !c->instanced) RT_FAIL(c, RT_ERR_NOT_READY, "%s: no instanced scene (rt_upload_instanced_scene)", what);
    if (n_remaps && !remaps) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: null remaps", what);
    if (n_instances && !remap_of_instance) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: null remap_of_instance", what);
    const uint64_t nm = c->n_materials;
    if (n_remaps && nm > 0xFFFFFFFEull / n_remaps)          // n_remaps * nm >= 2^32 - 1, without overflow
        RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: %u rows of %llu materials reach 2^32 - 1 entries", what, n_remaps, (unsigned long long)nm);
    const size_t entries = (size_t)n_remaps * nm;
    for (size_t e = 0; e < entries; ++e)
        if (remaps[e] >= nm)
            RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: row %llu maps material %llu to %u of %llu", what, (unsigned long long)(e / nm),
                    (unsigned long long)(e % nm), remaps[e], (unsigned long long)nm);
    for (uint32_t i = 0; i < n_instances; ++i)
        if (remap_of_instance[i] >= n_remaps && remap_of_instance[i] != RT_INVALID_ID)
            RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: instance %u names row %u of %u", what, i, remap_of_instance[i], n_remaps);
    RT_CUDA(c, cudaSetDevice(c->device));
    { int rc = join_shadow(c); if (rc) return rc; }     // a deferred shadow pass reads the instance records this call rewrites
    if (entries > c->mtl_cap)
    {   // a larger table (at least twice the old, as the instance buffer grows); frames in flight read the old one.  The launch
        // arguments change, so a captured frame graph is re-captured.
        RT_CUDA(c, cudaStreamSynchronize(c->stream));
        const size_t cap = std::max(entries, 2 * c->mtl_cap);
        DevAllocs g;
        uint32_t* p = nullptr;
        RT_CUDA(c, g.alloc(p, cap));
        c->mtl_mem = std::move(g); c->mtl_map = p; c->mtl_cap = cap;
        ++c->config_gen;
    }
    // the table and the record words, each one copy in render-stream order from the context's own host images (pageable, so
    // staged before the call returns; the caller's arrays may be pinned, and are not read after it)
    if (entries)
    {
        c->mtl_host.assign(remaps, remaps + entries);
        RT_CUDA(c, cudaMemcpyAsync(c->mtl_map, c->mtl_host.data(), entries * 4, cudaMemcpyHostToDevice, c->stream));
    }
    c->inst_mtl_row.resize(n_instances);
    for (uint32_t i = 0; i < n_instances; ++i)
        c->inst_mtl_row[i] = remap_of_instance[i] == RT_INVALID_ID ? RT_INVALID_ID : (uint32_t)(remap_of_instance[i] * nm);
    if (c->n_inst)
    {   // the instance records of the current list, as rt_set_instances wrote them but for the row offsets
        const size_t top = (size_t)std::max(c->inst_cap, 2u) - 1u;
        float4* rec = &c->inst_host[3 + top * 4];
        for (uint32_t i = 0; i < c->n_inst; ++i)
            rec[(size_t)i * 8 + 7].z = rtinst::int_bits((int)(i < n_instances ? c->inst_mtl_row[i] : RT_INVALID_ID));
        RT_CUDA(c, cudaMemcpyAsync(c->inst_rec, rec, (size_t)c->n_inst * 8 * 16, cudaMemcpyHostToDevice, c->stream));
    }
    return RT_OK;
}

// ---- geometry updates: rt_update_triangles[_device], rt_read_bvh (include/rt_b200.h)

// The refit map of the n_nodes nodes at `nodes` (device memory; references relative to them), built from their device copy (a
// refit rewrites only their boxes; blocking) into tree_mem: link and arrivals per node, the leaf list.
static int build_refit_map(rt_ctx* c, const float4* nodes_dev, uint64_t n_nodes, const char* what, uint2*& link, uint32_t*& leaves,
                           uint32_t*& arrivals, uint32_t& n_leaves)
{
    std::vector<RtLinearBVHNode> nodes(n_nodes);
    RT_CUDA(c, cudaMemcpyAsync(nodes.data(), nodes_dev, n_nodes * sizeof(RtLinearBVHNode), cudaMemcpyDeviceToHost, c->stream));
    RT_CUDA(c, cudaStreamSynchronize(c->stream));
    rtbvh::RefitMap m;
    rtbvh::build_refit_map(nodes.data(), n_nodes, m);
    DevAllocs g;
    uint2* l = nullptr; uint32_t *lv = nullptr, *ar = nullptr;
    cudaError_t e;
    if ((e = g.alloc(l, m.link.size() / 2)) || (e = g.alloc(lv, m.leaves.size())) || (e = g.alloc(ar, n_nodes)) ||
        (e = cudaMemcpy(l, m.link.data(), m.link.size() * 4, cudaMemcpyHostToDevice)) ||
        (e = cudaMemcpy(lv, m.leaves.data(), m.leaves.size() * 4, cudaMemcpyHostToDevice)))
        RT_FAIL(c, RT_ERR_CUDA, "%s: refit map: %s", what, cudaGetErrorString(e));
    c->tree_mem.adopt(std::move(g)); link = l; leaves = lv; arrivals = ar;
    n_leaves = (uint32_t)m.leaves.size();
    return RT_OK;
}

// The checks both variants share, then the refit map of the upload's tree (at the first update) and the ordering after earlier work.
static int begin_update(rt_ctx* c, const void* triangles, uint64_t n, const char* what)
{
    if (!c->scene_ready) RT_FAIL(c, RT_ERR_NOT_READY, "%s: rt_upload_scene has not been called", what);
    if (c->instanced) RT_FAIL(c, RT_ERR_UNSUPPORTED, "%s: not available on an instanced scene", what);
    if (!triangles) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: null triangles", what);
    if (n != c->n_tris) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: %llu triangles, the upload has %llu", what, (unsigned long long)n, (unsigned long long)c->n_tris);
    RT_CUDA(c, cudaSetDevice(c->device));
    { int rc = join_shadow(c); if (rc) return rc; }     // a deferred shadow pass reads the geometry this call rewrites
    if (c->refit_link) return RT_OK;
    return build_refit_map(c, c->scene.nodes_ref, c->n_nodes, what, c->refit_link, c->refit_leaves, c->refit_arrivals, c->refit_n_leaves);
}

static int launch_refit_records(rt_ctx* c, const void* src, uint32_t first, uint32_t n)
{
    DevScene& ds = c->scene;
    TimedLaunch t(c, RT_K_MISC);
    if (c->prev_pos)       // object motion: the positions this launch overwrites become the previous ones
        k_refit_records<true><<<grid_for(n), 256, 0, c->stream>>>((const float4*)src, first, n, (float4*)ds.tris_ref, (float4*)ds.wtris,
                                                                  (float4*)ds.tri_shade, c->prev_pos);
    else
        k_refit_records<false><<<grid_for(n), 256, 0, c->stream>>>((const float4*)src, first, n, (float4*)ds.tris_ref, (float4*)ds.wtris,
                                                                   (float4*)ds.tri_shade, nullptr);
    return post_launch(c, "k_refit_records");
}

// The refit, then the emitter table of the moved geometry.  The two refit kernels are plain launches and never execute
// griddepcontrol.launch_dependents: a traversal kernel launched with programmatic dependent launch stages the BVH before its
// pdl_wait() (rt_traverse.cuh), so an early trigger would let the next frame stage stale boxes.
static int launch_refit(rt_ctx* c, const uint32_t* leaves, uint32_t n_leaves, const uint2* link, uint32_t* arrivals, uint64_t n_nodes,
                        const float4* nodes_ref, const float4* tris_ref, const float4* wnodes)
{
    RT_CUDA(c, cudaMemsetAsync(arrivals, 0, n_nodes * 4, c->stream));
    TimedLaunch t(c, RT_K_MISC);
    k_refit<<<grid_for(n_leaves), 256, 0, c->stream>>>(leaves, n_leaves, link, arrivals, (float*)nodes_ref, tris_ref, (float*)wnodes);
    return post_launch(c, "k_refit");
}

static int finish_update(rt_ctx* c)
{
    {
        int rc = launch_refit(c, c->refit_leaves, c->refit_n_leaves, c->refit_link, c->refit_arrivals, c->n_nodes, c->scene.nodes_ref,
                              c->scene.tris_ref, c->scene.wnodes);
        if (rc) return rc;
    }
    // scene_mid, the origin of k_shade_queues' sort key, stays that of the upload: it orders the continuation rays, which
    // changes no result.  The buffers keep their addresses, so a captured frame graph stays valid.
    if (!c->emit_idx.empty()) c->emit_moved = true;
    return (c->emitter_sampling && !c->emit_idx.empty()) ? refresh_lights(c) : RT_OK;
}

// The record kernel over the caller's triangles[0 .. n), written to triangles first .. first + n - 1, through the staging
static int stage_records(rt_ctx* c, const RtTriangle* triangles, uint64_t n, uint64_t first_dst, const char* what)
{
    rt_ctx::Staging& sg = c->stage;
    if (!sg.host)
    {   // two halves of at most 32 MB each: the host copy into one half overlaps the upload and kernel of the other
        rt_ctx::Staging s;
        s.half = std::min<size_t>((size_t)n * sizeof(RtTriangle), (size_t)32 << 20) / sizeof(RtTriangle) * sizeof(RtTriangle);
        cudaError_t e;
        if ((e = s.mem.alloc(s.host, 2 * s.half, true)) || (e = s.mem.alloc(s.dev, 2 * s.half)) || (e = make_event(s.copied[0])) ||
            (e = make_event(s.copied[1])))
            RT_FAIL(c, RT_ERR_CUDA, "%s: staging buffers: %s", what, cudaGetErrorString(e));
        sg = std::move(s);
    }
    const uint64_t per_chunk = sg.half / sizeof(RtTriangle);
    for (uint64_t first = 0, k = 0; first < n; first += per_chunk, k ^= 1)
    {
        const uint32_t m = (uint32_t)std::min<uint64_t>(per_chunk, n - first);
        char* h = sg.host + k * sg.half; char* d = sg.dev + k * sg.half;
        RT_CUDA(c, cudaEventSynchronize(sg.copied[k]));          // the copy out of this half two chunks ago is done
        memcpy(h, triangles + first, (size_t)m * sizeof(RtTriangle));
        RT_CUDA(c, cudaMemcpyAsync(d, h, (size_t)m * sizeof(RtTriangle), cudaMemcpyHostToDevice, c->stream));
        RT_CUDA(c, cudaEventRecord(sg.copied[k], c->stream));
        int rc = launch_refit_records(c, d, (uint32_t)(first_dst + first), m); if (rc) return rc;
    }
    return RT_OK;
}

int rt_update_triangles(rt_ctx* c, const RtTriangle* triangles, uint64_t n)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_update_triangles(k, triangles, n));
    { int rc = begin_update(c, triangles, n, "rt_update_triangles"); if (rc) return rc; }
    { int rc = stage_records(c, triangles, n, 0, "rt_update_triangles"); if (rc) return rc; }
    return finish_update(c);
}

// The device variants take a single-device context and 16-byte aligned device memory of its device (a null pointer is left to the
// caller's own check)
static int check_device_triangles(rt_ctx* c, const void* triangles, const char* what, const char* host_variant)
{
    if (!c->children.empty())
        RT_FAIL(c, RT_ERR_UNSUPPORTED, "%s: a multi-device context: use %s (device memory belongs to one device)", what, host_variant);
    if (triangles)
    {
        cudaPointerAttributes a = {};
        if (cudaPointerGetAttributes(&a, triangles) != cudaSuccess) { cudaGetLastError(); a.type = cudaMemoryTypeUnregistered; }
        if (a.type != cudaMemoryTypeDevice || a.device != c->device || ((uintptr_t)triangles & 15u))
            RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: not 16-byte aligned device memory of device %d", what, c->device);
    }
    return RT_OK;
}

int rt_update_triangles_device(rt_ctx* c, const void* triangles, uint64_t n)
{
    RT_CHECK_CTX(c);
    { int rc = check_device_triangles(c, triangles, "rt_update_triangles_device", "rt_update_triangles"); if (rc) return rc; }
    { int rc = begin_update(c, triangles, n, "rt_update_triangles_device"); if (rc) return rc; }
    { int rc = launch_refit_records(c, triangles, 0, (uint32_t)n); if (rc) return rc; }
    return finish_update(c);
}

// ---- mesh updates in instanced scenes: rt_update_mesh_triangles[_device] (include/rt_b200.h)

// The argument checks both variants share (nothing is enqueued)
static int check_mesh_update(rt_ctx* c, uint32_t mesh, const void* triangles, uint64_t n, const char* what)
{
    if (!c->scene_ready || !c->instanced) RT_FAIL(c, RT_ERR_NOT_READY, "%s: no instanced scene (rt_upload_instanced_scene)", what);
    if (mesh >= c->meshes.size()) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: mesh %u of %zu", what, mesh, c->meshes.size());
    if (!triangles) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: null triangles", what);
    if (n != c->meshes[mesh].n_tris)
        RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: %llu triangles, mesh %u has %u", what, (unsigned long long)n, mesh, c->meshes[mesh].n_tris);
    return RT_OK;
}

// The ordering after earlier work, then the mesh's refit map (at its first update)
static int begin_mesh_update(rt_ctx* c, uint32_t mesh, const char* what)
{
    RT_CUDA(c, cudaSetDevice(c->device));
    { int rc = join_shadow(c); if (rc) return rc; }     // a deferred shadow pass reads the geometry this call rewrites
    rt_ctx::MeshRefit& r = c->mesh_refit[mesh];
    if (r.link) return RT_OK;
    return build_refit_map(c, c->scene.nodes_ref + (size_t)c->meshes[mesh].first_node * 3, r.n_nodes, what, r.link, r.leaves, r.arrivals,
                           r.n_leaves);
}

// The refit of the mesh's nodes (the records were written before), then its refit root box, read back (blocking), into the mesh's
// box; if an instance of the current list uses the mesh, the top-level tree of that list is rebuilt from the new box and only the
// header and the top-level records are rewritten: the instance records, the previous transforms and scene_mid stay.
static int finish_mesh_update(rt_ctx* c, uint32_t mesh, const char* what)
{
    rtinst::MeshInfo& mi = c->meshes[mesh];
    const rt_ctx::MeshRefit& r = c->mesh_refit[mesh];
    const float4* nodes = c->scene.nodes_ref + (size_t)mi.first_node * 3;
    {
        int rc = launch_refit(c, r.leaves, r.n_leaves, r.link, r.arrivals, r.n_nodes, nodes, c->scene.tris_ref + (size_t)mi.first_tri * 3,
                              c->scene.wnodes + mi.rec_f4);
        if (rc) return rc;
    }
    float4 box[2];
    RT_CUDA(c, cudaMemcpyAsync(box, nodes, sizeof(box), cudaMemcpyDeviceToHost, c->stream));
    RT_CUDA(c, cudaStreamSynchronize(c->stream));
    mi.lo[0] = box[0].x; mi.lo[1] = box[0].y; mi.lo[2] = box[0].z; mi.hi[0] = box[1].x; mi.hi[1] = box[1].y; mi.hi[2] = box[1].z;
    bool used = false;
    for (const RtInstance& in : c->inst_list) used = used || in.mesh == mesh;
    if (!used) return RT_OK;
    rtinst::Prepared pr;
    std::string err;
    if (!rtinst::prepare(c->inst_list.data(), (uint32_t)c->inst_list.size(), c->meshes, pr, err))
        RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: %s", what, err.c_str());     // not reached: the list passed rt_set_instances, the box is finite
    const size_t f4 = top_level_image(pr, (uint32_t)c->inst_list.size(), c->inst_host.data());
    RT_CUDA(c, cudaMemcpyAsync(c->inst_hdr, c->inst_host.data(), f4 * 16, cudaMemcpyHostToDevice, c->stream));
    return RT_OK;
}

int rt_update_mesh_triangles(rt_ctx* c, uint32_t mesh, const RtTriangle* triangles, uint64_t n)
{
    const char* what = "rt_update_mesh_triangles";
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_update_mesh_triangles(k, mesh, triangles, n));
    { int rc = check_mesh_update(c, mesh, triangles, n, what); if (rc) return rc; }
    for (uint64_t i = 0; i < n; ++i)
    {
        const RtTriangle& t = triangles[i];
        const float s[9] = { t.v1.position.x, t.v1.position.y, t.v1.position.z, t.v2.position.x, t.v2.position.y, t.v2.position.z,
                             t.v3.position.x, t.v3.position.y, t.v3.position.z };
        for (float v : s)
            if (!std::isfinite(v)) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: triangle %llu has a position that is not finite", what, (unsigned long long)i);
    }
    { int rc = begin_mesh_update(c, mesh, what); if (rc) return rc; }
    { int rc = stage_records(c, triangles, n, c->meshes[mesh].first_tri, what); if (rc) return rc; }
    return finish_mesh_update(c, mesh, what);
}

int rt_update_mesh_triangles_device(rt_ctx* c, uint32_t mesh, const void* triangles, uint64_t n)
{
    const char* what = "rt_update_mesh_triangles_device";
    RT_CHECK_CTX(c);
    { int rc = check_device_triangles(c, triangles, what, "rt_update_mesh_triangles"); if (rc) return rc; }
    { int rc = check_mesh_update(c, mesh, triangles, n, what); if (rc) return rc; }
    { int rc = begin_mesh_update(c, mesh, what); if (rc) return rc; }
    if (!c->mesh_bad)
    {
        DevAllocs g;
        uint32_t* bad = nullptr;
        RT_CUDA(c, g.alloc(bad, 1));
        c->tree_mem.adopt(std::move(g)); c->mesh_bad = bad;
    }
    uint32_t bad = 0;
    RT_CUDA(c, cudaMemsetAsync(c->mesh_bad, 0, 4, c->stream));
    {
        TimedLaunch t(c, RT_K_MISC);
        k_check_positions<<<grid_for((uint32_t)n), 256, 0, c->stream>>>((const float4*)triangles, (uint32_t)n, c->mesh_bad);
        int rc = post_launch(c, "k_check_positions"); if (rc) return rc;
    }
    RT_CUDA(c, cudaMemcpyAsync(&bad, c->mesh_bad, 4, cudaMemcpyDeviceToHost, c->stream));
    RT_CUDA(c, cudaStreamSynchronize(c->stream));
    if (bad) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "%s: a position is not finite", what);
    { int rc = launch_refit_records(c, triangles, c->meshes[mesh].first_tri, (uint32_t)n); if (rc) return rc; }
    return finish_mesh_update(c, mesh, what);
}

int rt_read_bvh(rt_ctx* c, RtLinearBVHNode* nodes, float* records, uint64_t* n_records)
{
    RT_CHECK_CTX(c); RT_NOT_ON_GROUP(c, "rt_read_bvh");
    if (!c->scene_ready) RT_FAIL(c, RT_ERR_NOT_READY, "rt_read_bvh: rt_upload_scene has not been called");
    if (c->instanced) RT_FAIL(c, RT_ERR_UNSUPPORTED, "rt_read_bvh: not available on an instanced scene");
    if (records && !n_records) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_read_bvh: records without n_records");
    RT_CUDA(c, cudaSetDevice(c->device));
    { int rc = join_shadow(c); if (rc) return rc; }
    if (nodes) RT_CUDA(c, cudaMemcpyAsync(nodes, c->scene.nodes_ref, c->n_nodes * sizeof(RtLinearBVHNode), cudaMemcpyDeviceToHost, c->stream));
    if (records) RT_CUDA(c, cudaMemcpyAsync(records, c->scene.wnodes, (size_t)c->scene.wnodes_f4 * 16, cudaMemcpyDeviceToHost, c->stream));
    if (n_records) *n_records = c->scene.wnodes_f4 / 4;
    RT_CUDA(c, cudaStreamSynchronize(c->stream));
    return RT_OK;
}

// ---- BVH rebuild: rt_rebuild_bvh and rt_rebuild_bvh_ploc (include/rt_b200.h, kernels in rt_lbvh.cuh and rt_ploc.cuh)

// A rebuilt tree's group, allocated but not yet in place: the nodes, records and refit map of a tree of 2n - 1 nodes and the
// linear BVH's temporaries.
struct TreeGroup
{
    DevAllocs mem;
    rt_ctx::Lbvh L;
    float4 *nodes = nullptr, *wnodes = nullptr; uint2* link = nullptr; uint32_t *leaves = nullptr, *arrivals = nullptr;
};

static cudaError_t alloc_tree(rt_ctx* c, TreeGroup& t)
{
    const size_t n = c->n_tris, nn = 2 * n - 1, n_rec = n > 1 ? n - 1 : 1;
    cudaError_t e = cudaSuccess;
    auto get = [&](auto*& view, size_t count) { if (e == cudaSuccess) e = t.mem.alloc(view, count); };
    rt_ctx::Lbvh& L = t.L;
    L.live = true;
    get(t.nodes, nn * 3); get(t.wnodes, n_rec * 4);                 // 3 float4 per RtLinearBVHNode, 4 per record
    get(t.link, nn); get(t.leaves, n); get(t.arrivals, nn);
    get(L.bounds, 6); get(L.top, RT_BVH_TOP_RECORDS); get(L.inner, n_rec);
    for (int k = 0; k < 2; ++k) { get(L.codes[k], n); get(L.ids[k], n); }
    if (e == cudaSuccess)
    {
        cub::DoubleBuffer<uint32_t> keys(L.codes[0], L.codes[1]), vals(L.ids[0], L.ids[1]);
        e = cub::DeviceRadixSort::SortPairs(nullptr, L.sort_bytes, keys, vals, (int)n, 0, 30, c->stream);
        get(L.sort_tmp, L.sort_bytes ? L.sort_bytes : 16);
    }
    return e;
}

// The new tree group replaces the current one (the caller has synchronised the render stream: a frame in flight may read it).
static void install_tree(rt_ctx* c, TreeGroup& t)
{
    c->tree_mem = std::move(t.mem);                    // frees the uploaded nodes, records and refit map
    c->scene.nodes_ref = t.nodes; c->scene.wnodes = t.wnodes;
    c->refit_link = t.link; c->refit_leaves = t.leaves; c->refit_arrivals = t.arrivals;
    c->lbvh = t.L;
    ++c->config_gen;                                   // new buffers and sizes: the frame graph is re-captured
}

// The first rebuild after an upload: the new tree group replaces the old one only once all of it is allocated, so a failure
// leaves the uploaded tree in place.
static int alloc_lbvh(rt_ctx* c)
{
    TreeGroup t;
    cudaError_t e = alloc_tree(c, t);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) RT_FAIL(c, RT_ERR_CUDA, "rt_rebuild_bvh: allocating the rebuilt tree: %s", cudaGetErrorString(e));
    install_tree(c, t);
    return RT_OK;
}

// The clustering temporaries of rt_rebuild_bvh_ploc, about 97 bytes per triangle plus the compaction's scratch; P is set only
// if all of them are allocated.
static cudaError_t alloc_ploc(rt_ctx* c, DevAllocs& g, rt_ctx::Lbvh::Ploc& out)
{
    const size_t n = c->n_tris;
    rt_ctx::Lbvh::Ploc P;
    cudaError_t e = cudaSuccess;
    auto get = [&](auto*& view, size_t count, bool host = false) { if (e == cudaSuccess) e = g.alloc(view, count, host); };
    get(P.clusters, 2 * n); get(P.nn, n); get(P.keep, n); get(P.inner, n); get(P.size, n); get(P.parent, 2 * n);
    get(P.made, 1); get(P.host, 2, true);
    if (e == cudaSuccess)
    {
        e = cub::DeviceSelect::Flagged(nullptr, P.select_bytes, P.clusters, P.keep, P.clusters + n, P.host, (int)n, c->stream);
        get(P.select_tmp, P.select_bytes ? P.select_bytes : 16);
    }
    if (e == cudaSuccess) out = P;
    return e;
}

// Steps 1-3 of the build rule: the key-point bounds, the keys and their sort into keys.Current() (codes) / vals.Current() (ids).
// k_lbvh_keys writes the end-of-leaf flags of the wtris records to `flags`.
static int sort_keys(rt_ctx* c, rt_ctx::Lbvh& L, float4* flags, cub::DoubleBuffer<uint32_t>& keys, cub::DoubleBuffer<uint32_t>& vals)
{
    const uint32_t n = (uint32_t)c->n_tris;
    RT_CUDA(c, cudaMemsetAsync(L.bounds, 0, 6 * 4, c->stream));
    int rc;
    {
        TimedLaunch t(c, RT_K_MISC);
        const uint32_t g = std::min<uint32_t>(grid_for(n).x, (uint32_t)c->num_sms * 8u);
        k_lbvh_bounds<<<g, 256, 0, c->stream>>>(c->scene.tris_ref, n, L.bounds);
        if ((rc = post_launch(c, "k_lbvh_bounds"))) return rc;
    }
    {
        TimedLaunch t(c, RT_K_MISC);
        k_lbvh_keys<<<grid_for(n), 256, 0, c->stream>>>(c->scene.tris_ref, n, L.bounds, L.codes[0], L.ids[0], flags);
        if ((rc = post_launch(c, "k_lbvh_keys"))) return rc;
    }
    // a stable sort of the 30-bit codes with the ids (ascending) as values orders the keys (code << 32) | id
    {
        TimedLaunch t(c, RT_K_MISC);
        size_t bytes = L.sort_bytes;
        RT_CUDA(c, cub::DeviceRadixSort::SortPairs(L.sort_tmp, bytes, keys, vals, (int)n, 0, 30, c->stream));
        if ((rc = post_launch(c, "DeviceRadixSort"))) return rc;
    }
    return RT_OK;
}

// Steps 5-6 from the tree in radix-tree form (lbvh.inner, ipre, ids: the triangle of each leaf in preorder; unused for n = 1):
// the top records, the nodes, records and refit map, then the boxes.
static int write_tree(rt_ctx* c, const uint32_t* ipre, const uint32_t* ids)
{
    rt_ctx::Lbvh& L = c->lbvh;
    DevScene& ds = c->scene;
    const uint32_t n = (uint32_t)c->n_tris, n_inner = n - 1;
    const uint32_t top_n = n_inner < RT_BVH_TOP_RECORDS ? n_inner : RT_BVH_TOP_RECORDS;
    float4* nodes = (float4*)ds.nodes_ref; float4* wnodes = (float4*)ds.wnodes; float4* wtris = (float4*)ds.wtris;
    int rc;
    if (n == 1)
    {
        TimedLaunch t(c, RT_K_MISC);
        k_lbvh_single<<<1, 1, 0, c->stream>>>(nodes, wnodes, wtris, c->refit_link, c->refit_leaves);
        if ((rc = post_launch(c, "k_lbvh_single"))) return rc;
    }
    else
    {
        {
            TimedLaunch t(c, RT_K_MISC);
            k_lbvh_top<<<1, 1024, 0, c->stream>>>(L.inner, ipre, top_n, L.top);
            if ((rc = post_launch(c, "k_lbvh_top"))) return rc;
        }
        {
            TimedLaunch t(c, RT_K_MISC);
            k_lbvh_write<<<grid_for(n_inner), 256, 0, c->stream>>>(L.inner, ipre, ids, L.top, top_n, n_inner, nodes, wnodes,
                                                                   c->refit_link, c->refit_leaves);
            if ((rc = post_launch(c, "k_lbvh_write"))) return rc;
        }
    }
    // the boxes: the refit of the new topology (k_refit keeps the box rule in one place)
    c->n_nodes = 2ull * n - 1; c->refit_n_leaves = n;
    ds.wnodes_f4 = 4 * (n_inner ? n_inner : 1); ds.top_n = top_n; ds.root_ref = n == 1 ? ~0 : 0;
    RT_CUDA(c, cudaMemsetAsync(c->refit_arrivals, 0, c->n_nodes * 4, c->stream));
    {
        TimedLaunch t(c, RT_K_MISC);
        k_refit<<<grid_for(n), 256, 0, c->stream>>>(c->refit_leaves, n, c->refit_link, c->refit_arrivals, (float*)nodes, ds.tris_ref,
                                                    (float*)wnodes);
        if ((rc = post_launch(c, "k_refit"))) return rc;
    }
    return RT_OK;
}

int rt_rebuild_bvh(rt_ctx* c, uint64_t* n_nodes)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_rebuild_bvh(k, n_nodes));
    if (!c->scene_ready) RT_FAIL(c, RT_ERR_NOT_READY, "rt_rebuild_bvh: rt_upload_scene has not been called");
    if (c->instanced) RT_FAIL(c, RT_ERR_UNSUPPORTED, "rt_rebuild_bvh: not available on an instanced scene");
    RT_CUDA(c, cudaSetDevice(c->device));
    { int rc = join_shadow(c); if (rc) return rc; }     // a deferred shadow pass reads the tree this call rewrites
    if (!c->lbvh.live) { int rc = alloc_lbvh(c); if (rc) return rc; }
    rt_ctx::Lbvh& L = c->lbvh;
    const uint32_t n = (uint32_t)c->n_tris, n_inner = n - 1;
    // Every launch below is a plain launch (none triggers dependent launches early), like the refit's: the next frame's
    // traversal kernel, even one launched with programmatic dependent launch, sees the finished tree.
    const uint32_t* ipre = nullptr; const uint32_t* ids = nullptr;
    int rc;
    if (n > 1)
    {
        cub::DoubleBuffer<uint32_t> keys(L.codes[0], L.codes[1]), vals(L.ids[0], L.ids[1]);
        if ((rc = sort_keys(c, L, (float4*)c->scene.wtris, keys, vals))) return rc;
        const uint32_t* codes = keys.Current(); ids = vals.Current();
        uint32_t* parent = keys.Alternate(); uint32_t* pre = vals.Alternate();       // the sort's inputs are dead
        {
            TimedLaunch t(c, RT_K_MISC);
            k_lbvh_karras<<<grid_for(n_inner), 256, 0, c->stream>>>(codes, ids, n, L.inner, parent);
            if ((rc = post_launch(c, "k_lbvh_karras"))) return rc;
        }
        {
            TimedLaunch t(c, RT_K_MISC);
            k_lbvh_number<<<grid_for(n_inner), 256, 0, c->stream>>>(L.inner, parent, n_inner, pre);
            if ((rc = post_launch(c, "k_lbvh_number"))) return rc;
        }
        ipre = pre;
    }
    if ((rc = write_tree(c, ipre, ids))) return rc;
    if (n_nodes) *n_nodes = c->n_nodes;
    return RT_OK;
}

int rt_rebuild_bvh_ploc(rt_ctx* c, uint64_t* n_nodes)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_rebuild_bvh_ploc(k, n_nodes));
    if (!c->scene_ready) RT_FAIL(c, RT_ERR_NOT_READY, "rt_rebuild_bvh_ploc: rt_upload_scene has not been called");
    if (c->instanced) RT_FAIL(c, RT_ERR_UNSUPPORTED, "rt_rebuild_bvh_ploc: not available on an instanced scene");
    RT_CUDA(c, cudaSetDevice(c->device));
    { int rc = join_shadow(c); if (rc) return rc; }     // a deferred shadow pass reads the tree this call rewrites
    // The first call after an upload builds in a new tree group, which replaces the uploaded tree only once the clustered tree is
    // known to fit the traversal stack.  The first call after rt_rebuild_bvh adds the clustering temporaries to its group.
    TreeGroup fresh;
    const bool install = !c->lbvh.live;
    rt_ctx::Lbvh& L = install ? fresh.L : c->lbvh;
    if (!L.ploc.clusters)
    {
        DevAllocs g;
        cudaError_t e = install ? alloc_tree(c, fresh) : cudaSuccess;
        if (e == cudaSuccess) e = alloc_ploc(c, g, L.ploc);
        if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
        if (e != cudaSuccess) RT_FAIL(c, RT_ERR_CUDA, "rt_rebuild_bvh_ploc: allocating the rebuilt tree: %s", cudaGetErrorString(e));
        (install ? fresh.mem : c->tree_mem).adopt(std::move(g));
    }
    rt_ctx::Lbvh::Ploc& P = L.ploc;
    const uint32_t n = (uint32_t)c->n_tris;
    // Plain launches only, as in rt_rebuild_bvh.
    const uint32_t* ipre = nullptr; const uint32_t* ids = nullptr;
    int rc;
    if (n > 1)
    {
        cub::DoubleBuffer<uint32_t> keys(L.codes[0], L.codes[1]), vals(L.ids[0], L.ids[1]);
        // k_lbvh_keys' end-of-leaf flags land in the cluster list (48 of its 64 bytes per triangle), which k_ploc_init then
        // overwrites: nothing of the current tree changes before the depth check (k_ploc_flags writes the flags after it)
        if ((rc = sort_keys(c, L, (float4*)P.clusters, keys, vals))) return rc;
        RT_CUDA(c, cudaMemsetAsync(P.parent, 0xFF, (2ull * n - 1) * 4, c->stream));
        RT_CUDA(c, cudaMemsetAsync(P.made, 0, 4, c->stream));
        {
            TimedLaunch t(c, RT_K_MISC);
            k_ploc_init<<<grid_for(n), 256, 0, c->stream>>>(vals.Current(), n, c->scene.tris_ref, P.clusters);
            if ((rc = post_launch(c, "k_ploc_init"))) return rc;
        }
        PlocCluster *cur = P.clusters, *next = P.clusters + n;
        for (uint32_t count = n; count > 1; std::swap(cur, next))
        {
            {
                TimedLaunch t(c, RT_K_MISC);
                k_ploc_nearest<<<grid_for(count, RT_PLOC_TILE), RT_PLOC_TILE, 0, c->stream>>>(cur, count, P.nn);
                if ((rc = post_launch(c, "k_ploc_nearest"))) return rc;
            }
            {
                TimedLaunch t(c, RT_K_MISC);
                k_ploc_merge<<<grid_for(count), 256, 0, c->stream>>>(cur, count, P.nn, P.keep, n, P.made, P.inner, P.size, P.parent);
                if ((rc = post_launch(c, "k_ploc_merge"))) return rc;
            }
            {
                TimedLaunch t(c, RT_K_MISC);
                size_t bytes = P.select_bytes;
                RT_CUDA(c, cub::DeviceSelect::Flagged(P.select_tmp, bytes, cur, P.keep, next, P.host, (int)count, c->stream));
                if ((rc = post_launch(c, "DeviceSelect"))) return rc;
            }
            RT_CUDA(c, cudaStreamSynchronize(c->stream));
            if (P.host[0] >= count) RT_FAIL(c, RT_ERR_CUDA, "rt_rebuild_bvh_ploc: an iteration merged no pair");
            count = P.host[0];
        }
        uint32_t* leaf_ids = keys.Current(); uint32_t* pre = vals.Alternate();      // the codes and the sort's inputs are dead
        P.host[1] = 0;
        {
            TimedLaunch t(c, RT_K_MISC);
            k_ploc_number<<<grid_for(2 * n - 1), 256, 0, c->stream>>>(n, P.inner, P.size, P.parent, leaf_ids, L.inner, pre, P.host + 1);
            if ((rc = post_launch(c, "k_ploc_number"))) return rc;
        }
        RT_CUDA(c, cudaStreamSynchronize(c->stream));
        if (P.host[1])
            RT_FAIL(c, RT_ERR_UNSUPPORTED, "rt_rebuild_bvh_ploc: the clustered tree is deeper than the 64 levels of the traversal "
                    "stack; the tree is unchanged (rt_rebuild_bvh builds a tree of at most 62 levels over any triangles)");
        ipre = pre; ids = leaf_ids;
    }
    if (install)
    {
        RT_CUDA(c, cudaStreamSynchronize(c->stream));
        install_tree(c, fresh);
    }
    if (n > 1)
    {
        TimedLaunch t(c, RT_K_MISC);
        k_ploc_flags<<<grid_for(n), 256, 0, c->stream>>>(n, (float4*)c->scene.wtris);
        if ((rc = post_launch(c, "k_ploc_flags"))) return rc;
    }
    if ((rc = write_tree(c, ipre, ids))) return rc;
    if (n_nodes) *n_nodes = c->n_nodes;
    return RT_OK;
}

int rt_set_camera(rt_ctx* c, const RtCamera* cam)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_set_camera(k, cam));
    if (!cam) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_set_camera: null camera");
    c->camera = *cam;
    c->aov_prev_camera = c->prev_camera;        // the AOV kernel sees the camera of the previous SetCameraData call
    c->prev_camera = *cam;                      // (cl_pt_integrator.cpp:365-371; zero-initialised before the first call)
    RayGenConsts& r = c->raygen;
    r.position = f3{ cam->position.x, cam->position.y, cam->position.z };
    r.front = f3{ cam->front.x, cam->front.y, cam->front.z };
    r.up = f3{ cam->up.x, cam->up.y, cam->up.z };
    // cross(front, up), raygeneration.cl:112 — plain float ops on the host (no contraction: -fmad=false
    // applies to host code too, and x86-64 has no implicit FMA)
    r.right = f3{ r.front.y * r.up.z - r.front.z * r.up.y, r.front.z * r.up.x - r.front.x * r.up.z, r.front.x * r.up.y - r.front.y * r.up.x };
    r.tan_half_fov = rt_tanf(0.5f * cam->fov);        // raygeneration.cl:108, uniform over the frame
    r.aspect_ratio = cam->aspect_ratio;
    r.aperture = cam->aperture; r.focus_distance = cam->focus_distance;
    r.inv_width = 1.0f / (float)c->width; r.inv_height = 1.0f / (float)c->height;
    c->camera_ready = true;
    return RT_OK;
}

int rt_set_option(rt_ctx* c, int key, uint32_t value)
{
    RT_CHECK_CTX(c);
    if (key == RT_OPT_PRESENT)
    {
        if (value > 1) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "present mode must be 0 (parallel read-back) or 1 (gather to the first device)");
        if (value == 1)
            for (rt_ctx* k : c->children)
                if (adaptive_wanted(k))
                    RT_FAIL(c, RT_ERR_UNSUPPORTED, "RT_OPT_PRESENT 1 is not available with adaptive sampling (the gathered resolve has no per-pixel sample counts)");
        c->present = (int)value;
        if (!c->children.empty())
        {   // gather presentation: the children push their pixels into a buffer on the first device while they render (fused gather)
            rt_ctx* k0 = c->children[0];
            void* buf = nullptr; uint64_t stride = 0;
            if (value == 1) { int rc = rt_gather_buffer(k0, &buf, &stride, nullptr); if (rc) { c->error = k0->error; return rc; } }
            for (rt_ctx* k : c->children) { int rc = rt_set_gather_target(k, value == 1 ? buf : nullptr, stride); if (rc) { c->error = k->error; return rc; } }
        }
        return RT_OK;
    }
    RT_FANOUT(c, rt_set_option(k, key, value));
    ++c->config_gen;
    switch (key)
    {
    case RT_OPT_WHITE_FURNACE:
        if ((value != 0) == (c->white_furnace != 0)) return RT_OK;
        c->white_furnace = value != 0;
        return (c->emitter_sampling || c->env_sampling) ? refresh_lights(c) : RT_OK;
    case RT_OPT_EMITTER_SAMPLING:
        if (value > 1) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "emitter sampling must be 0 (off) or 1 (emissive triangles with MIS)");
        if (value == 1 && c->scene_ready && c->instanced)
            RT_FAIL(c, RT_ERR_UNSUPPORTED, "emitter sampling is not available on instanced scenes");
        if (value == 1 && c->scene_ready)
        {
            std::string err;
            if (!rtemit::check_indices(c->emit_idx.data(), c->emit_idx.size(), c->emit_n_tris, err))
                RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "emitter sampling: the uploaded scene's %s", err.c_str());
        }
        if ((int)value == c->emitter_sampling) return RT_OK;
        c->emitter_sampling = (int)value;
        return refresh_lights(c);
    case RT_OPT_ENV_SAMPLING:
        if (value > 1) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "environment sampling must be 0 (off) or 1 (the environment map with MIS)");
        if ((int)value == c->env_sampling) return RT_OK;
        c->env_sampling = (int)value;
        return refresh_lights(c);
    case RT_OPT_OBJECT_MOTION:
        if (value > 1) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "object motion must be 0 (camera-only motion vectors) or 1 (triangle updates too)");
        if ((int)value == c->object_motion) return RT_OK;
        RT_CUDA(c, cudaSetDevice(c->device));
        if (value == 0)
        {   // a frame in flight may still read the previous positions
            RT_CUDA(c, cudaStreamSynchronize(c->stream));
            c->motion_mem.clear(); c->prev_pos = nullptr; c->object_motion = 0;
            return RT_OK;
        }
        c->object_motion = 1;
        return c->scene_ready ? set_prev_positions(c) : RT_OK;
    case RT_OPT_SAMPLER:
        if (value > 1) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "sampler type must be 0 (kRandom) or 1 (kBlueNoise)");
        if (value == 1 && !c->d_bn)
            RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "kBlueNoise needs the sampler tables: call rt_upload_sampler_tables first");
        c->sampler = (int)value; return RT_OK;
    case RT_OPT_AOV:
        if (value > 4) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "AOV index out of range");
        c->aov = (int)value;
        if (aov_wanted(c)) { RT_CUDA(c, cudaSetDevice(c->device)); return ensure_aov_buffers(c); }
        return RT_OK;
    case RT_OPT_DENOISER:
        if (value != 0 && c->world != 1)
            RT_FAIL(c, RT_ERR_UNSUPPORTED, "the temporal denoiser reprojects across the whole image and is not available with a multi-GPU partition");
        if (value != 0 && adaptive_wanted(c))
            RT_FAIL(c, RT_ERR_UNSUPPORTED, "the temporal denoiser is not available with adaptive sampling (it replaces the radiance every frame)");
        c->denoiser = value != 0;
        if (aov_wanted(c)) { RT_CUDA(c, cudaSetDevice(c->device)); return ensure_aov_buffers(c); }
        return RT_OK;
    case RT_OPT_AOV_ALWAYS:
        c->aov_always = value != 0;
        if (aov_wanted(c)) { RT_CUDA(c, cudaSetDevice(c->device)); return ensure_aov_buffers(c); }
        return RT_OK;
    case RT_OPT_COUNT_TRAVERSAL: c->count_traversal = value != 0; return RT_OK;
    case RT_OPT_KERNEL_TIMING: c->kernel_timing = value != 0; return RT_OK;
    case RT_OPT_GRAPH: c->use_graph = value != 0; return RT_OK;
    case RT_OPT_PDL: c->pdl = value != 0; return RT_OK;
    case RT_OPT_FRAME_THREADS:
        if (value != 0 && (value % 32 != 0 || value > RT_FRAME_MAX_THREADS)) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "frame-kernel CTA size must be 0 (automatic) or a multiple of 32 up to 1024");
        c->frame_threads = (int)value; return RT_OK;
    case RT_OPT_FRAME_KERNEL:
        if (value > 2) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "frame-kernel mode must be 0 (per-phase kernels), 1 (one kernel per frame) or 2 (by partition size)");
        c->frame_kernel = (int)value; return RT_OK;
    case RT_OPT_SMEM_BVH: c->smem_bvh = value != 0; return RT_OK;
    case RT_OPT_OCTANT_BVH: c->octant_bvh = value != 0; return RT_OK;
    case RT_OPT_TOP_SMEM:
        if (value > 640u) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "at most 640 top-of-tree records (40 KB per CTA) can be staged");
        c->top_smem_records = value; return RT_OK;
    case RT_OPT_OVERLAP:
    {
        if (value > 2) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "overlap mode must be 0, 1 or 2");
        int rt_j_ = join_shadow(c); if (rt_j_) return rt_j_;
        c->overlap = (int)value; return RT_OK;
    }
    case RT_OPT_TRAVERSAL:
        if (value > 1) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "traversal mode must be 0 (literal) or 1 (child-box layout)");
        { int rt_j_ = join_shadow(c); if (rt_j_) return rt_j_; }
        c->traversal = (int)value; return RT_OK;
    }
    RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "unknown option key %d", key);
}

int rt_upload_sampler_tables(rt_ctx* c, const int32_t* sobol, const int32_t* scrambling, const int32_t* ranking)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_upload_sampler_tables(k, sobol, scrambling, ranking));
    if (!sobol || !scrambling || !ranking) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_upload_sampler_tables: null table");
    for (int i = 0; i < RT_BN_TILE_COUNT; ++i)
        if (ranking[i] < 0 || ranking[i] > 255)
            RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_upload_sampler_tables: ranking entry %d is %d, outside 0..255", i, ranking[i]);
    RT_CUDA(c, cudaSetDevice(c->device));
    int rt_j_ = join_shadow(c); if (rt_j_) return rt_j_;
    RT_CUDA(c, cudaStreamSynchronize(c->stream));
    const size_t n = (size_t)RT_BN_SOBOL_COUNT + 2 * (size_t)RT_BN_TILE_COUNT;
    if (!c->d_bn) RT_CUDA(c, c->ctx_mem.alloc(c->d_bn, n));
    RT_CUDA(c, cudaMemcpy(c->d_bn, sobol, RT_BN_SOBOL_COUNT * sizeof(int), cudaMemcpyHostToDevice));
    RT_CUDA(c, cudaMemcpy(c->d_bn + RT_BN_SOBOL_COUNT, scrambling, RT_BN_TILE_COUNT * sizeof(int), cudaMemcpyHostToDevice));
    RT_CUDA(c, cudaMemcpy(c->d_bn + RT_BN_SOBOL_COUNT + RT_BN_TILE_COUNT, ranking, RT_BN_TILE_COUNT * sizeof(int), cudaMemcpyHostToDevice));
    ++c->config_gen;
    return RT_OK;
}

int rt_reset(rt_ctx* c)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_reset(k));
    { int rt_j_ = join_shadow(c); if (rt_j_) return rt_j_; }
    { int rc = frame_buffers_ready(c); if (rc) return rc; }
    RT_CUDA(c, cudaSetDevice(c->device));
    if (!c->denoiser) c->sample_count = 0;                                   // cl_pt_integrator.cpp:499-504
    // the adaptive-sampling setting takes effect here; a changed setting changes the frame's launch arguments
    if (c->ad_error != c->ad_req_error || c->ad_min != c->ad_req_min) ++c->config_gen;
    c->ad_error = c->ad_req_error; c->ad_min = c->ad_req_min;
    if (adaptive_on(c)) { int rc = reset_adaptive(c); if (rc) return rc; }
    else if (!c->ad_mem.empty())
    {   // the per-pixel state exists only while the setting is on
        cudaStreamSynchronize(c->stream);
        c->ad_mem.clear(); c->ad = {}; ++c->config_gen;
    }
    TimedLaunch t(c, RT_K_MISC);
    k_reset<<<grid_for(c->n_local), 256, 0, c->stream>>>(c->radiance, c->n_local);
    return post_launch(c, "k_reset");
}

int rt_advance_sample_count(rt_ctx* c)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_advance_sample_count(k));
    int rc = join_shadow(c); if (rc) return rc;     // end of the bounce loop: everything of this frame is ordered on the render stream
    if (adaptive_on(c))
    {
        if ((rc = frame_buffers_ready(c))) return rc;
        RT_CUDA(c, cudaSetDevice(c->device));
        if ((rc = launch_adaptive_update(c))) return rc;
    }
    ++c->sample_count;
    return RT_OK;
}

int rt_set_adaptive_sampling(rt_ctx* c, float max_error, uint32_t min_samples)
{
    RT_CHECK_CTX(c);
    const bool on = max_error > 0.0f;
    if (!(max_error == 0.0f || (on && std::isfinite(max_error) && min_samples >= 2)))
        RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_set_adaptive_sampling: need max_error == 0 (off), or a finite max_error > 0 and min_samples >= 2");
    if (on && c->denoiser)
        RT_FAIL(c, RT_ERR_UNSUPPORTED, "adaptive sampling is not available with the temporal denoiser (it replaces the radiance every frame)");
    if (on && !c->children.empty() && c->present == 1)
        RT_FAIL(c, RT_ERR_UNSUPPORTED, "adaptive sampling is not available with RT_OPT_PRESENT 1 (the gathered resolve has no per-pixel sample counts)");
    if (on && c->gather_slab)
        RT_FAIL(c, RT_ERR_UNSUPPORTED, "adaptive sampling is not available with a fused-gather target (stopped pixels are never pushed)");
    RT_FANOUT(c, rt_set_adaptive_sampling(k, max_error, min_samples));
    c->ad_req_error = on ? max_error : 0.0f; c->ad_req_min = on ? min_samples : 0u;
    return RT_OK;
}

int rt_set_spatial_denoiser(rt_ctx* c, uint32_t iterations, float sigma_color, float sigma_normal, float sigma_depth)
{
    RT_CHECK_CTX(c);
    auto ok = [](float s) { return std::isfinite(s) && s >= 0.0f; };
    if (iterations > 5 || !ok(sigma_color) || !ok(sigma_normal) || !ok(sigma_depth))
        RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_set_spatial_denoiser: need iterations <= 5 and finite sigmas >= 0");
    if (iterations != 0 && !c->children.empty())
        RT_FAIL(c, RT_ERR_UNSUPPORTED, "the spatial denoiser is not available on a multi-device context (neighbouring rows live on other devices)");
    if (iterations != 0 && c->world != 1)
        RT_FAIL(c, RT_ERR_UNSUPPORTED, "the spatial denoiser is not available with a multi-GPU partition (neighbouring rows live on other ranks)");
    RT_CUDA(c, cudaSetDevice(c->device));
    if ((iterations != 0) != (c->sd_iters != 0)) ++c->config_gen;   // the frames produce the AOVs or stop doing so: re-capture
    c->sd_iters = iterations;
    c->sd_sigma_c = sigma_color; c->sd_sigma_n = sigma_normal; c->sd_sigma_z = sigma_depth;
    if (iterations != 0) return ensure_aov_buffers(c);
    if (!c->sd_mem.empty())
    {   // the scratch planes exist only while the filter is on
        if (c->copy_stream) RT_CUDA(c, cudaStreamSynchronize(c->copy_stream));
        RT_CUDA(c, cudaStreamSynchronize(c->stream));
        c->sd_mem.clear();
        c->sd_col[0] = c->sd_col[1] = c->sd_guide = nullptr;
    }
    return RT_OK;
}

int rt_set_light_selection(rt_ctx* c, float analytic, float emitters, float environment)
{
    RT_CHECK_CTX(c);
    auto ok = [](float w) { return std::isfinite(w) && w > 0.0f; };
    if (!ok(analytic) || !ok(emitters) || !ok(environment) || !std::isfinite((analytic + emitters) + environment))
        RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_set_light_selection: every weight must be finite and > 0, and so must their sum");
    RT_FANOUT(c, rt_set_light_selection(k, analytic, emitters, environment));
    if (c->light_w[0] == analytic && c->light_w[1] == emitters && c->light_w[2] == environment) return RT_OK;
    c->light_w[0] = analytic; c->light_w[1] = emitters; c->light_w[2] = environment;
    return (c->emitter_sampling || c->env_sampling) ? refresh_lights(c) : RT_OK;
}

int rt_read_pixel_samples(rt_ctx* c, uint32_t* counts)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_read_pixel_samples(k, counts));
    { int rt_j_ = join_shadow(c); if (rt_j_) return rt_j_; }
    if (!counts) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_read_pixel_samples: null destination");
    if (!adaptive_on(c))
    {
        for (uint32_t r = 0; r < c->local_rows; ++r)
            std::fill_n(counts + ((size_t)c->rank + (size_t)r * c->world) * c->width, c->width, c->sample_count);
        return RT_OK;
    }
    RT_CUDA(c, cudaSetDevice(c->device));
    if (c->local_rows)
        RT_CUDA(c, cudaMemcpy2DAsync(counts + (size_t)c->rank * c->width, (size_t)c->world * c->width * 4, c->ad.count,
                                     (size_t)c->width * 4, (size_t)c->width * 4, c->local_rows, cudaMemcpyDeviceToHost, c->stream));
    RT_CUDA(c, cudaStreamSynchronize(c->stream));
    return RT_OK;
}

int rt_read_active_pixels(rt_ctx* c, uint32_t* n_active)
{
    RT_CHECK_CTX(c);
    if (!n_active) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_read_active_pixels: null destination");
    if (!c->children.empty())
    {
        uint32_t sum = 0, part = 0;
        for (rt_ctx* k : c->children) { int rc = rt_read_active_pixels(k, &part); if (rc) { c->error = k->error; return rc; } sum += part; }
        *n_active = sum;
        return RT_OK;
    }
    { int rt_j_ = join_shadow(c); if (rt_j_) return rt_j_; }
    if (!adaptive_on(c)) { *n_active = c->n_local; return RT_OK; }
    RT_CUDA(c, cudaSetDevice(c->device));
    RT_CUDA(c, cudaMemcpyAsync(n_active, &c->ad.ctl->n_active, 4, cudaMemcpyDeviceToHost, c->stream));
    RT_CUDA(c, cudaStreamSynchronize(c->stream));
    return RT_OK;
}

// A frame starts on one device: counters cleared, the frame constants set, and with `raygen` the full primary-ray queue (k_raygen).
// Without it the bounce-0 traversal of rt_extend_shade generates the primary rays itself (k_trace_primary).
static int begin_frame(rt_ctx* c, bool raygen)
{
    { int rt_j_ = join_shadow(c); if (rt_j_) return rt_j_; }
    int rc = require_ready(c); if (rc) return rc;
    RT_CUDA(c, cudaSetDevice(c->device));
    RT_CUDA(c, cudaMemsetAsync(c->counters, 0, sizeof(DevCounters), c->stream));
    c->stats_summed = false;
    TimedLaunch t(c, RT_K_RAYGEN);
    {
        FrameDyn dyn = frame_dyn(c);
        k_set_frame<<<1, 1, 0, c->stream>>>(c->d_dyn, dyn);
        ++c->launches;
    }
    if (raygen) k_raygen<<<grid_for(c->n_local), 256, 0, c->stream>>>(frame_params(c), c->q, c->counters, aov_params(c));
    note_frame_aovs(c);
    c->frame_started = true;
    c->primary_fused = !raygen;
    return post_launch(c, raygen ? "k_raygen" : "k_set_frame");
}

int rt_generate_rays(rt_ctx* c)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_generate_rays(k));
    return begin_frame(c, true);
}

#define RT_BOUNCE_CHECK(c, b)                                                                                   \
    do {                                                                                                        \
        int rt_rc_ = require_ready(c); if (rt_rc_) return rt_rc_;                                               \
        if ((b) > RT_MAX_BOUNCES) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "bounce %u exceeds RT_MAX_BOUNCES", (b)); \
        if (!(c)->frame_started) RT_FAIL(c, RT_ERR_NOT_READY, "rt_generate_rays has not been called");          \
        RT_CUDA(c, cudaSetDevice((c)->device));                                                                 \
    } while (0)

int rt_intersect(rt_ctx* c, uint32_t bounce)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_intersect(k, bounce));
    { int rt_j_ = join_shadow(c); if (rt_j_) return rt_j_; } RT_BOUNCE_CHECK(c, bounce);
    TimedLaunch t(c, RT_K_INTERSECT);
    launch_traversal<STEPWISE>(c, [&](auto count, auto smem, const auto& sc, size_t) {
        k_intersect<count.value, smem.value == RT_SMEM_INST><<<grid_for(c->n_local), 256, 0, c->stream>>>(frame_params(c), sc, c->traversal, c->q, c->counters, bounce);
    });
    return post_launch(c, "k_intersect");
}

/* ComputeAOVs: the AOV outputs are produced by the bounce-0 shading pass (it already holds the hit, the interpolated
 * normal and the unpacked material), so this step only makes sure the buffers exist when a view or the denoiser
 * needs them; with the default view (shaded colour, no denoiser) no AOV work is done at all. */
int rt_compute_aovs(rt_ctx* c)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_compute_aovs(k));
    if (!aov_wanted(c)) return RT_OK;
    RT_CUDA(c, cudaSetDevice(c->device));
    return ensure_aov_buffers(c);
}

int rt_shade_miss(rt_ctx* c, uint32_t bounce)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_shade_miss(k, bounce));
    { int rt_j_ = join_shadow(c); if (rt_j_) return rt_j_; } RT_BOUNCE_CHECK(c, bounce);
    TimedLaunch t(c, RT_K_MISS);
    (lights_sampled(c) ? k_shade_miss<true> : k_shade_miss<false>)<<<grid_for(c->n_local), 256, 0, c->stream>>>(frame_params(c), c->scene, c->q, c->counters, c->radiance, bounce);
    return post_launch(c, "k_shade_miss");
}

int rt_clear_outgoing_counter(rt_ctx* c, uint32_t) { RT_CHECK_CTX(c); return RT_OK; }
int rt_clear_shadow_counter(rt_ctx* c) { RT_CHECK_CTX(c); return RT_OK; }

int rt_shade_hits(rt_ctx* c, uint32_t bounce)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_shade_hits(k, bounce));
    { int rt_j_ = join_shadow(c); if (rt_j_) return rt_j_; } RT_BOUNCE_CHECK(c, bounce);
    c->cur_bounce = bounce;
    TimedLaunch t(c, RT_K_HIT);
    with_scene(c, [&](auto inst, const auto& sc) {
        (lights_sampled(c) ? k_shade_hits<true, inst.value> : k_shade_hits<false, inst.value>)<<<grid_for(c->n_local), 256, 0, c->stream>>>(frame_params(c), sc, c->q, c->counters, c->radiance, bounce, aov_params(c));
    });
    return post_launch(c, "k_shade_hits");
}

int rt_intersect_shadow(rt_ctx* c)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_intersect_shadow(k));
    { int rt_j_ = join_shadow(c); if (rt_j_) return rt_j_; } RT_BOUNCE_CHECK(c, c->cur_bounce);
    TimedLaunch t(c, RT_K_INTERSECT_SHADOW);
    launch_traversal<STEPWISE>(c, [&](auto count, auto smem, const auto& sc, size_t) {
        k_intersect_shadow<count.value, smem.value == RT_SMEM_INST><<<grid_for(c->n_local), 256, 0, c->stream>>>(frame_params(c), sc, c->traversal, c->q, c->counters, c->cur_bounce);
    });
    return post_launch(c, "k_intersect_shadow");
}

int rt_accumulate_direct(rt_ctx* c)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_accumulate_direct(k));
    { int rt_j_ = join_shadow(c); if (rt_j_) return rt_j_; } RT_BOUNCE_CHECK(c, c->cur_bounce);
    TimedLaunch t(c, RT_K_ACCUMULATE);
    k_accumulate<<<grid_for(c->n_local), 256, 0, c->stream>>>(frame_params(c), c->q, c->counters, c->radiance, c->cur_bounce);
    return post_launch(c, "k_accumulate");
}

int rt_denoise(rt_ctx* c)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_denoise(k));
    { int rt_j_ = join_shadow(c); if (rt_j_) return rt_j_; }
    if (!c->denoiser) return RT_OK;
    if (c->world != 1) RT_FAIL(c, RT_ERR_UNSUPPORTED, "temporal denoiser is single-GPU only");
    RT_CUDA(c, cudaSetDevice(c->device));
    int rc = frame_buffers_ready(c); if (rc || (rc = ensure_aov_buffers(c))) return rc;
    TimedLaunch t(c, RT_K_MISC);
    k_temporal<<<grid_for(c->n_local), 256, 0, c->stream>>>(c->width, c->height, c->radiance, c->prev_radiance, c->aov_depth, c->prev_depth, c->aov_velocity);
    return post_launch(c, "k_temporal");
}

int rt_copy_history(rt_ctx* c)
{   // cl_pt_integrator.cpp:670-675
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_copy_history(k));
    { int rt_j_ = join_shadow(c); if (rt_j_) return rt_j_; }
    if (!c->denoiser) return RT_OK;
    RT_CUDA(c, cudaSetDevice(c->device));
    int rc = frame_buffers_ready(c); if (rc || (rc = ensure_aov_buffers(c))) return rc;
    RT_CUDA(c, cudaMemcpyAsync(c->prev_radiance, c->radiance, (size_t)c->n_local * 16, cudaMemcpyDeviceToDevice, c->stream));
    RT_CUDA(c, cudaMemcpyAsync(c->prev_depth, c->aov_depth, (size_t)c->n_local * 4, cudaMemcpyDeviceToDevice, c->stream));
    return RT_OK;
}

int rt_extend_shade(rt_ctx* c, uint32_t bounce)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_extend_shade(k, bounce)); RT_BOUNCE_CHECK(c, bounce);
    c->cur_bounce = bounce;
    if (c->shadow_deferred && merged_trace_available(c))
    {   // this bounce's closest-hit traversal + the previous bounce's shadow pass in one kernel
        c->shadow_deferred = false;
        TimedLaunch t(c, RT_K_TRACE_BOTH);
        launch_traversal<MERGED>(c, [&](auto, auto smem, const auto& sc, size_t sm) {
            auto* k = k_trace_both<smem.value>;
            launch_chain(c, k, RT_PGRID(c, k, sm), sm, c->stream, frame_params(c), sc, c->traversal, c->q, c->counters, c->radiance, bounce, c->shadow_deferred_bounce);
        });
        int rc = post_launch(c, "k_trace_both"); if (rc) return rc;
    }
    else if (bounce == 0 && c->primary_fused)
    {   // the frame's primary rays are generated here (begin_frame without k_raygen)
        c->primary_fused = false;
        TimedLaunch t(c, RT_K_TRACE_CLOSEST);
        launch_traversal<PER_PHASE>(c, [&](auto count, auto smem, const auto& sc, size_t sm) {
            auto* k = k_trace_primary<count.value, smem.value>;
            if (count) k<<<RT_PGRID(c, k, sm), 256, sm, c->stream>>>(frame_params(c), sc, c->traversal, c->q, c->counters, aov_params(c));
            else launch_chain(c, k, RT_PGRID(c, k, sm), sm, c->stream, frame_params(c), sc, c->traversal, c->q, c->counters, aov_params(c));
        });
        int rc = post_launch(c, "k_trace_primary"); if (rc) return rc;
    }
    else
    {
        TimedLaunch t(c, RT_K_TRACE_CLOSEST);
        launch_traversal<PER_PHASE>(c, [&](auto count, auto smem, const auto& sc, size_t sm) {
            auto* k = k_trace_closest<count.value, smem.value>;
            if (count) k<<<RT_PGRID(c, k, sm), 256, sm, c->stream>>>(frame_params(c), sc, c->traversal, c->q, c->counters, bounce);
            else launch_chain(c, k, RT_PGRID(c, k, sm), sm, c->stream, frame_params(c), sc, c->traversal, c->q, c->counters, bounce);
        });
        int rc = post_launch(c, "k_trace_closest"); if (rc) return rc;
    }
    { int rc = join_shadow(c); if (rc) return rc; }     // the shading pass accumulates into radiance and refills the shadow queue
    TimedLaunch t(c, RT_K_SHADE_QUEUES);
    const bool sort = sorted_shading(c);
    const size_t sm = sort ? sizeof(ContStage) : 0;
    with_scene(c, [&](auto inst, const auto& sc) {
        auto* k = lights_sampled(c) ? (sort ? k_shade_queues<true, true, inst.value> : k_shade_queues<false, true, inst.value>)
                                     : (sort ? k_shade_queues<true, false, inst.value> : k_shade_queues<false, false, inst.value>);
        launch_chain(c, k, RT_PGRID(c, k, sm), sm, c->stream, frame_params(c), sc, c->q, c->counters, c->radiance, bounce, aov_params(c), c->scene_mid);
    });
    return post_launch(c, "k_shade_queues");
}

// the second stream of RT_OPT_OVERLAP 1 and its two events
static int ensure_shadow_stream(rt_ctx* c)
{
    if (c->shadow_stream) return RT_OK;
    RT_CUDA(c, make_event(c->ev_shaded)); RT_CUDA(c, make_event(c->ev_shadowed));
    RT_CUDA(c, make_stream(c->shadow_stream));          // last: the stream marks the set complete
    return RT_OK;
}

static int launch_shadow_pass(rt_ctx* c, uint32_t bounce, cudaStream_t st)
{
    TimedLaunch t(c, RT_K_SHADOW_ACCUMULATE, st);
    launch_traversal<PER_PHASE>(c, [&](auto count, auto smem, const auto& sc, size_t sm) {
        auto* k = k_shadow_accumulate<count.value, smem.value>;
        k<<<RT_PGRID(c, k, sm), 256, sm, st>>>(frame_params(c), sc, c->traversal, c->q, c->counters, c->radiance, bounce);
    });
    return post_launch(c, "k_shadow_accumulate");
}

int rt_shadow_accumulate(rt_ctx* c, uint32_t bounce)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_shadow_accumulate(k, bounce)); RT_BOUNCE_CHECK(c, bounce);
    int rc = join_shadow(c); if (rc) return rc;
    // The shadow pass of bounce b only shares the radiance buffer with LATER shading passes, so it may overlap the
    // closest-hit traversal of bounce b+1 (which touches neither).
    if (c->overlap == 2 && merged_trace_available(c))
    {   // deferred: rt_extend_shade(b+1) runs it inside its traversal kernel; join_shadow() launches it for anyone else
        c->shadow_deferred = true; c->shadow_deferred_bounce = bounce;
        return RT_OK;
    }
    if (c->overlap != 1) return launch_shadow_pass(c, bounce, c->stream);
    // overlap 1: second stream; join_shadow() orders it before the next kernel that needs its results.  Both kernels are
    // persistent, so the second fills the SMs as the first drains.
    if ((rc = ensure_shadow_stream(c))) return rc;
    cudaStream_t st = c->shadow_stream;
    RT_CUDA(c, cudaEventRecord(c->ev_shaded, c->stream));
    RT_CUDA(c, cudaStreamWaitEvent(st, c->ev_shaded, 0));
    rc = launch_shadow_pass(c, bounce, st); if (rc) return rc;
    RT_CUDA(c, cudaEventRecord(c->ev_shadowed, st));
    c->shadow_pending = true;
    return RT_OK;
}

static int integrate_body(rt_ctx* c, uint32_t max_bounces)
{
    int rc = begin_frame(c, false); if (rc) return rc;      // rt_extend_shade(0) generates the primary rays
    for (uint32_t b = 0; b <= max_bounces; ++b)          // inclusive, integrator.cpp:37
    {
        if ((rc = rt_extend_shade(c, b))) return rc;
        if ((rc = rt_shadow_accumulate(c, b))) return rc;
    }
    return rt_advance_sample_count(c);      // joins the shadow stream: the frame is complete in render-stream order
}

// Captures one frame (both streams) into a graph.  Nothing executes during capture; host-side frame state is restored.
static int capture_frame_graph(rt_ctx* c, uint32_t max_bounces)
{
    c->graph_exec.reset(); c->graph.reset(); c->graph_set_frame_node = nullptr; c->graph_gen = 0;
    int rc = join_shadow(c); if (rc) return rc;
    if (c->overlap == 1 && (rc = ensure_shadow_stream(c))) return rc;      // created outside the capture
    const uint32_t saved_samples = c->sample_count, saved_bounce = c->cur_bounce;
    const uint64_t saved_launches = c->launches;
    const bool saved_started = c->frame_started, saved_aov_ready = c->aov_ready, saved_ad_fresh = c->ad_fresh;
    RT_CUDA(c, cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeThreadLocal));
    rc = integrate_body(c, max_bounces);
    cudaGraph_t captured = nullptr;
    cudaError_t e = cudaStreamEndCapture(c->stream, &captured);
    Owned<cudaGraph_t> graph(captured);
    c->graph_launches = c->launches - saved_launches;
    c->sample_count = saved_samples; c->cur_bounce = saved_bounce; c->launches = saved_launches; c->frame_started = saved_started;
    c->aov_ready = saved_aov_ready; c->ad_fresh = saved_ad_fresh;
    c->shadow_pending = false; c->shadow_deferred = false; c->primary_fused = false;
    if (rc) return rc;
    if (e != cudaSuccess) RT_FAIL(c, RT_ERR_CUDA, "cudaStreamEndCapture failed: %s", cudaGetErrorString(e));
    size_t n_nodes = 0;
    RT_CUDA(c, cudaGraphGetNodes(graph, nullptr, &n_nodes));
    std::vector<cudaGraphNode_t> nodes(n_nodes);
    RT_CUDA(c, cudaGraphGetNodes(graph, nodes.data(), &n_nodes));
    for (cudaGraphNode_t nd : nodes)
    {
        cudaGraphNodeType ty;
        RT_CUDA(c, cudaGraphNodeGetType(nd, &ty));
        if (ty != cudaGraphNodeTypeKernel) continue;
        cudaKernelNodeParams kp;
        RT_CUDA(c, cudaGraphKernelNodeGetParams(nd, &kp));
        if (kp.gridDim.x == 1 && kp.blockDim.x == 1 && !c->graph_set_frame_node)
        {   // k_set_frame is the only <<<1,1>>> launch of the frame and the first kernel of it
            c->graph_set_frame_node = nd; c->graph_set_frame_func = kp.func;
        }
    }
    if (!c->graph_set_frame_node) RT_FAIL(c, RT_ERR_CUDA, "frame graph has no k_set_frame node");
    cudaGraphExec_t exec = nullptr;
    e = cudaGraphInstantiate(&exec, graph, 0);
    if (e != cudaSuccess) RT_FAIL(c, RT_ERR_CUDA, "cudaGraphInstantiate failed: %s", cudaGetErrorString(e));
    c->graph_exec.reset(exec); c->graph = std::move(graph);
    c->graph_gen = c->config_gen; c->graph_max_bounces = max_bounces;
    return RT_OK;
}

// Which schedule rt_integrate runs, and the CTA shape of the one-kernel frame.  With a whole 1080p frame per GPU the per-phase
// kernels are at least as fast (specialised register budgets — 5 CTAs/SM of 48 registers for traversal — and one kind of code per
// SM at a time; on one H100 80GB HBM3: a tie within 1.5 % on CornellBox, 1 % ahead on ShaderBalls, DESIGN.md section 4); from
// half a 1080p frame down the
// launch boundaries and kernel tails of 20+ dependent launches cost more and the one-kernel frame wins.  RT_OPT_FRAME_KERNEL = 2
// switches at 7168 pixels per SM (0.95 M pixels on 132 SMs).
static bool frame_kernel_selected(const rt_ctx* c)
{
    if (c->instanced) return false;                // instanced scenes always run the per-phase kernels
    if (c->frame_kernel == 2) return (size_t)c->n_local <= (size_t)c->num_sms * 7168u;
    return c->frame_kernel == 1;
}

// CTA size of k_frame (measured during development on partitions of 1-8 GPUs, not re-measured on H100).  One 1024-thread CTA per SM keeps all 32 warps of an SM in the same phase — one kind
// of code in the instruction caches — and is the best shape when the BVH lives in shared memory (CornellBox, every partition
// size) or every warp still has several items per phase; scenes traversed through L1/L2 on small partitions (<= 4096 pixels
// per SM) prefer 4 CTAs of 256 threads per SM whose phases interleave.
static int frame_kernel_threads(const rt_ctx* c)
{
    if (c->frame_threads) return c->frame_threads;
    const int mode = bvh_stage(c).mode;
    if (mode == 1 || mode == 3) return 1024;      // the whole BVH in shared memory
    return (size_t)c->n_local > (size_t)c->num_sms * 4096u ? 1024 : 256;
}

// Fused gather, end of a frame: k_frame has pushed every pixel already (copy_slab false); the per-phase schedule pushes its whole
// slab with one device-to-device copy.  Then the completion flag.
static int gather_signal(rt_ctx* c, bool copy_slab)
{
    if (!c->gather_slab) return RT_OK;
    if (copy_slab && c->n_local)
        RT_CUDA(c, cudaMemcpyAsync(c->gather_slab, c->radiance, (size_t)c->n_local * 16, cudaMemcpyDefault, c->stream));
    ++c->gather_frame;
    c->gather_sample = c->sample_count;
    k_gather_signal<<<1, 1, 0, c->stream>>>(c->gather_flag, c->gather_frame);
    ++c->launches;
    return post_launch(c, "k_gather_signal");
}

// Launch shape of the one-kernel frame (k_frame): the CTAs that are resident at once, at most one per group of 32 pixels, and the
// slots of each CTA's region of every queue.
static int frame_kernel_grid(rt_ctx* c, const void* k, int threads, size_t sm, uint32_t& grid, uint32_t& slots_per_cta)
{
    const int per_sm = std::min(resident_per_sm(c, k, threads, sm), 32);
    const uint32_t n_groups = (c->n_local + 31u) / 32u;
    grid = (uint32_t)(c->num_sms * per_sm / c->grid_div);
    if (grid < (uint32_t)c->num_sms) grid = (uint32_t)c->num_sms;
    if (grid > n_groups) grid = n_groups;
    if (grid < 1) grid = 1;
    slots_per_cta = ((n_groups + grid - 1u) / grid) * 32u;
    if ((size_t)grid * slots_per_cta > c->n_alloc) RT_FAIL(c, RT_ERR_CUDA, "frame kernel: queue regions exceed the allocation");
    return RT_OK;
}

// Does a frame run as the one-kernel frame?  (The traversal counters and the kernel timing need the per-phase kernels.)
static bool one_kernel_frame(const rt_ctx* c) { return frame_kernel_selected(c) && !c->kernel_timing && !c->count_traversal; }

// The whole frame as ONE persistent kernel (k_frame): a counter clear and a launch.  It pushes the fused gather's pixels itself
// when `push`.  accumulate: the counters are not cleared, so k_frame's statistics add up over consecutive frames (every counter of
// k_frame is an atomic add except n_primary, which it sets, or adds to with adaptive sampling).  With adaptive sampling the
// convergence update follows the frame.
static int integrate_frame_kernel(rt_ctx* c, uint32_t max_bounces, bool accumulate = false, bool push = true)
{
    int rc = require_ready(c); if (rc) return rc;
    if ((rc = join_shadow(c))) return rc;
    RT_CUDA(c, cudaSetDevice(c->device));
    if (!accumulate) RT_CUDA(c, cudaMemsetAsync(c->counters, 0, sizeof(DevCounters), c->stream));
    const int threads = frame_kernel_threads(c);
    const FrameDyn dyn = frame_dyn(c);
    FrameParams fp = frame_params(c);
    fp.gather = push ? c->gather_slab : nullptr;
    rc = launch_traversal<FRAME>(c, [&](auto, auto smem, const DevScene& sc, size_t sm) -> int {
        auto* k = lights_sampled(c) ? k_frame<smem.value, true> : k_frame<smem.value>;
        uint32_t grid, slots_per_cta;
        int rc2 = frame_kernel_grid(c, (const void*)k, threads, sm, grid, slots_per_cta); if (rc2) return rc2;
        TimedLaunch t(c, RT_K_MISC);
        k<<<grid, threads, sm, c->stream>>>(fp, sc, c->traversal, c->q, c->counters, c->radiance, aov_params(c), max_bounces, slots_per_cta, dyn);
        return RT_OK;
    });
    if (rc || (rc = post_launch(c, "k_frame"))) return rc;
    note_frame_aovs(c);
    if (adaptive_on(c) && (rc = launch_adaptive_update(c))) return rc;
    c->frame_started = true; c->cur_bounce = max_bounces;
    ++c->sample_count;
    return RT_OK;
}

// One frame on the schedule rt_integrate selects, without the fused gather's completion signal.  *pushed: the frame kernel has
// pushed every pixel to the gather target already (otherwise the radiance slab has to be copied).
static int integrate_frame(rt_ctx* c, uint32_t max_bounces, bool* pushed)
{
    *pushed = false;
    if (one_kernel_frame(c)) { *pushed = true; return integrate_frame_kernel(c, max_bounces); }
    if (!c->use_graph || c->kernel_timing || c->count_traversal) return integrate_body(c, max_bounces);
    int rc = require_ready(c); if (rc) return rc;
    RT_CUDA(c, cudaSetDevice(c->device));
    if (!c->graph_exec || c->graph_gen != c->config_gen || c->graph_max_bounces != max_bounces)
        if ((rc = capture_frame_graph(c, max_bounces))) return rc;
    if ((rc = join_shadow(c))) return rc;
    // the one per-frame update: k_set_frame's by-value argument (sample index + camera constants)
    FrameDyn dyn = frame_dyn(c);
    FrameDyn* dst = c->d_dyn;
    void* args[2] = { &dst, &dyn };
    cudaKernelNodeParams kp;
    memset(&kp, 0, sizeof(kp));
    kp.func = c->graph_set_frame_func; kp.gridDim = dim3(1); kp.blockDim = dim3(1); kp.sharedMemBytes = 0; kp.kernelParams = args; kp.extra = nullptr;
    RT_CUDA(c, cudaGraphExecKernelNodeSetParams(c->graph_exec, c->graph_set_frame_node, &kp));
    RT_CUDA(c, cudaGraphLaunch(c->graph_exec, c->stream));
    note_frame_aovs(c);
    c->launches += c->graph_launches;
    c->frame_started = true; c->cur_bounce = max_bounces;
    ++c->sample_count;
    return RT_OK;
}

int rt_integrate(rt_ctx* c, uint32_t max_bounces)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_integrate(k, max_bounces));
    if (max_bounces > RT_MAX_BOUNCES) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "max_bounces %u exceeds RT_MAX_BOUNCES", max_bounces);
    c->stats_summed = false;
    c->emit_max_bounces = max_bounces;
    bool pushed = false;
    int rc = integrate_frame(c, max_bounces, &pushed); if (rc) return rc;
    return gather_signal(c, !pushed);
}

// A multi-sample call leaves its summed statistics in counters_sum, which only rt_read_frame_stats reads: the counters that the
// taps (rt_read_rays, rt_read_hits) take their entry counts from never exceed one frame's rays.
int rt_integrate_samples(rt_ctx* c, uint32_t max_bounces, uint32_t n_samples)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_integrate_samples(k, max_bounces, n_samples));
    if (max_bounces > RT_MAX_BOUNCES) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "max_bounces %u exceeds RT_MAX_BOUNCES", max_bounces);
    if (n_samples == 0) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_integrate_samples: n_samples must be at least 1");
    if (n_samples > 0xFFFFFFFFu - c->sample_count)
        RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_integrate_samples: the sample count %u + %u would wrap", c->sample_count, n_samples);
    if (n_samples > 1 && c->denoiser)
        RT_FAIL(c, RT_ERR_UNSUPPORTED, "rt_integrate_samples: the temporal denoiser runs once per sample; render one sample per call with it");
    if (n_samples == 1) return rt_integrate(c, max_bounces);
    c->emit_max_bounces = max_bounces;
    int rc = require_ready(c); if (rc) return rc;
    if ((rc = join_shadow(c))) return rc;
    RT_CUDA(c, cudaSetDevice(c->device));
    if (!c->counters_sum) RT_CUDA(c, c->ctx_mem.alloc(c->counters_sum, 1));
    RT_CUDA(c, cudaMemsetAsync(c->counters_sum, 0, sizeof(DevCounters), c->stream));
    c->stats_summed = false;
    bool pushed = true;
    if (one_kernel_frame(c))
    {   // n k_frame launches that add up their statistics in c->counters, folded into counters_sum once per batch (a batch stays
        // small enough that no 32-bit half of the packed 64-bit counters can carry into the other); only the last frame pushes
        // to the gather target
        const uint32_t batch = 0xFFFFFFFFu / std::max(c->n_local, 1u);
        for (uint32_t s = 0; s < n_samples; ++s)
        {
            if (s % batch == 0) RT_CUDA(c, cudaMemsetAsync(c->counters, 0, sizeof(DevCounters), c->stream));
            if ((rc = integrate_frame_kernel(c, max_bounces, true, s + 1 == n_samples))) return rc;
            if ((s + 1) % batch == 0 || s + 1 == n_samples)
            {   // with adaptive sampling k_frame adds up n_primary itself (it varies from frame to frame)
                TimedLaunch t(c, RT_K_MISC);
                k_add_counters<<<1, 256, 0, c->stream>>>(c->counters_sum, c->counters, adaptive_on(c) ? 1u : s % batch + 1);
                if ((rc = post_launch(c, "k_add_counters"))) return rc;
            }
        }
        RT_CUDA(c, cudaMemsetAsync(c->counters, 0, sizeof(DevCounters), c->stream));   // the taps find no rays of this call
    }
    else
    {   // n frames of the per-phase schedule: they clear the counters at the start of every frame (their queue cursors), so each
        // frame's statistics are added into counters_sum after it; the counters keep the last frame's, as after rt_integrate
        for (uint32_t s = 0; s < n_samples; ++s)
        {
            if ((rc = integrate_frame(c, max_bounces, &pushed))) return rc;
            TimedLaunch t(c, RT_K_MISC);
            k_add_counters<<<1, 256, 0, c->stream>>>(c->counters_sum, c->counters, 1u);
            if ((rc = post_launch(c, "k_add_counters"))) return rc;
        }
    }
    c->stats_summed = true;
    return gather_signal(c, !pushed);
}

// the resolve kernel of this context's rows into `out`, on its stream
// With the spatial denoiser on and the shaded-colour view, k_resolve writes into a scratch plane, a pack kernel gathers the guides,
// and the passes ping-pong between the scratch planes; the last pass writes `out`.  Every launch counts under RT_K_RESOLVE.
static int launch_resolve(rt_ctx* c, float4* out)
{
    const AovParams ap = aov_params(c);
    const int view = ap.enabled ? c->aov : 0;
    const bool filter = c->sd_iters != 0 && view == 0;
    if (filter)
    {
        if (!c->aov_ready)
            RT_FAIL(c, RT_ERR_NOT_READY, "the spatial denoiser needs the AOVs of a frame rendered with it on: render a frame first");
        const size_t n = std::max(c->n_local, 1u);
        for (float4** p : { &c->sd_col[0], &c->sd_col[1], &c->sd_guide })
            if (!*p) RT_CUDA(c, c->sd_mem.alloc(*p, n));
    }
    {
        TimedLaunch t(c, RT_K_RESOLVE);
        k_resolve<<<grid_for(c->n_local), 256, 0, c->stream>>>(c->radiance, filter ? c->sd_col[0] : out, c->n_local, c->sample_count, c->denoiser,
                                                               view, ap, adaptive_on(c) ? c->ad.count : nullptr);
        int rc = post_launch(c, "k_resolve"); if (rc) return rc;
    }
    if (!filter) return RT_OK;
    {
        TimedLaunch t(c, RT_K_RESOLVE);
        k_sd_pack<<<grid_for(c->n_local), 256, 0, c->stream>>>(c->aov_normal, c->aov_depth, c->sd_guide, c->n_local);
        int rc = post_launch(c, "k_sd_pack"); if (rc) return rc;
    }
    const float kc = c->sd_sigma_c > 0.0f ? 1.0f / (c->sd_sigma_c * c->sd_sigma_c) : 0.0f;
    const float kn = c->sd_sigma_n > 0.0f ? 1.0f / (c->sd_sigma_n * c->sd_sigma_n) : 0.0f;
    const dim3 block(32, 8), grid((c->width + 31u) / 32u, (c->local_rows + 7u) / 8u);
    for (uint32_t i = 0; i < c->sd_iters; ++i)
    {
        const float4* src = c->sd_col[i & 1u];
        float4* dst = (i + 1 == c->sd_iters) ? out : c->sd_col[(i + 1) & 1u];
        TimedLaunch t(c, RT_K_RESOLVE);
        if (c->local_rows)
            k_sd_pass<<<grid, block, 0, c->stream>>>(src, dst, c->sd_guide, c->width, c->local_rows, 1 << i, kc * (float)(1u << i), kn, c->sd_sigma_z);
        int rc = post_launch(c, "k_sd_pass"); if (rc) return rc;
    }
    return RT_OK;
}

// the pipelined read-back's copy stream and its events
static int ensure_copy_stream(rt_ctx* c)
{
    if (c->copy_stream) return RT_OK;
    for (int i = 0; i < 2; ++i) { RT_CUDA(c, make_event(c->resolve_done[i])); RT_CUDA(c, make_event(c->copy_done[i])); }
    RT_CUDA(c, make_stream(c->copy_stream));            // last: the stream marks the set complete
    return RT_OK;
}

// resolve kernel + device->host copy of this context's rows, enqueued on its stream (no synchronisation)
static int resolve_enqueue(rt_ctx* c, float* dst)
{
    { int rt_j_ = join_shadow(c); if (rt_j_) return rt_j_; }
    { int rc = frame_buffers_ready(c); if (rc) return rc; }
    RT_CUDA(c, cudaSetDevice(c->device));
    if (c->copy_pending[0]) RT_CUDA(c, cudaStreamWaitEvent(c->stream, c->copy_done[0], 0));   // rt_resolve_async may still copy out of c->resolved
    { int rc = launch_resolve(c, c->resolved); if (rc) return rc; }
    if (dst && c->local_rows)
        RT_CUDA(c, cudaMemcpy2DAsync(dst + (size_t)c->rank * c->width * 4, (size_t)c->world * c->width * 16, c->resolved,
                                     (size_t)c->width * 16, (size_t)c->width * 16, c->local_rows, cudaMemcpyDeviceToHost, c->stream));
    return RT_OK;
}

int rt_resolve(rt_ctx* c, float* dst)
{
    RT_CHECK_CTX(c);
    if (!c->children.empty())
    {
        if (c->present == 1 && dst)
        {   // the frame's ONE collective: radiance slabs -> first device over NVLink, resolved and read back there
            rt_ctx* k0 = c->children[0];
            bool pushed = true;              // did the frame kernels push this frame already (fused gather)?
            for (rt_ctx* k : c->children) pushed = pushed && k->gather_slab && k->gather_sample == k->sample_count;
            int rc;
            if (pushed)
            {
                rc = rt_gather_wait(k0);
                if (!rc) rc = rt_resolve_gathered(k0, k0->own_gather, (uint64_t)k0->own_gather_stride, dst);
            }
            else
            {   // frames rendered before the option was set: explicit peer copies
                rc = rt_gather_radiance(c); if (rc) return rc;
                rc = rt_resolve_gathered(k0, c->gather_buf, (uint64_t)c->gather_stride_f4 * 16, dst);
            }
            if (rc) c->error = k0->error;
            return rc;
        }
        // parallel read-back: every device resolves its rows and copies them into the caller's image over its own PCIe
        // link (page-lock the image, rt_host_register, for the copies to overlap); all enqueued first, then awaited
        for (rt_ctx* k : c->children) { int rc = resolve_enqueue(k, dst); if (rc) { c->error = k->error; return rc; } }
        for (rt_ctx* k : c->children)
        {
            if (cudaSetDevice(k->device) != cudaSuccess || cudaStreamSynchronize(k->stream) != cudaSuccess)
                RT_FAIL(c, RT_ERR_CUDA, "rt_resolve: device %d failed: %s", k->device, cudaGetErrorString(cudaGetLastError()));
        }
        return RT_OK;
    }
    int rc = resolve_enqueue(c, dst); if (rc) return rc;
    RT_CUDA(c, cudaStreamSynchronize(c->stream));
    return RT_OK;
}

/* Pipelined variant of rt_resolve for frame loops that do not need the image before submitting the next frame:
 * resolves on the render stream, then copies device->host on a second stream so that the PCIe transfer of frame i
 * overlaps the kernels of frame i+1.  Two resolve buffers alternate; the host buffer handed to call i must stay
 * untouched until rt_resolve_wait() (or the second-next rt_resolve_async) returns. */
int rt_resolve_async(rt_ctx* c, float* dst)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_resolve_async(k, dst));
    { int rt_j_ = join_shadow(c); if (rt_j_) return rt_j_; }
    if (!dst) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_resolve_async: null destination");
    { int rc = frame_buffers_ready(c); if (rc) return rc; }
    RT_CUDA(c, cudaSetDevice(c->device));
    { int rc = ensure_copy_stream(c); if (rc) return rc; }
    if (!c->resolved2) RT_CUDA(c, c->frame_mem.alloc(c->resolved2, c->n_local ? c->n_local : 1));
    const int k = (int)(c->async_index++ & 1u);
    float4* buf = k ? c->resolved2 : c->resolved;
    if (c->copy_pending[k]) RT_CUDA(c, cudaStreamWaitEvent(c->stream, c->copy_done[k], 0));   // buffer k is being re-used
    { int rc = launch_resolve(c, buf); if (rc) return rc; }
    RT_CUDA(c, cudaEventRecord(c->resolve_done[k], c->stream));
    RT_CUDA(c, cudaStreamWaitEvent(c->copy_stream, c->resolve_done[k], 0));
    if (c->local_rows)
        RT_CUDA(c, cudaMemcpy2DAsync(dst + (size_t)c->rank * c->width * 4, (size_t)c->world * c->width * 16, buf,
                                     (size_t)c->width * 16, (size_t)c->width * 16, c->local_rows, cudaMemcpyDeviceToHost, c->copy_stream));
    RT_CUDA(c, cudaEventRecord(c->copy_done[k], c->copy_stream));
    c->copy_pending[k] = true;
    return RT_OK;
}

static int resolve_gathered_impl(rt_ctx* c, const void* slabs, uint64_t stride_bytes, float* dst, bool async)
{
    RT_CHECK_CTX(c); RT_NOT_ON_GROUP(c, "rt_resolve_gathered");
    { int rt_j_ = join_shadow(c); if (rt_j_) return rt_j_; }
    if (!slabs || !dst) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_resolve_gathered: null pointer");
    const size_t rows_max = ((size_t)c->height + c->world - 1) / c->world;
    if (stride_bytes % 16 != 0 || stride_bytes < rows_max * c->width * 16)
        RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_resolve_gathered: slab stride must be a multiple of 16 and hold %zu rows", rows_max);
    if (c->aov != 0 || c->denoiser) RT_FAIL(c, RT_ERR_UNSUPPORTED, "rt_resolve_gathered resolves the shaded colour only (AOV views and the denoiser are single-GPU)");
    if (adaptive_wanted(c)) RT_FAIL(c, RT_ERR_UNSUPPORTED, "rt_resolve_gathered divides by one sample count: not available with adaptive sampling");
    if (c->sd_iters) RT_FAIL(c, RT_ERR_UNSUPPORTED, "rt_resolve_gathered has no guides of other ranks: not available with the spatial denoiser");
    RT_CUDA(c, cudaSetDevice(c->device));
    const size_t n = (size_t)c->width * c->height;
    int k = 0;
    if (async)
    {
        { int rc = ensure_copy_stream(c); if (rc) return rc; }
        k = (int)(c->async_index++ & 1u);
        if (c->copy_pending[k]) RT_CUDA(c, cudaStreamWaitEvent(c->stream, c->copy_done[k], 0));
    }
    if (!c->resolved_full[k]) RT_CUDA(c, c->ctx_mem.alloc(c->resolved_full[k], n));
    {
        TimedLaunch t(c, RT_K_RESOLVE);
        k_resolve_gathered<<<grid_for((uint32_t)n), 256, 0, c->stream>>>((const float4*)slabs, (size_t)(stride_bytes / 16), c->resolved_full[k],
                                                                            c->width, c->height, c->world, c->sample_count);
        int rc = post_launch(c, "k_resolve_gathered"); if (rc) return rc;
    }
    if (!async)
    {
        RT_CUDA(c, cudaMemcpyAsync(dst, c->resolved_full[k], n * 16, cudaMemcpyDeviceToHost, c->stream));
        RT_CUDA(c, cudaStreamSynchronize(c->stream));
        return RT_OK;
    }
    RT_CUDA(c, cudaEventRecord(c->resolve_done[k], c->stream));
    RT_CUDA(c, cudaStreamWaitEvent(c->copy_stream, c->resolve_done[k], 0));
    RT_CUDA(c, cudaMemcpyAsync(dst, c->resolved_full[k], n * 16, cudaMemcpyDeviceToHost, c->copy_stream));
    RT_CUDA(c, cudaEventRecord(c->copy_done[k], c->copy_stream));
    c->copy_pending[k] = true;
    return RT_OK;
}
int rt_resolve_gathered(rt_ctx* c, const void* slabs, uint64_t stride_bytes, float* dst) { return resolve_gathered_impl(c, slabs, stride_bytes, dst, false); }
int rt_resolve_gathered_async(rt_ctx* c, const void* slabs, uint64_t stride_bytes, float* dst) { return resolve_gathered_impl(c, slabs, stride_bytes, dst, true); }

int rt_resolve_wait(rt_ctx* c)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_resolve_wait(k));
    RT_CUDA(c, cudaSetDevice(c->device));
    if (c->copy_stream) RT_CUDA(c, cudaStreamSynchronize(c->copy_stream));
    c->copy_pending[0] = c->copy_pending[1] = false;
    return RT_OK;
}

int rt_sync(rt_ctx* c)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_sync(k));
    { int rt_j_ = join_shadow(c); if (rt_j_) return rt_j_; }
    RT_CUDA(c, cudaSetDevice(c->device));
    RT_CUDA(c, cudaStreamSynchronize(c->stream));
    return RT_OK;
}

int rt_read_hits(rt_ctx* c, uint32_t bounce, RtHit* hits, uint32_t* pixels, uint32_t* n_out)
{
    RT_CHECK_CTX(c); RT_NOT_ON_GROUP(c, "rt_read_hits");
    { int rt_j_ = join_shadow(c); if (rt_j_) return rt_j_; }
    if (bounce > RT_MAX_BOUNCES || !n_out) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_read_hits: bad arguments");
    { int rc = frame_buffers_ready(c); if (rc) return rc; }
    RT_CUDA(c, cudaSetDevice(c->device));
    RT_CUDA(c, cudaStreamSynchronize(c->stream));
    uint32_t n = 0;
    RT_CUDA(c, cudaMemcpy(&n, in_count_ptr(c->counters, bounce), 4, cudaMemcpyDeviceToHost));
    *n_out = n;
    if (hits && n) RT_CUDA(c, cudaMemcpy(hits, c->q.hits, (size_t)n * 16, cudaMemcpyDeviceToHost));   // same 16-byte layout as RtHit
    if (pixels && n)
    {
        std::vector<float4> a(n);
        RT_CUDA(c, cudaMemcpy(a.data(), c->q.B[bounce & 1], (size_t)n * 16, cudaMemcpyDeviceToHost));     // B.w: the packed pixel
        for (uint32_t i = 0; i < n; ++i) { uint32_t pxy; memcpy(&pxy, &a[i].w, 4); pixels[i] = (pxy >> 16) * c->width + (pxy & 0xFFFFu); }
    }
    return RT_OK;
}

int rt_read_rays(rt_ctx* c, uint32_t bounce, RtRay* rays, uint32_t* pixels, uint32_t* n_out)
{
    RT_CHECK_CTX(c); RT_NOT_ON_GROUP(c, "rt_read_rays");
    { int rt_j_ = join_shadow(c); if (rt_j_) return rt_j_; }
    if (bounce > RT_MAX_BOUNCES || !n_out || !rays || !pixels) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_read_rays: bad arguments");
    int rc = frame_buffers_ready(c); if (rc) return rc;
    RT_CUDA(c, cudaSetDevice(c->device));
    if ((rc = ensure_scratch(c, (size_t)c->n_local * (sizeof(RtRay) + 4) + 64))) return rc;
    RtRay* drays = (RtRay*)c->scratch;
    uint32_t* dpix = (uint32_t*)(c->scratch + (size_t)c->n_local * sizeof(RtRay));
    k_unpack_rays<<<grid_for(c->n_local), 256, 0, c->stream>>>(c->q.A[bounce & 1], c->q.B[bounce & 1], in_count_ptr(c->counters, bounce), c->width, drays, dpix);
    ++c->launches;
    if ((rc = post_launch(c, "k_unpack_rays"))) return rc;
    RT_CUDA(c, cudaStreamSynchronize(c->stream));
    uint32_t n = 0;
    RT_CUDA(c, cudaMemcpy(&n, in_count_ptr(c->counters, bounce), 4, cudaMemcpyDeviceToHost));
    *n_out = n;
    if (n)
    {
        RT_CUDA(c, cudaMemcpy(rays, drays, (size_t)n * sizeof(RtRay), cudaMemcpyDeviceToHost));
        RT_CUDA(c, cudaMemcpy(pixels, dpix, (size_t)n * 4, cudaMemcpyDeviceToHost));
    }
    return RT_OK;
}

int rt_read_radiance(rt_ctx* c, float* dst)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_read_radiance(k, dst));
    { int rt_j_ = join_shadow(c); if (rt_j_) return rt_j_; }
    if (!dst) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_read_radiance: null destination");
    { int rc = frame_buffers_ready(c); if (rc) return rc; }
    RT_CUDA(c, cudaSetDevice(c->device));
    if (c->local_rows)
        RT_CUDA(c, cudaMemcpy2DAsync(dst + (size_t)c->rank * c->width * 4, (size_t)c->world * c->width * 16, c->radiance,
                                     (size_t)c->width * 16, (size_t)c->width * 16, c->local_rows, cudaMemcpyDeviceToHost, c->stream));
    RT_CUDA(c, cudaStreamSynchronize(c->stream));
    return RT_OK;
}

int rt_read_frame_stats(rt_ctx* c, RtFrameStats* out)
{
    RT_CHECK_CTX(c);
    if (!c->children.empty())
    {   // whole-frame counters = sums over the partitions
        if (!out) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_read_frame_stats: null destination");
        static thread_local RtFrameStats part;
        memset(out, 0, sizeof(*out));
        for (rt_ctx* k : c->children)
        {
            int rc = rt_read_frame_stats(k, &part); if (rc) { c->error = k->error; return rc; }
            for (uint32_t b = 0; b <= RT_MAX_BOUNCES; ++b)
            {
                out->n_ext[b] += part.n_ext[b]; out->n_miss[b] += part.n_miss[b]; out->n_emissive_hits[b] += part.n_emissive_hits[b];
                out->n_shadow[b] += part.n_shadow[b]; out->n_cont[b] += part.n_cont[b]; out->n_unoccluded[b] += part.n_unoccluded[b];
                out->nodes_ext[b] += part.nodes_ext[b]; out->tris_ext[b] += part.tris_ext[b];
                out->nodes_shadow[b] += part.nodes_shadow[b]; out->tris_shadow[b] += part.tris_shadow[b];
            }
        }
        return RT_OK;
    }
    { int rt_j_ = join_shadow(c); if (rt_j_) return rt_j_; }
    if (!out) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_read_frame_stats: null destination");
    RT_CUDA(c, cudaSetDevice(c->device));
    RT_CUDA(c, cudaStreamSynchronize(c->stream));
    static thread_local DevCounters h;
    RT_CUDA(c, cudaMemcpy(&h, c->stats_summed ? c->counters_sum : c->counters, sizeof(DevCounters), cudaMemcpyDeviceToHost));
    memset(out, 0, sizeof(*out));
    for (uint32_t b = 0; b <= RT_MAX_BOUNCES; ++b)
    {
        out->n_ext[b] = (b == 0) ? h.n_primary : h.emit[b - 1].next; out->n_miss[b] = h.hm[b].miss; out->n_emissive_hits[b] = h.n_emissive[b];
        out->n_shadow[b] = h.emit[b].shadow; out->n_cont[b] = h.emit[b].next; out->n_unoccluded[b] = h.n_unoccluded[b];
        out->nodes_ext[b] = h.nodes_ext[b]; out->tris_ext[b] = h.tris_ext[b];
        out->nodes_shadow[b] = h.nodes_shadow[b]; out->tris_shadow[b] = h.tris_shadow[b];
    }
    return RT_OK;
}

int rt_read_sample_count(rt_ctx* c, uint32_t* out) { RT_CHECK_CTX(c); if (!out) return RT_ERR_INVALID_ARGUMENT; *out = c->children.empty() ? c->sample_count : c->children[0]->sample_count; return RT_OK; }

int rt_read_aovs(rt_ctx* c, float* albedo, float* depth, float* normal, float* velocity)
{
    RT_CHECK_CTX(c); RT_FANOUT(c, rt_read_aovs(k, albedo, depth, normal, velocity));
    { int rt_j_ = join_shadow(c); if (rt_j_) return rt_j_; }
    if (!c->aov_albedo) RT_FAIL(c, RT_ERR_NOT_READY, "AOV buffers do not exist: select an AOV view, enable the denoiser or set RT_OPT_AOV_ALWAYS first");
    RT_CUDA(c, cudaSetDevice(c->device));
    auto rows = [&](void* dst, const void* src, size_t elem) -> int {
        if (dst && c->local_rows)
            RT_CUDA(c, cudaMemcpy2DAsync((char*)dst + (size_t)c->rank * c->width * elem, (size_t)c->world * c->width * elem, src,
                                         (size_t)c->width * elem, (size_t)c->width * elem, c->local_rows, cudaMemcpyDeviceToHost, c->stream));
        return RT_OK;
    };
    int rc;
    if ((rc = rows(albedo, c->aov_albedo, 16)) || (rc = rows(depth, c->aov_depth, 4)) || (rc = rows(normal, c->aov_normal, 16)) || (rc = rows(velocity, c->aov_velocity, 8))) return rc;
    RT_CUDA(c, cudaStreamSynchronize(c->stream));
    return RT_OK;
}

int rt_kernel_times(rt_ctx* c, float* ms, uint32_t* launches)
{
    RT_CHECK_CTX(c);
    if (!c->children.empty())
    {   // the devices run concurrently: per class the slowest device's time, launches summed
        float m[RT_K_CLASS_COUNT]; uint32_t n[RT_K_CLASS_COUNT];
        for (int i = 0; i < RT_K_CLASS_COUNT; ++i) { if (ms) ms[i] = 0.0f; if (launches) launches[i] = 0; }
        for (rt_ctx* k : c->children)
        {
            int rc = rt_kernel_times(k, m, n); if (rc) { c->error = k->error; return rc; }
            for (int i = 0; i < RT_K_CLASS_COUNT; ++i) { if (ms && m[i] > ms[i]) ms[i] = m[i]; if (launches) launches[i] += n[i]; }
        }
        return RT_OK;
    }
    { int rt_j_ = join_shadow(c); if (rt_j_) return rt_j_; }
    RT_CUDA(c, cudaSetDevice(c->device));
    RT_CUDA(c, cudaStreamSynchronize(c->stream));
    for (auto& t : c->timed)
    {
        float m = 0.0f;
        RT_CUDA(c, cudaEventElapsedTime(&m, t.a, t.b));
        c->ms[t.cls] += m; c->nlaunch[t.cls] += 1;
        c->event_pool.push_back(std::move(t.a)); c->event_pool.push_back(std::move(t.b));
    }
    c->timed.clear();
    for (int k = 0; k < RT_K_CLASS_COUNT; ++k)
    {
        if (ms) ms[k] = c->ms[k];
        if (launches) launches[k] = c->nlaunch[k];
        c->ms[k] = 0.0f; c->nlaunch[k] = 0;
    }
    return RT_OK;
}

int rt_bvh_staging(rt_ctx* c, uint32_t* mode, uint64_t* bytes)
{
    RT_CHECK_CTX(c); if (!mode && !bytes) return RT_ERR_INVALID_ARGUMENT;
    const Stage sg = bvh_stage(c->children.empty() ? c : c->children[0]);
    if (mode) *mode = (uint32_t)sg.mode;
    if (bytes) *bytes = sg.bytes;
    return RT_OK;
}

int rt_launch_count(rt_ctx* c, uint64_t* out)
{
    RT_CHECK_CTX(c); if (!out) return RT_ERR_INVALID_ARGUMENT;
    *out = c->launches;
    for (rt_ctx* k : c->children) *out += k->launches;
    return RT_OK;
}
int rt_local_pixel_count(rt_ctx* c, uint32_t* out)
{
    RT_CHECK_CTX(c); if (!out) return RT_ERR_INVALID_ARGUMENT;
    *out = c->n_local;
    for (rt_ctx* k : c->children) *out += k->n_local;
    return RT_OK;
}

int rt_radiance_device_ptr(rt_ctx* c, void** out_ptr, uint64_t* out_bytes)
{
    RT_CHECK_CTX(c); RT_NOT_ON_GROUP(c, "rt_radiance_device_ptr");
    if (!out_ptr || !out_bytes) return RT_ERR_INVALID_ARGUMENT;
    *out_ptr = c->radiance; *out_bytes = (uint64_t)c->n_local * 16;
    return RT_OK;
}

int rt_stream_handle(rt_ctx* c, void** out) { RT_CHECK_CTX(c); RT_NOT_ON_GROUP(c, "rt_stream_handle"); if (!out) return RT_ERR_INVALID_ARGUMENT; *out = (void*)c->stream; return RT_OK; }

/* One context over several devices of the node (SURVEY 8b: "multi-GPU fan-out internal to the shim"; the reference's CLContext
 * enumerates every device of its platform, cl_context.cpp:64-89, and uses one).  devices[i] renders rank i of an n-way scanline
 * partition with the scene replicated; the caller stays single-threaded and every call fans out.  A device may be listed more
 * than once (two partitions time-share it). */
int rt_create_multi(uint32_t width, uint32_t height, const int* devices, uint32_t n_devices, rt_ctx** out_ctx)
{
    if (!out_ctx || !devices || n_devices == 0 || n_devices > 64)
    {
        g_create_error = "rt_create_multi: bad arguments (need 1..64 devices)"; return RT_ERR_INVALID_ARGUMENT;
    }
    *out_ctx = nullptr;
    if (n_devices == 1) return rt_create(width, height, devices[0], out_ctx);
    rt_ctx* g = new rt_ctx;
    g->width = width; g->height = height; g->world = n_devices; g->device = devices[0];
    for (uint32_t i = 0; i < n_devices; ++i)
    {
        rt_ctx* k = nullptr;
        int rc = rt_create(width, height, devices[i], &k);
        if (rc == RT_OK) { rc = rt_set_partition(k, i, n_devices); if (rc != RT_OK) { g_create_error = k->error; rt_destroy(k); } }
        if (rc != RT_OK) { for (rt_ctx* o : g->children) rt_destroy(o); delete g; return rc; }
        g->children.push_back(k);
    }
    // contexts that time-share one device split its resident CTA slots, so that their persistent kernels run side by side
    for (rt_ctx* k : g->children)
    {
        int same = 0;
        for (rt_ctx* o : g->children) same += o->device == k->device;
        k->grid_div = same;
    }
    // peer access towards the first device for the NVLink gather (ignored where it is already on / not available:
    // cudaMemcpyPeerAsync then stages through the host)
    for (uint32_t i = 1; i < n_devices; ++i)
        if (devices[i] != devices[0])
        {
            int can = 0;
            if (cudaDeviceCanAccessPeer(&can, devices[i], devices[0]) == cudaSuccess && can)
            {
                cudaSetDevice(devices[i]);
                cudaError_t e = cudaDeviceEnablePeerAccess(devices[0], 0);
                if (e != cudaSuccess) cudaGetLastError();       // cudaErrorPeerAccessAlreadyEnabled included
            }
        }
    *out_ctx = g;
    return RT_OK;
}

/* The single collective of a multi-device frame (north_star): every device's radiance slab is copied to the first device
 * (cudaMemcpyPeerAsync on the source device's stream: NVLink / NVSwitch between peers), into world slabs of stride
 * rows_max * width float4 — the layout rt_resolve_gathered reads.  The first device's stream then waits for all copies. */
int rt_gather_radiance(rt_ctx* c)
{
    RT_CHECK_CTX(c);
    if (c->children.empty()) RT_FAIL(c, RT_ERR_UNSUPPORTED, "rt_gather_radiance needs a multi-device context (rt_create_multi)");
    rt_ctx* k0 = c->children[0];
    const size_t rows_max = ((size_t)c->height + c->world - 1) / c->world;
    const size_t stride = rows_max * c->width;
    RT_CUDA(c, cudaSetDevice(k0->device));
    if (!c->gather_buf)
    {
        RT_CUDA(c, c->gather_mem.alloc(c->gather_buf, stride * c->world));
        RT_CUDA(c, cudaMemsetAsync(c->gather_buf, 0, stride * c->world * 16, k0->stream));
        RT_CUDA(c, cudaStreamSynchronize(k0->stream));
        c->gather_stride_f4 = stride;
        c->gather_events.resize(c->world);
    }
    for (uint32_t i = 0; i < c->world; ++i)
    {
        rt_ctx* k = c->children[i];
        { int rc = join_shadow(k); if (rc) { c->error = k->error; return rc; } }
        RT_CUDA(c, cudaSetDevice(k->device));
        if (!c->gather_events[i]) RT_CUDA(c, make_event(c->gather_events[i]));
        if (k->n_local)
            RT_CUDA(c, cudaMemcpyPeerAsync(c->gather_buf + (size_t)i * stride, k0->device, k->radiance, k->device, (size_t)k->n_local * 16, k->stream));
        RT_CUDA(c, cudaEventRecord(c->gather_events[i], k->stream));
    }
    RT_CUDA(c, cudaSetDevice(k0->device));
    for (uint32_t i = 1; i < c->world; ++i) RT_CUDA(c, cudaStreamWaitEvent(k0->stream, c->gather_events[i], 0));
    return RT_OK;
}

int rt_device_count(int* out)
{
    if (!out) return RT_ERR_INVALID_ARGUMENT;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); n = 0; }
    *out = n;
    return RT_OK;
}

/* Page-locks / releases a caller-owned host buffer (the image handed to rt_resolve): device->host copies into page-locked
 * memory are asynchronous, which is what lets the devices of a multi-device context read back in parallel. */
int rt_host_register(void* ptr, uint64_t bytes)
{
    if (!ptr || !bytes) return RT_ERR_INVALID_ARGUMENT;
    cudaError_t e = cudaHostRegister(ptr, bytes, cudaHostRegisterPortable);
    if (e != cudaSuccess) { cudaGetLastError(); g_create_error = std::string("rt_host_register: ") + cudaGetErrorString(e); return RT_ERR_CUDA; }
    return RT_OK;
}
int rt_host_unregister(void* ptr)
{
    if (!ptr) return RT_ERR_INVALID_ARGUMENT;
    cudaError_t e = cudaHostUnregister(ptr);
    if (e != cudaSuccess) { cudaGetLastError(); g_create_error = std::string("rt_host_unregister: ") + cudaGetErrorString(e); return RT_ERR_CUDA; }
    return RT_OK;
}

/* ---- fused gather over peer memory ------------------------------------------------------------------------------------------
 * The frame's one collective done by the frame kernel itself: every rank pushes the radiance of a pixel into its slab of a buffer
 * on the presenting device (NVLink peer stores) the moment the pixel's path ends, so the transfer is spread over the whole frame
 * instead of following it; a per-rank flag signals completion.  The buffer holds world slabs of rows_max * width float4 (the layout
 * rt_resolve_gathered reads) followed by the flags.  One process per GPU: the owner exports the buffer with rt_ipc_export, the
 * other ranks map it with rt_ipc_open; one process over several devices (rt_create_multi): peer access, no handles needed. */
int rt_gather_buffer(rt_ctx* c, void** dev_ptr, uint64_t* stride_bytes, uint64_t* total_bytes)
{
    RT_CHECK_CTX(c); RT_NOT_ON_GROUP(c, "rt_gather_buffer");
    if (!dev_ptr || !stride_bytes) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_gather_buffer: null output");
    const size_t rows_max = ((size_t)c->height + c->world - 1) / c->world;
    const size_t stride = rows_max * c->width * 16;
    const size_t total = stride * c->world + 256;
    RT_CUDA(c, cudaSetDevice(c->device));
    if (c->own_gather && c->own_gather_stride != stride) { c->gather_mem.clear(); c->own_gather = nullptr; }
    if (!c->own_gather)
    {
        RT_CUDA(c, c->gather_mem.alloc(c->own_gather, total));
        RT_CUDA(c, cudaMemset(c->own_gather, 0, total));
        c->own_gather_stride = stride;
    }
    *dev_ptr = c->own_gather; *stride_bytes = stride;
    if (total_bytes) *total_bytes = total;
    return RT_OK;
}

int rt_ipc_export(const void* dev_ptr, void* handle64)
{
    if (!dev_ptr || !handle64) return RT_ERR_INVALID_ARGUMENT;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handles are 64 bytes");
    cudaIpcMemHandle_t h;
    cudaError_t e = cudaIpcGetMemHandle(&h, const_cast<void*>(dev_ptr));
    if (e != cudaSuccess) { cudaGetLastError(); g_create_error = std::string("rt_ipc_export: ") + cudaGetErrorString(e); return RT_ERR_CUDA; }
    memcpy(handle64, &h, 64);
    return RT_OK;
}

int rt_ipc_open(rt_ctx* c, const void* handle64, void** dev_ptr)
{
    RT_CHECK_CTX(c); RT_NOT_ON_GROUP(c, "rt_ipc_open");
    if (!handle64 || !dev_ptr) RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_ipc_open: null argument");
    RT_CUDA(c, cudaSetDevice(c->device));
    cudaIpcMemHandle_t h; memcpy(&h, handle64, 64);
    void* p = nullptr;
    RT_CUDA(c, cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    c->ipc_opened.emplace_back(p);
    *dev_ptr = p;
    return RT_OK;
}

/* base = the buffer of rt_gather_buffer as THIS process addresses it (own pointer, peer pointer or rt_ipc_open mapping);
 * NULL turns the fused gather off.  Takes effect with the next frame. */
int rt_set_gather_target(rt_ctx* c, void* base, uint64_t stride_bytes)
{
    RT_CHECK_CTX(c); RT_NOT_ON_GROUP(c, "rt_set_gather_target");
    { int rc = join_shadow(c); if (rc) return rc; }
    if (!base) { c->gather_slab = nullptr; c->gather_flag = nullptr; return RT_OK; }
    if (adaptive_wanted(c)) RT_FAIL(c, RT_ERR_UNSUPPORTED, "a fused-gather target is not available with adaptive sampling (stopped pixels are never pushed)");
    const size_t rows_max = ((size_t)c->height + c->world - 1) / c->world;
    if (stride_bytes % 16 != 0 || stride_bytes < rows_max * c->width * 16)
        RT_FAIL(c, RT_ERR_INVALID_ARGUMENT, "rt_set_gather_target: slab stride must be a multiple of 16 and hold %zu rows", rows_max);
    c->gather_slab = (float4*)((char*)base + (size_t)c->rank * stride_bytes);
    c->gather_flag = (uint32_t*)((char*)base + (size_t)c->world * stride_bytes) + c->rank;
    return RT_OK;
}

/* On the context that presents (it must have a gather target itself, i.e. take part in the frames): makes its stream wait until
 * every rank has signalled the frame this context rendered last. */
int rt_gather_wait(rt_ctx* c)
{
    RT_CHECK_CTX(c); RT_NOT_ON_GROUP(c, "rt_gather_wait");
    if (!c->gather_flag) RT_FAIL(c, RT_ERR_NOT_READY, "rt_gather_wait: no gather target set");
    RT_CUDA(c, cudaSetDevice(c->device));
    k_gather_wait<<<1, 64, 0, c->stream>>>(c->gather_flag - c->rank, c->world, c->gather_frame);
    ++c->launches;
    return post_launch(c, "k_gather_wait");
}

/* Parity tap: out[i] = f(a[i], b[i]) for a function of include/rt_math.h, evaluated on `device` (host pointers; blocking).
 * fn: 0 sin 1 cos 2 tan 3 atan2(a, b) 4 acos 5 pow(a, b) 6 fmin 7 fmax 8 1/sqrt(a) 9 a / b. */
int rt_math_eval(int device, int fn, const float* a, const float* b, float* out, uint64_t n)
{
    if (!a || !b || !out || fn < 0 || fn > 10) return RT_ERR_INVALID_ARGUMENT;
    if (n == 0) return RT_OK;
    if (cudaSetDevice(device) != cudaSuccess) { cudaGetLastError(); g_create_error = "rt_math_eval: no such CUDA device"; return RT_ERR_NO_DEVICE; }
    DevAllocs g;
    float *da = nullptr, *db = nullptr, *dout = nullptr;
    cudaError_t e = g.alloc(da, n);
    if (e == cudaSuccess) e = g.alloc(db, n);
    if (e == cudaSuccess) e = g.alloc(dout, n);
    if (e == cudaSuccess) e = cudaMemcpy(da, a, n * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(db, b, n * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess)
    {
        k_math_eval<<<(unsigned)((n + 255) / 256), 256>>>(fn, da, db, dout, n);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(out, dout, n * 4, cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) { g_create_error = std::string("rt_math_eval: ") + cudaGetErrorString(e); return RT_ERR_CUDA; }
    return RT_OK;
}

} // extern "C"
