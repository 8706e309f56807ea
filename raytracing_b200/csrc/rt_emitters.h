/*
 * rt_emitters.h — the emitter table of RT_OPT_EMITTER_SAMPLING (include/rt_b200.h), built once on the host from the upload.
 * Shared by the library (rt_upload_scene / rt_set_option) and the CPU model the tests compare the kernels with, so both sample
 * the same discrete distribution bit for bit.  Plain float arithmetic in the order written; compile with -ffp-contract=off.
 *
 *   emitters   the uploaded emissive_indices (indices into the leaf-ordered triangles), in upload order
 *   A_t        0.5f * sqrtf((cx*cx + cy*cy) + cz*cz),  c = cross(p2 - p1, p3 - p1) as rt_bvh_layout.h's geometric normal
 *   w_t        A_t * luma(E),  E = the material's constant emission (mat_rec), luma = (E.r*0.299f + E.g*0.587f) + E.b*0.114f;
 *              a w_t that is not finite and > 0 counts as 0
 *   cdf[i]     S_i / S_n with S_i = w_0 + ... + w_i summed in list order; cdf[n-1] = 1 exactly
 *   pmf_i      cdf[i] - cdf[i-1] (cdf[-1] = 0)
 *   P_e        0 if S_n is not finite and > 0, or in white-furnace mode; 1 if every analytic light has zero radiance; else 0.5
 *   pdfA[t]    (P_e * pmf_i) / A_t for emitter t = emitters[i] with pmf_i > 0, else 0 (every other triangle too)
 */
#pragma once

#include <cmath>
#include <cstdint>
#include <string>
#include <vector>

#include "rt_types.h"

namespace rtemit
{

struct Table
{
    std::vector<uint32_t> list;   // emitter triangle ids, upload order
    std::vector<float> cdf;       // one per emitter, last entry 1
    std::vector<float> pdfA;      // one per triangle
    float p_e = 0.0f;             // probability of sampling an emitter instead of an analytic light
};

// With emitter sampling on, every index must name a triangle and appear once.
inline bool check_indices(const uint32_t* idx, uint64_t n, uint64_t n_tris, std::string& err)
{
    std::vector<uint8_t> seen(n_tris, 0);
    for (uint64_t i = 0; i < n; ++i)
    {
        if (idx[i] >= n_tris) { err = "emissive index " + std::to_string(idx[i]) + " is not a triangle"; return false; }
        if (seen[idx[i]]) { err = "emissive index " + std::to_string(idx[i]) + " is listed twice"; return false; }
        seen[idx[i]] = 1;
    }
    return true;
}

inline float tri_area(const RtTriangle& t)
{
    const RtFloat3 &p1 = t.v1.position, &p2 = t.v2.position, &p3 = t.v3.position;
    float e1x = p2.x - p1.x, e1y = p2.y - p1.y, e1z = p2.z - p1.z;
    float e2x = p3.x - p1.x, e2y = p3.y - p1.y, e2z = p3.z - p1.z;
    float cx = e1y * e2z - e1z * e2y, cy = e1z * e2x - e1x * e2z, cz = e1x * e2y - e1y * e2x;
    return 0.5f * sqrtf((cx * cx + cy * cy) + cz * cz);
}

// The constant emission of a packed material, unpacked as rt_bvh_layout.h's build_mat_rec (= load_material without textures)
inline float emission_luma(const RtPackedMaterial& m)
{
    float f = ldexpf(1.0f, (int)(m.emission >> 24) - (128 + 8));
    float r = (float)(int)(m.emission & 0xFF) * f, g = (float)(int)((m.emission >> 8) & 0xFF) * f, b = (float)(int)((m.emission >> 16) & 0xFF) * f;
    return (r * 0.299f + g * 0.587f) + b * 0.114f;
}

// tri(i) returns the RtTriangle of emitters[i] (the caller has checked the indices).  p_e_sel >= 0: the P_e of the light-selection
// rule (rt_envmap.h rtenv::select) replaces the default 1 / 0.5 of an active table.
template <class TriOf>
inline void build(TriOf tri, const uint32_t* idx, uint64_t n, uint64_t n_tris, const RtPackedMaterial* mats,
                  const RtLight* lights, uint32_t n_analytic, bool white_furnace, Table& out, float p_e_sel = -1.0f)
{
    out.list.assign(idx, idx + n);
    out.cdf.assign(n, 0.0f);
    out.pdfA.assign(n_tris, 0.0f);
    out.p_e = 0.0f;
    std::vector<float> area(n), w(n);
    float s = 0.0f;
    for (uint64_t i = 0; i < n; ++i)
    {
        const RtTriangle& t = tri(i);
        area[i] = tri_area(t);
        float wi = area[i] * emission_luma(mats[t.mtlIndex]);
        w[i] = (std::isfinite(wi) && wi > 0.0f) ? wi : 0.0f;
        s += w[i];
    }
    if (!(std::isfinite(s) && s > 0.0f) || white_furnace) { out.cdf.clear(); out.list.clear(); return; }
    float run = 0.0f;
    for (uint64_t i = 0; i < n; ++i) { run += w[i]; out.cdf[i] = run / s; }
    out.cdf[n - 1] = 1.0f;
    bool dark = true;
    for (uint32_t l = 0; l < n_analytic; ++l)
        if (lights[l].radiance.x != 0.0f || lights[l].radiance.y != 0.0f || lights[l].radiance.z != 0.0f) dark = false;
    out.p_e = p_e_sel >= 0.0f ? p_e_sel : (dark ? 1.0f : 0.5f);
    for (uint64_t i = 0; i < n; ++i)
    {
        float pmf = out.cdf[i] - (i ? out.cdf[i - 1] : 0.0f);
        if (pmf > 0.0f) out.pdfA[idx[i]] = (out.p_e * pmf) / area[i];
    }
}

} // namespace rtemit
