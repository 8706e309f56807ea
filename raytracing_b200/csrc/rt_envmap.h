/*
 * rt_envmap.h — the environment table of RT_OPT_ENV_SAMPLING and the light-kind selection of rt_set_light_selection
 * (include/rt_b200.h).  The table is built once on the host from the uploaded environment image; the direction <-> texel-cell
 * mapping and the sampling walk are RT_HD, so the kernels and the CPU model the tests compare them with (tests/light_model.cpp)
 * run the same code.  Plain float arithmetic in the order written; compile with -ffp-contract=off / -fmad=false.
 *
 *   W_ij      luma(texel i of row j) * rt_sinf(RT_PI * (((float)j + 0.5f) / (float)h)),  luma = (r*0.299f + g*0.587f) + b*0.114f;
 *             a luma that is not finite and >= 0 counts as 0
 *   R_j       W_0j + ... + W_(w-1)j (running float sum);  T = R_0 + ... + R_(h-1) (running float sum)
 *   marg[j]   (R_0 + ... + R_j) / T, marg[h-1] = 1;   cond[j][i] = (W_0j + ... + W_ij) / R_j, cond[j][w-1] = 1 (every entry 1
 *             in a row with R_j = 0, which is never drawn but by rounding, and then has density 0)
 *   pdf[j][i] P_v * (((float)w * (float)h) * W_ij / T): P_v times the density in (u, v) = (cx, cy) texture space
 *   active    T finite and > 0, the option on and white-furnace mode off
 */
#pragma once

#include <cmath>
#include <cstdint>
#include <vector>

#include "rt_math.h"
#include "rt_types.h"

#if defined(__CUDA_ARCH__)
#define RT_ENV_LD(p) __ldg(p)
#else
#define RT_ENV_LD(p) (*(p))
#endif

#define RT_ENV_2PI2 19.7392088f        // 2 pi^2: d(omega) = 2 pi^2 sin(theta) du dv

namespace rtenv
{

// sample_sky's texture coordinates of a direction (rt_device.cuh, oracle SampleSky: miss.cl:28-39), before the repeat wrap
RT_HD void sky_coords(float x, float y, float z, float& cx, float& cy)
{
    cx = rt_atan2f(x, y) + RT_PI;
    cy = rt_acosf(z);
    cx = cx < 0.0f ? cx + RT_TWO_PI : cx;
    cx *= RT_INV_TWO_PI;
    cy *= RT_INV_PI;
}

// p_v(dir): the density per solid angle with which the environment strategy draws `dir`, including P_v (pdf = the device or host
// table).  The cell is the texel whose square holds sample_sky's (u, v); sin(theta) = sqrtf(max(1 - z*z, 0)).  0 / inf at the poles
// (where the MIS weight of the other strategy then takes it all).
RT_HD float pdf_dir(const float* pdf, int w, int h, float x, float y, float z)
{
    float cx, cy;
    sky_coords(x, y, z, cx, cy);
    const float wt = (float)w, ht = (float)h;
    const float u = (cx - floorf(cx)) * wt, v = (cy - floorf(cy)) * ht;
    const int i = u > 0.0f ? (u < wt ? (int)u : w - 1) : 0;          // NaN -> 0
    const int j = v > 0.0f ? (v < ht ? (int)v : h - 1) : 0;
    const float st = sqrtf(rt_fmaxf(1.0f - z * z, 0.0f));
    return RT_ENV_LD(pdf + (size_t)j * w + i) / (RT_ENV_2PI2 * st);
}

// The direction of texture coordinates (u, v): the inverse of sky_coords.  phi = u * 2pi - pi, theta = v * pi;
// dir = (sin(theta) * sin(phi), sin(theta) * cos(phi), cos(theta)) with rt_math's sin / cos.
RT_HD void dir_of(float u, float v, float& x, float& y, float& z)
{
    const float phi = u * RT_TWO_PI - RT_PI, theta = v * RT_PI;
    double sp, cp, st, ct;
    rt_sincos_d((double)phi, &sp, &cp);
    rt_sincos_d((double)theta, &st, &ct);
    const float s = (float)st;
    x = s * (float)sp; y = s * (float)cp; z = (float)ct;
}

// One environment sample: row j = first marg entry above min(r1, 0x1.fffffep-1), column i = first entry of row j's cond above
// min(r2, 0x1.fffffep-1); u = ((float)i + r3) / (float)w, v = ((float)j + r4) / (float)h; dir = dir_of(u, v).
RT_HD void sample(const float* marg, const float* cond, int w, int h, float r1, float r2, float r3, float r4, float& x, float& y, float& z)
{
    r1 = rt_fminf(r1, 0.99999994f);
    r2 = rt_fminf(r2, 0.99999994f);
    uint32_t lo = 0, hi = (uint32_t)h - 1u;
    while (lo < hi)
    {
        const uint32_t mid = (lo + hi) >> 1;
        if (RT_ENV_LD(marg + mid) > r1) hi = mid; else lo = mid + 1u;
    }
    const uint32_t j = lo;
    const float* row = cond + (size_t)j * w;
    lo = 0; hi = (uint32_t)w - 1u;
    while (lo < hi)
    {
        const uint32_t mid = (lo + hi) >> 1;
        if (RT_ENV_LD(row + mid) > r2) hi = mid; else lo = mid + 1u;
    }
    const float u = ((float)lo + r3) / (float)w, v = ((float)j + r4) / (float)h;
    dir_of(u, v, x, y, z);
}

// The light-kind probabilities of rt_set_light_selection.  A kind's weight counts only while the kind is active; S = (a + e) + v,
// P_e = e / S, P_v = v / S, p_ev = P_e + P_v, no_analytic = (a == 0).  All 0 when nothing is active.
struct Selection
{
    float p_e = 0.0f, p_v = 0.0f, p_ev = 0.0f;
    bool no_analytic = false;
};

inline Selection select(bool analytic, bool emitters, bool env, float w_analytic, float w_emitters, float w_env)
{
    Selection s;
    const float a = analytic ? w_analytic : 0.0f, e = emitters ? w_emitters : 0.0f, v = env ? w_env : 0.0f;
    const float sum = (a + e) + v;
    if (!(sum > 0.0f)) return s;
    s.p_e = e / sum; s.p_v = v / sum; s.p_ev = s.p_e + s.p_v;
    s.no_analytic = a == 0.0f;
    return s;
}

// Whether an analytic light has non-zero radiance (the analytic kind is active)
inline bool analytic_lit(const RtLight* lights, uint32_t n_analytic)
{
    for (uint32_t l = 0; l < n_analytic; ++l)
        if (lights[l].radiance.x != 0.0f || lights[l].radiance.y != 0.0f || lights[l].radiance.z != 0.0f) return true;
    return false;
}

struct Table
{
    std::vector<float> marg;       // h entries
    std::vector<float> cond;       // w * h entries, row-major
    std::vector<float> pdf;        // w * h entries: P_v * p_uv once scaled
};

// Builds the CDFs and p_uv (pdf without P_v) of an RGBA32F image; returns whether T is finite and > 0 (else the table is empty).
inline bool build(const float* rgba, uint32_t w, uint32_t h, Table& out)
{
    const size_t n = (size_t)w * h;
    out.marg.assign(h, 0.0f); out.cond.assign(n, 0.0f); out.pdf.assign(n, 0.0f);
    std::vector<float> row_sum(h);
    float total = 0.0f;
    for (uint32_t j = 0; j < h; ++j)
    {
        const float s = rt_sinf(RT_PI * (((float)j + 0.5f) / (float)h));
        float run = 0.0f;
        for (uint32_t i = 0; i < w; ++i)
        {
            const float* p = rgba + ((size_t)j * w + i) * 4;
            float l = (p[0] * 0.299f + p[1] * 0.587f) + p[2] * 0.114f;
            l = (std::isfinite(l) && l >= 0.0f) ? l : 0.0f;
            const float wij = l * s;
            out.pdf[(size_t)j * w + i] = wij;
            run += wij;
            out.cond[(size_t)j * w + i] = run;
        }
        row_sum[j] = run;
        total += run;
        out.marg[j] = total;
    }
    if (!(std::isfinite(total) && total > 0.0f)) { out.marg.clear(); out.cond.clear(); out.pdf.clear(); return false; }
    const float area = (float)w * (float)h;
    for (uint32_t j = 0; j < h; ++j)
    {
        out.marg[j] = out.marg[j] / total;
        float* row = out.cond.data() + (size_t)j * w;
        for (uint32_t i = 0; i < w; ++i)
        {
            row[i] = row_sum[j] > 0.0f ? row[i] / row_sum[j] : 1.0f;
            float& p = out.pdf[(size_t)j * w + i];
            p = (area * p) / total;
        }
        row[w - 1] = 1.0f;
    }
    out.marg[h - 1] = 1.0f;
    return true;
}

// pdf[k] = P_v * p_uv[k]
inline void scale(Table& t, float p_v)
{
    for (float& p : t.pdf) p = p_v * p;
}

} // namespace rtenv
