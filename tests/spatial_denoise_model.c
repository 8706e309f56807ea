/*
 * spatial_denoise_model.c — the scalar model of this project's spatial denoiser (rt_set_spatial_denoiser, include/rt_b200.h),
 * written from the rule stated there, independently of the kernels in raytracing_b200/csrc/rt_kernels.cu.  It is a model of this
 * project's filter (an edge-avoiding a-trous wavelet filter after Dammertz et al. 2010), not of reference code.  Plain float
 * arithmetic in the stated order, rt_expf from include/rt_math.h; compiled with -ffp-contract=off so that it gives the kernels'
 * bits.  The tests build it into a temporary shared library.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "rt_math.h"

void sdm_expf(const float* x, float* out, uint64_t n)
{
    for (uint64_t i = 0; i < n; ++i) out[i] = rt_expf(x[i]);
}

static int finite3(const float* c) { return isfinite(c[0]) && isfinite(c[1]) && isfinite(c[2]); }

/* a term of the distance: its difference times its factor, added only when both are positive */
static float term(float diff, float k) { return (k > 0.0f && diff > 0.0f) ? diff * k : 0.0f; }

/* ldr, normal: width*height RGBA float (row-major), depth: width*height float; out: width*height RGBA (alpha 1).  iterations 0..5;
 * out may not alias ldr. */
void sdm_filter(uint32_t width, uint32_t height, const float* ldr, const float* normal, const float* depth, uint32_t iterations,
                float sigma_color, float sigma_normal, float sigma_depth, float* out)
{
    static const float h[5] = { 0.0625f, 0.25f, 0.375f, 0.25f, 0.0625f };
    const size_t n = (size_t)width * height;
    float* a = (float*)malloc(n * 16);
    float* b = (float*)malloc(n * 16);
    for (size_t i = 0; i < n; ++i) { memcpy(a + 4 * i, ldr + 4 * i, 12); a[4 * i + 3] = 1.0f; }
    const float kc = sigma_color > 0.0f ? 1.0f / (sigma_color * sigma_color) : 0.0f;
    const float kn = sigma_normal > 0.0f ? 1.0f / (sigma_normal * sigma_normal) : 0.0f;
    for (uint32_t it = 0; it < iterations; ++it)
    {
        const int step = 1 << it;
        const float kci = kc * (float)step;
        for (uint32_t y = 0; y < height; ++y)
            for (uint32_t x = 0; x < width; ++x)
            {
                const size_t p = (size_t)y * width + x;
                const float* cp = a + 4 * p;
                const int cfin = finite3(cp);
                const float c0[3] = { cfin ? cp[0] : 0.0f, cfin ? cp[1] : 0.0f, cfin ? cp[2] : 0.0f };
                const float kcp = cfin ? kci : 0.0f;
                const float* np_ = normal + 4 * p;
                const float zp = depth[p];
                const float kz = sigma_depth > 0.0f ? 1.0f / (sigma_depth * zp) : 0.0f;
                float wsum = 0.0f, s0 = 0.0f, s1 = 0.0f, s2 = 0.0f;
                for (int ty = -2; ty <= 2; ++ty)
                {
                    const long qy = (long)y + (long)ty * step;
                    if (qy < 0 || qy >= (long)height) continue;
                    for (int tx = -2; tx <= 2; ++tx)
                    {
                        const long qx = (long)x + (long)tx * step;
                        if (qx < 0 || qx >= (long)width) continue;
                        const size_t q = (size_t)qy * width + (size_t)qx;
                        const float* cq = a + 4 * q;
                        if (!finite3(cq)) continue;
                        const float* nq = normal + 4 * q;
                        const float dr = c0[0] - cq[0], dg = c0[1] - cq[1], db = c0[2] - cq[2];
                        const float dc = (dr * dr + dg * dg) + db * db;
                        const float nx = np_[0] - nq[0], ny = np_[1] - nq[1], nz = np_[2] - nq[2];
                        const float dn = (nx * nx + ny * ny) + nz * nz;
                        const float dz = fabsf(zp - depth[q]);
                        float d = term(dc, kcp);
                        d = d + term(dn, kn);
                        d = d + term(dz, kz);
                        const float w = (h[ty + 2] * h[tx + 2]) * rt_expf(-d);
                        if (w > 0.0f)
                        {
                            wsum = wsum + w;
                            s0 = s0 + w * cq[0]; s1 = s1 + w * cq[1]; s2 = s2 + w * cq[2];
                        }
                    }
                }
                float* o = b + 4 * p;
                if (wsum > 0.0f) { o[0] = s0 / wsum; o[1] = s1 / wsum; o[2] = s2 / wsum; }
                else { o[0] = cp[0]; o[1] = cp[1]; o[2] = cp[2]; }
                o[3] = 1.0f;
            }
        float* t = a; a = b; b = t;
    }
    memcpy(out, a, n * 16);
    free(a); free(b);
}
