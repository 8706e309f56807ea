/*
 * rt_math.h — deterministic elementary functions shared by the CUDA kernels
 * (raytracing_b200/csrc) and the CPU oracle (oracle/), so that both sides
 * produce bit-identical float results.
 *
 * Why this exists: the reference's arithmetic lives in OpenCL C and uses the
 * OpenCL driver's built-in `tan, sin, cos, acos, atan2, pow, normalize`
 * (raygeneration.cl:108, bxdf.h:33-54,71-74,157-168, miss.cl:28-39) whose
 * results are implementation-defined at the ulp level.  CUDA's libdevice and
 * glibc's libm also differ from each other by an ulp here and there, and a
 * path tracer is chaotic (one flipped comparison changes a pixel completely).
 * So the transcendental functions are restated ONCE, here, using only IEEE-754
 * +,-,*,/,sqrt on doubles (correctly rounded on both x86-64 and sm_90a when
 * FMA contraction is off: gcc -ffp-contract=off, nvcc -fmad=false) and a final
 * round to float.  Results are within 1 ulp (almost always correctly rounded),
 * well inside the OpenCL 1.2 accuracy requirements (sin/cos/acos 4 ulp, tan 5,
 * atan2 6, pow 16).
 *
 * Valid argument ranges (the ones the path uses): |x| < 1e5 for sin/cos/tan.
 */
#ifndef RT_MATH_H
#define RT_MATH_H

#include <math.h>
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define RT_HD __host__ __device__ __forceinline__
#else
#define RT_HD static inline
#endif

RT_HD uint32_t rt_float_bits(float f)
{
#if defined(__CUDA_ARCH__)
    return __float_as_uint(f);
#else
    uint32_t u; memcpy(&u, &f, 4); return u;
#endif
}

RT_HD float rt_bits_float(uint32_t u)
{
#if defined(__CUDA_ARCH__)
    return __uint_as_float(u);
#else
    float f; memcpy(&f, &u, 4); return f;
#endif
}

/* fminf/fmaxf with IEEE-754 minNum/maxNum semantics (NaN operand is ignored,
 * -0 < +0): exactly what PTX min.f32/max.f32 and CUDA fminf/fmaxf do.  The
 * reference's OpenCL `min`/`max` leave NaN behaviour undefined (SURVEY A.4-5);
 * this is the documented choice for oracle and kernels alike. */
RT_HD float rt_fminf(float a, float b)
{
#if defined(__CUDA_ARCH__)
    return fminf(a, b);
#else
    if (a != a) return b;
    if (b != b) return a;
    if (a < b) return a;
    if (b < a) return b;
    return rt_bits_float(rt_float_bits(a) | rt_float_bits(b));
#endif
}

RT_HD float rt_fmaxf(float a, float b)
{
#if defined(__CUDA_ARCH__)
    return fmaxf(a, b);
#else
    if (a != a) return b;
    if (b != b) return a;
    if (a > b) return a;
    if (b > a) return b;
    return rt_bits_float(rt_float_bits(a) & rt_float_bits(b));
#endif
}

/* sin and cos of a double argument, |x| < 1e5: Cody-Waite reduction by pi/2
 * (two-term split) and Taylor polynomials on [-pi/4, pi/4] (truncation error
 * < 1e-18). */
RT_HD void rt_sincos_d(double x, double* s_out, double* c_out)
{
    if (!(fabs(x) < 1.0e5))
    {
        /* out of the supported range (or NaN/inf): return NaN deterministically */
        double z = x - x;
        *s_out = z / z; *c_out = z / z;
        return;
    }
    const double two_over_pi = 0.6366197723675814;
    const double pio2_hi = 1.57079632673412561417e+00;  /* first 33 bits of pi/2 */
    const double pio2_lo = 6.07710050650619224932e-11;  /* pi/2 - pio2_hi */
    double kd = rint(x * two_over_pi);
    int k = (int)kd;
    double r = x - kd * pio2_hi;
    r = r - kd * pio2_lo;
    double r2 = r * r;
    double ps = 2.8114572543455206e-15;
    ps = ps * r2 + -7.647163731819816e-13;
    ps = ps * r2 + 1.6059043836821613e-10;
    ps = ps * r2 + -2.505210838544172e-08;
    ps = ps * r2 + 2.7557319223985893e-06;
    ps = ps * r2 + -0.0001984126984126984;
    ps = ps * r2 + 0.008333333333333333;
    ps = ps * r2 + -0.16666666666666666;
    double sr = r + r * (r2 * ps);
    double pc = -1.5619206968586225e-16;
    pc = pc * r2 + 4.779477332387385e-14;
    pc = pc * r2 + -1.1470745597729725e-11;
    pc = pc * r2 + 2.08767569878681e-09;
    pc = pc * r2 + -2.755731922398589e-07;
    pc = pc * r2 + 2.48015873015873e-05;
    pc = pc * r2 + -0.001388888888888889;
    pc = pc * r2 + 0.041666666666666664;
    pc = pc * r2 + -0.5;
    double cr = 1.0 + r2 * pc;
    switch (k & 3)
    {
    case 0:  *s_out = sr;  *c_out = cr;  break;
    case 1:  *s_out = cr;  *c_out = -sr; break;
    case 2:  *s_out = -sr; *c_out = -cr; break;
    default: *s_out = -cr; *c_out = sr;  break;
    }
}

RT_HD float rt_sinf(float x) { double s, c; rt_sincos_d((double)x, &s, &c); return (float)s; }
RT_HD float rt_cosf(float x) { double s, c; rt_sincos_d((double)x, &s, &c); return (float)c; }
RT_HD float rt_tanf(float x) { double s, c; rt_sincos_d((double)x, &s, &c); return (float)(s / c); }

/* atan of a non-negative finite double: breakpoint reduction
 * atan(a) = atan(c) + atan((a-c)/(1+a*c)), c in {0,1/4,1/2,3/4,1}, then the
 * alternating Taylor series on |t| <= 1/8 (truncation error < 1e-23). */
RT_HD double rt_atan_pos_d(double a)
{
    double base, c;
    int inverted = 0;
    if (a > 1.0) { a = 1.0 / a; inverted = 1; }
    /* one division for all five breakpoints (same operations per breakpoint as the five-way branch: c = 0 gives
     * (a - 0) / (1 + a * 0) = a exactly, c = 1 gives (a - 1) / (1 + a)), so the compiled code holds one divide */
    if (a < 0.125)      { base = 0.0;                 c = 0.0; }
    else if (a < 0.375) { base = 0.24497866312686414; c = 0.25; }
    else if (a < 0.625) { base = 0.4636476090008061;  c = 0.5; }
    else if (a < 0.875) { base = 0.6435011087932844;  c = 0.75; }
    else                { base = 0.7853981633974483;  c = 1.0; }
    double t = (a - c) / (1.0 + a * c);
    double t2 = t * t;
    double p = 0.04;
    p = p * t2 + -0.043478260869565216;
    p = p * t2 + 0.047619047619047616;
    p = p * t2 + -0.05263157894736842;
    p = p * t2 + 0.058823529411764705;
    p = p * t2 + -0.06666666666666667;
    p = p * t2 + 0.07692307692307693;
    p = p * t2 + -0.09090909090909091;
    p = p * t2 + 0.1111111111111111;
    p = p * t2 + -0.14285714285714285;
    p = p * t2 + 0.2;
    p = p * t2 + -0.3333333333333333;
    double r = base + (t + t * (t2 * p));
    return inverted ? (1.5707963267948966 - r) : r;
}

/* atan2(y, x) in double for finite (or NaN) arguments; IEEE sign conventions
 * for zeros (atan2(+-0, +x) = +-0, atan2(+-0, -x) = +-pi). */
RT_HD double rt_atan2_d(double y, double x, int y_negative, int x_negative)
{
    double ax = fabs(x), ay = fabs(y);
    double r;
    if (ax != ax || ay != ay) return ax + ay;             /* NaN in, NaN out */
    if (ay == 0.0)            r = 0.0;
    else if (ax == 0.0)       r = 1.5707963267948966;
    else
    {   /* one quotient <= 1 and one polynomial for both octants (same operations as two separate calls) */
        const int steep = !(ay <= ax);
        const double q = steep ? ax / ay : ay / ax;
        r = rt_atan_pos_d(q);
        if (steep) r = 1.5707963267948966 - r;
    }
    if (x_negative) r = 3.141592653589793 - r;
    return y_negative ? -r : r;
}

RT_HD float rt_atan2f(float y, float x)
{
    return (float)rt_atan2_d((double)y, (double)x,
                             (int)(rt_float_bits(y) >> 31), (int)(rt_float_bits(x) >> 31));
}

/* acos(x) = atan2(sqrt((1-x)(1+x)), x); NaN outside [-1,1]. */
RT_HD float rt_acosf(float x)
{
    double xd = (double)x;
    double q = (1.0 - xd) * (1.0 + xd);   /* exact products/sums of floats fit a double */
    double s = sqrt(q);                   /* q < 0 -> NaN, as acos requires */
    return (float)rt_atan2_d(s, xd, 0, xd < 0.0);
}

/* natural log of a positive finite double */
RT_HD double rt_log_pos_d(double x)
{
    int e;
    double m = frexp(x, &e);              /* m in [0.5, 1) */
    if (m < 0.70710678118654752) { m = m * 2.0; e = e - 1; }
    double s = (m - 1.0) / (m + 1.0);     /* |s| <= 0.1716 */
    double s2 = s * s;
    double p = 0.08695652173913043;
    p = p * s2 + 0.09523809523809523;
    p = p * s2 + 0.10526315789473684;
    p = p * s2 + 0.11764705882352941;
    p = p * s2 + 0.13333333333333333;
    p = p * s2 + 0.15384615384615385;
    p = p * s2 + 0.18181818181818182;
    p = p * s2 + 0.2222222222222222;
    p = p * s2 + 0.2857142857142857;
    p = p * s2 + 0.4;
    p = p * s2 + 0.6666666666666666;
    p = p * s2 + 2.0;
    return (double)e * 0.6931471805599453 + s * p;
}

/* exp of a double with |t| < 700 */
RT_HD double rt_exp_d(double t)
{
    const double ln2_hi = 6.93147180369123816490e-01;
    const double ln2_lo = 1.90821492927058770002e-10;
    double kd = rint(t * 1.4426950408889634);
    double r = t - kd * ln2_hi;
    r = r - kd * ln2_lo;
    double p = 1.1470745597729725e-11;
    p = p * r + 1.6059043836821613e-10;
    p = p * r + 2.08767569878681e-09;
    p = p * r + 2.505210838544172e-08;
    p = p * r + 2.755731922398589e-07;
    p = p * r + 2.7557319223985893e-06;
    p = p * r + 2.48015873015873e-05;
    p = p * r + 0.0001984126984126984;
    p = p * r + 0.001388888888888889;
    p = p * r + 0.008333333333333333;
    p = p * r + 0.041666666666666664;
    p = p * r + 0.16666666666666666;
    p = p * r + 0.5;
    p = p * r + 1.0;
    p = p * r + 1.0;
    return ldexp(p, (int)kd);
}

/* exp of a float in float arithmetic only (the edge-stopping weights of the spatial denoiser: one per tap, 25 taps x 5 passes per
 * pixel, where a double exp would cost more than the filter's memory traffic).  Cody-Waite reduction x = k ln2 + r, |r| <= ln2/2
 * (ln2_hi has 16 significant bits, so k * ln2_hi is exact for |k| <= 256), the degree-7 Taylor polynomial of exp(r) (truncation
 * error < 5e-9 relative) in Horner form, and a scale by 2^k built from its exponent bits.  Below ln(FLT_MIN) the result is 0
 * (no subnormals), above ln(FLT_MAX) it is +inf; NaN in, NaN out.  Within 1.25 ulp of the exact exp over [-87.3, 88.7] (the bound
 * tests/test_spatial_denoise_cpu.py checks). */
RT_HD float rt_expf(float x)
{
    if (x != x) return x + x;
    if (x > 88.72283935546875f) return INFINITY;
    if (x < -87.33654022216797f) return 0.0f;
    const float ln2_hi = 0.693145751953125f;
    const float ln2_lo = 1.42860682030941723212e-06f;
    const float kf = rintf(x * 1.44269502162933349609f);
    float r = x - kf * ln2_hi;
    r = r - kf * ln2_lo;
    float p = 1.98412701e-04f;        /* 1/5040 */
    p = p * r + 1.38888892e-03f;      /* 1/720 */
    p = p * r + 8.33333377e-03f;      /* 1/120 */
    p = p * r + 4.16666679e-02f;      /* 1/24 */
    p = p * r + 1.66666672e-01f;      /* 1/6 */
    p = p * r + 0.5f;
    p = p * r + 1.0f;
    p = p * r + 1.0f;
    const int k = (int)kf;            /* -126 .. 128 */
    if (k > 127) return (p * rt_bits_float(254u << 23)) * 2.0f;
    return p * rt_bits_float((uint32_t)(k + 127) << 23);
}

/* pow(x, y).  The path only needs pow(x, 5.0f) (Schlick Fresnel, bxdf.h:71-74,
 * any sign of x) and pow(x in [0,1], 2.2f) (texture gamma, material.h:251-264).
 * y == 5 is evaluated as an exact-in-double product (also right for x < 0);
 * other exponents use exp(y*log(x)) for x > 0. */
RT_HD float rt_powf(float x, float y)
{
    double xd = (double)x;
    if (y == 5.0f)
    {
        double x2 = xd * xd;
        return (float)((x2 * x2) * xd);
    }
    if (y == 0.0f) return 1.0f;
    if (x != x || y != y) return x + y;
    if (x == 0.0f) return (y > 0.0f) ? 0.0f : INFINITY;
    if (x < 0.0f) return (x - x) / (x - x);               /* NaN: not on the path */
    if (xd > 1.0e300) return (y > 0.0f) ? x : 0.0f;       /* +inf */
    double t = (double)y * rt_log_pos_d(xd);
    if (t > 700.0) return INFINITY;
    if (t < -700.0) return 0.0f;
    return (float)rt_exp_d(t);
}

#endif /* RT_MATH_H */
