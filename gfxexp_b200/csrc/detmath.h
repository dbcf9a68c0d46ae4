// detmath.h — deterministic single-precision transcendentals shared by the CUDA kernels and
// the CPU oracle.
//
// Why this exists: the reference calls sincosf/acos/atan2 inside encodeNormal/decodeNormal,
// toPolarYUp/fromPolarYUp and the GGX sampler (common/common_device.cuh:14-65,470-504).
// glibc's libm and CUDA's libdevice differ by 1-2 ULP on those, which flips 16-bit polar
// codes and reservoir decisions.  Every function below uses only IEEE +,-,*,/ and sqrt in a
// fixed order (no FMA contraction: nvcc -fmad=false, gcc -ffp-contract=off), so the same
// input gives the same bits on the host and on sm_90a.  The polynomials are the published
// Cephes single-precision kernels (sinf/cosf/asinf/atanf); tests/test_detmath.py bounds the
// error against libm (<= 4 ULP away from the zeros, same monotone 16-bit quantisation).
#pragma once
#include <stdint.h>
#include <math.h>
#include <string.h>

#if defined(__CUDACC__)
#define DM_HD __host__ __device__ __forceinline__
#else
#define DM_HD static inline
#endif

#define DM_PI 3.14159265358979323846f
#define DM_2PI 6.28318530717958647692f
#define DM_PI_2 1.57079632679489661923f
#define DM_PI_4 0.78539816339744830962f

DM_HD uint32_t dm_f2u(float f) {
#if defined(__CUDA_ARCH__)
    return __float_as_uint(f);
#else
    uint32_t u; memcpy(&u, &f, 4); return u;
#endif
}
DM_HD float dm_u2f(uint32_t u) {
#if defined(__CUDA_ARCH__)
    return __uint_as_float(u);
#else
    float f; memcpy(&f, &u, 4); return f;
#endif
}

// float -> uint32 conversion with the CUDA saturating semantics on both sides
// (C++ leaves negative/NaN inputs undefined; x86 cvttss2si would give 0x80000000).
DM_HD uint32_t dm_f2uint(float f) {
    if (!(f > 0.0f)) return 0u;              // negative, -0, NaN
    if (f >= 4294967296.0f) return 0xFFFFFFFFu;
    return (uint32_t)f;
}
DM_HD int32_t dm_f2int(float f) {
    if (f != f) return 0;
    if (f >= 2147483648.0f) return 2147483647;
    if (f <= -2147483648.0f) return (int32_t)0x80000000;
    return (int32_t)f;
}

// Radical inverse of idx in base `base`, the float loop of svgf_main.cpp:1410-1421 that fills the SVGF app's table of TAA
// sub-pixel offsets.  The reference's build rounds every step (MSVC /fp:precise); so must every compiler here.
DM_HD float dm_halton(uint32_t base, uint32_t idx) {
    const float recBase = 1.0f / base;
    float ret = 0.0f;
    float scale = 1.0f;
    while (idx) {
        scale *= recBase;
        ret += (idx % base) * scale;
        idx /= base;
    }
    return ret;
}

// sin and cos of x (|x| up to a few thousand; the path only feeds [-pi, 4pi]).
// Quadrant reduction by pi/2 with a three-term Cody-Waite split, then the Cephes minimax
// polynomials on [-pi/4, pi/4].
DM_HD void dm_sincos(float x, float* s, float* c) {
    const float twoOverPi = 0.63661977236758134308f;
    const float k = floorf(x * twoOverPi + 0.5f);
    // pi/2 = C1 + C2 + C3, C1 and C2 have short mantissas so k*C1, k*C2 are exact.
    const float C1 = 1.5703125f;
    const float C2 = 4.837512969970703125e-4f;
    const float C3 = 7.54978995489188216e-8f;
    float r = x - k * C1;
    r = r - k * C2;
    r = r - k * C3;
    const float z = r * r;
    float ps = -1.9515295891e-4f * z + 8.3321608736e-3f;
    ps = ps * z - 1.6666654611e-1f;
    ps = ps * z * r + r;
    float pc = 2.443315711809948e-5f * z - 1.388731625493765e-3f;
    pc = pc * z + 4.166664568298827e-2f;
    pc = pc * z * z - 0.5f * z + 1.0f;
    const int32_t q = ((int32_t)k) & 3;
    float ss, cc;
    if (q == 0) { ss = ps; cc = pc; }
    else if (q == 1) { ss = pc; cc = -ps; }
    else if (q == 2) { ss = -ps; cc = -pc; }
    else { ss = -pc; cc = ps; }
    *s = ss;
    *c = cc;
}
DM_HD float dm_sin(float x) { float s, c; dm_sincos(x, &s, &c); return s; }
DM_HD float dm_cos(float x) { float s, c; dm_sincos(x, &s, &c); return c; }

// asin on [-1, 1] (Cephes asinf).
DM_HD float dm_asin(float x) {
    const float a = fabsf(x);
    if (a > 1.0f) return x > 0 ? DM_PI_2 : -DM_PI_2;
    float z, w;
    const bool big = a > 0.5f;
    if (big) {
        z = 0.5f * (1.0f - a);
        w = sqrtf(z);
    }
    else {
        w = a;
        z = w * w;
    }
    float p = 4.2163199048e-2f * z + 2.4181311049e-2f;
    p = p * z + 4.5470025998e-2f;
    p = p * z + 7.4953002686e-2f;
    p = p * z + 1.6666752422e-1f;
    p = p * z * w + w;
    if (big)
        p = DM_PI_2 - (p + p);
    return x < 0 ? -p : p;
}

// acos on [-1, 1] (Cephes acosf).
DM_HD float dm_acos(float x) {
    if (x < -1.0f) x = -1.0f;
    if (x > 1.0f) x = 1.0f;
    if (x > 0.5f)
        return 2.0f * dm_asin(sqrtf(0.5f * (1.0f - x)));
    if (x < -0.5f)
        return DM_PI - 2.0f * dm_asin(sqrtf(0.5f * (1.0f + x)));
    return DM_PI_2 - dm_asin(x);
}

// atan for x >= 0 (Cephes atanf kernel).
DM_HD float dm_atan_pos(float x) {
    float y;
    if (x > 2.414213562373095f) { // tan(3pi/8)
        y = DM_PI_2;
        x = -(1.0f / x);
    }
    else if (x > 0.4142135623730950f) { // tan(pi/8)
        y = DM_PI_4;
        x = (x - 1.0f) / (x + 1.0f);
    }
    else {
        y = 0.0f;
    }
    const float z = x * x;
    float p = 8.05374449538e-2f * z - 1.38776856032e-1f;
    p = p * z + 1.99777106478e-1f;
    p = p * z - 3.33329491539e-1f;
    p = p * z * x + x;
    return y + p;
}

// atan(x) for every x: odd extension of dm_atan_pos (the sign bit is kept, so atan(-0) = -0; +-inf -> +-pi/2, NaN -> NaN).
// applyBumpMapping's tiltAngle = atan(projLength / z) (common_device.cuh:184), where z may be 0 or negative.
DM_HD float dm_atan(float x) {
    if (x != x) return x;
    const float a = dm_atan_pos(fabsf(x));
    return (dm_f2u(x) >> 31) ? -a : a;
}

// atan2(y, x) in [-pi, pi].
DM_HD float dm_atan2(float y, float x) {
    if (x == 0.0f) {
        if (y > 0.0f) return DM_PI_2;
        if (y < 0.0f) return -DM_PI_2;
        // atan2(+-0, +-0): follow the sign of x like libm (+0 -> 0, -0 -> pi).
        return (dm_f2u(x) >> 31) ? ((dm_f2u(y) >> 31) ? -DM_PI : DM_PI) : y;
    }
    if (y == 0.0f)
        return x > 0.0f ? y : ((dm_f2u(y) >> 31) ? -DM_PI : DM_PI);
    const float a = dm_atan_pos(fabsf(y) / fabsf(x));
    float r = x > 0.0f ? a : DM_PI - a;
    return y < 0.0f ? -r : r;
}

// exp(x) for the NRC roughness remap (1 - e^{-r}); Cephes expf.
DM_HD float dm_exp(float x) {
    if (x > 88.0f) return INFINITY;
    if (x < -103.0f) return 0.0f;
    const float LOG2E = 1.44269504088896341f;
    const float k = floorf(x * LOG2E + 0.5f);
    float r = x - k * 0.693359375f;
    r = r - k * -2.12194440e-4f;
    const float z = r * r;
    float p = 1.9875691500e-4f * r + 1.3981999507e-3f;
    p = p * r + 8.3334519073e-3f;
    p = p * r + 4.1665795894e-2f;
    p = p * r + 1.6666665459e-1f;
    p = p * r + 5.0000001201e-1f;
    p = p * z + r + 1.0f;
    // scale by 2^k through the exponent field (k in [-149, 127] after the range checks).
    const int32_t ki = (int32_t)k;
    if (ki < -126) {
        const float s1 = dm_u2f((uint32_t)(ki + 100 + 127) << 23);
        return p * s1 * dm_u2f((uint32_t)(127 - 100) << 23);
    }
    return p * dm_u2f((uint32_t)(ki + 127) << 23);
}

// log(x) for x > 0 (normal or subnormal); Cephes logf.  Used by dm_pow for the sRGB transfer function of the output side.
DM_HD float dm_log(float x) {
    if (!(x > 0.0f)) return x == 0.0f ? -INFINITY : NAN;
    if (x == INFINITY) return INFINITY;
    // frexp through the exponent field: x = m * 2^e with m in [0.5, 1)
    int32_t e = 0;
    uint32_t bits = dm_f2u(x);
    if ((bits >> 23) == 0u) { // subnormal: scale by 2^24 first
        x = x * 16777216.0f;
        bits = dm_f2u(x);
        e = -24;
    }
    e += (int32_t)(bits >> 23) - 126;
    float m = dm_u2f((bits & 0x007FFFFFu) | 0x3F000000u);
    if (m < 0.707106781186547524f) {
        e -= 1;
        m = m + m - 1.0f;
    }
    else {
        m = m - 1.0f;
    }
    const float z = m * m;
    float y = 7.0376836292e-2f * m + -1.1514610310e-1f;
    y = y * m + 1.1676998740e-1f;
    y = y * m + -1.2420140846e-1f;
    y = y * m + 1.4249322787e-1f;
    y = y * m + -1.6668057665e-1f;
    y = y * m + 2.0000714765e-1f;
    y = y * m + -2.4999993993e-1f;
    y = y * m + 3.3333331174e-1f;
    y = y * m * z;
    const float fe = (float)e;
    y = y + -2.12194440e-4f * fe;
    y = y + -0.5f * z;
    float r = m + y;
    r = r + 0.693359375f * fe;
    return r;
}

// x^y for x >= 0 as exp(y log x): accurate to a few ULP for the exponents of the sRGB curves (|y log x| < 10), which is
// far below one 8-bit code; what matters is that both sides compute the same bits.
DM_HD float dm_pow(float x, float y) {
    if (x == 0.0f) return y > 0.0f ? 0.0f : (y == 0.0f ? 1.0f : INFINITY);
    return dm_exp(y * dm_log(x));
}
