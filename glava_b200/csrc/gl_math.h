/* gl_math.h — deterministic float32 transcendentals for the GLSL-semantics kernels.
 *
 * The reference's visualiser modules are GLSL 330 fragment shaders
 * (shaders/glava/{radial,circle}/1.frag use atan/sin, util/smooth.glsl:13-15,36 uses
 * log/sin).  GLSL leaves the precision of these built-ins implementation-defined, so a
 * from-scratch implementation has to pick one.  We pick functions built ONLY from
 * correctly-rounded IEEE-754 binary32 operations (+ - * / and fused multiply-add), so
 * that the sm_90a kernels (compiled --fmad=false, explicit __fmaf_rn) and a host
 * build (-ffp-contract=off, fmaf()) produce bit-identical results.  Accuracy is
 * <= 2 ulp over the ranges the shaders use, far inside GLSL's own allowance.
 *
 * Polynomials: classic Cephes single-precision minimax coefficients (sinf/cosf/atanf/
 * logf), argument reduction by two-constant Cody-Waite for sin.
 *
 * Usable from C (gnu11), C++ and CUDA.  All functions are static inline.
 */
#ifndef GLAVA_B200_GL_MATH_H
#define GLAVA_B200_GL_MATH_H

#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define GLM_FN __host__ __device__ static __forceinline__
#else
#include <math.h>
#define GLM_FN static inline
#endif

GLM_FN float glm_fma(float a, float b, float c) {
#if defined(__CUDA_ARCH__)
    return __fmaf_rn(a, b, c);
#else
    return fmaf(a, b, c);
#endif
}
GLM_FN float glm_mul(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
GLM_FN float glm_add(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}
GLM_FN float glm_div(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fdiv_rn(a, b);
#else
    return a / b;
#endif
}
/* correctly rounded square root (IEEE-754 requires it of both) */
GLM_FN float glm_sqrt(float x) {
#if defined(__CUDA_ARCH__)
    return __fsqrt_rn(x);
#else
    return sqrtf(x);
#endif
}
GLM_FN uint32_t glm_f2u(float f) {
#if defined(__CUDA_ARCH__)
    return __float_as_uint(f);
#else
    uint32_t u; memcpy(&u, &f, 4); return u;
#endif
}
GLM_FN float glm_u2f(uint32_t u) {
#if defined(__CUDA_ARCH__)
    return __uint_as_float(u);
#else
    float f; memcpy(&f, &u, 4); return f;
#endif
}
GLM_FN float glm_abs(float x) { return glm_u2f(glm_f2u(x) & 0x7fffffffu); }
/* round to nearest, ties to even (GLSL round() as llvmpipe/NVIDIA implement it) */
GLM_FN float glm_rint(float x) {
#if defined(__CUDA_ARCH__)
    return rintf(x);
#else
    return rintf(x);
#endif
}

/* sin(x), |x| <~ 8192.  k = nearest multiple of pi/2, r = x - k*pi/2 in two steps. */
GLM_FN float glm_sin(float x) {
    const float TWO_OVER_PI = 0.6366197466850281f;
    const float PIO2_HI = 1.57079637050628662109375f;   /* float(pi/2)                   */
    const float PIO2_LO = -4.37113900018624283e-08f;    /* pi/2 - PIO2_HI                */
    float kf = glm_rint(glm_mul(x, TWO_OVER_PI));
    float r  = glm_fma(-kf, PIO2_HI, x);
    r        = glm_fma(-kf, PIO2_LO, r);
    int   k  = (int) kf;
    float z  = glm_mul(r, r);
    float s, c;
    /* sin(r) on [-pi/4, pi/4] */
    s = glm_fma(z, -1.9515295891e-4f, 8.3321608736e-3f);
    s = glm_fma(z, s, -1.6666654611e-1f);
    s = glm_fma(glm_mul(s, z), r, r);
    /* cos(r) on [-pi/4, pi/4] */
    c = glm_fma(z, 2.443315711809948e-5f, -1.388731625493765e-3f);
    c = glm_fma(z, c, 4.166664568298827e-2f);
    c = glm_fma(glm_mul(c, z), z, glm_fma(-0.5f, z, 1.0f));
    float res = (k & 1) ? c : s;
    return (k & 2) ? -res : res;
}

/* atan(t) for t in [0, 1] */
GLM_FN float glm_atan01(float t) {
    float base = 0.0f;
    if (t > 0.4142135679721832275390625f) {             /* tan(pi/8) */
        t = glm_div(glm_add(t, -1.0f), glm_add(t, 1.0f));
        base = 0.785398185253143310546875f;             /* pi/4 */
    }
    float z = glm_mul(t, t);
    float p = glm_fma(z, 8.05374449538e-2f, -1.38776856032e-1f);
    p = glm_fma(z, p, 1.99777106478e-1f);
    p = glm_fma(z, p, -3.33329491539e-1f);
    p = glm_fma(glm_mul(p, z), t, t);
    return glm_add(base, p);
}

/* GLSL atan(y, x): angle of (x, y) in (-pi, pi]; atan(0, 0) := 0. */
GLM_FN float glm_atan2(float y, float x) {
    const float PI_F   = 3.1415927410125732421875f;
    const float PIO2_F = 1.57079637050628662109375f;
    float ax = glm_abs(x), ay = glm_abs(y);
    float mx = ax > ay ? ax : ay;
    float mn = ax > ay ? ay : ax;
    float r;
    if (mx == 0.0f) r = 0.0f;
    else {
        r = glm_atan01(glm_div(mn, mx));
        if (ay > ax) r = glm_add(PIO2_F, -r);
        if (x < 0.0f) r = glm_add(PI_F, -r);
    }
    return (glm_f2u(y) & 0x80000000u) ? -r : r;
}

/* natural log, x > 0, normal range (subnormals are not produced by the callers) */
GLM_FN float glm_log(float x) {
    uint32_t u = glm_f2u(x);
    int e = (int) ((u >> 23) & 0xffu) - 126;                 /* x = m * 2^e, m in [0.5, 1) */
    float m = glm_u2f((u & 0x007fffffu) | 0x3f000000u);
    if (m < 0.707106769084930419921875f) { e -= 1; m = glm_add(glm_add(m, m), -1.0f); }
    else m = glm_add(m, -1.0f);
    float z = glm_mul(m, m);
    float p = glm_fma(m, 7.0376836292e-2f, -1.1514610310e-1f);
    p = glm_fma(m, p, 1.1676998740e-1f);
    p = glm_fma(m, p, -1.2420140846e-1f);
    p = glm_fma(m, p, 1.4249322787e-1f);
    p = glm_fma(m, p, -1.6668057665e-1f);
    p = glm_fma(m, p, 2.0000714765e-1f);
    p = glm_fma(m, p, -2.4999993993e-1f);
    p = glm_fma(m, p, 3.3333331174e-1f);
    p = glm_mul(glm_mul(p, m), z);
    float fe = (float) e;
    p = glm_fma(fe, -2.12194440e-4f, p);
    p = glm_fma(-0.5f, z, p);
    float r = glm_add(m, p);
    return glm_fma(fe, 0.693359375f, r);
}

/* e^x (Cephes expf scheme: x = n ln2 + r, degree-5 polynomial, exact scaling by 2^n); overflow -> +inf, underflow -> 0 */
GLM_FN float glm_exp(float x) {
    if (x != x) return x;
    if (x > 88.7228317f) return glm_u2f(0x7f800000u);
    if (x < -103.278929f) return 0.0f;
    const float n = glm_rint(glm_mul(x, 1.44269504088896341f));
    float r = glm_fma(n, -0.693359375f, x);
    r = glm_fma(n, 2.12194440e-4f, r);
    const float z = glm_mul(r, r);
    float p = glm_fma(r, 1.9875691500e-4f, 1.3981999507e-3f);
    p = glm_fma(r, p, 8.3334519073e-3f);
    p = glm_fma(r, p, 4.1665795894e-2f);
    p = glm_fma(r, p, 1.6666665459e-1f);
    p = glm_fma(r, p, 5.0000001201e-1f);
    float y = glm_add(glm_fma(p, z, r), 1.0f);
    /* y * 2^n in two exact steps (n may exceed one exponent field's reach near the ends of the range) */
    int k = (int) n;
    const int k1 = k / 2; k -= k1;
    y = glm_mul(y, glm_u2f((uint32_t) (k1 + 127) << 23));
    return glm_mul(y, glm_u2f((uint32_t) (k + 127) << 23));
}
/* 2^x: the integer part is exact, the fraction goes through glm_exp */
GLM_FN float glm_exp2(float x) {
    if (x != x) return x;
    if (x > 128.0f) return glm_u2f(0x7f800000u);
    if (x < -150.0f) return 0.0f;
    const float n = glm_rint(x);
    float y = glm_exp(glm_mul(glm_add(x, -n), 0.693147180559945309f));   /* |x - n| <= 0.5, the subtraction is exact */
    int k = (int) n;
    const int k1 = k / 2; k -= k1;
    y = glm_mul(y, glm_u2f((uint32_t) (k1 + 127) << 23));
    return glm_mul(y, glm_u2f((uint32_t) (k + 127) << 23));
}
/* x^y for x > 0 as GLSL defines it (exp2(y * log2(x)) up to precision; undefined for x < 0): exp(y * log(x)); 0^y = 0 for y > 0 */
GLM_FN float glm_pow(float x, float y) {
    if (x == 0.0f) return y > 0.0f ? 0.0f : glm_u2f(0x7fc00000u);
    return glm_exp(glm_mul(y, glm_log(x)));
}

#endif /* GLAVA_B200_GL_MATH_H */
