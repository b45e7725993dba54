// spectrum_core.h — element-wise maths of the spectrum path, shared by the CUDA kernel
// and the host-emulation tests.  Compiled with --fmad=false (device) / -ffp-contract=off
// (host): every float op is a separately rounded IEEE binary32 op.
//
// Reference for every function is cited at its definition.
#ifndef GLAVA_B200_SPECTRUM_CORE_H
#define GLAVA_B200_SPECTRUM_CORE_H

#include "../../include/glava_b200.h"
#include "fft_core.h"

#include <math.h>

namespace glb {

// ---- GLSL helper semantics (DESIGN.md "GLSL semantics") ---------------------------------------
GLB_HD float g_clamp(float v, float lo, float hi) { return v < lo ? lo : (v > hi ? hi : v); }
GLB_HD float g_min(float a, float b) { return b < a ? b : a; }
GLB_HD float g_max(float a, float b) { return a < b ? b : a; }
GLB_HD float g_mod(float x, float y) { return x - y * floorf(x / y); }
GLB_HD float g_sign(float x) { return x > 0.0f ? 1.0f : (x < 0.0f ? -1.0f : 0.0f); }
// float -> unorm store: clamp, then ONE rounding of the float32 product, ties to even (Mesa's _mesa_float_to_unorm; the
// llvmpipe goldens pin it: the reference's R16 uploads are reproduced bit for bit), NaN -> 0.
// cvt.rni on the device, lrintf on the host (default rounding mode): the same bits.
#if defined(__CUDA_ARCH__)
GLB_HD uint32_t g_rne(float v) { return (uint32_t) __float2int_rn(v); }
#else
GLB_HD uint32_t g_rne(float v) { return (uint32_t) lrintf(v); }
#endif
GLB_HD uint32_t unorm8(float c)  { return c > 0.0f ? (c < 1.0f ? g_rne(c * 255.0f) : 255u) : 0u; }
GLB_HD uint32_t unorm16(float c) { return c > 0.0f ? (c < 1.0f ? g_rne(c * 65535.0f) : 65535u) : 0u; }
// unorm fetch = (float) u / MAX, correctly rounded.  Computed as a reciprocal multiply plus one
// fma residual correction, which equals the IEEE quotient for every u in range
// (exhaustively checked: tests/test_emul_parity.py::test_unorm_fetch_is_exact_division).
GLB_HD float from8(uint32_t u) {
    const float x = (float) u, r = 1.0f / 255.0f;
    float q = x * r;
    return glm_fma(glm_fma(-q, 255.0f, x), r, q);
}
GLB_HD float from16(uint32_t u) {
    const float x = (float) u, r = 1.0f / 65535.0f;
    float q = x * r;
    return glm_fma(glm_fma(-q, 65535.0f, x), r, q);
}

#define GLB_PI    3.14159265359f
#define GLB_TWOPI 6.28318530718f

// ---- transform_fft tail: |.|, log(x+1)/3, index ramp — render.c:842-846 ------------------------
// `data[n] + 1` is a float add in the reference too; its log() and /3 run in double and round to
// float once.  Here both run in float (glm_log: <= 1 ulp; IEEE divide), i.e. within ~2.5e-7 relative
// of the reference's value — 40x inside the 1e-5 tolerance and far below the FFT's own rounding —
// at a fifth of the instruction count of a software double log.  i / n is exact (n is a power of two).
GLB_HD float fft_post(float v, int i, int n, float fft_scale, float fft_cutoff) {
    v = fabsf(v);
    v = glm_log(v + 1.0f) / 3.0f;
    float ramp = (((float) i * (1.0f / (float) n)) * fft_scale) + (1.0f - fft_cutoff);
    return v * (ramp > 1.0f ? ramp : 1.0f);
}

// ---- pipeline A: transform_gravity (render.c:720-736) -------------------------------------------
GLB_HD float gravity_a(float b, float* applied, float g) {
    float a = *applied;
    a = (b >= a) ? (b - g) : (a - g);
    *applied = a;
    return a;
}
// transform_average weight (render.c:661,766): window_frame(f, avg_frames - 1) expands to
// 0.6 - 0.4*cos(TWOPI*f/F - 1), double.  Host-computed LUT, once per build: derive() in capi.cu.

// ---- pipeline B (R16 GL passes) ------------------------------------------------------------------
// K1 + K2: GL_MAX blend into gr_store then gravity_pass.frag:8, render.c:2199-2228
GLB_HD uint32_t gravity_b(uint32_t uploaded, uint32_t gr_store, float diff) {
    uint32_t g = gr_store > uploaded ? gr_store : uploaded;
    return unorm16(from16(g) - diff);
}

// ---- K5: util/smooth.glsl:13-64 via util/smooth_pass.frag:14-16 -----------------------------------
struct SmoothParams {
    float smooth_factor, sample_range, sample_scale, hybrid_weight;
    int   sample_mode, round_formula;
};
GLB_HD SmoothParams smooth_params(const glava_b200_params& p) {
    return { p.smooth_factor, p.sample_range, p.sample_scale, p.hybrid_weight, p.sample_mode, p.round_formula };
}
GLB_HD float scale_audio(const SmoothParams& p, float idx) {                 // smooth.glsl:13-15
    return -glm_log((-(p.sample_range) * idx) + 1.0f) / p.sample_scale;
}
GLB_HD float round_formula(const SmoothParams& p, float x) {                 // common.glsl:17-21
    switch (p.round_formula) {
        case 1:  return x;
        case 2:  return sqrtf(1.0f - ((x - 1.0f) * (x - 1.0f)));
        default: return (0.5f * glm_sin((GLB_PI * x) - (GLB_PI / 2.0f))) + 0.5f;
    }
}
// tex: R16 texels (n of them) as uint16; texelFetch out of range reads 0
GLB_HD float fetch16(const uint16_t* tex, int n, int i) {
    return (i < 0 || i >= n) ? 0.0f : from16(tex[i]);
}
// The taps of smooth_audio() for one output position: texel index round(s) and weight
// ROUND_FORMULA(clamp((m - |rm - s|) / m, 0, 1)) for s = smin, smin + 1, ... (<= smax in `average`
// mode, < smax otherwise; smooth.glsl:33,44,55).  Index and weight depend only on the parameters and
// on idx — NOT on the audio — which is what lets the kernel precompute them once (SmoothTable).
template <class Tap>
GLB_HD void smooth_enumerate(const SmoothParams& p, int n, float idx, Tap tap) {
    float fn = (float) n;
    float smin = scale_audio(p, g_clamp(idx - p.smooth_factor, 0.0f, 1.0f)) * fn;
    float smax = scale_audio(p, g_clamp(idx + p.smooth_factor, 0.0f, 1.0f)) * fn;
    float m = ((smax - smin) / 2.0f), s;
    float rm = smin + m;
    if (p.sample_mode == 0) {
        for (s = smin; s <= smax; s += 1.0f) tap((int) glm_rint(s), round_formula(p, g_clamp((m - fabsf(rm - s)) / m, 0.0f, 1.0f)));
    } else {
        for (s = smin; s < smax; s += 1.0f) tap((int) glm_rint(s), round_formula(p, g_clamp((m - fabsf(rm - s)) / m, 0.0f, 1.0f)));
    }
}
// running state of the three SAMPLE_MODEs, fed tap by tap in the GLSL loop's order
struct SmoothAcc {
    float avg, weight, vmax;
    GLB_HD void init() { avg = 0.0f; weight = 0.0f; vmax = 0.0f; }
    GLB_HD void add(float texel, float w) {          // smooth.glsl:34-37 / 45-50 / 56-58
        weight += w;
        float v = texel * w;
        avg += v;
        if (vmax < v) vmax = v;
    }
    GLB_HD void add_noweight(float texel, float w) { // same, `weight` supplied separately (precomputed)
        float v = texel * w;
        avg += v;
        if (vmax < v) vmax = v;
    }
    GLB_HD float result(const SmoothParams& p) const {
        if (p.sample_mode == 0) return avg / weight;
        if (p.sample_mode == 2) return (vmax * (1.0f - p.hybrid_weight)) + ((avg / weight) * p.hybrid_weight);
        return vmax;
    }
};
GLB_HD float smooth_audio_raw(const SmoothParams& p, const uint16_t* tex, int n, float idx) {
    SmoothAcc acc; acc.init();
    smooth_enumerate(p, n, idx, [&](int i, float w) { acc.add(fetch16(tex, n, i), w); });
    return acc.result(p);
}
// one output texel of the smooth pass: viewport n x 1, gl_FragCoord.x = x + 0.5, uniform w = n
GLB_HD uint32_t smooth_pass_texel(const SmoothParams& p, const uint16_t* tex, int n, int x) {
    return unorm16(smooth_audio_raw(p, tex, n, ((float) x + 0.5f) / (float) n));
}

}  // namespace glb
#endif
