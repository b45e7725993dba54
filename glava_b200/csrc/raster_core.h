// raster_core.h — the visualiser modules' per-pixel maths as __host__ __device__ functions.
//
// Each function restates one GLSL fragment shader of the reference (cited at the function)
// under the GLSL semantics listed in DESIGN.md.  Column-only and row-only sub-expressions
// are factored out (bars_column / bars_row, graph_height / graph_row, wave_column) so the
// CUDA kernels can hoist them; the generic per-pixel entry points recombine them, so the
// hoisted and the per-pixel evaluation are the same arithmetic by construction.
//
// All multi-stage modules are evaluated in ONE pass: stages that read the previous RGBA8
// surface (premultiply, 8-neighbour stencils) are reproduced by re-deriving the neighbour's
// 8-bit-quantised stage-1 value in registers — no intermediate surface touches HBM.
#ifndef GLAVA_B200_RASTER_CORE_H
#define GLAVA_B200_RASTER_CORE_H

#include "spectrum_core.h"

namespace glb {

struct f4 { float r, g, b, a; };
GLB_HD f4 mk4(float r, float g, float b, float a) { f4 v = { r, g, b, a }; return v; }
GLB_HD f4 mk4a(const float* c) { return mk4(c[0], c[1], c[2], c[3]); }
GLB_HD uint32_t pack8(f4 c) { return unorm8(c.r) | (unorm8(c.g) << 8) | (unorm8(c.b) << 16) | (unorm8(c.a) << 24); }
GLB_HD f4 unpack8(uint32_t u) { return mk4(from8(u & 255u), from8((u >> 8) & 255u), from8((u >> 16) & 255u), from8(u >> 24)); }
GLB_HD f4 g_mix(f4 a, f4 b, float t) {
    float s = 1.0f - t;
    return mk4(a.r * s + b.r * t, a.g * s + b.g * t, a.b * s + b.b * t, a.a * s + b.a * t);
}
// ---- compiled colour expressions (glava_b200_color_prog): any COLOR / BAR_OUTLINE macro the closed forms do not cover ----
// One instruction = one lane-wise float operation, each individually rounded like the GLSL it was compiled from.
#define GLB_COP1(expr) { const f4 A = reg[o.a]; float v; f4 R; \
    v = A.r; R.r = (expr); v = A.g; R.g = (expr); v = A.b; R.b = (expr); v = A.a; R.a = (expr); reg[o.dst] = R; } break
#define GLB_COP2(expr) { const f4 A = reg[o.a], B = reg[o.b]; float v, w; f4 R; \
    v = A.r; w = B.r; R.r = (expr); v = A.g; w = B.g; R.g = (expr); v = A.b; w = B.b; R.b = (expr); v = A.a; w = B.a; R.a = (expr); \
    reg[o.dst] = R; } break
#define GLB_COP3(expr) { const f4 A = reg[o.a], B = reg[o.b], Cc = reg[((int) o.imm) & (GLAVA_B200_COLOR_REGS - 1)]; float v, w, u; f4 R; \
    v = A.r; w = B.r; u = Cc.r; R.r = (expr); v = A.g; w = B.g; u = Cc.g; R.g = (expr); \
    v = A.b; w = B.b; u = Cc.b; R.b = (expr); v = A.a; w = B.a; u = Cc.a; R.a = (expr); reg[o.dst] = R; } break
GLB_HD float cop_smoothstep(float e0, float e1, float x) {
    const float t = g_clamp((x - e0) / (e1 - e0), 0.0f, 1.0f);
    return (t * t) * (3.0f - (2.0f * t));
}
GLB_HD float& cop_lane(f4& r, int k) { return k == 0 ? r.r : (k == 1 ? r.g : (k == 2 ? r.b : r.a)); }
// ---- the colour VM's transcendentals over the whole float range (DESIGN §4.5) ----
// The module kernels call gl_math.h with bounded, positive arguments; a user's expression can pass any float.  These
// wrappers give gl_math.h's results where its reductions hold, and IEEE's answers beyond: sin / cos / tan of any finite x
// lie in [-1, 1] (Payne-Hanek past |x| = 8192), log is -inf at +-0, NaN below 0 and at NaN, +inf at +inf and finite on
// subnormals, atan(+-inf, +-inf) is +-pi/4 or +-3pi/4.  Integer and correctly rounded float operations only, so the
// device and the host build agree bit for bit.
GLB_HD float cvm_inf() { return glm_u2f(0x7f800000u); }
GLB_HD float cvm_nan() { return glm_u2f(0x7fffffffu); }
// bits 32 (j - 1) + 1 .. 32 j after the binary point of 2/pi; word 0 stands for 32 zero bits before it
GLB_HD uint32_t cvm_2opi_word(int j) {
    switch (j) {
        case 1: return 0xa2f9836eu; case 2: return 0x4e441529u; case 3: return 0xfc2757d1u; case 4: return 0xf534ddc0u;
        case 5: return 0xdb629599u; case 6: return 0x3c439041u; case 7: return 0xfe5163abu; default: return 0u;
    }
}
GLB_HD uint32_t cvm_funnel(uint32_t hi, uint32_t lo, int s) { return s ? (hi << s) | (lo >> (32 - s)) : hi; }
// x = r + q pi/2 (mod 2 pi), |r| <= pi/4, for finite |x| > 8192.  |x| = m 2^e with m < 2^24, so x 2/pi = m sum_k t_k 2^(e - k)
// over the bits t_k of 2/pi; the terms k <= e - 2 are multiples of 4.  The 96 bits from k = e - 1 on form W, and
// x 2/pi = m W 2^-94 (mod 4) up to less than 2^-71 from the bits past W.
GLB_HD float cvm_reduce_large(float x, int* q) {
    const uint32_t u = glm_f2u(x);
    const uint64_t m = (u & 0x007fffffu) | 0x00800000u;
    const int k0 = (int) ((u >> 23) & 0xffu) - 120, i = k0 >> 5, s = k0 & 31;   // k0 = (e - 1) + 31: bit offset in the words
    const uint32_t t0 = cvm_2opi_word(i), t1 = cvm_2opi_word(i + 1), t2 = cvm_2opi_word(i + 2), t3 = cvm_2opi_word(i + 3);
    const uint64_t p2 = m * cvm_funnel(t2, t3, s);
    const uint64_t p1 = m * cvm_funnel(t1, t2, s) + (p2 >> 32);
    const uint64_t p0 = m * cvm_funnel(t0, t1, s) + (p1 >> 32);
    int k = (int) ((p0 >> 30) & 3u);
    int64_t f = (int64_t) (((p0 & 0x3fffffffu) << 32) | (p1 & 0xffffffffu));  // the fraction in units of 2^-62
    if (f >= ((int64_t) 1 << 61)) { f -= (int64_t) 1 << 62; k += 1; }        // to the nearest quadrant
    // r = f 2^-62 pi/2, with f split into two floats and pi/2 into PIO2_HI + PIO2_LO (as glm_sin)
    const float fh = (float) f, fl = (float) (f - (int64_t) fh);
    float r = glm_fma(fh, 1.57079637050628662109375f, glm_fma(fh, -4.37113900018624283e-08f, glm_mul(fl, 1.57079637050628662109375f)));
    r = glm_mul(r, 0x1p-62f);
    if (u >> 31) { r = -r; k = -k; }
    *q = k & 3;
    return r;
}
// any x: glm_sin's own reduction up to |x| = 8192, Payne-Hanek beyond, NaN for inf and NaN
GLB_HD float cvm_reduce(float x, int* q) {
    const float ax = glm_abs(x);
    if (ax <= 8192.0f) {
        const float kf = glm_rint(glm_mul(x, 0.6366197466850281f));
        float r = glm_fma(-kf, 1.57079637050628662109375f, x);
        r = glm_fma(-kf, -4.37113900018624283e-08f, r);
        *q = (int) kf & 3;
        return r;
    }
    if (!(ax < cvm_inf())) { *q = 0; return cvm_nan(); }
    return cvm_reduce_large(x, q);
}
// sin(r + q pi/2), |r| <= pi/4: glm_sin's polynomials
GLB_HD float cvm_sin_q(float r, int q) {
    const float z = glm_mul(r, r);
    float s = glm_fma(z, -1.9515295891e-4f, 8.3321608736e-3f);
    s = glm_fma(z, s, -1.6666654611e-1f);
    s = glm_fma(glm_mul(s, z), r, r);
    float c = glm_fma(z, 2.443315711809948e-5f, -1.388731625493765e-3f);
    c = glm_fma(z, c, 4.166664568298827e-2f);
    c = glm_fma(glm_mul(c, z), z, glm_fma(-0.5f, z, 1.0f));
    const float res = (q & 1) ? c : s;
    return (q & 2) ? -res : res;
}
GLB_HD float cvm_sin(float x) {
    if (glm_abs(x) <= 8192.0f) return glm_sin(x);
    int q; const float r = cvm_reduce(x, &q);
    return cvm_sin_q(r, q);
}
GLB_HD float cvm_cos(float x) { int q; const float r = cvm_reduce(x, &q); return cvm_sin_q(r, q + 1); }
GLB_HD float cvm_tan(float x) { int q; const float r = cvm_reduce(x, &q); return glm_div(cvm_sin_q(r, q), cvm_sin_q(r, q + 1)); }
GLB_HD float cvm_log(float x) {
    if (!(x > 0.0f)) return x == 0.0f ? -cvm_inf() : cvm_nan();
    if (x == cvm_inf()) return x;
    if (x < 1.17549435e-38f) return glm_add(glm_log(glm_mul(x, 16777216.0f)), -16.63553233343868742f);   // subnormal: log(x 2^24) - 24 ln 2
    return glm_log(x);
}
// glm_exp returns 0 below ln 2^-149; e^x rounds to 2^-149 down to ln 2^-150
GLB_HD float cvm_exp(float x) { return (x < -103.278929f && x > -103.972077f) ? glm_u2f(1u) : glm_exp(x); }
GLB_HD float cvm_pow(float x, float y) { return x == 0.0f ? glm_pow(x, y) : cvm_exp(glm_mul(y, cvm_log(x))); }
GLB_HD float cvm_atan2(float y, float x) {
    if (glm_abs(x) == cvm_inf() && glm_abs(y) == cvm_inf()) {
        const float r = x > 0.0f ? 0.785398185253143310546875f : 2.35619449615478515625f;   // float(pi/4), float(3 pi/4)
        return (glm_f2u(y) & 0x80000000u) ? -r : r;
    }
    return glm_atan2(y, x);
}
GLB_HD_NOINLINE f4 eval_color_prog(const glava_b200_color_prog& c, float x) {
    f4 reg[GLAVA_B200_COLOR_REGS];
    for (int i = 0; i < GLAVA_B200_COLOR_REGS; ++i) reg[i] = mk4(0.0f, 0.0f, 0.0f, 0.0f);
    const int n = c.n_ops < GLAVA_B200_COLOR_OPS ? c.n_ops : GLAVA_B200_COLOR_OPS;
    for (int i = 0; i < n; ++i) {
        glava_b200_color_op o = c.ops[i];
        o.dst &= GLAVA_B200_COLOR_REGS - 1; o.a &= GLAVA_B200_COLOR_REGS - 1; o.b &= GLAVA_B200_COLOR_REGS - 1;
        switch (o.op) {
            case GLAVA_B200_COP_SPLAT: reg[o.dst] = mk4(o.imm, o.imm, o.imm, o.imm); break;
            case GLAVA_B200_COP_VAR:   reg[o.dst] = mk4(x, x, x, x); break;
            case GLAVA_B200_COP_LANE:  cop_lane(reg[o.dst], o.a & 3) = o.imm; break;
            case GLAVA_B200_COP_SHUF: {
                const f4 A = reg[o.a]; f4 R = reg[o.dst];
                const int m = (int) o.imm;
                for (int k = 0; k < 4; ++k) {
                    const int sel = (m >> (3 * k)) & 7;
                    if (sel < 4) { f4 T = A; cop_lane(R, k) = cop_lane(T, sel); }
                }
                reg[o.dst] = R;
            } break;
            case GLAVA_B200_COP_ADD:   GLB_COP2(v + w);
            case GLAVA_B200_COP_SUB:   GLB_COP2(v - w);
            case GLAVA_B200_COP_MUL:   GLB_COP2(v * w);
            case GLAVA_B200_COP_DIV:   GLB_COP2(v / w);
            case GLAVA_B200_COP_MIN:   GLB_COP2(g_min(v, w));
            case GLAVA_B200_COP_MAX:   GLB_COP2(g_max(v, w));
            case GLAVA_B200_COP_MOD:   GLB_COP2(g_mod(v, w));
            case GLAVA_B200_COP_STEP:  GLB_COP2(w < v ? 0.0f : 1.0f);
            case GLAVA_B200_COP_NEG:   GLB_COP1(-v);
            case GLAVA_B200_COP_ABS:   GLB_COP1(fabsf(v));
            case GLAVA_B200_COP_FLOOR: GLB_COP1(floorf(v));
            case GLAVA_B200_COP_CEIL:  GLB_COP1(ceilf(v));
            case GLAVA_B200_COP_FRACT: GLB_COP1(v - floorf(v));
            case GLAVA_B200_COP_SQRT:  GLB_COP1(sqrtf(v));
            case GLAVA_B200_COP_SIN:   GLB_COP1(cvm_sin(v));
            case GLAVA_B200_COP_COS:   GLB_COP1(cvm_cos(v));
            case GLAVA_B200_COP_LOG:   GLB_COP1(cvm_log(v));
            case GLAVA_B200_COP_SIGN:  GLB_COP1(g_sign(v));
            case GLAVA_B200_COP_TRUNC: GLB_COP1(truncf(v));
            case GLAVA_B200_COP_MIX:   GLB_COP3((v * (1.0f - u)) + (w * u));
            case GLAVA_B200_COP_CLAMP: GLB_COP3(g_min(g_max(v, w), u));
            case GLAVA_B200_COP_SMOOTHSTEP: GLB_COP3(cop_smoothstep(v, w, u));
            case GLAVA_B200_COP_LT:    GLB_COP2(v < w ? 1.0f : 0.0f);
            case GLAVA_B200_COP_LE:    GLB_COP2(v <= w ? 1.0f : 0.0f);
            case GLAVA_B200_COP_EQ:    GLB_COP2(v == w ? 1.0f : 0.0f);
            case GLAVA_B200_COP_NE:    GLB_COP2(v != w ? 1.0f : 0.0f);
            case GLAVA_B200_COP_AND:   GLB_COP2((v != 0.0f && w != 0.0f) ? 1.0f : 0.0f);
            case GLAVA_B200_COP_OR:    GLB_COP2((v != 0.0f || w != 0.0f) ? 1.0f : 0.0f);
            case GLAVA_B200_COP_NOT:   GLB_COP1(v != 0.0f ? 0.0f : 1.0f);
            case GLAVA_B200_COP_SELECT: GLB_COP3(u != 0.0f ? v : w);
            case GLAVA_B200_COP_EXP:   GLB_COP1(cvm_exp(v));
            case GLAVA_B200_COP_EXP2:  GLB_COP1(glm_exp2(v));
            case GLAVA_B200_COP_LOG2:  GLB_COP1(cvm_log(v) * 1.44269504088896341f);
            case GLAVA_B200_COP_POW:   GLB_COP2(cvm_pow(v, w));
            case GLAVA_B200_COP_ATAN2: GLB_COP2(cvm_atan2(v, w));
            case GLAVA_B200_COP_TAN:   GLB_COP1(cvm_tan(v));
            default: break;
        }
    }
    return reg[c.result & (GLAVA_B200_COLOR_REGS - 1)];
}
GLB_HD f4 eval_color(const glava_b200_color& c, const glava_b200_color_prog& prog, float x) {
    if (c.mode == 1) return mk4a(c.lo);
    if (c.mode == 2) return eval_color_prog(prog, x);
    return g_mix(mk4a(c.lo), mk4a(c.hi), g_clamp(x / c.gradient, 0.0f, 1.0f));
}
GLB_HD uint32_t premultiply8(uint32_t px) {                              // util/premultiply.frag:12-15
    f4 f = unpack8(px);
    return pack8(mk4(f.r * f.a, f.g * f.a, f.b * f.a, f.a));
}

// ---- non-native opacity (`setopacity "none"` / "xroot": premultiply_alpha == 0) --------------------------------------
// The reference then enables GL_BLEND with glBlendFunc(GL_SRC_ALPHA, GL_ONE_MINUS_SRC_ALPHA) for every module stage
// (render.c:1467-1470), each drawn into a target glClear'd to the `setbg` colour (render.c:1700, 2028), and skips the
// premultiply stages (util/premultiply.frag:2-4).  Blending happens in the target's own 8-bit normalised fixed point, as
// llvmpipe does it (tests/golden/llvmpipe_golden.npz: the reference's non-native-opacity frames are reproduced bit for bit):
// the fragment is converted to unorm8 first, then C = mul_norm(Cs, As) + mul_norm(Cd, 255 - As) per channel, alpha
// included, saturating; mul_norm(a, b) = (t + (t >> 8)) >> 8 with t = a * b + 128 (a * b / 255 rounded).
// NATIVE = true is the shipped mode and compiles to exactly the code it was before this existed.
GLB_HD uint32_t mul_norm8(uint32_t a, uint32_t b) { const uint32_t t = a * b + 128u; return (t + (t >> 8)) >> 8; }
GLB_HD uint32_t blend_store(const glava_b200_params& p, f4 s) {
    const uint32_t S = pack8(s), D = pack8(mk4a(p.clear_color));
    const uint32_t a = S >> 24, ia = 255u - a;
    uint32_t out = 0;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        uint32_t r = mul_norm8((S >> (8 * c)) & 255u, a) + mul_norm8((D >> (8 * c)) & 255u, ia);
        out |= (r > 255u ? 255u : r) << (8 * c);
    }
    return out;
}
template <bool NATIVE> GLB_HD uint32_t stage_store(const glava_b200_params& p, f4 s) { return NATIVE ? pack8(s) : blend_store(p, s); }
template <bool NATIVE> GLB_HD uint32_t stage_bg(const glava_b200_params& p) { return NATIVE ? 0u : blend_store(p, mk4(0.0f, 0.0f, 0.0f, 0.0f)); }

// the 1-D textures bound as audio_l / audio_r for one stream
struct AudioTex {
    const uint16_t* l; const uint16_t* r;
    int n; int pre_smoothed; SmoothParams sp;
};
// smooth_audio() as the module sees it (smooth.glsl:23-64 with _PRE_SMOOTHED_AUDIO, render.c:292)
GLB_HD float sample_audio(const AudioTex& t, const uint16_t* tex, float idx) {
    if (t.pre_smoothed) return fetch16(tex, t.n, (int) glm_rint(idx * (float) t.n));
    return smooth_audio_raw(t.sp, tex, t.n, idx);
}
GLB_HD float sample_audio_adj(const AudioTex& t, const uint16_t* tex, float idx, float pixel) {   // smooth.glsl:67-73
    float al = sample_audio(t, tex, g_max(idx - pixel, 0.0f)),
          am = sample_audio(t, tex, idx),
          ar = sample_audio(t, tex, g_min(idx + pixel, 1.0f));
    return (al + am + ar) / 3.0f;
}

// =================================== bars (bars/1.frag:36-135) ===================================
struct BarsCol { int cls; float v, vm; };      // cls 0: gap/out of range, 1: bar interior column, 2: bar edge column
struct BarsRow { uint32_t fill, outl; };

// ax = AREA_X (gl_FragCoord.x, or .y when MIRROR_YX), aw = AREA_WIDTH.
// Geometry half of the column: which texture (0 = audio_l, 1 = audio_r) is sampled at which
// normalised position pp; returns false in gaps / outside [-1, 1].  `md_inner` = interior column.
GLB_HD bool bars_column_coord(const glava_b200_params& p, float ax, int aw, int* chan, float* pp_out, bool* md_inner) {
    float dx;
    if (p.channels == 2) dx = ax - (float) (aw / 2);
    else dx = p.bars_invert == 1 ? (float) aw - ax : ax;
    float section = p.bars_width + p.bars_gap;
    float center = section / 2.0f;
    float m = fabsf(g_mod(dx, section));
    float md = m - center;
    float nbars = floorf(((float) aw * 0.5f) / section) * 2.0f;
    float hi = ceilf(p.bars_width / 2.0f), lo = -floorf(p.bars_width / 2.0f);
    if (!(md < hi && md >= lo)) return false;
    float s = dx / section;
    float pp = (g_sign(s) == 1.0f ? ceilf(s) : floorf(s));
    if (p.channels == 2) pp /= (nbars / 2.0f); else pp /= nbars;
    pp += g_sign(pp) * ((0.5f + center) / (float) aw);
    if (pp > 1.0f || pp < -1.0f) return false;
    if (pp > 0.0f) {
        if (p.bars_direction == 1) pp = 1.0f - pp;
        *chan = (p.channels == 1 || p.bars_invert > 0) ? 0 : 1;
    } else {
        pp = fabsf(pp);
        if (p.bars_direction == 1) pp = 1.0f - pp;
        *chan = (p.channels == 1) ? 0 : (p.bars_invert > 0 ? 1 : 0);
    }
    *pp_out = pp;
    *md_inner = !(p.bars_outline_width > 0.0f) ||
                (md < hi - p.bars_outline_width && md >= lo + p.bars_outline_width);
    return true;
}
GLB_HD BarsCol bars_column(const glava_b200_params& p, const AudioTex& t, float ax, int aw) {
    BarsCol c = { 0, 0.0f, 0.0f };
    int chan; float pp; bool inner;
    if (!bars_column_coord(p, ax, aw, &chan, &pp, &inner)) return c;
    float v = sample_audio(t, chan ? t.r : t.l, pp);
    v *= p.bars_amplify;
    c.v = v; c.vm = v - p.bars_outline_width;
    c.cls = inner ? 1 : 2;
    return c;
}
template <bool NATIVE> GLB_HD BarsRow bars_row_t(const glava_b200_params& p, float d) {
    f4 col = eval_color(p.bars_color, p.bars_color_prog, d);
    f4 outl = p.bars_outline_mode == 0 ? mk4(col.r * 1.5f, col.g * 1.5f, col.b * 1.5f, col.a)
            : (p.bars_outline_mode == 2 ? eval_color_prog(p.bars_outline_prog, d) : mk4a(p.bars_outline));
    BarsRow r = { stage_store<NATIVE>(p, col), stage_store<NATIVE>(p, outl) };
    return r;
}
GLB_HD BarsRow bars_row(const glava_b200_params& p, float d) { return bars_row_t<true>(p, d); }
// bg: what a fragment left at vec4(0) stores (0 natively, the blended clear colour otherwise)
GLB_HD uint32_t bars_combine(const glava_b200_params& p, const BarsCol& c, const BarsRow& r, float d, uint32_t bg = 0u) {
    if (c.cls == 0) return bg;
    if (d < c.vm) return c.cls == 1 ? r.fill : r.outl;
    if (p.bars_outline_width > 0.0f && d <= c.v) return r.outl;
    return bg;
}
GLB_HD uint32_t bars_px(const glava_b200_params& p, const AudioTex& t, int x, int y) {
    float fx = (float) x + 0.5f, fy = (float) y + 0.5f;
    int   aw = p.bars_mirror_yx ? p.h : p.w, ah = p.bars_mirror_yx ? p.w : p.h;
    float ax = p.bars_mirror_yx ? fy : fx,  ay = p.bars_mirror_yx ? fx : fy;
    float d = p.bars_flip ? (float) ah - ay : ay;
    if (!p.premultiply_alpha) return bars_combine(p, bars_column(p, t, ax, aw), bars_row_t<false>(p, d), d, stage_bg<false>(p));
    return bars_combine(p, bars_column(p, t, ax, aw), bars_row(p, d), d);
}

// ================================= radial (radial/1.frag:32-116, 2.frag) =========================
GLB_HD f4 apply_frag(f4 f, f4 c) {                                         // radial/1.frag:35 (_USE_ALPHA > 0)
    float k = 1.0f - g_clamp(f.a, 0.0f, 1.0f);
    return mk4(f.r * f.a + c.r * k, f.g * f.a + c.g * k, f.b * f.a + c.b * k, g_max(c.a, f.a));
}
// Everything radial/1.frag + radial/2.frag compute for a pixel EXCEPT the audio lookup: the only
// audio-dependent step is the test `d <= v` for a pixel inside a bar, so a pixel is fully described by
// its two possible final RGBA8 values, the bar it belongs to and its d (= distance - C_RADIUS).
// raster_radial_kernel caches this per renderer (the same for every stream and frame).
struct RadialGeo {
    uint32_t lit;      // final value if the bar reaches this pixel (d <= v - BAR_OUTLINE_WIDTH)
    uint32_t unlit;    // final value otherwise (ring or 0)
    float    dR;       // d - C_RADIUS
    int      bar;      // -1: not on a bar; else (side << 16) | k with side 0 = audio_l, 1 = audio_r, pos = k / (NBARS/2)
    uint32_t band;     // BAR_OUTLINE_WIDTH > 0 only: final value in the bar's end cap, v - BAR_OUTLINE_WIDTH < d <= v
};
// `BAR_WIDTH / 2` as radial/1.frag:62,79,88 evaluate it: an integer division when the macro is an integer literal
GLB_HD float radial_bar_half(const glava_b200_params& p) {
    return p.radial_bar_width_int ? (float) ((int) p.radial_bar_width / 2) : p.radial_bar_width / 2.0f;
}
GLB_HD uint32_t radial_finish(const glava_b200_params& p, f4 frag) {
    if (!p.premultiply_alpha) return blend_store(p, frag);                 // stage 1 blended, radial/2.frag skipped
    return premultiply8(pack8(frag));                                      // radial/2.frag
}
GLB_HD RadialGeo radial_geometry(const glava_b200_params& p, int x, int y) {
    RadialGeo g = { 0u, 0u, 0.0f, -1, 0u };
    f4 frag = mk4(0, 0, 0, 0);
    float dx = ((float) x + 0.5f) - (float) (p.w / 2) + p.radial_off_x,
          dy = ((float) y + 0.5f) - (float) (p.h / 2) + p.radial_off_y;
    float theta = glm_atan2(dy, dx);
    float d = sqrtf((dx * dx) + (dy * dy));
    float R = p.radial_radius, hl = p.radial_line / 2.0f;
    if (d > R - hl && d < R + hl) {
        frag = apply_frag(frag, mk4a(p.radial_outline));
        frag.a *= g_clamp((p.radial_line_half - fabsf(R - d)) * p.radial_c_alias, 0.0f, 1.0f);
    }
    if (d > R) {
        const float section = (GLB_TWOPI / (float) p.radial_nbars);
        const float center = ((GLB_TWOPI / (float) p.radial_nbars) / 2.0f);
        float m = g_mod(theta, section);
        float ym = d * glm_sin(center - m);
        const float bw2 = radial_bar_half(p), ow = p.radial_bar_outline_width;
        if (fabsf(ym) < bw2) {
            float idx = theta + p.radial_rotate;
            float dir = g_mod(fabsf(idx), GLB_TWOPI);
            if (dir > GLB_PI) idx = -g_sign(idx) * (GLB_TWOPI - dir);
            if (p.radial_invert == 0) idx = -idx;
            g.bar = ((idx > 0.0f ? 0 : 1) << 16) | (int) (fabsf(idx) / section);
            d -= R;
            g.dR = d;
            // radial/1.frag:85-110: COLOR, or BAR_OUTLINE along the bar's sides and in its end cap when BAR_OUTLINE_WIDTH > 0
            f4 r = (!(ow > 0.0f) || fabsf(ym) < bw2 - ow) ? eval_color(p.radial_color, p.radial_color_prog, d) : mk4a(p.radial_bar_outline);
            r.a *= ((bw2 - fabsf(ym)) * p.radial_bar_alias);
            g.lit = radial_finish(p, apply_frag(frag, r));
            if (ow > 0.0f) {
                f4 o = mk4a(p.radial_bar_outline);
                o.a *= ((bw2 - fabsf(ym)) * p.radial_bar_alias);
                g.band = radial_finish(p, apply_frag(frag, o));
            }
        }
    }
    // neither ring nor lit bar: apply_frag(0, 0) = 0 and stage 2 keeps 0 — skip the arithmetic
    if (p.premultiply_alpha && frag.r == 0.0f && frag.g == 0.0f && frag.b == 0.0f && frag.a == 0.0f) g.unlit = 0u;
    else g.unlit = radial_finish(p, apply_frag(frag, mk4(0, 0, 0, 0)));
    return g;
}
// bar height of bar `bar` (radial/1.frag:68-73): pos = int(abs(idx) / section) / float(NBARS / 2)
GLB_HD float radial_bar_value(const glava_b200_params& p, const AudioTex& t, int bar) {
    float pos = (float) (bar & 0xffff) / (float) (p.radial_nbars / 2);
    float v = sample_audio(t, (bar >> 16) ? t.r : t.l, pos);
    return v * p.radial_amplify;
}
GLB_HD uint32_t radial_px(const glava_b200_params& p, const AudioTex& t, int x, int y) {
    RadialGeo g = radial_geometry(p, x, y);
    if (g.bar < 0) return g.unlit;
    const float v = radial_bar_value(p, t, g.bar);
    if (!(p.radial_bar_outline_width > 0.0f)) return (g.dR <= v) ? g.lit : g.unlit;
    if (g.dR <= v - p.radial_bar_outline_width) return g.lit;
    return (g.dR <= v) ? g.band : g.unlit;
}
// conservative test: can pixel (x, y) be non-zero?  outside this disc radial_px() is exactly 0
GLB_HD float radial_reach(const glava_b200_params& p) {
    // bars reach d <= C_RADIUS + AMPLIFY * max(tex) with tex <= 1; ring reaches C_RADIUS + C_LINE/2
    return p.radial_radius + g_max(fabsf(p.radial_amplify), fabsf(p.radial_line)) + 2.0f;
}

// ================================= circle (circle/1.frag, 2.frag, 3.frag) ========================
GLB_HD float circle_apply_smooth(const glava_b200_params& p, const AudioTex& t, float theta) {   // circle/1.frag:34-49
    float idx = theta + p.circle_rotate;
    float dir = g_mod(fabsf(idx), GLB_TWOPI);
    if (dir > GLB_PI) idx = -g_sign(idx) * (GLB_TWOPI - dir);
    if (p.circle_invert > 0) idx = -idx;
    float pos = fabsf(idx) / (GLB_PI + 0.001f);
    float v = sample_audio(t, idx > 0.0f ? t.l : t.r, pos);
    v *= p.circle_amplify;
    return v;
}
// stage 1, pixel_center_integer (circle/1.frag:1,51-84): returns the RGBA8 value of the stage surface
template <bool NATIVE> GLB_HD uint32_t circle_stage1_t(const glava_b200_params& p, const AudioTex& t, int x, int y) {
    if (x < 0 || y < 0 || x >= p.w || y >= p.h) return 0u;                 // texelFetch outside the surface
    float dx = (float) x - (float) (p.w / 2), dy = (float) y - (float) (p.h / 2);
    float theta = glm_atan2(dy, dx);
    float d = sqrtf((dx * dx) + (dy * dy));
    float adv = (1.0f / d) * (p.circle_line * 0.5f);
    float adj0 = theta + adv, adj1 = theta - adv;
    d -= p.circle_radius;
    float hl = p.circle_line / 2.0f;
    if (d >= -hl) {
        float v = circle_apply_smooth(p, t, theta);
        adj0 = circle_apply_smooth(p, t, adj0) - v;
        adj1 = circle_apply_smooth(p, t, adj1) - v;
        float dmax = g_max(adj0, adj1), dmin = g_min(adj0, adj1);
        d -= v;
        bool in = p.circle_fill ? (d < hl) : ((d > -hl && d < hl) || (d <= dmax && d >= dmin));
        if (in) return stage_store<NATIVE>(p, mk4a(p.circle_outline));
    }
    return stage_bg<NATIVE>(p);
}
GLB_HD uint32_t circle_stage1(const glava_b200_params& p, const AudioTex& t, int x, int y) { return circle_stage1_t<true>(p, t, x, y); }
// The audio-independent part of circle/1.frag for one pixel (valid when the textures are pre-smoothed,
// i.e. smooth_audio() is a single texelFetch): d - C_RADIUS and, for the three angles theta,
// theta +- adv, which texel of which channel apply_smooth() fetches.  Cached per renderer by
// raster_circle_kernel.  e* = -1: pixel cannot be lit (inside the inner circle / outside the surface);
// else (channel << 30) | texel, texel == 0x3fffffff meaning "out of range, reads 0".
struct CircleGeo { float dR; int e0, e1, e2; };
GLB_HD int circle_texel_ref(const glava_b200_params& p, float theta) {     // circle/1.frag:34-45 without the fetch
    float idx = theta + p.circle_rotate;
    float dir = g_mod(fabsf(idx), GLB_TWOPI);
    if (dir > GLB_PI) idx = -g_sign(idx) * (GLB_TWOPI - dir);
    if (p.circle_invert > 0) idx = -idx;
    float pos = fabsf(idx) / (GLB_PI + 0.001f);
    int i = (int) glm_rint(pos * (float) p.n);
    if (i < 0 || i >= p.n) i = 0x3fffffff;
    return ((idx > 0.0f ? 0 : 1) << 30) | i;
}
GLB_HD CircleGeo circle_geometry(const glava_b200_params& p, int x, int y) {
    CircleGeo g = { 0.0f, -1, -1, -1 };
    if (x < 0 || y < 0 || x >= p.w || y >= p.h) return g;
    float dx = (float) x - (float) (p.w / 2), dy = (float) y - (float) (p.h / 2);
    float theta = glm_atan2(dy, dx);
    float d = sqrtf((dx * dx) + (dy * dy));
    float adv = (1.0f / d) * (p.circle_line * 0.5f);
    float adj0 = theta + adv, adj1 = theta - adv;
    d -= p.circle_radius;
    if (d >= -(p.circle_line / 2.0f)) {
        g.dR = d;
        g.e0 = circle_texel_ref(p, theta); g.e1 = circle_texel_ref(p, adj0); g.e2 = circle_texel_ref(p, adj1);
    }
    return g;
}
GLB_HD float circle_ref_value(const glava_b200_params& p, const AudioTex& t, int e) {
    const int i = e & 0x3fffffff;
    const uint16_t* tex = (e >> 30) ? t.r : t.l;
    float v = (i >= t.n) ? 0.0f : from16(tex[i]);
    return v * p.circle_amplify;
}
// the per-frame constants of stage 1, hoisted out of the per-cell path by the kernel
struct CircleConsts { float amplify, hl; int fill; uint32_t outline_px; };
GLB_HD CircleConsts circle_consts(const glava_b200_params& p) {
    CircleConsts c = { p.circle_amplify, p.circle_line / 2.0f, p.circle_fill, pack8(mk4a(p.circle_outline)) };
    return c;
}
GLB_HD float circle_ref_value_c(const CircleConsts& c, const uint16_t* tl, const uint16_t* tr, int n, int e) {
    const int i = e & 0x3fffffff;
    const uint16_t* tex = (e >> 30) ? tr : tl;
    float v = (i >= n) ? 0.0f : from16(tex[i]);
    return v * c.amplify;
}
GLB_HD uint32_t circle_stage1_c(const CircleConsts& c, const uint16_t* tl, const uint16_t* tr, int n, const CircleGeo& g) {
    if (g.e0 < 0) return 0u;
    float v = circle_ref_value_c(c, tl, tr, n, g.e0);
    float adj0 = circle_ref_value_c(c, tl, tr, n, g.e1) - v;
    float adj1 = circle_ref_value_c(c, tl, tr, n, g.e2) - v;
    float dmax = g_max(adj0, adj1), dmin = g_min(adj0, adj1);
    float d = g.dR - v;
    bool in = c.fill ? (d < c.hl) : ((d > -c.hl && d < c.hl) || (d <= dmax && d >= dmin));
    return in ? c.outline_px : 0u;
}
GLB_HD uint32_t circle_stage1_geo(const glava_b200_params& p, const AudioTex& t, const CircleGeo& g) {
    return circle_stage1_c(circle_consts(p), t.l, t.r, t.n, g);
}
// 8-tap neighbour mean as written in circle/2.frag:18-27, graph/2.frag:21-30, wave/2.frag:18-27:
// taps a3 and a7 repeat a0 and a4.  nb[] = stage values at (x+1,y) (x+1,y+1) (x,y+1) (x-1,y) (x-1,y-1) (x,y-1)
GLB_HD f4 neigh_avg(const uint32_t nb[6]) {
    f4 a0 = unpack8(nb[0]), a1 = unpack8(nb[1]), a2 = unpack8(nb[2]), a3 = a0,
       a4 = unpack8(nb[3]), a5 = unpack8(nb[4]), a6 = unpack8(nb[5]), a7 = a4;
    return mk4((a0.r + a1.r + a2.r + a3.r + a4.r + a5.r + a6.r + a7.r) / 8.0f,
               (a0.g + a1.g + a2.g + a3.g + a4.g + a5.g + a6.g + a7.g) / 8.0f,
               (a0.b + a1.b + a2.b + a3.b + a4.b + a5.b + a6.b + a7.b) / 8.0f,
               (a0.a + a1.a + a2.a + a3.a + a4.a + a5.a + a6.a + a7.a) / 8.0f);
}
GLB_HD float neigh_avg_alpha(const uint32_t nb[6]) {
    float a0 = from8(nb[0] >> 24), a1 = from8(nb[1] >> 24), a2 = from8(nb[2] >> 24),
          a4 = from8(nb[3] >> 24), a5 = from8(nb[4] >> 24), a6 = from8(nb[5] >> 24);
    return (a0 + a1 + a2 + a0 + a4 + a5 + a6 + a4) / 8.0f;
}
GLB_HD uint32_t circle_finish(const glava_b200_params& p, uint32_t own, const uint32_t nb[6]) {
    uint32_t px = own;
    if (p.circle_smooth) {                                                 // circle/2.frag:14-32
        if ((own >> 24) == 0u) px = pack8(neigh_avg(nb));
    }
    return p.premultiply_alpha ? premultiply8(px) : px;                    // circle/3.frag
}
GLB_HD float circle_reach(const glava_b200_params& p) {
    return p.circle_radius + fabsf(p.circle_amplify) + fabsf(p.circle_line) + 3.0f;
}
// non-native: stage 2 (when C_SMOOTH) is blended like stage 1, stage 3 (premultiply) is skipped
GLB_HD uint32_t circle_finish_blend(const glava_b200_params& p, uint32_t own, const uint32_t nb[6]) {
    // with C_SMOOTH 0 circle/2.frag is not disabled, it copies its input (:12): one more blend over the clear colour
    return blend_store(p, (p.circle_smooth && (own >> 24) == 0u) ? neigh_avg(nb) : unpack8(own));
}
template <bool NATIVE> GLB_HD uint32_t circle_px_t(const glava_b200_params& p, const AudioTex& t, int x, int y) {
    uint32_t nb[6] = { 0, 0, 0, 0, 0, 0 };
    uint32_t own = circle_stage1_t<NATIVE>(p, t, x, y);
    if (p.circle_smooth && (own >> 24) == 0u) {
        nb[0] = circle_stage1_t<NATIVE>(p, t, x + 1, y);     nb[1] = circle_stage1_t<NATIVE>(p, t, x + 1, y + 1);
        // circle/2.frag: half-integer gl_FragCoord, ivec2(x + 0.5 - 1) = 0 at x = 0 (see graph_px_cols)
        const int xm = x > 0 ? x - 1 : x, ym = y > 0 ? y - 1 : y;
        nb[2] = circle_stage1_t<NATIVE>(p, t, x, y + 1);     nb[3] = circle_stage1_t<NATIVE>(p, t, xm, y);
        nb[4] = circle_stage1_t<NATIVE>(p, t, xm, ym);       nb[5] = circle_stage1_t<NATIVE>(p, t, x, ym);
    }
    return NATIVE ? circle_finish(p, own, nb) : circle_finish_blend(p, own, nb);
}
GLB_HD uint32_t circle_px(const glava_b200_params& p, const AudioTex& t, int x, int y) {
    return p.premultiply_alpha ? circle_px_t<true>(p, t, x, y) : circle_px_t<false>(p, t, x, y);
}

// ================================= graph (graph/1.frag, 2.frag) ==================================
// column function: line height s(x), graph/1.frag:87-105 + side selection :124-132; pixel_center_integer
// which texture (0 = audio_l, 1 = audio_r) and which normalised position column x samples
GLB_HD float graph_column_coord(const glava_b200_params& p, int x, int* chan) {
    float fx = (float) x, W = (float) p.w;
    float half_w = (float) (p.w / 2);
    float idx;
    if (fx < half_w) { *chan = 0; idx = p.graph_direction < 0 ? fx : (half_w - fx); }
    else             { *chan = 1; idx = p.graph_direction < 0 ? (-fx + W) : (fx - half_w); }
    return idx / half_w;
}
// JOIN = JOIN_CHANNELS (graph/1.frag:93-96,126): towards the centre the two halves are pulled to `middle`, the mean of the
// left channel's last and the right channel's first sample, along a smoothstep of the centre taper.  pow(fact, 3) and
// pow(fact, 2) are evaluated as exact products (GLSL leaves pow's precision open).
template <bool JOIN> GLB_HD float graph_height_t(const glava_b200_params& p, const AudioTex& t, int x) {
    float fx = (float) x, W = (float) p.w;
    float pixel = 1.0f / W;
    int chan;
    float coord = graph_column_coord(p, x, &chan);
    float s = sample_audio_adj(t, chan ? t.r : t.l, coord, pixel);
    s *= p.graph_vscale;
    float fact = g_clamp((fabsf((float) (p.w / 2) - fx) / W) * 48.0f, 0.0f, 1.0f);
    if (JOIN) {
        const float middle = (p.graph_vscale * (sample_audio_adj(t, t.l, 1.0f, pixel) + sample_audio_adj(t, t.r, 0.0f, pixel))) / 2.0f;
        fact = (-2.0f * ((fact * fact) * fact)) + (3.0f * (fact * fact));
        s = (fact * s) + ((1.0f - fact) * middle);
    } else s *= fact;
    s *= g_clamp((g_min(fx, W - fx) / W) * 48.0f, 0.0f, 1.0f);
    return s;
}
GLB_HD float graph_height(const glava_b200_params& p, const AudioTex& t, int x) { return graph_height_t<false>(p, t, x); }
GLB_HD float graph_height_any(const glava_b200_params& p, const AudioTex& t, int x) {
    return p.graph_join_channels ? graph_height_t<true>(p, t, x) : graph_height_t<false>(p, t, x);
}
GLB_HD float graph_d(const glava_b200_params& p, int y) { return p.graph_invert > 0 ? (float) p.h - (float) y : (float) y; }
template <bool NATIVE> GLB_HD uint32_t graph_row_t(const glava_b200_params& p, int y) {
    return stage_store<NATIVE>(p, eval_color(p.graph_color, p.graph_color_prog, graph_d(p, y)));
}
GLB_HD uint32_t graph_row(const glava_b200_params& p, int y) { return graph_row_t<true>(p, y); }
// stage-1 surface value at (x, y) given the column height s and the row colour (bg: what `fragment = vec4(0)` stores)
GLB_HD uint32_t graph_stage1(const glava_b200_params& p, float s, uint32_t rowcol, int y, uint32_t bg = 0u) {
    return (graph_d(p, y) + 1.5f <= s) ? rowcol : bg;                       // graph/1.frag:116
}
GLB_HD uint32_t graph_finish(const glava_b200_params& p, uint32_t own, const uint32_t nb[6]) {   // graph/2.frag:19-44
    if (!(p.graph_draw_outline || p.graph_draw_highlight)) return own;
    float avg_a = neigh_avg_alpha(nb);
    if (avg_a > 0.0f) {
        f4 f = unpack8(own);
        if (f.a <= 0.0f) { if (p.graph_draw_outline) return pack8(mk4a(p.graph_outline)); }
        else if (avg_a < 1.0f) {
            if (p.graph_draw_highlight) { float k = avg_a * 2.0f; return pack8(mk4(f.r * k, f.g * k, f.b * k, f.a)); }
        }
    }
    return own;
}
// non-native: stage 2's result is blended over the clear colour like stage 1's
GLB_HD uint32_t graph_finish_blend(const glava_b200_params& p, uint32_t own, const uint32_t nb[6]) {
    if (!(p.graph_draw_outline || p.graph_draw_highlight)) return own;     // graph/2.frag disabled
    f4 f = unpack8(own);
    const float avg_a = neigh_avg_alpha(nb);
    if (avg_a > 0.0f) {
        if (f.a <= 0.0f) { if (p.graph_draw_outline) f = mk4a(p.graph_outline); }
        else if (avg_a < 1.0f) {
            if (p.graph_draw_highlight) { const float k = avg_a * 2.0f; f = mk4(f.r * k, f.g * k, f.b * k, f.a); }
        }
    }
    return blend_store(p, f);
}
// generic per-pixel: s3 = heights of columns x-1, x, x+1 (out-of-surface columns: any value, masked here)
template <bool NATIVE> GLB_HD uint32_t graph_px_cols_t(const glava_b200_params& p, const float s3[3], const uint32_t row3[3], int x, int y) {
    // row3 = row colours of y-1, y, y+1
    // graph/2.frag addresses its taps as ivec2(gl_FragCoord.x - 1, gl_FragCoord.y - 1) with the DEFAULT half-integer
    // gl_FragCoord (stage 2 does not declare pixel_center_integer): at x = 0 that is int(-0.5) = 0 — float -> int drops
    // the fraction (GLSL 3.30 5.4.1) — so the "x - 1" / "y - 1" taps of column 0 / row 0 read column 0 / row 0
    // themselves; only the "+ 1" taps can leave the surface.
    const uint32_t bg = stage_bg<NATIVE>(p);
    bool xr = x + 1 < p.w, yu = y + 1 < p.h;
    const int cl = x > 0 ? 0 : 1, rd = y > 0 ? 0 : 1;                       // s3 / row3 slot of the "- 1" taps
    const int ym = y > 0 ? y - 1 : y;
    uint32_t own = graph_stage1(p, s3[1], row3[1], y, bg);
    uint32_t nb[6];
    nb[0] = xr ? graph_stage1(p, s3[2], row3[1], y, bg) : 0u;
    nb[1] = (xr && yu) ? graph_stage1(p, s3[2], row3[2], y + 1, bg) : 0u;
    nb[2] = yu ? graph_stage1(p, s3[1], row3[2], y + 1, bg) : 0u;
    nb[3] = graph_stage1(p, s3[cl], row3[1], y, bg);
    nb[4] = graph_stage1(p, s3[cl], row3[rd], ym, bg);
    nb[5] = graph_stage1(p, s3[1], row3[rd], ym, bg);
    return NATIVE ? graph_finish(p, own, nb) : graph_finish_blend(p, own, nb);
}
GLB_HD uint32_t graph_px_cols(const glava_b200_params& p, const float s3[3], const uint32_t row3[3], int x, int y) {
    return graph_px_cols_t<true>(p, s3, row3, x, y);
}
// ---- graph/3.frag (ANTI_ALIAS 1): the step between neighbouring columns of the line is faded --------------------------
// Evaluated per pixel without a surface: S(x, y) below is the previous stage's value re-derived from the column heights.
// graph/4.frag (premultiply) tests `#if ANTI_ALIAS == 0` without including graph.glsl — the macro is undefined there, the
// test is true and the stage is always disabled — so stage 3 is the last one, in native mode too.
template <bool NATIVE> struct GraphCols {            // heights of columns x-2 .. x+2 around the pixel's column
    const glava_b200_params& p; int x; float h5[5];
    GLB_HD uint32_t S(int col, int y) const {         // stage-2 (or stage-1) surface value, 0 outside (texelFetch)
        if (col < 0 || y < 0 || col >= p.w || y >= p.h) return 0u;
        const int k = col - x + 2;                    // slot of `col` in h5 (callers stay within x-1 .. x+1)
        const float s3[3] = { h5[k - 1], h5[k], h5[k + 1] };
        const uint32_t row3[3] = { y > 0 ? graph_row_t<NATIVE>(p, y - 1) : 0u, graph_row_t<NATIVE>(p, y),
                                   y + 1 < p.h ? graph_row_t<NATIVE>(p, y + 1) : 0u };
        return graph_px_cols_t<NATIVE>(p, s3, row3, col, y);
    }
    GLB_HD float up(float xf, float oy) const {       // get_col_height_up, graph/3.frag:21-44
        float y = oy;
        if (p.graph_invert > 0) { while (y >= 0.0f) { if ((S((int) xf, (int) y) >> 24) == 0u) { y += 1.0f; break; } y -= 1.0f; } }
        else { while (y < (float) p.h) { if ((S((int) xf, (int) y) >> 24) == 0u) { y -= 1.0f; break; } y += 1.0f; } }
        return y;
    }
    GLB_HD float down(float xf, float oy) const {     // get_col_height_down, graph/3.frag:48-69
        float y = oy;
        if (p.graph_invert > 0) { while (y < (float) p.h) { if ((S((int) xf, (int) y) >> 24) != 0u) break; y += 1.0f; } }
        else { while (y >= 0.0f) { if ((S((int) xf, (int) y) >> 24) != 0u) break; y -= 1.0f; } }
        return y;
    }
};
template <bool NATIVE> GLB_HD_NOINLINE uint32_t graph_px_aa(const glava_b200_params& p, const AudioTex& t, int x, int y) {
    GraphCols<NATIVE> c = { p, x, { 0.0f, 0.0f, 0.0f, 0.0f, 0.0f } };
    for (int k = 0; k < 5; ++k) { const int col = x - 2 + k; if (col >= 0 && col < p.w) c.h5[k] = graph_height_any(p, t, col); }
    const float X = (float) x + 0.5f, Y = (float) y + 0.5f;               // default (half-integer) gl_FragCoord
    const uint32_t own = c.S(x, y);
    f4 f = unpack8(own);
    if (f.a <= 0.0f) {
        bool left_done = false;
        float h2 = 0.0f, a_fact = 0.0f;
        if ((c.S((int) (X - 1.0f), y) >> 24) != 0u) {                     // ivec2(-0.5) = 0: column 0 tests itself
            const float h1 = c.up(X - 1.0f, Y);
            h2 = c.down(X, Y);
            f = unpack8(c.S(x, (int) h2));
            a_fact = g_clamp(fabsf((h1 - Y) / (h2 - h1)), 0.0f, 1.0f);
            left_done = true;
        }
        if ((c.S((int) (X + 1.0f), y) >> 24) != 0u) {
            if (!left_done) { h2 = c.down(X, Y); f = unpack8(c.S(x, (int) h2)); }
            const float h3 = c.up(X + 1.0f, Y);
            a_fact = g_max(a_fact, g_clamp(fabsf((h3 - Y) / (h2 - h3)), 0.0f, 1.0f));
        }
        f.a *= a_fact;
    }
    return stage_store<NATIVE>(p, f);
}
GLB_HD uint32_t graph_px(const glava_b200_params& p, const AudioTex& t, int x, int y) {
    if (p.graph_anti_alias) return p.premultiply_alpha ? graph_px_aa<true>(p, t, x, y) : graph_px_aa<false>(p, t, x, y);
    float s3[3] = { x > 0 ? graph_height_any(p, t, x - 1) : 0.0f, graph_height_any(p, t, x), x + 1 < p.w ? graph_height_any(p, t, x + 1) : 0.0f };
    if (!p.premultiply_alpha) {
        uint32_t rowb[3] = { y > 0 ? graph_row_t<false>(p, y - 1) : 0u, graph_row_t<false>(p, y), y + 1 < p.h ? graph_row_t<false>(p, y + 1) : 0u };
        return graph_px_cols_t<false>(p, s3, rowb, x, y);
    }
    uint32_t row3[3] = { y > 0 ? graph_row(p, y - 1) : 0u, graph_row(p, y), y + 1 < p.h ? graph_row(p, y + 1) : 0u };
    return graph_px_cols(p, s3, row3, x, y);
}

// ================================= wave (wave/1.frag, 2.frag) ====================================
struct WaveCol { float s, dmin, dmax, thick; uint32_t color; };
GLB_HD int wave_tex_index(int n, float coord) {                             // texture(): NEAREST + REPEAT (render.c:514-517)
    float u = coord * (float) n;
    int i = (int) floorf(u);
    i %= n; if (i < 0) i += n;
    return i;
}
GLB_HD float wave_tex(const AudioTex& t, float coord) { return from16(t.l[wave_tex_index(t.n, coord)]); }
GLB_HD WaveCol wave_column(const glava_b200_params& p, const AudioTex& t, int x) {   // wave/1.frag:17-31, pixel_center_integer
    float fx = (float) x, W = (float) p.w, H = (float) p.h;
    float os   = ((wave_tex(t, (fx + 0.0f) / W) - 0.5f) * p.wave_amplify) + 0.5f;
    float adj0 = ((wave_tex(t, (fx + -1.0f) / W) - 0.5f) * p.wave_amplify) + 0.5f;
    float adj1 = ((wave_tex(t, (fx + 1.0f) / W) - 0.5f) * p.wave_amplify) + 0.5f;
    float s0 = adj0 - os, s1 = adj1 - os;
    WaveCol c;
    c.dmax = g_max(s0, s1); c.dmin = g_min(s0, s1);
    c.s = (os + (H * 0.5f) - 0.5f);
    c.thick = g_clamp(fabsf(c.s - (H * 0.5f)) * 6.0f, p.wave_min_thickness, p.wave_max_thickness);
    float k = (fabsf((H * 0.5f) - c.s) * 0.02f);
    c.color = pack8(mk4(p.wave_base_color[0] + k, p.wave_base_color[1] + k, p.wave_base_color[2] + k, p.wave_base_color[3] + k));
    return c;
}
GLB_HD uint32_t wave_stage1(const WaveCol& c, int y, uint32_t bg = 0u) {     // wave/1.frag:32-38
    float diff = (float) y - c.s;
    return (fabsf(diff) < c.thick || (diff <= c.dmax && diff >= c.dmin)) ? c.color : bg;
}
// c3 = columns x-1, x, x+1
template <bool NATIVE> GLB_HD uint32_t wave_px_cols_t(const glava_b200_params& p, const WaveCol c3[3], int x, int y) {   // wave/2.frag:14-33
    const uint32_t bg = stage_bg<NATIVE>(p);
    bool xl = x - 1 >= 0, xr = x + 1 < p.w, yd = y - 1 >= 0, yu = y + 1 < p.h;
    uint32_t own = wave_stage1(c3[1], y, bg);
    uint32_t nb[6];
    nb[0] = xr ? wave_stage1(c3[2], y, bg) : 0u;
    nb[1] = (xr && yu) ? wave_stage1(c3[2], y + 1, bg) : 0u;
    nb[2] = yu ? wave_stage1(c3[1], y + 1, bg) : 0u;
    nb[3] = xl ? wave_stage1(c3[0], y, bg) : 0u;
    nb[4] = (xl && yd) ? wave_stage1(c3[0], y - 1, bg) : 0u;
    nb[5] = yd ? wave_stage1(c3[1], y - 1, bg) : 0u;
    if (neigh_avg_alpha(nb) > 0.0f) {
        if ((own >> 24) == 0u || x == 0 || x == p.w - 1) return stage_store<NATIVE>(p, mk4a(p.wave_outline));
    }
    return NATIVE ? own : blend_store(p, unpack8(own));                    // stage 2 is drawn (and blended) for every pixel
}
GLB_HD uint32_t wave_px_cols(const glava_b200_params& p, const WaveCol c3[3], int x, int y) { return wave_px_cols_t<true>(p, c3, x, y); }
// non-native: the column's stage-1 colour goes through the blend before it is stored
GLB_HD WaveCol wave_column_blend(const glava_b200_params& p, const AudioTex& t, int x) {
    WaveCol c = wave_column(p, t, x);
    const float H = (float) p.h;
    const float k = (fabsf((H * 0.5f) - c.s) * 0.02f);
    c.color = blend_store(p, mk4(p.wave_base_color[0] + k, p.wave_base_color[1] + k, p.wave_base_color[2] + k, p.wave_base_color[3] + k));
    return c;
}
GLB_HD uint32_t wave_px(const glava_b200_params& p, const AudioTex& t, int x, int y) {
    WaveCol c3[3];
    if (!p.premultiply_alpha) {
        c3[1] = wave_column_blend(p, t, x);
        c3[0] = x > 0 ? wave_column_blend(p, t, x - 1) : c3[1];
        c3[2] = x + 1 < p.w ? wave_column_blend(p, t, x + 1) : c3[1];
        return wave_px_cols_t<false>(p, c3, x, y);
    }
    c3[1] = wave_column(p, t, x);
    c3[0] = x > 0 ? wave_column(p, t, x - 1) : c3[1];
    c3[2] = x + 1 < p.w ? wave_column(p, t, x + 1) : c3[1];
    return wave_px_cols(p, c3, x, y);
}

// ================================= test (test/1.frag:32, 2.frag, 3.frag) ==========================
GLB_HD uint32_t test_px(const glava_b200_params& p) {
    if (!p.premultiply_alpha)                                               // stages 1 and 2 blended, test/3.frag skipped
        return blend_store(p, unpack8(blend_store(p, mk4(1.0f, 0.0f, 0.0f, (float) 1 / (float) 3))));
    uint32_t px = pack8(mk4(1.0f, 0.0f, 0.0f, (float) 1 / (float) 3));
    px = pack8(unpack8(px));                                                // test/2.frag passthrough
    return premultiply8(px);                                                // test/3.frag
}

// ================================= dirty-row marks (bars, graph, wave) ============================
// Every framebuffer slot keeps one word per (row band, 128-pixel warp strip) of the raster launch that last wrote it:
// rows [lo, hi) of the band may be non-zero in memory, every other row of the band is 0 (lo = low 16 bits, hi = high
// 16 bits; h <= 16384, validate_params).  A kernel stores a zero row only where it falls inside the old interval — a row
// that is 0 in memory and 0 in the new frame needs no store — and then records the rows it stored non-zero content in.
GLB_HD uint32_t dirty_pack(int lo, int hi) { return lo < hi ? ((uint32_t) lo | ((uint32_t) hi << 16)) : 0u; }
// Zero rows [za, zb) of a band, old mark `old` -> the rows [*a, *b) of them that must be stored (*a == *b: none).
GLB_HD void dirty_zero_span(uint32_t old, int za, int zb, int* a, int* b) {
    const int lo = (int) (old & 0xffffu), hi = (int) (old >> 16);
    const int s = za > lo ? za : lo, e = zb < hi ? zb : hi;
    *a = s; *b = e > s ? e : s;
}

// generic per-pixel dispatcher
GLB_HD_NOINLINE uint32_t module_px(const glava_b200_params& p, const AudioTex& t, int x, int y) {
    switch (p.module) {
        case GLAVA_B200_MOD_BARS:   return bars_px(p, t, x, y);
        case GLAVA_B200_MOD_RADIAL: return radial_px(p, t, x, y);
        case GLAVA_B200_MOD_CIRCLE: return circle_px(p, t, x, y);
        case GLAVA_B200_MOD_GRAPH:  return graph_px(p, t, x, y);
        case GLAVA_B200_MOD_WAVE:   return wave_px(p, t, x, y);
        default:                    return test_px(p);
    }
}

}  // namespace glb
#endif
