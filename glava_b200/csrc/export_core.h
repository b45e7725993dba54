// export_core.h — the pixel arithmetic of glava_b200_export_frames (DESIGN 4.10) as __host__ __device__ functions: the
// composite over an opaque background, RGB -> Y / Cb / Cr in integer fixed point (BT.709 or BT.601, limited or full range), the 2x2 chroma
// average, and which framebuffer rows the dirty-row marks say must be read.  export_kernels.cu and the host test tier
// (tests/test_export_core.py) compile this same code.
#ifndef GLAVA_B200_EXPORT_CORE_H
#define GLAVA_B200_EXPORT_CORE_H

#include "raster_core.h"

namespace glb {

// What one export call does to every pixel: the public format, whether it composites, the renderer's opacity
// (premultiply_alpha != 0: native, the frame is premultiplied over a transparent target) and the background 0x00BBGGRR
struct ExportFmt {
    int      format;            // GLAVA_B200_EXPORT_*
    int      over;              // composite (always for the YUV formats)
    int      native;
    uint32_t bg;
};

// ---- composite ---------------------------------------------------------------------------------------------------------
// The opaque colour GLava's window shows for a stored pixel (R in the low byte).  Native opacity: the premultiplied pixel
// over `bg`, C = min(255, c + mul_norm8(bg, 255 - a)) per channel, the unorm8 product the blend path uses (raster_core.h).
// Any other opacity: the window ignores alpha, the colour is as stored.  Alpha becomes 255.
GLB_HD uint32_t export_over(uint32_t px, uint32_t bg, int native) {
    if (!native) return px | 0xff000000u;
    const uint32_t ia = 255u - (px >> 24);
    uint32_t out = 0xff000000u;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const uint32_t v = ((px >> (8 * c)) & 255u) + mul_norm8((bg >> (8 * c)) & 255u, ia);
        out |= (v > 255u ? 255u : v) << (8 * c);
    }
    return out;
}
GLB_HD uint32_t export_swap_rb(uint32_t px) { return (px & 0xff00ff00u) | ((px & 0xffu) << 16) | ((px >> 16) & 0xffu); }
// one RGBA / BGRA output pixel
GLB_HD uint32_t export_px(const ExportFmt& f, uint32_t px) {
    if (f.over) px = export_over(px, f.bg, f.native);
    return f.format == GLAVA_B200_EXPORT_BGRA ? export_swap_rb(px) : px;
}

// ---- BT.709, limited range ---------------------------------------------------------------------------------------------
// Kr = 0.2126, Kb = 0.0722; Y' = Kr R + Kg G + Kb B, Y = 16 + 219/255 Y', Cb = 128 + 224/255 (B - Y') / (2 (1 - Kb)),
// Cr = 128 + 224/255 (R - Y') / (2 (1 - Kr)).  Coefficients scaled by 2^16 and rounded; the blue coefficient of Cb and the
// red one of Cr are minus the sum of the other two, so every grey has Cb = Cr = 128 exactly.  Black gives (16, 128, 128),
// white (235, 128, 128); over all 2^24 colours the result is within 0.503 code values of the float64 formula.
#define GLB_YUV_SHIFT 16
#define GLB_YUV_HALF (1 << (GLB_YUV_SHIFT - 1))
#define GLB_Y_R 11966
#define GLB_Y_G 40254
#define GLB_Y_B 4064
#define GLB_CB_R (-6596)
#define GLB_CB_G (-22189)
#define GLB_CB_B (-(GLB_CB_R + GLB_CB_G))
#define GLB_CR_G (-26145)
#define GLB_CR_B (-2639)
#define GLB_CR_R (-(GLB_CR_G + GLB_CR_B))

// ---- colour encodings (DESIGN 4.15) --------------------------------------------------------------------------------------
// The Y'CbCr formats write one of four encodings, chosen by the descriptor's GLAVA_B200_EXPORT_FULL_RANGE (0x100) and
// GLAVA_B200_EXPORT_BT601 (0x200) bits: E = flags >> 8 & 3, 0 BT.709 limited range (flags 0, the literals above and
// below), 1 BT.709 full range, 2 BT.601 limited, 3 BT.601 full.  Every set is built by yuv_coef from (Kr, Kb, range, bits):
// limited range Y = 16 + 219/255 Y', C = 128 + 224/255 P (10 bits: 64 + 876/255 Y', 512 + 896/255 P); full range (H.273,
// JFIF) Y = Y', C = 128 + P (10 bits: 1023/255 Y', 512 + 1023/255 P), P = (B - Y') / (2 (1 - Kb)) for Cb, (R - Y') /
// (2 (1 - Kr)) for Cr.  Coefficients scaled by 2^16 and rounded half away from zero; the blue coefficient of Cb and the red
// one of Cr are minus the sum of the other two, so every grey has Cb = Cr = 128 (512) exactly.  Full range reaches 255.5
// (1023.5) before rounding in blue's Cb and red's Cr, so its codes are clamped to 255 (1023); limited range never leaves
// [16, 240] ([64, 960]) and is not.  Accumulators, 8 bits: |coefficient sums| <= 2^16 (full), so a code's sum is within
// 255 * 2^16 + (128 << 16) + 2^15 < 2^25; 10 bits, per pixel <= 262915 * 255 + (512 << 16) + 2^15 < 2^27, P010 chroma over
// block sums (<= 1020, shift 18) <= 131458 * 1020 + (512 << 18) + 2^17 < 2^29; every minimum is >= 0 (DESIGN 4.15).
struct YuvCoef { int yr, yg, yb, cbr, cbg, cbb, crr, crg, crb, yoff, coff, top; bool full; };
constexpr int yuv_round(double x) { return x < 0 ? -(int) (-x + 0.5) : (int) (x + 0.5); }
constexpr YuvCoef yuv_coef(double kr, double kb, bool full, int bits) {
    const double kg = 1 - kr - kb, s = 1 << GLB_YUV_SHIFT;
    const double top = bits == 10 ? 1023 : 255;
    const double ys = full ? top / 255 : (bits == 10 ? 876.0 : 219.0) / 255;
    const double cs = full ? top / 255 : (bits == 10 ? 896.0 : 224.0) / 255;
    const int cbr = yuv_round(-kr / (2 * (1 - kb)) * cs * s), cbg = yuv_round(-kg / (2 * (1 - kb)) * cs * s);
    const int crg = yuv_round(-kg / (2 * (1 - kr)) * cs * s), crb = yuv_round(-kb / (2 * (1 - kr)) * cs * s);
    return { yuv_round(kr * ys * s), yuv_round(kg * ys * s), yuv_round(kb * ys * s), cbr, cbg, -(cbr + cbg), -(crg + crb), crg,
             crb, full ? 0 : bits == 10 ? 64 : 16, bits == 10 ? 512 : 128, (int) top, full };
}
// the set of encoding E (0..3) at 8 or 10 bits: BT.709 Kr, Kb = 0.2126, 0.0722; BT.601 0.299, 0.114
constexpr YuvCoef yuv_enc(int E, int bits) { return yuv_coef(E & 2 ? 0.299 : 0.2126, E & 2 ? 0.114 : 0.0722, (E & 1) != 0, bits); }
constexpr bool yuv_same(const YuvCoef& a, int yr, int yg, int yb, int cbr, int cbg, int crg, int crb) {
    return a.yr == yr && a.yg == yg && a.yb == yb && a.cbr == cbr && a.cbg == cbg && a.cbb == -(cbr + cbg) && a.crg == crg &&
           a.crb == crb && a.crr == -(crg + crb);
}
static_assert(yuv_same(yuv_enc(0, 8), GLB_Y_R, GLB_Y_G, GLB_Y_B, GLB_CB_R, GLB_CB_G, GLB_CR_G, GLB_CR_B), "BT.709 limited 8-bit");
// the encoding index of a descriptor's flags: 0..3 as above, 4 for GLAVA_B200_EXPORT_PQ and 5 for GLAVA_B200_EXPORT_HLG
// (DESIGN 4.22; the host refuses either with the other bits)
GLB_HD int export_enc(uint32_t flags) {
    const uint32_t hdr = (flags >> 11) & 3u;
    return hdr ? (int) (3u + hdr) : (int) ((flags >> 8) & 3u);
}
// a code of set S from its accumulator (scaled by 2^shift, rounding included): full range clamps to the top code
template <int E, int Bits>
GLB_HD uint32_t yuv_code(int acc, int shift) {
    constexpr YuvCoef S = yuv_enc(E, Bits);
    const int v = acc >> shift;
    if constexpr (S.full) return (uint32_t) (v > S.top ? S.top : v);
    return (uint32_t) v;
}

// ---- BT.2020 HDR: PQ and HLG at 10 bits (DESIGN 4.22) --------------------------------------------------------------------
// GLAVA_B200_EXPORT_PQ (0x800) and GLAVA_B200_EXPORT_HLG (0x1000) select encodings E = 4 and 5: BT.2020 non-constant-
// luminance Y'CbCr, limited range, with that transfer function, on P010, YUV420P10, YUV444P10 and YUV422P10 only.  An
// 8-bit R'G'B' triple v (BT.709 primaries) is shown as SDR graphics at BT.2408's 203 cd/m^2, display-referred:
//   L = (v / 255)^2.4 (BT.1886, L_B = 0; hdr_lin's table of float64 rounded to float32),
//   F = 203 M L, M the BT.709 -> BT.2020 matrix from the primaries and D65 (BT.2087's to 4 decimals),
//   PQ: E' = PQ^-1(F / 10000) (ST 2084); HLG: BT.2100's inverse OOTF for a 1000 cd/m^2 display (gamma 1.2, L_B = 0), then
//   its OETF; Y' = 0.2627 R' + 0.6780 G' + 0.0593 B', Y = 64 + 876 Y', Cb = 512 + 896 (B' - Y') / 1.8814, Cr = 512 + 896
//   (R' - Y') / 1.4746, rounded half up.  Subsampled chroma is that of the mean of the pixels' E' (hdr_mean4, a fixed order).
// Only correctly rounded float32 operations and gl_math.h's glm_log / glm_exp / glm_pow, so the host build and the kernels
// (--fmad=false) agree bit for bit.  No channel passes 203 cd/m^2, so MaxCLL <= 203.  These encodings run only in
// instantiations E = 4, 5 of the 10-bit items (export_y10 and the quads branch on E at compile time).
#define GLB_ENC_PQ 4
#define GLB_ENC_HLG 5
GLB_HD bool export_hdr_format(int format) {             // the formats the HDR bits apply to
    return format == GLAVA_B200_EXPORT_P010 || format == GLAVA_B200_EXPORT_YUV420P10 || format == GLAVA_B200_EXPORT_YUV444P10 ||
           format == GLAVA_B200_EXPORT_YUV422P10;
}
#define GLB_HDR_LIN_TABLE { \
    0.0f, 1.67611404e-06f, 8.84658311e-06f, 2.34096315e-05f, 4.66925449e-05f, 7.97685279e-05f, 0.000123556776f, 0.000178870556f, \
    0.000246444717f, 0.000326953188f, 0.000421020814f, 0.000529231911f, 0.000652136572f, 0.000790255668f, 0.000944084488f, 0.00111409591f, \
    0.00130074308f, 0.00150446116f, 0.00172566937f, 0.00196477212f, 0.00222216127f, 0.0024982153f, 0.00279330276f, 0.00310778082f, \
    0.00344199757f, 0.00379629177f, 0.00417099427f, 0.00456642779f, 0.00498290779f, 0.00542074209f, 0.00588023337f, 0.00636167731f, \
    0.0068653631f, 0.00739157572f, 0.00794059318f, 0.00851269066f, 0.00910813734f, 0.00972719677f, 0.0103701297f, 0.0110371923f, \
    0.0117286369f, 0.0124447113f, 0.0131856594f, 0.0139517235f, 0.01474314f, 0.0155601436f, 0.0164029654f, 0.0172718335f, \
    0.0181669723f, 0.0190886036f, 0.0200369488f, 0.0210122224f, 0.0220146403f, 0.023044413f, 0.0241017509f, 0.0251868591f, \
    0.0262999441f, 0.0274412073f, 0.0286108498f, 0.029809067f, 0.0310360584f, 0.0322920159f, 0.033577133f, 0.0348916017f, \
    0.0362356044f, 0.0376093313f, 0.0390129685f, 0.0404466987f, 0.0419107042f, 0.043405164f, 0.0449302532f, 0.0464861542f, \
    0.0480730385f, 0.049691081f, 0.0513404533f, 0.0530213267f, 0.0547338724f, 0.0564782582f, 0.0582546517f, 0.0600632168f, \
    0.0619041175f, 0.0637775213f, 0.0656835809f, 0.0676224604f, 0.0695943311f, 0.0715993345f, 0.0736376345f, 0.0757093951f, \
    0.0778147578f, 0.0799538866f, 0.0821269304f, 0.0843340382f, 0.0865753666f, 0.0888510644f, 0.0911612809f, 0.0935061574f, \
    0.0958858505f, 0.0983005017f, 0.100750253f, 0.103235252f, 0.10575565f, 0.108311571f, 0.110903174f, 0.113530591f, \
    0.116193965f, 0.118893437f, 0.121629141f, 0.124401219f, 0.127209798f, 0.130055025f, 0.132937044f, 0.135855973f, \
    0.138811946f, 0.141805097f, 0.144835562f, 0.147903472f, 0.151008964f, 0.15415217f, 0.15733321f, 0.160552204f, \
    0.163809299f, 0.167104617f, 0.17043829f, 0.173810437f, 0.177221179f, 0.180670649f, 0.184158966f, 0.187686265f, \
    0.191252664f, 0.194858283f, 0.198503241f, 0.202187672f, 0.205911696f, 0.209675416f, 0.213478968f, 0.217322454f, \
    0.221206024f, 0.225129768f, 0.22909382f, 0.233098283f, 0.237143293f, 0.241228953f, 0.245355383f, 0.249522701f, \
    0.253731012f, 0.257980436f, 0.262271076f, 0.266603082f, 0.270976543f, 0.275391549f, 0.279848248f, 0.28434673f, \
    0.288887113f, 0.293469518f, 0.298094034f, 0.30276081f, 0.307469904f, 0.312221438f, 0.317015558f, 0.321852326f, \
    0.32673189f, 0.33165434f, 0.336619765f, 0.341628283f, 0.346680015f, 0.35177505f, 0.356913507f, 0.362095475f, \
    0.367321074f, 0.372590393f, 0.377903551f, 0.383260638f, 0.388661772f, 0.394107074f, 0.399596572f, 0.405130446f, \
    0.410708755f, 0.416331619f, 0.421999156f, 0.427711427f, 0.43346855f, 0.439270616f, 0.445117742f, 0.451010019f, \
    0.456947535f, 0.462930411f, 0.468958735f, 0.475032598f, 0.481152117f, 0.487317383f, 0.493528455f, 0.499785483f, \
    0.506088555f, 0.512437761f, 0.51883316f, 0.525274873f, 0.531763017f, 0.538297653f, 0.54487896f, 0.551506877f, \
    0.558181643f, 0.564903319f, 0.571671903f, 0.578487635f, 0.585350454f, 0.592260599f, 0.599218071f, 0.606222987f, \
    0.613275409f, 0.620375514f, 0.627523303f, 0.634718955f, 0.641962469f, 0.649253964f, 0.656593561f, 0.663981318f, \
    0.671417356f, 0.678901732f, 0.686434567f, 0.69401592f, 0.701645911f, 0.709324598f, 0.717052102f, 0.724828482f, \
    0.732653797f, 0.740528226f, 0.748451769f, 0.756424546f, 0.764446676f, 0.772518218f, 0.780639231f, 0.788809836f, \
    0.797030091f, 0.805300117f, 0.813620031f, 0.821989834f, 0.830409646f, 0.838879526f, 0.847399592f, 0.855969965f, \
    0.864590704f, 0.873261809f, 0.881983459f, 0.890755713f, 0.899578691f, 0.908452392f, 0.917376935f, 0.926352441f, \
    0.935378969f, 0.944456577f, 0.953585386f, 0.962765455f, 0.971996844f, 0.981279731f, 0.990614057f, 1.0f \
}
#ifdef __CUDACC__
__device__ static const float glb_hdr_lin_dev[256] = GLB_HDR_LIN_TABLE;
#endif
static const float glb_hdr_lin_host[256] = GLB_HDR_LIN_TABLE;
// (v / 255)^2.4 of an 8-bit code
GLB_HD float hdr_lin(uint32_t v) {
#ifdef __CUDA_ARCH__
    return __ldg(glb_hdr_lin_dev + v);
#else
    return glb_hdr_lin_host[v];
#endif
}
// 203 M / 10000 (PQ's F / 10000) and 203 M / 1000 (HLG's F / 1000), float64 rounded to float32, row-major
#define GLB_HDR_M_PQ { 0.0127362991f, 0.00668444578f, 0.00087925524f, 0.00140267494f, 0.0186666697f, 0.000230655001f, \
                       0.000332746218f, 0.00178667018f, 0.0181805845f }
#define GLB_HDR_M_HLG { 0.127362996f, 0.0668444559f, 0.00879255217f, 0.0140267499f, 0.186666697f, 0.00230655004f, \
                        0.00332746212f, 0.0178667009f, 0.181805834f }
struct HdrRgb { float r, g, b; };                           // E' = (R', G', B')
struct HdrM { float rr, rg, rb, gr, gg, gb, br, bg, bb; };
// ST 2084's inverse EOTF of y = F / 10000 >= 0; m1, m2, c1, c2, c3 are exact in float32
GLB_HD float hdr_pq(float y) {
    const float p = glm_pow(y, 0.1593017578125f);
    return glm_pow(glm_div(glm_fma(18.8515625f, p, 0.8359375f), glm_fma(18.6875f, p, 1.0f)), 78.84375f);
}
// BT.2100's HLG OETF of scene light e >= 0 (a = 0.17883277, b = 1 - 4a, c = 0.5 - a ln 4a)
GLB_HD float hdr_hlg(float e) {
    if (e <= 1.0f / 12.0f) return glm_sqrt(glm_mul(3.0f, e));
    return glm_fma(0.17883277f, glm_log(glm_fma(12.0f, e, -0.28466892f)), 0.55991073f);
}
// E' of an 8-bit triple c (R low; the top byte is ignored) under E = 4 (PQ) or 5 (HLG)
template <int E>
GLB_HD HdrRgb hdr_rgb(uint32_t c) {
    constexpr HdrM m = E == GLB_ENC_PQ ? HdrM GLB_HDR_M_PQ : HdrM GLB_HDR_M_HLG;
    const float lr = hdr_lin(c & 255u), lg = hdr_lin((c >> 8) & 255u), lb = hdr_lin((c >> 16) & 255u);
    const float fr = glm_fma(m.rb, lb, glm_fma(m.rg, lg, glm_mul(m.rr, lr)));
    const float fg = glm_fma(m.gb, lb, glm_fma(m.gg, lg, glm_mul(m.gr, lr)));
    const float fb = glm_fma(m.bb, lb, glm_fma(m.bg, lg, glm_mul(m.br, lr)));
    if constexpr (E == GLB_ENC_PQ) {
        return { hdr_pq(fr), hdr_pq(fg), hdr_pq(fb) };
    } else {
        // inverse OOTF: E = (F / 1000) (Y_D / 1000)^(-1/6), E = 0 where Y_D = 0 (black: every F is 0)
        const float yd = glm_fma(0.0593f, fb, glm_fma(0.6780f, fg, glm_mul(0.2627f, fr)));
        if (yd <= 0.0f) return { 0.0f, 0.0f, 0.0f };
        const float s = glm_pow(yd, -1.0f / 6.0f);
        return { hdr_hlg(glm_mul(fr, s)), hdr_hlg(glm_mul(fg, s)), hdr_hlg(glm_mul(fb, s)) };
    }
}
// BT.2020's Y' of E'
GLB_HD float hdr_luma(const HdrRgb& e) { return glm_fma(0.0593f, e.b, glm_fma(0.6780f, e.g, glm_mul(0.2627f, e.r))); }
// the unrounded 10-bit codes: Y, and Cb / Cr (896 / 1.8814 and 896 / 1.4746 folded)
GLB_HD float hdr_yf(const HdrRgb& e) { return glm_fma(876.0f, hdr_luma(e), 64.0f); }
GLB_HD float hdr_cbf(const HdrRgb& e) { return glm_fma(476.241097f, glm_add(e.b, -hdr_luma(e)), 512.0f); }
GLB_HD float hdr_crf(const HdrRgb& e) { return glm_fma(607.622406f, glm_add(e.r, -hdr_luma(e)), 512.0f); }
// a code rounded half up; every value passed lies in [0, 1023]
GLB_HD uint32_t hdr_code(float x) { return (uint32_t) glm_add(x, 0.5f); }
GLB_HD uint32_t hdr_y10(const HdrRgb& e) { return hdr_code(hdr_yf(e)); }
// (Cb, Cr) codes of E', Cb in the low 16 bits (as export_cbcr10)
GLB_HD uint32_t hdr_cbcr10(const HdrRgb& e) { return hdr_code(hdr_cbf(e)) | (hdr_code(hdr_crf(e)) << 16); }
// the mean E' of a 2x2 block (a, b the top row) in a fixed order; a 4:2:2 pair (a, b) is the block (a, b, a, b), whose mean
// is exactly (a + b) / 2, and one pixel the block (a, a, a, a), whose mean is exactly a
GLB_HD HdrRgb hdr_mean4(const HdrRgb& a, const HdrRgb& b, const HdrRgb& c, const HdrRgb& d) {
    return { glm_mul(glm_add(glm_add(a.r, b.r), glm_add(c.r, d.r)), 0.25f), glm_mul(glm_add(glm_add(a.g, b.g), glm_add(c.g, d.g)), 0.25f),
             glm_mul(glm_add(glm_add(a.b, b.b), glm_add(c.b, d.b)), 0.25f) };
}

// the Y code of a composited pixel under encoding E (E = 0: the BT.709 limited byte above)
template <int E = 0>
GLB_HD uint32_t export_y(uint32_t c) {
    constexpr YuvCoef S = yuv_enc(E, 8);
    const int r = (int) (c & 255u), g = (int) ((c >> 8) & 255u), b = (int) ((c >> 16) & 255u);
    return yuv_code<E, 8>(S.yr * r + S.yg * g + S.yb * b + (S.yoff << GLB_YUV_SHIFT) + GLB_YUV_HALF, GLB_YUV_SHIFT);
}
// (Cb, Cr) as the two bytes of NV12's interleaved plane: Cb low, Cr high
template <int E = 0>
GLB_HD uint32_t export_cbcr(uint32_t c) {
    constexpr YuvCoef S = yuv_enc(E, 8);
    const int r = (int) (c & 255u), g = (int) ((c >> 8) & 255u), b = (int) ((c >> 16) & 255u);
    const uint32_t cb = yuv_code<E, 8>(S.cbr * r + S.cbg * g + S.cbb * b + (S.coff << GLB_YUV_SHIFT) + GLB_YUV_HALF, GLB_YUV_SHIFT);
    const uint32_t cr = yuv_code<E, 8>(S.crr * r + S.crg * g + S.crb * b + (S.coff << GLB_YUV_SHIFT) + GLB_YUV_HALF, GLB_YUV_SHIFT);
    return cb | (cr << 8);
}
// The chroma sample of a 2x2 block: the per-channel average (s + 2) >> 2 of its four composited pixels
GLB_HD uint32_t export_avg4(uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    uint32_t out = 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const uint32_t s = ((a >> (8 * k)) & 255u) + ((b >> (8 * k)) & 255u) + ((c >> (8 * k)) & 255u) + ((d >> (8 * k)) & 255u);
        out |= ((s + 2u) >> 2) << (8 * k);
    }
    return out;
}
// NV12 of a quad of output rows 2j (top) and 2j + 1 (bot): four Y bytes per row, and the (Cb, Cr) pairs of the quad's two
// 2x2 blocks as one little-endian word (Cb0, Cr0, Cb1, Cr1)
template <int E = 0>
GLB_HD uint32_t export_nv12_quad(const ExportFmt& f, const uint32_t top[4], const uint32_t bot[4], uint32_t* y_top, uint32_t* y_bot) {
    uint32_t t[4], b[4];
    *y_top = 0u; *y_bot = 0u;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        t[k] = export_over(top[k], f.bg, f.native);
        b[k] = export_over(bot[k], f.bg, f.native);
        *y_top |= export_y<E>(t[k]) << (8 * k);
        *y_bot |= export_y<E>(b[k]) << (8 * k);
    }
    return export_cbcr<E>(export_avg4(t[0], t[1], b[0], b[1])) | (export_cbcr<E>(export_avg4(t[2], t[3], b[2], b[3])) << 16);
}

// ---- I420, YUV 4:4:4 and P010 (DESIGN 4.14) ------------------------------------------------------------------------------
GLB_HD bool export_yuv(int format) {                   // a format with chroma planes
    return format == GLAVA_B200_EXPORT_NV12 || format == GLAVA_B200_EXPORT_I420 || format == GLAVA_B200_EXPORT_YUV444 ||
           format == GLAVA_B200_EXPORT_P010;
}
// The planar 10-bit formats (DESIGN 4.16) run kernels of their own, so export_yuv, which the existing ladder kernels evaluate
// at run time, does not name them; the host checks take export_ycbcr, every format with chroma planes
GLB_HD bool export_p10(int format) { return format == GLAVA_B200_EXPORT_YUV420P10 || format == GLAVA_B200_EXPORT_YUV444P10; }
// The 4:2:2 formats (DESIGN 4.18), likewise kernels of their own: chroma per horizontal pixel pair, w even, any h
GLB_HD bool export_422(int format) {
    return format == GLAVA_B200_EXPORT_YUV422P || format == GLAVA_B200_EXPORT_YUV422P10 || format == GLAVA_B200_EXPORT_UYVY;
}
// The formats with an alpha plane (DESIGN 4.19), kernels of their own again: never composited, planar, A after Cr
GLB_HD bool export_yuva(int format) { return format == GLAVA_B200_EXPORT_YUVA420P || format == GLAVA_B200_EXPORT_YUVA444P10; }
// every Y'CbCr format, the ones the colour flags apply to; export_chroma_planes: those with chroma planes (UYVY packs its
// chroma into its one plane)
GLB_HD bool export_ycbcr(int format) { return export_yuv(format) || export_p10(format) || export_422(format) || export_yuva(format); }
GLB_HD bool export_chroma_planes(int format) { return export_ycbcr(format) && format != GLAVA_B200_EXPORT_UYVY; }
GLB_HD bool export_420(int format) {                   // chroma per 2x2 block: w and h even, items are row pairs
    return format == GLAVA_B200_EXPORT_NV12 || format == GLAVA_B200_EXPORT_I420 || format == GLAVA_B200_EXPORT_P010 ||
           format == GLAVA_B200_EXPORT_YUV420P10 || format == GLAVA_B200_EXPORT_YUVA420P;
}
GLB_HD bool export_planar(int format) {
    return format == GLAVA_B200_EXPORT_I420 || format == GLAVA_B200_EXPORT_YUV444 || export_p10(format) ||
           format == GLAVA_B200_EXPORT_YUV422P || format == GLAVA_B200_EXPORT_YUV422P10 || export_yuva(format);
}

// Where the chroma of a destination lies, from the descriptor and the output height: `cb`, the bytes from the luma to the
// chroma plane (NV12 / P010: the CbCr plane, uv_offset or pitch * h; the planar formats: the Cb plane, right after the
// luma); `cr`, the bytes from Cb to Cr (planar only: uv_offset, or 0 for one chroma plane, back to back; a YUVA format's
// A plane lies as far again past Cr); `plane`, the bytes of one planar chroma plane (I420 / YUV420P10 / YUVA420P: h / 2
// rows of pitch / 2; YUV422P / YUV422P10: h rows of pitch / 2)
struct ExportPlanes { size_t cb, cr, plane; };
GLB_HD ExportPlanes export_planes(int format, size_t pitch, size_t uv_offset, int h) {
    ExportPlanes p = { uv_offset ? uv_offset : pitch * (size_t) h, 0, 0 };
    if (export_planar(format)) {
        p.plane = format == GLAVA_B200_EXPORT_I420 || format == GLAVA_B200_EXPORT_YUV420P10 || format == GLAVA_B200_EXPORT_YUVA420P
                      ? (pitch / 2) * (size_t) (h / 2)
                  : format == GLAVA_B200_EXPORT_YUV422P || format == GLAVA_B200_EXPORT_YUV422P10 ? (pitch / 2) * (size_t) h
                                                                                                 : pitch * (size_t) h;
        p.cb = pitch * (size_t) h;
        p.cr = uv_offset ? uv_offset : p.plane;
    }
    return p;
}

// I420: NV12's CbCr word (Cb0, Cr0, Cb1, Cr1) as the two Cb bytes and the two Cr bytes
GLB_HD uint32_t export_cb_pair(uint32_t uv) { return (uv & 0xffu) | ((uv >> 8) & 0xff00u); }
GLB_HD uint32_t export_cr_pair(uint32_t uv) { return ((uv >> 8) & 0xffu) | ((uv >> 16) & 0xff00u); }

// YUV 4:4:4 of one row's quad: Y, Cb and Cr of each composited pixel, four bytes each
template <int E = 0>
GLB_HD void export_444_quad(const ExportFmt& f, const uint32_t in[4], uint32_t* y, uint32_t* cb, uint32_t* cr) {
    *y = 0u; *cb = 0u; *cr = 0u;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const uint32_t c = export_over(in[k], f.bg, f.native), uv = export_cbcr<E>(c);
        *y |= export_y<E>(c) << (8 * k);
        *cb |= (uv & 255u) << (8 * k);
        *cr |= (uv >> 8) << (8 * k);
    }
}

// P010: BT.709 limited range at 10 bits, Y = 64 + 876/255 Y', C = 512 + 896/255 (...), built as the 8-bit coefficients are
// (scaled by 2^16 and rounded; the blue coefficient of Cb and the red one of Cr minus the sum of the other two, so every grey
// has Cb = Cr = 512).  Black gives (64, 512, 512), white (940, 512, 512); over all 2^24 colours each code is within 0.503 code
// values of float64 (tests/test_export_formats_core.py).
#define GLB_Y10_R 47864
#define GLB_Y10_G 161017
#define GLB_Y10_B 16255
#define GLB_CB10_R (-26383)
#define GLB_CB10_G (-88755)
#define GLB_CB10_B (-(GLB_CB10_R + GLB_CB10_G))
#define GLB_CR10_G (-104580)
#define GLB_CR10_B (-10557)
#define GLB_CR10_R (-(GLB_CR10_G + GLB_CR10_B))
static_assert(yuv_same(yuv_enc(0, 10), GLB_Y10_R, GLB_Y10_G, GLB_Y10_B, GLB_CB10_R, GLB_CB10_G, GLB_CR10_G, GLB_CR10_B),
              "BT.709 limited 10-bit");
// the 10-bit Y code of a composited pixel
template <int E = 0>
GLB_HD uint32_t export_y10(uint32_t c) {
    if constexpr (E >= GLB_ENC_PQ) {
        return hdr_y10(hdr_rgb<E>(c));
    } else {
        constexpr YuvCoef S = yuv_enc(E, 10);
        const int r = (int) (c & 255u), g = (int) ((c >> 8) & 255u), b = (int) ((c >> 16) & 255u);
        return yuv_code<E, 10>(S.yr * r + S.yg * g + S.yb * b + (S.yoff << GLB_YUV_SHIFT) + GLB_YUV_HALF, GLB_YUV_SHIFT);
    }
}
// The per-channel sums (0..1020) of a 2x2 block's four composited pixels, 10 bits each (R low).  P010 chroma takes these
// exact sums, not NV12's (s + 2) >> 2 byte: the two bits that average rounds away are what 10 bits carry.
GLB_HD uint32_t export_sum4(uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    uint32_t out = 0;
#pragma unroll
    for (int k = 0; k < 3; ++k)
        out |= (((a >> (8 * k)) & 255u) + ((b >> (8 * k)) & 255u) + ((c >> (8 * k)) & 255u) + ((d >> (8 * k)) & 255u)) << (10 * k);
    return out;
}
// the 10-bit (Cb, Cr) codes of block sums s (export_sum4), Cb in the low 16 bits: the 16-bit coefficients over sums four
// times the average, so shift 18; every accumulator stays in [0, 2^31)
template <int E = 0>
GLB_HD uint32_t export_cbcr10(uint32_t s) {
    constexpr YuvCoef S = yuv_enc(E, 10);
    const int r = (int) (s & 1023u), g = (int) ((s >> 10) & 1023u), b = (int) (s >> 20);
    const uint32_t cb = yuv_code<E, 10>(S.cbr * r + S.cbg * g + S.cbb * b + (S.coff << 18) + (1 << 17), 18);
    const uint32_t cr = yuv_code<E, 10>(S.crr * r + S.crg * g + S.crb * b + (S.coff << 18) + (1 << 17), 18);
    return cb | (cr << 16);
}
// The 10-bit (Cb, Cr) codes of the 2x2 block of composited pixels a, b (top row), c, d, Cb low: export_cbcr10 of their sums,
// or under an HDR encoding the chroma of their mean E' (the scaled items, which hold one pixel per lane, take this)
template <int E = 0>
GLB_HD uint32_t export_block10(uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    if constexpr (E >= GLB_ENC_PQ) return hdr_cbcr10(hdr_mean4(hdr_rgb<E>(a), hdr_rgb<E>(b), hdr_rgb<E>(c), hdr_rgb<E>(d)));
    else return export_cbcr10<E>(export_sum4(a, b, c, d));
}
// P010 of a quad of output rows 2j (top) and 2j + 1 (bot): per row its four Y samples as two words (little-endian uint16,
// code << 6), and the (Cb, Cr) sample pairs of the quad's two 2x2 blocks, one word each
template <int E = 0>
GLB_HD void export_p010_quad(const ExportFmt& f, const uint32_t top[4], const uint32_t bot[4], uint32_t yt[2], uint32_t yb[2],
                             uint32_t uv[2]) {
    if constexpr (E >= GLB_ENC_PQ) {                        // DESIGN 4.22: each pixel's E' once, the block's mean for chroma
        HdrRgb t[4], b[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            t[k] = hdr_rgb<E>(export_over(top[k], f.bg, f.native));
            b[k] = hdr_rgb<E>(export_over(bot[k], f.bg, f.native));
        }
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            yt[k] = (hdr_y10(t[2 * k]) << 6) | (hdr_y10(t[2 * k + 1]) << 22);
            yb[k] = (hdr_y10(b[2 * k]) << 6) | (hdr_y10(b[2 * k + 1]) << 22);
            uv[k] = hdr_cbcr10(hdr_mean4(t[2 * k], t[2 * k + 1], b[2 * k], b[2 * k + 1])) << 6;
        }
    } else {
        uint32_t t[4], b[4];
    #pragma unroll
        for (int k = 0; k < 4; ++k) {
            t[k] = export_over(top[k], f.bg, f.native);
            b[k] = export_over(bot[k], f.bg, f.native);
        }
    #pragma unroll
        for (int k = 0; k < 2; ++k) {
            yt[k] = (export_y10<E>(t[2 * k]) << 6) | (export_y10<E>(t[2 * k + 1]) << 22);
            yb[k] = (export_y10<E>(b[2 * k]) << 6) | (export_y10<E>(b[2 * k + 1]) << 22);
            uv[k] = export_cbcr10<E>(export_sum4(t[2 * k], t[2 * k + 1], b[2 * k], b[2 * k + 1])) << 6;
        }
    }
}

// What zero pixels become in a new format's quad, for the kernels' all-zero shortcut: y, the luma word of a row (P010: one
// of its two equal words); u and v, I420's Cb and Cr pairs, YUV 4:4:4's Cb and Cr words, P010's CbCr word (v unused)
struct ExportZero { uint32_t y, u, v; };
template <int E = 0>
GLB_HD ExportZero export_zero(const ExportFmt& f) {
    const uint32_t z[4] = { 0u, 0u, 0u, 0u };
    ExportZero o = { 0u, 0u, 0u };
    if (f.format == GLAVA_B200_EXPORT_YUV444) {
        export_444_quad<E>(f, z, &o.y, &o.u, &o.v);
    } else if (f.format == GLAVA_B200_EXPORT_P010) {
        uint32_t yt[2], yb[2], uv[2];
        export_p010_quad<E>(f, z, z, yt, yb, uv);
        o.y = yt[0]; o.u = uv[0];
    } else {
        uint32_t yb;
        const uint32_t uv = export_nv12_quad<E>(f, z, z, &o.y, &yb);
        o.u = export_cb_pair(uv); o.v = export_cr_pair(uv);
    }
    return o;
}

// ---- planar 10-bit: yuv420p10le and yuv444p10le (DESIGN 4.16) -------------------------------------------------------------
// Little-endian uint16 samples holding the 10-bit code in their low bits.  Y is export_y10 (P010's code without the << 6).
// 4:2:0 chroma is P010's, export_cbcr10 of the exact block sums.  4:4:4 chroma is export_cbcr10 of the pixel's channels
// times 4, the sums of a 2x2 block of that pixel: with X = coef c + (off << 16), (4 X + 2^17) >> 18 = (X + 2^15) >> 16, the
// per-pixel 10-bit code, so no new rounding enters.
template <int E = 0>
GLB_HD uint32_t export_cbcr10_px(uint32_t c) {
    if constexpr (E >= GLB_ENC_PQ) {
        return hdr_cbcr10(hdr_rgb<E>(c));
    } else {
        const uint32_t s = (c & 255u) | (((c >> 8) & 255u) << 10) | (((c >> 16) & 255u) << 20);
        return export_cbcr10<E>(s << 2);
    }
}
// yuv420p10le of a quad of output rows 2j (top) and 2j + 1 (bot): per row its four Y samples as two words (two uint16
// each), and the Cb samples and the Cr samples of the quad's two 2x2 blocks, one word each
template <int E = 0>
GLB_HD void export_i010_quad(const ExportFmt& f, const uint32_t top[4], const uint32_t bot[4], uint32_t yt[2], uint32_t yb[2],
                             uint32_t* cb, uint32_t* cr) {
    if constexpr (E >= GLB_ENC_PQ) {                        // as export_p010_quad's, in the planar layout
        HdrRgb t[4], b[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            t[k] = hdr_rgb<E>(export_over(top[k], f.bg, f.native));
            b[k] = hdr_rgb<E>(export_over(bot[k], f.bg, f.native));
        }
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            yt[k] = hdr_y10(t[2 * k]) | (hdr_y10(t[2 * k + 1]) << 16);
            yb[k] = hdr_y10(b[2 * k]) | (hdr_y10(b[2 * k + 1]) << 16);
        }
        const uint32_t c0 = hdr_cbcr10(hdr_mean4(t[0], t[1], b[0], b[1])), c1 = hdr_cbcr10(hdr_mean4(t[2], t[3], b[2], b[3]));
        *cb = (c0 & 0xffffu) | (c1 << 16);
        *cr = (c0 >> 16) | (c1 & 0xffff0000u);
    } else {
        uint32_t t[4], b[4];
    #pragma unroll
        for (int k = 0; k < 4; ++k) {
            t[k] = export_over(top[k], f.bg, f.native);
            b[k] = export_over(bot[k], f.bg, f.native);
        }
    #pragma unroll
        for (int k = 0; k < 2; ++k) {
            yt[k] = export_y10<E>(t[2 * k]) | (export_y10<E>(t[2 * k + 1]) << 16);
            yb[k] = export_y10<E>(b[2 * k]) | (export_y10<E>(b[2 * k + 1]) << 16);
        }
        const uint32_t c0 = export_cbcr10<E>(export_sum4(t[0], t[1], b[0], b[1]));
        const uint32_t c1 = export_cbcr10<E>(export_sum4(t[2], t[3], b[2], b[3]));
        *cb = (c0 & 0xffffu) | (c1 << 16);
        *cr = (c0 >> 16) | (c1 & 0xffff0000u);
    }
}
// yuv444p10le of one row's quad: the Y, Cb and Cr samples of each composited pixel, two words each
template <int E = 0>
GLB_HD void export_444p10_quad(const ExportFmt& f, const uint32_t in[4], uint32_t y[2], uint32_t cb[2], uint32_t cr[2]) {
    if constexpr (E >= GLB_ENC_PQ) {                        // DESIGN 4.22: each pixel's E' once
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const HdrRgb e0 = hdr_rgb<E>(export_over(in[2 * k], f.bg, f.native)), e1 = hdr_rgb<E>(export_over(in[2 * k + 1], f.bg, f.native));
            const uint32_t uv0 = hdr_cbcr10(e0), uv1 = hdr_cbcr10(e1);
            y[k] = hdr_y10(e0) | (hdr_y10(e1) << 16);
            cb[k] = (uv0 & 0xffffu) | (uv1 << 16);
            cr[k] = (uv0 >> 16) | (uv1 & 0xffff0000u);
        }
    } else {
    #pragma unroll
        for (int k = 0; k < 2; ++k) {
            const uint32_t c0 = export_over(in[2 * k], f.bg, f.native), c1 = export_over(in[2 * k + 1], f.bg, f.native);
            const uint32_t uv0 = export_cbcr10_px<E>(c0), uv1 = export_cbcr10_px<E>(c1);
            y[k] = export_y10<E>(c0) | (export_y10<E>(c1) << 16);
            cb[k] = (uv0 & 0xffffu) | (uv1 << 16);
            cr[k] = (uv0 >> 16) | (uv1 & 0xffff0000u);
        }
    }
}
// export_zero of the planar 10-bit formats: y, one of a row's two equal luma words; u and v, the Cb and Cr words (YUV420P10:
// the quad's two blocks; YUV444P10: one of a row's two equal words)
template <int E = 0>
GLB_HD ExportZero export_zero10(const ExportFmt& f) {
    const uint32_t z[4] = { 0u, 0u, 0u, 0u };
    uint32_t y[2], yb[2], u[2], v[2];
    if (f.format == GLAVA_B200_EXPORT_YUV444P10) {
        export_444p10_quad<E>(f, z, y, u, v);
    } else {
        export_i010_quad<E>(f, z, z, y, yb, &u[0], &v[0]);
    }
    return { y[0], u[0], v[0] };
}

// ---- 4:2:2: yuv422p, yuv422p10le and UYVY (DESIGN 4.18) -------------------------------------------------------------------
// The chroma of a horizontal pixel pair (c0, c1) is the 4:2:0 chroma of the 2x2 block whose two rows are that pair, so no
// new rounding enters: 8 bits export_cbcr of export_avg4(c0, c1, c0, c1) (per channel (2a + 2b + 2) >> 2 = (a + b + 1) >> 1,
// NV12's chroma), 10 bits export_cbcr10 of export_sum4(c0, c1, c0, c1) (P010's exact-sum chroma, sums <= 1020).  Y is
// export_y / export_y10 per pixel.
// YUV422P of one row's quad: its four Y bytes, and the (Cb, Cr) pairs of its two pixel pairs as NV12's word (Cb0, Cr0, Cb1,
// Cr1; export_cb_pair / export_cr_pair split it into the planes' bytes)
template <int E = 0>
GLB_HD uint32_t export_422_quad(const ExportFmt& f, const uint32_t in[4], uint32_t* y) {
    uint32_t c[4];
    *y = 0u;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        c[k] = export_over(in[k], f.bg, f.native);
        *y |= export_y<E>(c[k]) << (8 * k);
    }
    return export_cbcr<E>(export_avg4(c[0], c[1], c[0], c[1])) | (export_cbcr<E>(export_avg4(c[2], c[3], c[2], c[3])) << 16);
}
// UYVY of the same: the Y word and the CbCr word interleaved as Cb, Y0, Cr, Y1 per pixel pair, one word per pair
GLB_HD void export_uyvy_words(uint32_t y, uint32_t uv, uint32_t w[2]) {
    w[0] = (uv & 0xffu) | ((y & 0xffu) << 8) | ((uv & 0xff00u) << 8) | ((y & 0xff00u) << 16);
    w[1] = ((uv >> 16) & 0xffu) | (((y >> 16) & 0xffu) << 8) | (((uv >> 24) & 0xffu) << 16) | (y & 0xff000000u);
}
// and back: the Y word and the CbCr word of two UYVY words
GLB_HD void export_uyvy_split(const uint32_t w[2], uint32_t* y, uint32_t* uv) {
    *y = ((w[0] >> 8) & 0xffu) | ((w[0] >> 16) & 0xff00u) | ((w[1] << 8) & 0xff0000u) | (w[1] & 0xff000000u);
    *uv = (w[0] & 0xffu) | ((w[0] >> 8) & 0xff00u) | ((w[1] & 0xffu) << 16) | ((w[1] << 8) & 0xff000000u);
}
// yuv422p10le of one row's quad: its four Y samples as two words, and the Cb samples and the Cr samples of its two pixel
// pairs, one word each
template <int E = 0>
GLB_HD void export_422p10_quad(const ExportFmt& f, const uint32_t in[4], uint32_t y[2], uint32_t* cb, uint32_t* cr) {
    if constexpr (E >= GLB_ENC_PQ) {                        // DESIGN 4.22: each pixel's E' once, a pair's chroma its block's
        HdrRgb e[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) e[k] = hdr_rgb<E>(export_over(in[k], f.bg, f.native));
#pragma unroll
        for (int k = 0; k < 2; ++k) y[k] = hdr_y10(e[2 * k]) | (hdr_y10(e[2 * k + 1]) << 16);
        const uint32_t c0 = hdr_cbcr10(hdr_mean4(e[0], e[1], e[0], e[1])), c1 = hdr_cbcr10(hdr_mean4(e[2], e[3], e[2], e[3]));
        *cb = (c0 & 0xffffu) | (c1 << 16);
        *cr = (c0 >> 16) | (c1 & 0xffff0000u);
    } else {
        uint32_t c[4];
    #pragma unroll
        for (int k = 0; k < 4; ++k) c[k] = export_over(in[k], f.bg, f.native);
    #pragma unroll
        for (int k = 0; k < 2; ++k) y[k] = export_y10<E>(c[2 * k]) | (export_y10<E>(c[2 * k + 1]) << 16);
        const uint32_t c0 = export_cbcr10<E>(export_sum4(c[0], c[1], c[0], c[1]));
        const uint32_t c1 = export_cbcr10<E>(export_sum4(c[2], c[3], c[2], c[3]));
        *cb = (c0 & 0xffffu) | (c1 << 16);
        *cr = (c0 >> 16) | (c1 & 0xffff0000u);
    }
}
// export_zero of the 4:2:2 formats: YUV422P y the Y word, u and v the Cb and Cr pairs; YUV422P10 y one of the two equal Y
// words, u and v the Cb and Cr words; UYVY y the word of a pixel pair (u, v unused)
template <int E = 0>
GLB_HD ExportZero export_zero422(const ExportFmt& f) {
    const uint32_t z[4] = { 0u, 0u, 0u, 0u };
    ExportZero o = { 0u, 0u, 0u };
    if (f.format == GLAVA_B200_EXPORT_YUV422P10) {
        uint32_t y[2];
        export_422p10_quad<E>(f, z, y, &o.u, &o.v);
        o.y = y[0];
    } else {
        uint32_t y, w[2];
        const uint32_t uv = export_422_quad<E>(f, z, &y);
        export_uyvy_words(y, uv, w);
        if (f.format == GLAVA_B200_EXPORT_UYVY) o.y = w[0];
        else { o.y = y; o.u = export_cb_pair(uv); o.v = export_cr_pair(uv); }
    }
    return o;
}

// ---- transparency: straight RGBA / BGRA, yuva420p and yuva444p10le (DESIGN 4.19) --------------------------------------------
// Under native opacity a stored pixel (c, a) is premultiplied over a transparent target.  Its straight (unassociated)
// colour, per channel, is S = a == 0 ? 0 : min(255, (c 255 + a / 2) / a): the integer quotient rounded half up, exact on
// host and device (plain unsigned division).  Wherever c <= a, mul_norm8(S, a) == c, so premultiplying S with the blend
// path's own product gives the stored pixel back (tests/test_export_alpha_core.py, all 65536 pairs).  The min and the
// a == 0 case only act where c > a: Graph runs no premultiply stage, so a translucent graph colour can store more
// colour than alpha, an additive part straight alpha cannot hold; it is clamped.
// The alpha formats are never composited: ExportFmt.over is set for them only under any other opacity than native, where
// the frame is opaque and export_over makes every pixel (c, 255), whose straight colour is c.  So STRAIGHT is then
// EXPORT_OVER's bytes, and the YUVA formats I420's / YUV444P10's Y, Cb and Cr with A = 255 (1023).
// Straight RGBA / BGRA run these kernels under a format code of their own, the public format with GLB_EXPORT_STRAIGHT set
// (public formats stay below it), chosen on the host by export_kernel_format.
#define GLB_EXPORT_STRAIGHT 0x100
GLB_HD bool export_straight(int format) { return (format & GLB_EXPORT_STRAIGHT) != 0; }
GLB_HD bool export_alpha(int format) { return export_yuva(format) || export_straight(format); }   // the alpha kernels' formats
inline int export_kernel_format(int format, uint32_t flags) {   // host code
    return flags & GLAVA_B200_EXPORT_STRAIGHT ? format | GLB_EXPORT_STRAIGHT : format;
}
// one straight channel of stored colour c and alpha a
GLB_HD uint32_t export_unpremul(uint32_t c, uint32_t a) {
    if (!a) return 0u;
    const uint32_t s = (c * 255u + (a >> 1)) / a;
    return s > 255u ? 255u : s;
}
// the straight pixel (S_r, S_g, S_b, a) of a stored one; opaque and zero pixels need no division
GLB_HD uint32_t export_straight_px(uint32_t px) {
    const uint32_t a = px >> 24;
    if (a == 255u || !px) return px;
    uint32_t out = px & 0xff000000u;
#pragma unroll
    for (int c = 0; c < 3; ++c) out |= export_unpremul((px >> (8 * c)) & 255u, a) << (8 * c);
    return out;
}
// the pixel the alpha arithmetic starts from: stored, or composited (any other opacity than native: (c, 255))
GLB_HD uint32_t export_alpha_in(const ExportFmt& f, uint32_t px) { return f.over ? export_over(px, f.bg, f.native) : px; }
// the 10-bit alpha code: (a 1023 + 127) / 255, no ties, 0 -> 0, 255 -> 1023, within 0.495 of a 1023 / 255
GLB_HD uint32_t export_a10(uint32_t a) { return (a * 1023u + 127u) / 255u; }
// The straight colour of a 2x2 block for its 4:2:0 chroma, weighted by alpha: per channel min(255, (sum c 255 + sum a / 2)
// / sum a), 0 when sum a = 0, i.e. the un-premultiplied block average.  Four opaque pixels give export_avg4 exactly:
// (s 255 + 510) / 1020 = (s + 2) >> 2.  Zero-alpha pixels hold black and so weigh nothing, which keeps bar edges free of
// dark fringes.
GLB_HD uint32_t export_block_straight(uint32_t p0, uint32_t p1, uint32_t p2, uint32_t p3) {
    const uint32_t sa = (p0 >> 24) + (p1 >> 24) + (p2 >> 24) + (p3 >> 24);
    if (!sa) return 0u;
    uint32_t out = 0u;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const uint32_t s = ((p0 >> (8 * k)) & 255u) + ((p1 >> (8 * k)) & 255u) + ((p2 >> (8 * k)) & 255u) + ((p3 >> (8 * k)) & 255u);
        const uint32_t v = (s * 255u + (sa >> 1)) / sa;
        out |= (v > 255u ? 255u : v) << (8 * k);
    }
    return out;
}
// straight RGBA / BGRA of one stored pixel (fmt: the kernel format code)
GLB_HD uint32_t export_straight_out(const ExportFmt& f, int fmt, uint32_t px) {
    const uint32_t s = export_straight_px(export_alpha_in(f, px));
    return (fmt & ~GLB_EXPORT_STRAIGHT) == GLAVA_B200_EXPORT_BGRA ? export_swap_rb(s) : s;
}
// yuva420p of a quad of output rows 2j (top) and 2j + 1 (bot): per row four Y bytes and four A bytes, and the Cb and Cr
// bytes of the quad's two 2x2 blocks (I420's pairs)
template <int E = 0>
GLB_HD void export_yuva420_quad(const ExportFmt& f, const uint32_t top[4], const uint32_t bot[4], uint32_t* yt, uint32_t* yb,
                                uint32_t* cb, uint32_t* cr, uint32_t* at, uint32_t* ab) {
    uint32_t t[4], b[4];
    *yt = 0u; *yb = 0u; *at = 0u; *ab = 0u;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        t[k] = export_alpha_in(f, top[k]);
        b[k] = export_alpha_in(f, bot[k]);
        *yt |= export_y<E>(export_straight_px(t[k])) << (8 * k);
        *yb |= export_y<E>(export_straight_px(b[k])) << (8 * k);
        *at |= (t[k] >> 24) << (8 * k);
        *ab |= (b[k] >> 24) << (8 * k);
    }
    const uint32_t uv = export_cbcr<E>(export_block_straight(t[0], t[1], b[0], b[1])) |
                        (export_cbcr<E>(export_block_straight(t[2], t[3], b[2], b[3])) << 16);
    *cb = export_cb_pair(uv); *cr = export_cr_pair(uv);
}
// yuva444p10le of one row's quad: the Y, Cb, Cr and A samples of each pixel, two words each
template <int E = 0>
GLB_HD void export_yuva444p10_quad(const ExportFmt& f, const uint32_t in[4], uint32_t y[2], uint32_t cb[2], uint32_t cr[2],
                                   uint32_t a[2]) {
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        const uint32_t p0 = export_alpha_in(f, in[2 * k]), p1 = export_alpha_in(f, in[2 * k + 1]);
        const uint32_t s0 = export_straight_px(p0), s1 = export_straight_px(p1);
        const uint32_t uv0 = export_cbcr10_px<E>(s0), uv1 = export_cbcr10_px<E>(s1);
        y[k] = export_y10<E>(s0) | (export_y10<E>(s1) << 16);
        cb[k] = (uv0 & 0xffffu) | (uv1 << 16);
        cr[k] = (uv0 >> 16) | (uv1 & 0xffff0000u);
        a[k] = export_a10(p0 >> 24) | (export_a10(p1 >> 24) << 16);
    }
}
// What zero pixels become in an alpha format, for the kernels' all-zero shortcut: YUVA420P y / a the Y / A word of a row,
// u / v the Cb / Cr pairs; YUVA444P10 y, u, v, a one of a row's two equal words per plane; straight RGBA / BGRA y the pixel
struct ExportZeroA { uint32_t y, u, v, a; };
template <int E = 0>
GLB_HD ExportZeroA export_zero_alpha(const ExportFmt& f) {
    const uint32_t z[4] = { 0u, 0u, 0u, 0u };
    ExportZeroA o = { 0u, 0u, 0u, 0u };
    if (f.format == GLAVA_B200_EXPORT_YUVA420P) {
        uint32_t yb, ab;
        export_yuva420_quad<E>(f, z, z, &o.y, &yb, &o.u, &o.v, &o.a, &ab);
    } else if (f.format == GLAVA_B200_EXPORT_YUVA444P10) {
        uint32_t y[2], u[2], v[2], a[2];
        export_yuva444p10_quad<E>(f, z, y, u, v, a);
        o = { y[0], u[0], v[0], a[0] };
    } else {
        o.y = export_straight_out(f, f.format, 0u);
    }
    return o;
}

// ---- mark-aware reads ----------------------------------------------------------------------------------------------------
// When the last raster pass kept dirty-row marks (capi.cu mark_key != 0), slot s of the framebuffer has one word per (band of
// `rows` rows, 128-pixel strip) at the band's first row (raster_core.h dirty_pack): rows [lo, hi) of the band may be non-zero,
// every other row of it is 0 in memory.  The export reads a row of a strip only when its band's word says so.
GLB_HD size_t export_mark_index(int slot, int w, int h, int rows, int y, int strip) {
    return ((size_t) slot * h + (size_t) (y - y % rows)) * (size_t) ((w + 127) >> 7) + (size_t) strip;
}
GLB_HD bool export_row_read(uint32_t mark, int y) { return y >= (int) (mark & 0xffffu) && y < (int) (mark >> 16); }

// ---- scaled export (DESIGN 4.11): exact integer area average ------------------------------------------------------------
// Along one axis `n` source pixels shrink to `m` outputs (1 <= m <= n <= 16384): output X covers [X n, (X + 1) n) and source
// i covers [i m, (i + 1) m); the weight of i in X is the length of their overlap.  The span of X is [first, last]; interior
// weights are all m, the two edge weights are given (first == last only when n == m, weight n).  Every product fits 32 bits.
struct ExportSpan { int first, last; uint32_t w_first, w_last; };
GLB_HD ExportSpan export_span(int X, int n, int m) {
    const uint32_t a = (uint32_t) X * (uint32_t) n, b = a + (uint32_t) n;
    ExportSpan s;
    s.first = (int) (a / (uint32_t) m);
    s.last = (int) ((b - 1u) / (uint32_t) m);
    const uint32_t e = (uint32_t) (s.first + 1) * (uint32_t) m;
    s.w_first = (e < b ? e : b) - a;
    s.w_last = b - (uint32_t) s.last * (uint32_t) m;
    return s;
}
// the weight of source index i (first <= i <= last) in the span
GLB_HD uint32_t export_span_weight(const ExportSpan& s, int i, int m) {
    return i == s.first ? s.w_first : i == s.last ? s.w_last : (uint32_t) m;
}
// Crop coordinates are top-down as the export writes them: crop row r is framebuffer row h - 1 - (src_y + r), and crop
// column i is framebuffer column src_x + i, whose mark word is that of strip (src_x + i) >> 7 (export_mark_index).  A
// footprint can straddle strips, so it is walked strip by strip.
GLB_HD int export_fb_row(int h, int src_y, int r) { return h - 1 - src_y - r; }
// The mark-aware walk of a footprint's framebuffer rows [y, y_end) in one strip goes band by band: the band that holds y
// ends at the returned row, and of its rows only [*ra, *rb) may be non-zero (`mark`: the band's word; rows == 0, no marks:
// one band, every row read).  A band the marks call empty costs one word, however many footprint rows it holds.
GLB_HD int export_band_rows(int y, int y_end, int rows, uint32_t mark, int* ra, int* rb) {
    if (!rows) { *ra = y; *rb = y_end; return y_end; }
    const int band_end = y - y % rows + rows, end = band_end < y_end ? band_end : y_end;
    const int lo = (int) (mark & 0xffffu), hi = (int) (mark >> 16);
    *ra = lo > y ? lo : y;
    *rb = hi < end ? hi : end;
    return end;
}

// floor(x / d) for every x < 2^63 as umulhi(x, mul) >> shift, d >= 2: shift = floor(log2(d - 1)), mul = ceil(2^(64 + shift) / d)
// (< 2^64 because d > 2^shift).  With e = mul d - 2^(64 + shift) in [0, d), x mul / 2^(64 + shift) = x / d + x e / (d 2^(64 +
// shift)), and x e < 2^63 2^(shift + 1) = 2^(64 + shift), so the error stays under 1 / d and never crosses an integer.
// d == 1: mul = 0, the quotient is x.
struct ExportRecip { uint64_t mul; int shift; };
inline ExportRecip export_recip(uint64_t d) {                 // host code
    if (d < 2) return { 0, 0 };
    int s = 63;
    while (!((d - 1) >> s)) --s;
    const unsigned __int128 k = (unsigned __int128) 1 << (64 + s);
    return { (uint64_t) ((k + d - 1) / d), s };
}
GLB_HD uint64_t export_div(uint64_t x, const ExportRecip& r) {
    if (!r.mul) return x;
#ifdef __CUDA_ARCH__
    return __umul64hi(x, r.mul) >> r.shift;
#else
    return (uint64_t) (((unsigned __int128) x * r.mul) >> 64) >> r.shift;
#endif
}

// One output pixel's sums: per channel sum of w * (composited) pixel and the total weight w of the pixels summed.  Only
// non-zero pixels are summed: a zero pixel, read or skipped by the marks, stands for `zc` = what a zero pixel becomes
// (export_px of 0 before any R / B swap), and export_scaled_px adds those in with the weight the sums lack.
// Per source row the sums are 32-bit (at most 255 * src_w); the fold over rows is 64-bit (at most 255 * d < 2^36).
GLB_HD void export_acc(const ExportFmt& f, uint32_t px, uint32_t w, uint32_t acc[4], uint32_t* wsum) {
    if (!px) return;
    if (f.over) px = export_over(px, f.bg, f.native);
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[c] += w * ((px >> (8 * c)) & 255u);
    *wsum += w;
}
GLB_HD void export_fold(const uint32_t row[4], uint32_t row_w, uint32_t wy, uint64_t acc[4], uint64_t* wsum) {
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[c] += (uint64_t) wy * row[c];
    *wsum += (uint64_t) wy * row_w;
}
// The output pixel (before any R / B swap): per channel (sum + (d - wsum) zc + d / 2) / d, d = src_w * src_h, the sum of all
// weights; composited, alpha is 255.  All sums zero: zc itself.
GLB_HD uint32_t export_scaled_px(const ExportFmt& f, const uint64_t acc[4], uint64_t wsum, uint64_t d, const ExportRecip& r, uint32_t zc) {
    if (!wsum) return zc;
    uint32_t out = f.over ? 0xff000000u : 0u;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        if (c == 3 && f.over) break;
        const uint64_t x = acc[c] + (d - wsum) * ((zc >> (8 * c)) & 255u) + (d >> 1);
        out |= (uint32_t) export_div(x, r) << (8 * c);
    }
    return out;
}

// ---- encoder ladder (DESIGN 4.13): one unit of the schedule ------------------------------------------------------------
// A unit is one item of a rung's standalone kernel: (rung, row, col) with row = output row pair and col = 128-pixel strip of
// a whole-frame rung (export_kernel), row = output row (NV12: row pair) and col = run of 32 output columns otherwise
// (export_scaled_kernel).  Packed as rung << 56 | row << 28 | col.
GLB_HD uint64_t ladder_unit(int rung, int row, int col) { return ((uint64_t) rung << 56) | ((uint64_t) row << 28) | (uint64_t) col; }
GLB_HD int ladder_unit_rung(uint64_t u) { return (int) (u >> 56); }
GLB_HD int ladder_unit_row(uint64_t u) { return (int) ((u >> 28) & 0xfffffffu); }
GLB_HD int ladder_unit_col(uint64_t u) { return (int) (u & 0xfffffffu); }
// The kernel a ladder launches, from its rungs' formats (kernel format codes) and encodings (host code):
// export_ladder_yuva_kernel when a rung is YUVA or straight RGBA / BGRA, else export_ladder_422_kernel when one is 4:2:2,
// else export_ladder_p10_kernel when one is planar 10-bit, else export_ladder_enc_kernel when one has an encoding other
// than 0, else export_ladder_yuv_kernel when one is I420, YUV444 or P010, else export_ladder_kernel; before all of them
// export_ladder_hdr_kernel when a rung has an HDR encoding (DESIGN 4.22)
enum LadderKernel { ladder_plain = 0, ladder_yuv = 1, ladder_enc = 2, ladder_p10 = 3, ladder_422 = 4, ladder_yuva = 5, ladder_hdr = 6 };
inline int ladder_kernel(const int* format, const int* enc, int n) {
    bool yuv = false, e = false, p10 = false, k422 = false, alpha = false;
    for (int j = 0; j < n; ++j)
        if (enc[j] >= GLB_ENC_PQ) return ladder_hdr;
    for (int j = 0; j < n; ++j) {
        yuv |= format[j] != GLAVA_B200_EXPORT_NV12 && export_yuv(format[j]);
        e |= enc[j] != 0;
        p10 |= export_p10(format[j]);
        k422 |= export_422(format[j]);
        alpha |= export_alpha(format[j]);
    }
    return alpha ? ladder_yuva : k422 ? ladder_422 : p10 ? ladder_p10 : e ? ladder_enc : yuv ? ladder_yuv : ladder_plain;
}

// ---- overlay (DESIGN 4.12): the frame composited onto the caller's image ----------------------------------------------------
// Native opacity only (any other opacity writes export_frames' opaque bytes).  The premultiplied "over" GLava's window
// performs on the desktop, with the caller's pixel d as the desktop, in all four channels: C = min(255, c + mul_norm8(d_c,
// 255 - a)), alpha likewise.  px and d in the same byte order (a BGRA destination takes export_swap_rb(px)).  A zero pixel
// leaves d as it is: mul_norm8(d, 255) = d.
GLB_HD uint32_t overlay_px(uint32_t px, uint32_t d) {
    const uint32_t ia = 255u - (px >> 24);
    uint32_t out = 0u;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const uint32_t v = ((px >> (8 * c)) & 255u) + mul_norm8((d >> (8 * c)) & 255u, ia);
        out |= (v > 255u ? 255u : v) << (8 * c);
    }
    return out;
}
// NV12 blends in Y'CbCr: the limited-range transform is affine, so the composite of premultiplied c (alpha a) over a pixel
// whose code value is V_D is off a/255 + M c + (1 - a/255) V_D exactly.  In the 16-bit fixed point of export_y /
// export_cbcr the first and last terms are one fraction T / 255, T = off a + (255 - a) V_D <= 255 * 255, rounded down in
// 2^-16 units (T 2^16 + 127 < 2^32).  a = 255 gives export_y / export_cbcr; a = 0 with c = 0 gives V_D back.
GLB_HD uint32_t overlay_frac(uint32_t off, uint32_t a, uint32_t vd) {
    return (((off * a + (255u - a) * vd) << GLB_YUV_SHIFT) + 127u) / 255u;
}
GLB_HD uint32_t overlay_clamp(int v) { return v < 0 ? 0u : v > 255 ? 255u : (uint32_t) v; }
// the Y byte of pixel px (stored, premultiplied) over a Y byte yd, the destination in encoding E (DESIGN 4.15: the offset
// is 16 in limited range, 0 in full range; every set keeps "a zero pixel leaves yd" and "an opaque pixel gives export_y")
template <int E = 0>
GLB_HD uint32_t overlay_y(uint32_t px, uint32_t yd) {
    constexpr YuvCoef S = yuv_enc(E, 8);
    const int r = (int) (px & 255u), g = (int) ((px >> 8) & 255u), b = (int) ((px >> 16) & 255u);
    const int t = (int) overlay_frac((uint32_t) S.yoff, px >> 24, yd);
    return overlay_clamp((S.yr * r + S.yg * g + S.yb * b + t + GLB_YUV_HALF) >> GLB_YUV_SHIFT);
}
// the (Cb, Cr) pair of a block average m (overlay_avg4: alpha included) over the pair uvd (Cb low byte, Cr high)
template <int E = 0>
GLB_HD uint32_t overlay_cbcr(uint32_t m, uint32_t uvd) {
    constexpr YuvCoef S = yuv_enc(E, 8);
    const int r = (int) (m & 255u), g = (int) ((m >> 8) & 255u), b = (int) ((m >> 16) & 255u);
    const uint32_t a = m >> 24;
    const int tb = (int) overlay_frac((uint32_t) S.coff, a, uvd & 255u), tr = (int) overlay_frac((uint32_t) S.coff, a, (uvd >> 8) & 255u);
    const int cb = (S.cbr * r + S.cbg * g + S.cbb * b + tb + GLB_YUV_HALF) >> GLB_YUV_SHIFT;
    const int cr = (S.crr * r + S.crg * g + S.crb * b + tr + GLB_YUV_HALF) >> GLB_YUV_SHIFT;
    return overlay_clamp(cb) | (overlay_clamp(cr) << 8);
}
// export_avg4 in all four channels: the chroma block of the overlay averages the stored pixels, alpha included
GLB_HD uint32_t overlay_avg4(uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    uint32_t out = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const uint32_t s = ((a >> (8 * k)) & 255u) + ((b >> (8 * k)) & 255u) + ((c >> (8 * k)) & 255u) + ((d >> (8 * k)) & 255u);
        out |= ((s + 2u) >> 2) << (8 * k);
    }
    return out;
}
// NV12 of a quad (rows 2j and 2j + 1, four pixels each) over the destination's Y words yt / yb and CbCr word uv (two pairs):
// updates them in place
template <int E = 0>
GLB_HD void overlay_nv12_quad(const uint32_t top[4], const uint32_t bot[4], uint32_t* yt, uint32_t* yb, uint32_t* uv) {
    uint32_t t = 0u, b = 0u;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        t |= overlay_y<E>(top[k], (*yt >> (8 * k)) & 255u) << (8 * k);
        b |= overlay_y<E>(bot[k], (*yb >> (8 * k)) & 255u) << (8 * k);
    }
    *yt = t; *yb = b;
    *uv = overlay_cbcr<E>(overlay_avg4(top[0], top[1], bot[0], bot[1]), *uv & 0xffffu) |
          (overlay_cbcr<E>(overlay_avg4(top[2], top[3], bot[2], bot[3]), *uv >> 16) << 16);
}
// NV12 under dirty-row marks, one warp per band [b0, b1) of a strip: the output row pairs it visits are [*ja, *jb) (pair j =
// framebuffer rows h - 1 - 2j and h - 2 - 2j), those that hold a row of [lo, hi), the rows the band's word lets through
// (lo < hi).  With odd band heights a pair can straddle a band edge; it belongs to the band of its upper framebuffer row if
// that row is marked, else to the other band.  So the band drops its top pair when that pair's upper row is b1 (the first
// row of the band above, overlay_top_straddles) and the band above marks it, and its bottom pair's lower row, below b0, is
// read when the band below marks it.  Returns whether the bottom pair straddles (the band below's word is then needed).
GLB_HD bool overlay_band_pairs(int h, int b0, int lo, int hi, int* ja, int* jb) {
    *ja = (h - hi) >> 1;
    *jb = ((h - 1 - lo) >> 1) + 1;
    return h - 2 - 2 * (*jb - 1) < b0;
}
GLB_HD bool overlay_top_straddles(int h, int b1, int ja) { return h - 1 - 2 * ja >= b1; }

// ---- overlay opacity (DESIGN 4.20) ------------------------------------------------------------------------------------------
// The pixel an overlay at opacity K (0..255) composites: all four channels of the premultiplied pixel scaled by K / 255 in
// the blend path's unorm8 product, then blended by the format's own native blend.  mul_norm8(x, 255) = x and mul_norm8(x,
// 0) = 0, so K = 255 is the plain overlay and K = 0 a zero pixel; the product is monotonic, so c <= a stays c' <= a'.
GLB_HD uint32_t fade_px(uint32_t px, uint32_t k) {
    uint32_t out = 0u;
#pragma unroll
    for (int c = 0; c < 4; ++c) out |= mul_norm8((px >> (8 * c)) & 255u, k) << (8 * c);
    return out;
}
// Any other opacity than native: GLava's window is opaque, the pixel is the stored colour with alpha 255 (export_over), faded
GLB_HD uint32_t fade_opaque(uint32_t px, uint32_t k) { return fade_px(px | 0xff000000u, k); }

// ---- overlay onto decoded pictures (DESIGN 4.17): I420, YUV 4:4:4 and the 10-bit formats ------------------------------------
// 8-bit I420 is NV12's arithmetic (overlay_y, overlay_cbcr of the block's overlay_avg4); YUV 4:4:4 takes overlay_cbcr of
// each pixel (the average of a 2x2 block of one pixel is that pixel).  10 bits build the same fraction at 10 bits:
//   Y   = clamp((coef c + F + 2^15) >> 16),      F = floor((T 2^16 + 127) / 255),   T = off a + (255 - a) V_D <= 1023 * 255
//   4:2:0 chroma from the block's exact sums S (export_sum4) and alpha sum S_a (0..1020), as P010's export chroma:
//   C   = clamp((coef S + 4 G + 2^17) >> 18),    G = floor((T' 2^16 + 509) / 1020), T' = off S_a + (1020 - S_a) V_D
//   4:4:4 chroma: the same of the pixel's channels and alpha times 4 (as export_cbcr10_px).
// T 2^16 passes 2^32, so F and G are taken exactly in 32 bits from T = 255 q + r (T' = 1020 q + r): F = q 2^16 + floor((r
// 2^16 + 127) / 255).  A zero pixel (block) gives V_D back, an opaque one (a = 255, S_a = 1020) export_y10 / export_cbcr10.
// Accumulators are signed: |coef c| <= 262915 * 255 and F <= 1023 * 2^16 keep Y's under 2^28; |coef S| <= 131458 * 1020
// and 4 G <= 1023 * 2^18 keep chroma's under 2^29.  Codes clamp to [0, 1023]: stored colours above their alpha (not
// premultiplied) can leave the range, as they can at 8 bits (overlay_clamp).
GLB_HD uint32_t overlay_frac10(uint32_t off, uint32_t a, uint32_t vd) {
    const uint32_t t = off * a + (255u - a) * vd, q = t / 255u;
    return (q << GLB_YUV_SHIFT) + (((t - 255u * q) << GLB_YUV_SHIFT) + 127u) / 255u;
}
GLB_HD uint32_t overlay_frac10_4(uint32_t off, uint32_t sa, uint32_t vd) {
    const uint32_t t = off * sa + (1020u - sa) * vd, q = t / 1020u;
    return (q << GLB_YUV_SHIFT) + (((t - 1020u * q) << GLB_YUV_SHIFT) + 509u) / 1020u;
}
GLB_HD uint32_t overlay_clamp10(int v) { return v < 0 ? 0u : v > 1023 ? 1023u : (uint32_t) v; }
// the 10-bit Y code of pixel px (stored, premultiplied) over the code yd, in encoding E
template <int E = 0>
GLB_HD uint32_t overlay_y10(uint32_t px, uint32_t yd) {
    constexpr YuvCoef S = yuv_enc(E, 10);
    const int r = (int) (px & 255u), g = (int) ((px >> 8) & 255u), b = (int) ((px >> 16) & 255u);
    const int t = (int) overlay_frac10((uint32_t) S.yoff, px >> 24, yd);
    return overlay_clamp10((S.yr * r + S.yg * g + S.yb * b + t + GLB_YUV_HALF) >> GLB_YUV_SHIFT);
}
// the 10-bit (Cb, Cr) codes, Cb in the low 16 bits, of block sums s (export_sum4) with alpha sum sa over the codes cbd, crd
template <int E = 0>
GLB_HD uint32_t overlay_cbcr10(uint32_t s, uint32_t sa, uint32_t cbd, uint32_t crd) {
    constexpr YuvCoef S = yuv_enc(E, 10);
    const int r = (int) (s & 1023u), g = (int) ((s >> 10) & 1023u), b = (int) (s >> 20);
    const int gb = (int) overlay_frac10_4((uint32_t) S.coff, sa, cbd), gr = (int) overlay_frac10_4((uint32_t) S.coff, sa, crd);
    const int cb = (S.cbr * r + S.cbg * g + S.cbb * b + 4 * gb + (1 << 17)) >> 18;
    const int cr = (S.crr * r + S.crg * g + S.crb * b + 4 * gr + (1 << 17)) >> 18;
    return overlay_clamp10(cb) | (overlay_clamp10(cr) << 16);
}
GLB_HD uint32_t overlay_asum4(uint32_t a, uint32_t b, uint32_t c, uint32_t d) { return (a >> 24) + (b >> 24) + (c >> 24) + (d >> 24); }

// A 10-bit sample of the caller's picture holds its code as v >> 6 (P010: Msb) or v & 1023 (planar); a blended sample is
// written with the other bits zero, and a sample no non-zero pixel covers keeps all 16 bits.
template <bool Msb> GLB_HD uint32_t overlay_code10(uint32_t v) { return Msb ? (v & 0xffffu) >> 6 : v & 1023u; }
template <bool Msb> GLB_HD uint32_t overlay_sample10(uint32_t code) { return Msb ? code << 6 : code; }
// Y of pixel px over sample v
template <int E, bool Msb>
GLB_HD uint32_t overlay_y10_sample(uint32_t px, uint32_t v) {
    return px ? overlay_sample10<Msb>(overlay_y10<E>(px, overlay_code10<Msb>(v))) : v & 0xffffu;
}
// Y of pixels p0, p1 over a word of two samples (p0's low)
template <int E, bool Msb>
GLB_HD uint32_t overlay_y10_word(uint32_t p0, uint32_t p1, uint32_t v) {
    return overlay_y10_sample<E, Msb>(p0, v) | (overlay_y10_sample<E, Msb>(p1, v >> 16) << 16);
}
// the (Cb, Cr) samples of a 2x2 block over the samples cb, cr: Cb low, Cr high
template <int E, bool Msb>
GLB_HD uint32_t overlay_block10(uint32_t p0, uint32_t p1, uint32_t p2, uint32_t p3, uint32_t cb, uint32_t cr) {
    if ((p0 | p1 | p2 | p3) == 0u) return (cb & 0xffffu) | (cr << 16);
    const uint32_t c = overlay_cbcr10<E>(export_sum4(p0, p1, p2, p3), overlay_asum4(p0, p1, p2, p3), overlay_code10<Msb>(cb),
                                         overlay_code10<Msb>(cr));
    return overlay_sample10<Msb>(c & 0xffffu) | (overlay_sample10<Msb>(c >> 16) << 16);
}
// the (Cb, Cr) samples of one pixel (4:4:4) over the samples cb, cr: a 2x2 block of that pixel
template <int E, bool Msb>
GLB_HD uint32_t overlay_px10(uint32_t px, uint32_t cb, uint32_t cr) { return overlay_block10<E, Msb>(px, px, px, px, cb, cr); }

// ---- overlay onto HDR pictures (DESIGN 4.22) ------------------------------------------------------------------------------
// The blend happens in the picture's code domain, as at SDR, from each pixel's straight colour S (export_straight_px) and its
// alpha a: Y = round((a Y_f(S) + (255 - a) Y_D) / 255), Y_f the unrounded code; the chroma of n pixels (a 2x2 block, a
// pair as the block (p0, p1, p0, p1), one pixel as the block of four) with A = sum a_i is round(512 + sum a_i (C_f(S_i) -
// 512) / (255 n) + (1 - A / (255 n)) (C_D - 512)), taken as the chroma of the weighted mean P = sum (a_i / 255) E'_i / n
// (linear in E') plus (1 - A / (255 n)) (C_D - 512).  An opaque pixel (block) has weights 1 and 0 exactly, so it gives the
// HDR export's codes bit for bit; zero pixels and blocks are left to the callers, which keep their samples.
struct HdrPx { HdrRgb e; float w; };                        // E' of the straight colour, and a / 255
template <int E>
GLB_HD HdrPx hdr_px(uint32_t px) { return { hdr_rgb<E>(export_straight_px(px)), glm_div((float) (px >> 24), 255.0f) }; }
// the Y code of pixel p over the code yd
GLB_HD uint32_t hdr_over_y(const HdrPx& p, uint32_t yd) {
    const uint32_t v = hdr_code(glm_add(glm_mul(hdr_yf(p.e), p.w), glm_mul((float) yd, glm_add(1.0f, -p.w))));
    return v > 1023u ? 1023u : v;
}
// the (Cb, Cr) codes, Cb low, of the block a, b (top row), c, d over the codes cbd, crd
GLB_HD uint32_t hdr_over_cbcr(const HdrPx& a, const HdrPx& b, const HdrPx& c, const HdrPx& d, uint32_t cbd, uint32_t crd) {
    const HdrRgb m = hdr_mean4({ glm_mul(a.e.r, a.w), glm_mul(a.e.g, a.w), glm_mul(a.e.b, a.w) },
                               { glm_mul(b.e.r, b.w), glm_mul(b.e.g, b.w), glm_mul(b.e.b, b.w) },
                               { glm_mul(c.e.r, c.w), glm_mul(c.e.g, c.w), glm_mul(c.e.b, c.w) },
                               { glm_mul(d.e.r, d.w), glm_mul(d.e.g, d.w), glm_mul(d.e.b, d.w) });
    const float k = glm_add(1.0f, -glm_mul(glm_add(glm_add(a.w, b.w), glm_add(c.w, d.w)), 0.25f));
    const uint32_t cb = hdr_code(glm_add(hdr_cbf(m), glm_mul(k, glm_add((float) cbd, -512.0f))));
    const uint32_t cr = hdr_code(glm_add(hdr_crf(m), glm_mul(k, glm_add((float) crd, -512.0f))));
    return (cb > 1023u ? 1023u : cb) | ((cr > 1023u ? 1023u : cr) << 16);
}
// Y of pixel px (E' and weight p) over sample v: a zero pixel keeps all 16 bits
template <bool Msb>
GLB_HD uint32_t hdr_over_y_sample(uint32_t px, const HdrPx& p, uint32_t v) {
    return px ? overlay_sample10<Msb>(hdr_over_y(p, overlay_code10<Msb>(v))) : v & 0xffffu;
}

// I420 of a quad (rows 2j and 2j + 1) over the Y words yt / yb and the Cb and Cr pairs cb / cr (two bytes each): NV12's
// overlay_nv12_quad on the interleaved pairs, so I420 is NV12 deinterleaved bit for bit
template <int E = 0>
GLB_HD void overlay_i420_quad(const uint32_t top[4], const uint32_t bot[4], uint32_t* yt, uint32_t* yb, uint32_t* cb, uint32_t* cr) {
    uint32_t uv = (*cb & 0xffu) | ((*cr & 0xffu) << 8) | ((*cb & 0xff00u) << 8) | ((*cr & 0xff00u) << 16);
    overlay_nv12_quad<E>(top, bot, yt, yb, &uv);
    *cb = export_cb_pair(uv); *cr = export_cr_pair(uv);
}
// YUV 4:4:4 of one row's quad over the Y, Cb and Cr words (four bytes each)
template <int E = 0>
GLB_HD void overlay_444_quad(const uint32_t in[4], uint32_t* y, uint32_t* cb, uint32_t* cr) {
    uint32_t oy = 0u, ou = 0u, ov = 0u;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        oy |= overlay_y<E>(in[k], (*y >> (8 * k)) & 255u) << (8 * k);
        const uint32_t uv = overlay_cbcr<E>(in[k], ((*cb >> (8 * k)) & 255u) | (((*cr >> (8 * k)) & 255u) << 8));
        ou |= (uv & 255u) << (8 * k);
        ov |= (uv >> 8) << (8 * k);
    }
    *y = oy; *cb = ou; *cr = ov;
}
// P010 (Msb) or YUV420P10 of a quad over the Y words yt[2] / yb[2] (two samples each) and the chroma of its two blocks:
// P010 uv[2], one (Cb, Cr) word per block; YUV420P10 uv[0] the two Cb samples, uv[1] the two Cr samples
template <int E, bool Msb>
GLB_HD void overlay_p10_quad(const uint32_t top[4], const uint32_t bot[4], uint32_t yt[2], uint32_t yb[2], uint32_t uv[2]) {
    if constexpr (E >= GLB_ENC_PQ) {                        // DESIGN 4.22: each pixel's E' once
        HdrPx t[4], b[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) { t[k] = hdr_px<E>(top[k]); b[k] = hdr_px<E>(bot[k]); }
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            yt[k] = hdr_over_y_sample<Msb>(top[2 * k], t[2 * k], yt[k]) | (hdr_over_y_sample<Msb>(top[2 * k + 1], t[2 * k + 1], yt[k] >> 16) << 16);
            yb[k] = hdr_over_y_sample<Msb>(bot[2 * k], b[2 * k], yb[k]) | (hdr_over_y_sample<Msb>(bot[2 * k + 1], b[2 * k + 1], yb[k] >> 16) << 16);
        }
        // sample by sample, as the planar chroma below: P010 uv[k] is block k's (Cb, Cr) word, YUV420P10 uv[0] / uv[1] the
        // two Cb / Cr samples
        uint32_t cb[2], cr[2];
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            cb[k] = Msb ? uv[k] & 0xffffu : (uv[0] >> (16 * k)) & 0xffffu;
            cr[k] = Msb ? uv[k] >> 16 : (uv[1] >> (16 * k)) & 0xffffu;
            if ((top[2 * k] | top[2 * k + 1] | bot[2 * k] | bot[2 * k + 1]) != 0u) {
                const uint32_t c = hdr_over_cbcr(t[2 * k], t[2 * k + 1], b[2 * k], b[2 * k + 1], overlay_code10<Msb>(cb[k]),
                                                 overlay_code10<Msb>(cr[k]));
                cb[k] = overlay_sample10<Msb>(c & 0xffffu);
                cr[k] = overlay_sample10<Msb>(c >> 16);
            }
        }
        if (Msb) { uv[0] = cb[0] | (cr[0] << 16); uv[1] = cb[1] | (cr[1] << 16); }
        else { uv[0] = cb[0] | (cb[1] << 16); uv[1] = cr[0] | (cr[1] << 16); }
    } else {
    #pragma unroll
        for (int k = 0; k < 2; ++k) {
            yt[k] = overlay_y10_word<E, Msb>(top[2 * k], top[2 * k + 1], yt[k]);
            yb[k] = overlay_y10_word<E, Msb>(bot[2 * k], bot[2 * k + 1], yb[k]);
        }
        if (Msb) {
    #pragma unroll
            for (int k = 0; k < 2; ++k) uv[k] = overlay_block10<E, true>(top[2 * k], top[2 * k + 1], bot[2 * k], bot[2 * k + 1], uv[k], uv[k] >> 16);
        } else {
            // sample by sample: packing both blocks' results through overlay_block10's words let nvcc 12.9 (sm_90a) merge a
            // kept Cr sample's bits into the blended one; tests/test_gpu_overlay_planes.py pins the result on the device
            uint32_t cb[2], cr[2];
    #pragma unroll
            for (int k = 0; k < 2; ++k) {
                cb[k] = (uv[0] >> (16 * k)) & 0xffffu;
                cr[k] = (uv[1] >> (16 * k)) & 0xffffu;
                if ((top[2 * k] | top[2 * k + 1] | bot[2 * k] | bot[2 * k + 1]) != 0u) {
                    const uint32_t c = overlay_cbcr10<E>(export_sum4(top[2 * k], top[2 * k + 1], bot[2 * k], bot[2 * k + 1]),
                                                         overlay_asum4(top[2 * k], top[2 * k + 1], bot[2 * k], bot[2 * k + 1]),
                                                         cb[k] & 1023u, cr[k] & 1023u);
                    cb[k] = c & 0xffffu;
                    cr[k] = c >> 16;
                }
            }
            uv[0] = cb[0] | (cb[1] << 16);
            uv[1] = cr[0] | (cr[1] << 16);
        }
    }
}
// YUV444P10 of one row's quad over the Y, Cb and Cr words y[2], cb[2], cr[2] (two samples each)
template <int E = 0>
GLB_HD void overlay_444p10_quad(const uint32_t in[4], uint32_t y[2], uint32_t cb[2], uint32_t cr[2]) {
    if constexpr (E >= GLB_ENC_PQ) {                        // DESIGN 4.22: each pixel's chroma its own block of four
        uint32_t oy[4], u[4], v[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint32_t ys = (y[k >> 1] >> (16 * (k & 1))) & 0xffffu;
            u[k] = (cb[k >> 1] >> (16 * (k & 1))) & 0xffffu;
            v[k] = (cr[k >> 1] >> (16 * (k & 1))) & 0xffffu;
            oy[k] = ys;
            if (in[k]) {
                const HdrPx p = hdr_px<E>(in[k]);
                oy[k] = hdr_over_y(p, ys & 1023u);
                const uint32_t c = hdr_over_cbcr(p, p, p, p, u[k] & 1023u, v[k] & 1023u);
                u[k] = c & 0xffffu;
                v[k] = c >> 16;
            }
        }
        y[0] = oy[0] | (oy[1] << 16); y[1] = oy[2] | (oy[3] << 16);
        cb[0] = u[0] | (u[1] << 16); cb[1] = u[2] | (u[3] << 16);
        cr[0] = v[0] | (v[1] << 16); cr[1] = v[2] | (v[3] << 16);
    } else {
    #pragma unroll
        for (int k = 0; k < 2; ++k) y[k] = overlay_y10_word<E, false>(in[2 * k], in[2 * k + 1], y[k]);
        // sample by sample, as overlay_p10_quad's planar chroma
        uint32_t u[4], v[4];
    #pragma unroll
        for (int k = 0; k < 4; ++k) {
            u[k] = (cb[k >> 1] >> (16 * (k & 1))) & 0xffffu;
            v[k] = (cr[k >> 1] >> (16 * (k & 1))) & 0xffffu;
            if (in[k]) {
                const uint32_t c = overlay_cbcr10<E>(export_sum4(in[k], in[k], in[k], in[k]), 4u * (in[k] >> 24), u[k] & 1023u, v[k] & 1023u);
                u[k] = c & 0xffffu;
                v[k] = c >> 16;
            }
        }
        cb[0] = u[0] | (u[1] << 16); cb[1] = u[2] | (u[3] << 16);
        cr[0] = v[0] | (v[1] << 16); cr[1] = v[2] | (v[3] << 16);
    }
}

// ---- overlay onto 4:2:2 pictures (DESIGN 4.18) ----------------------------------------------------------------------------
// The chroma of a pixel pair (p0, p1) is the 4:2:0 blend of the block whose two rows are that pair: 8 bits overlay_cbcr of
// overlay_avg4(p0, p1, p0, p1), 10 bits overlay_cbcr10 of its sums.  A zero pair leaves its chroma (8 bits: overlay_cbcr of
// 0 is uvd exactly), an opaque pair gives export_422_quad's / export_422p10_quad's chroma.
// YUV422P (and UYVY, through export_uyvy_split) of one row's quad over the Y word y and the CbCr word uv (NV12's layout)
template <int E = 0>
GLB_HD void overlay_422_quad(const uint32_t in[4], uint32_t* y, uint32_t* uv) {
    uint32_t oy = 0u;
#pragma unroll
    for (int k = 0; k < 4; ++k) oy |= overlay_y<E>(in[k], (*y >> (8 * k)) & 255u) << (8 * k);
    *y = oy;
    *uv = overlay_cbcr<E>(overlay_avg4(in[0], in[1], in[0], in[1]), *uv & 0xffffu) |
          (overlay_cbcr<E>(overlay_avg4(in[2], in[3], in[2], in[3]), *uv >> 16) << 16);
}
// YUV422P10 of one row's quad over the Y words y[2] and the Cb and Cr words cb, cr (two samples each); the chroma sample by
// sample, as overlay_p10_quad's planar chroma
template <int E = 0>
GLB_HD void overlay_422p10_quad(const uint32_t in[4], uint32_t y[2], uint32_t* cb, uint32_t* cr) {
    if constexpr (E >= GLB_ENC_PQ) {                        // DESIGN 4.22: each pixel's E' once, a pair's chroma its block's
        HdrPx p[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) p[k] = hdr_px<E>(in[k]);
#pragma unroll
        for (int k = 0; k < 2; ++k)
            y[k] = hdr_over_y_sample<false>(in[2 * k], p[2 * k], y[k]) | (hdr_over_y_sample<false>(in[2 * k + 1], p[2 * k + 1], y[k] >> 16) << 16);
        uint32_t u[2], v[2];
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            u[k] = (*cb >> (16 * k)) & 0xffffu;
            v[k] = (*cr >> (16 * k)) & 0xffffu;
            if ((in[2 * k] | in[2 * k + 1]) != 0u) {
                const uint32_t c = hdr_over_cbcr(p[2 * k], p[2 * k + 1], p[2 * k], p[2 * k + 1], u[k] & 1023u, v[k] & 1023u);
                u[k] = c & 0xffffu;
                v[k] = c >> 16;
            }
        }
        *cb = u[0] | (u[1] << 16);
        *cr = v[0] | (v[1] << 16);
    } else {
    #pragma unroll
        for (int k = 0; k < 2; ++k) y[k] = overlay_y10_word<E, false>(in[2 * k], in[2 * k + 1], y[k]);
        uint32_t u[2], v[2];
    #pragma unroll
        for (int k = 0; k < 2; ++k) {
            const uint32_t p0 = in[2 * k], p1 = in[2 * k + 1];
            u[k] = (*cb >> (16 * k)) & 0xffffu;
            v[k] = (*cr >> (16 * k)) & 0xffffu;
            if ((p0 | p1) != 0u) {
                const uint32_t c = overlay_cbcr10<E>(export_sum4(p0, p1, p0, p1), overlay_asum4(p0, p1, p0, p1), u[k] & 1023u, v[k] & 1023u);
                u[k] = c & 0xffffu;
                v[k] = c >> 16;
            }
        }
        *cb = u[0] | (u[1] << 16);
        *cr = v[0] | (v[1] << 16);
    }
}

}  // namespace glb
#endif
