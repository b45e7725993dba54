"""Transparent exports, straight RGBA / BGRA, YUVA420P and YUVA444P10 (DESIGN 4.19), on the host: the un-premultiply of
export_core.h over all 65536 (c, a) pairs (the integer formula, within 0.5 of c 255 / a and re-premultiplied by the blend
path's mul_norm8 to c wherever c <= a), the 10-bit alpha code, the alpha-weighted block chroma, the Y'CbCr bounds against
float64 of the exact straight colour per encoding, host walks of export_yuva_kernel's and export_scaled_yuva_kernel's
loops against tests/export_alpha_np.py with sentinel bytes around and between all four planes, the identities with the
opaque exports, and the refusals, byte counts and ladder kernel choice through the fake runtime."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from tests.export_alpha_np import (a10_np, alpha_in_np, block_straight_np, export_alpha_np, frame_alpha_np,
                                   scaled_alpha_np, unpremul_np)
from tests.export_fake import desc_of
from tests.test_export_core import CSRC, marked_frame, over_np, pack, premultiplied
from tests.test_export_formats_core import call, device_buf, memcpys, renderer
from tests.test_export_formats_core import fake  # noqa: F401 (the fake-runtime fixture)
from tests.test_export_ladder_core import rungs_of, scale_of
from tests.test_export_matrix_core import ENCODINGS
from tests.test_export_p10_core import p10_np
from tests.test_export_scaled_core import area_np

RGBA, BGRA, NV12, I420, YUV444P10, YUVA420P, YUVA444P10 = 0, 1, 2, 4, 8, 14, 15
OVER, STRAIGHT = 1, 4
RGBA_S, BGRA_S = RGBA | 0x100, BGRA | 0x100                   # the kernel format codes of straight RGBA / BGRA
SENTINEL = 0xA5
# every (format, encoding) the kernels are instantiated for: straight RGBA / BGRA have no encoding
FMT_E = [(f, e) for f in (YUVA420P, YUVA444P10) for e in range(4)] + [(RGBA_S, 0), (BGRA_S, 0)]
# the largest distance of each code from float64 on the exact straight colour (c 255 / a per channel) over the sample of
# t_bounds, per (encoding, bits): [Y, Cb, Cr], as DESIGN 4.19 records them
BOUND = {(0, 8): (0.9298, 0.9285, 0.9255), (1, 8): (1.0001, 0.9970, 0.9919), (2, 8): (0.9304, 0.9256, 0.9222),
         (3, 8): (1.0000, 0.9970, 0.9919), (0, 10): (2.2193, 2.2110, 2.2293), (1, 10): (2.5065, 2.4708, 2.4634),
         (2, 10): (2.2168, 2.2176, 2.2293), (3, 10): (2.5072, 2.4703, 2.4594)}

SHIM = r"""
#include "export_core.h"
using namespace glb;
#define DISPATCH(fn, ...) switch (e) { case 1: fn<1>(__VA_ARGS__); break; case 2: fn<2>(__VA_ARGS__); break; \
                                       case 3: fn<3>(__VA_ARGS__); break; default: fn<0>(__VA_ARGS__); }
static void put(uint8_t* p, uint32_t v, int n) { memcpy(p, &v, n); }      // the first n bytes of v, little-endian
static void put16(uint8_t* p, const uint32_t* v, int n) {                  // the first n uint16 samples of the words v[]
    for (int k = 0; k < n; ++k) { const uint16_t s = (uint16_t) (v[k >> 1] >> (16 * (k & 1))); memcpy(p + 2 * k, &s, 2); }
}
extern "C" void t_pairs(uint32_t* s, uint32_t* m) {                        // every (c, a): S and mul_norm8(S, a)
    for (uint32_t a = 0; a < 256; ++a)
        for (uint32_t c = 0; c < 256; ++c) { s[a * 256 + c] = export_unpremul(c, a); m[a * 256 + c] = mul_norm8(s[a * 256 + c], a); }
}
extern "C" void t_px(const uint32_t* px, size_t n, uint32_t* out) { for (size_t i = 0; i < n; ++i) out[i] = export_straight_px(px[i]); }
extern "C" void t_a10(uint32_t* out) { for (uint32_t a = 0; a < 256; ++a) out[a] = export_a10(a); }
extern "C" void t_block(const uint32_t* p, size_t n, uint32_t* out, uint32_t* avg) {
    for (size_t i = 0; i < n; ++i) {
        out[i] = export_block_straight(p[4 * i], p[4 * i + 1], p[4 * i + 2], p[4 * i + 3]);
        avg[i] = export_avg4(p[4 * i], p[4 * i + 1], p[4 * i + 2], p[4 * i + 3]);
    }
}
// one slot [h][w] -> the planes, as export_yuva_kernel walks it (yuva_item): row pairs, 128-pixel strips, a quad per lane
template <int E> static void walk(const uint32_t* fb, int w, int h, const uint32_t* marks, int rows, int fmt, int over, int native,
                                  uint32_t bg, uint8_t* dst, size_t pitch, uint8_t* cb, size_t cr) {
    const ExportFmt f = { fmt, over, native, bg };
    const ExportZeroA z = export_zero_alpha<E>(f);
    for (int j = 0; j < (h + 1) / 2; ++j)
        for (int strip = 0; strip < (w + 127) >> 7; ++strip)
            for (int lane = 0; lane < 32; ++lane) {
                const int x = strip * 128 + lane * 4;
                if (x >= w) continue;
                const int y0 = h - 1 - 2 * j, y1 = y0 - 1;
                uint32_t q[2][4] = { { 0u, 0u, 0u, 0u }, { 0u, 0u, 0u, 0u } };
                for (int r = 0; r < 2; ++r) {
                    const int y = r ? y1 : y0;
                    if (y < 0 || (marks && !export_row_read(marks[export_mark_index(0, w, h, rows, y, strip)], y))) continue;
                    for (int k = 0; k < 4; ++k) q[r][k] = x + k < w ? fb[(size_t) y * w + x + k] : 0u;
                }
                const int n = x + 4 <= w ? 4 : w - x;
                for (int r = 0; r < 2 && (r == 0 || y1 >= 0); ++r) {
                    const bool any = (q[r][0] | q[r][1] | q[r][2] | q[r][3]) != 0u;
                    if (export_straight(fmt)) {
                        for (int k = 0; k < n; ++k) put(dst + (size_t) (2 * j + r) * pitch + 4 * (size_t) (x + k), any ? export_straight_out(f, fmt, q[r][k]) : z.y, 4);
                    } else if (fmt == GLAVA_B200_EXPORT_YUVA444P10) {
                        uint32_t y[2] = { z.y, z.y }, u[2] = { z.u, z.u }, v[2] = { z.v, z.v }, a[2] = { z.a, z.a };
                        if (any) export_yuva444p10_quad<E>(f, q[r], y, u, v, a);
                        const size_t o = (size_t) (2 * j + r) * pitch + 2 * (size_t) x;
                        put16(dst + o, y, n); put16(cb + o, u, n); put16(cb + cr + o, v, n); put16(cb + 2 * cr + o, a, n);
                    }
                }
                if (fmt != GLAVA_B200_EXPORT_YUVA420P) continue;
                uint32_t yt = z.y, yb = z.y, u = z.u, v = z.v, at = z.a, ab = z.a;
                if (q[0][0] | q[0][1] | q[0][2] | q[0][3] | q[1][0] | q[1][1] | q[1][2] | q[1][3]) export_yuva420_quad<E>(f, q[0], q[1], &yt, &yb, &u, &v, &at, &ab);
                const size_t o = (size_t) (2 * j) * pitch + x;
                uint8_t* pu = cb + (size_t) j * (pitch / 2) + x / 2;
                put(dst + o, yt, n); put(dst + o + pitch, yb, n); put(pu, u, n / 2); put(pu + cr, v, n / 2);
                put(cb + 2 * cr + o, at, n); put(cb + 2 * cr + o + pitch, ab, n);
            }
}
// the scaled image img [out_h][out_w] (scaled_px of each output pixel) -> the planes, as export_scaled_yuva_kernel walks it
// (scaled_yuva_item): units of one output row (YUVA420P: a row pair), runs of 32 lanes, the 2x2 chroma from lane + 1
template <int E> static void scaled(const uint32_t* img, int out_w, int out_h, int fmt, uint8_t* dst, size_t pitch, uint8_t* cb, size_t cr) {
    const bool pairs = fmt == GLAVA_B200_EXPORT_YUVA420P;
    auto at = [&](int Y, int X) { return X < out_w ? img[(size_t) Y * out_w + X] : 0u; };
    for (int u = 0; u < (pairs ? out_h / 2 : out_h); ++u)
        for (int run = 0; run < (out_w + 31) / 32; ++run)
            for (int lane = 0; lane < 32 && run * 32 + lane < out_w; ++lane) {
                const int X = run * 32 + lane;
                if (export_straight(fmt)) {
                    const uint32_t s = export_straight_px(at(u, X));
                    put(dst + (size_t) u * pitch + 4 * (size_t) X, (fmt & 0xff) == GLAVA_B200_EXPORT_BGRA ? export_swap_rb(s) : s, 4);
                } else if (!pairs) {
                    const uint32_t px = at(u, X), s = export_straight_px(px), uv = export_cbcr10_px<E>(s);
                    const size_t o = (size_t) u * pitch + 2 * (size_t) X;
                    put(dst + o, export_y10<E>(s), 2); put(cb + o, uv, 2); put(cb + cr + o, uv >> 16, 2);
                    put(cb + 2 * cr + o, export_a10(px >> 24), 2);
                } else {
                    const uint32_t top = at(2 * u, X), bot = at(2 * u + 1, X);
                    const size_t o = (size_t) (2 * u) * pitch + X;
                    put(dst + o, export_y<E>(export_straight_px(top)), 1); put(dst + o + pitch, export_y<E>(export_straight_px(bot)), 1);
                    put(cb + 2 * cr + o, top >> 24, 1); put(cb + 2 * cr + o + pitch, bot >> 24, 1);
                    if (!(lane & 1)) {
                        const uint32_t uv = export_cbcr<E>(export_block_straight(top, at(2 * u, X + 1), bot, at(2 * u + 1, X + 1)));
                        uint8_t* pu = cb + (size_t) u * (pitch / 2) + X / 2;
                        put(pu, uv, 1); put(pu + cr, uv >> 8, 1);
                    }
                }
            }
}
template <int E> static void zero(int fmt, int over, int native, uint32_t bg, uint32_t* out) {
    const ExportFmt f = { fmt, over, native, bg };
    const ExportZeroA z = export_zero_alpha<E>(f);
    out[0] = z.y; out[1] = z.u; out[2] = z.v; out[3] = z.a;
}
// Y'CbCr of the straight colour against float64 of the exact one (c 255 / a), over every grey and a fixed sample of
// premultiplied colours: err[0..2] the largest |code - float| of Y, Cb, Cr at `bits` (10: YUVA444P10, 8: YUVA420P's Y and
// the chroma of a block of four equal pixels)
template <int E> static void bounds(int bits, double* err) {
    const double kr = E & 2 ? 0.299 : 0.2126, kb = E & 2 ? 0.114 : 0.0722, kg = 1 - kr - kb;
    const bool full = E & 1;
    const double top = bits == 10 ? 1023 : 255, ys = full ? top / 255 : (bits == 10 ? 876.0 : 219.0) / 255;
    const double cs = full ? top / 255 : (bits == 10 ? 896.0 : 224.0) / 255, yoff = full ? 0 : bits == 10 ? 64 : 16, coff = bits == 10 ? 512 : 128;
    uint64_t st = 0x9e3779b97f4a7c15ull;
    auto rnd = [&]() { st ^= st << 13; st ^= st >> 7; st ^= st << 17; return (uint32_t) st; };
    err[0] = err[1] = err[2] = 0;
    for (long i = 0; i < (1L << 22) + 256 * 256; ++i) {
        uint32_t a, c[3];
        if (i < 256 * 256) { a = (uint32_t) (i >> 8); c[0] = c[1] = c[2] = (uint32_t) (i & 255) > a ? a : (uint32_t) (i & 255); }
        else { a = 1 + rnd() % 255; for (int k = 0; k < 3; ++k) c[k] = rnd() % (a + 1); }
        if (!a) continue;
        const uint32_t px = c[0] | (c[1] << 8) | (c[2] << 16) | (a << 24);
        uint32_t yv, cbv, crv;
        if (bits == 10) {
            const ExportFmt f = { GLAVA_B200_EXPORT_YUVA444P10, 0, 1, 0u };
            const uint32_t q[4] = { px, px, px, px };
            uint32_t y[2], u[2], v[2], al[2];
            export_yuva444p10_quad<E>(f, q, y, u, v, al);
            yv = y[0] & 0xffffu; cbv = u[0] & 0xffffu; crv = v[0] & 0xffffu;
        } else {
            const ExportFmt f = { GLAVA_B200_EXPORT_YUVA420P, 0, 1, 0u };
            const uint32_t q[4] = { px, px, px, px };
            uint32_t yt, yb, u, v, at, ab;
            export_yuva420_quad<E>(f, q, q, &yt, &yb, &u, &v, &at, &ab);
            yv = yt & 255u; cbv = u & 255u; crv = v & 255u;
        }
        const double r = c[0] * 255.0 / a, g = c[1] * 255.0 / a, b = c[2] * 255.0 / a, yp = kr * r + kg * g + kb * b;
        double fy = yoff + ys * yp, fcb = coff + cs * (b - yp) / (2 * (1 - kb)), fcr = coff + cs * (r - yp) / (2 * (1 - kr));
        fy = fy > top ? top : fy; fcb = fcb > top ? top : fcb; fcr = fcr > top ? top : fcr;
        const double d[3] = { std::fabs(yv - fy), std::fabs(cbv - fcb), std::fabs(crv - fcr) };
        for (int k = 0; k < 3; ++k) err[k] = d[k] > err[k] ? d[k] : err[k];
    }
}
extern "C" void t_walk(int e, const uint32_t* fb, int w, int h, const uint32_t* marks, int rows, int fmt, int over, int native,
                       uint32_t bg, uint8_t* dst, size_t pitch, uint8_t* cb, size_t cr) {
    DISPATCH(walk, fb, w, h, marks, rows, fmt, over, native, bg, dst, pitch, cb, cr)
}
extern "C" void t_scaled_walk(int e, const uint32_t* img, int out_w, int out_h, int fmt, uint8_t* dst, size_t pitch, uint8_t* cb, size_t cr) {
    DISPATCH(scaled, img, out_w, out_h, fmt, dst, pitch, cb, cr)
}
extern "C" void t_zero(int e, int fmt, int over, int native, uint32_t bg, uint32_t* out) { DISPATCH(zero, fmt, over, native, bg, out) }
extern "C" void t_bounds(int e, int bits, double* err) { DISPATCH(bounds, bits, err) }
extern "C" void t_predicates(int format, size_t pitch, int h, long long* out) {
    out[0] = export_yuva(format); out[1] = export_alpha(format); out[2] = export_ycbcr(format); out[3] = export_chroma_planes(format);
    out[4] = export_420(format); out[5] = export_planar(format); out[6] = (long long) export_planes(format, pitch, 0, h).plane;
    out[7] = export_straight(format); out[8] = export_yuv(format) || export_p10(format) || export_422(format);
}
extern "C" int t_kernel_format(int format, uint32_t flags) { return export_kernel_format(format, flags); }
extern "C" int t_ladder_kernel(const int* format, const int* enc, int n) { return ladder_kernel(format, enc, n); }
"""


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("export_alpha_core")
    src, so = d / "shim.cpp", d / "shim.so"
    src.write_text(SHIM)
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I", CSRC,
                    "-include", "cstring", "-include", "cmath", "-o", str(so), str(src)], check=True)
    L = C.CDLL(str(so))
    vp, sz, i32, u32 = C.c_void_p, C.c_size_t, C.c_int, C.c_uint32
    L.t_pairs.argtypes = [vp, vp]
    L.t_px.argtypes = [vp, sz, vp]
    L.t_a10.argtypes = [vp]
    L.t_block.argtypes = [vp, sz, vp, vp]
    L.t_walk.argtypes = [i32, vp, i32, i32, vp, i32, i32, i32, i32, u32, vp, sz, vp, sz]
    L.t_scaled_walk.argtypes = [i32, vp, i32, i32, i32, vp, sz, vp, sz]
    L.t_zero.argtypes = [i32, i32, i32, i32, u32, vp]
    L.t_bounds.argtypes = [i32, i32, vp]
    L.t_predicates.argtypes = [i32, sz, i32, vp]
    L.t_kernel_format.argtypes = [i32, u32]
    L.t_ladder_kernel.argtypes = [vp, vp, i32]
    return L


def words(c):
    """[..., 4] ints -> uint32 pixel words"""
    c = np.asarray(c, np.int64)
    return np.ascontiguousarray(pack(c[..., 0], c[..., 1], c[..., 2], c[..., 3]), np.uint32)


def channels(wd):
    wd = np.asarray(wd, np.uint32)
    return np.stack([(wd >> (8 * k)) & 255 for k in range(4)], axis=-1).astype(np.int64)


# ---- arithmetic -------------------------------------------------------------------------------------------------------------
def test_unpremultiply_every_pair(shim):
    """all 65536 (c, a): the integer formula; within 0.5 of c 255 / a where c <= a; mul_norm8(S, a) == c where c <= a"""
    s, m = np.zeros(65536, np.uint32), np.zeros(65536, np.uint32)
    shim.t_pairs(s.ctypes.data, m.ctypes.data)
    a, c = np.divmod(np.arange(65536, dtype=np.int64), 256)
    s, m = s.astype(np.int64), m.astype(np.int64)
    assert np.array_equal(s, unpremul_np(c, a))
    ok = (c <= a) & (a > 0)
    assert np.abs(s[ok] - c[ok] * 255.0 / a[ok]).max() <= 0.5
    assert np.array_equal(m[ok], c[ok]), "re-premultiplying the straight colour gives the stored pixel back"
    # mul_norm8 restated: round(S a / 255) half up
    assert np.array_equal(m, (2 * s * a + 255) // 510)
    assert (s[a == 0] == 0).all() and (s[(c > a)] == np.where(a[c > a] == 0, 0, 255)).all()


def test_straight_pixels_and_alpha_codes(shim):
    rng = np.random.default_rng(3)
    c = rng.integers(0, 256, (50000, 4))
    c[:1000, 3] = 255
    c[1000:2000] = 0
    c[2000:3000, 3] = 0
    px = words(c)
    out = np.zeros_like(px)
    shim.t_px(px.ctypes.data, px.size, out.ctypes.data)
    want = c.copy()
    want[..., :3] = unpremul_np(c[..., :3], c[..., 3:4])
    assert np.array_equal(channels(out), want)
    a10 = np.zeros(256, np.uint32)
    shim.t_a10(a10.ctypes.data)
    a = np.arange(256)
    assert np.array_equal(a10, a10_np(a)) and a10[0] == 0 and a10[255] == 1023
    assert np.abs(a10 - a * 1023 / 255).max() < 0.495
    assert ((a * 1023 * 2) % 510 != 255).all(), "no ties"


def test_block_chroma(shim):
    """the alpha-weighted block colour on random blocks, zero-alpha blocks, one opaque pixel, c > a, and all opaque (= avg4)"""
    rng = np.random.default_rng(5)
    blocks = [premultiplied(rng, (20000, 4)).astype(np.int64)]
    z = premultiplied(rng, (500, 4)).astype(np.int64)
    z[..., 3] = 0
    blocks.append(z)                                                   # sum a = 0 (graph pixels may keep colour)
    one = np.zeros((500, 4, 4), np.int64)
    one[:, 0] = rng.integers(0, 256, (500, 4))
    one[:, 0, 3] = 255
    blocks.append(one)                                                 # one opaque pixel: its colour
    blocks.append(rng.integers(0, 256, (5000, 4, 4)))                  # c > a
    op = rng.integers(0, 256, (5000, 4, 4))
    op[..., 3] = 255
    blocks.append(op)
    b = np.concatenate(blocks)
    px = words(b)
    out, avg = np.zeros(len(b), np.uint32), np.zeros(len(b), np.uint32)
    shim.t_block(px.ctypes.data, len(b), out.ctypes.data, avg.ctypes.data)
    img = b.reshape(len(b), 2, 2, 4).transpose(1, 0, 2, 3).reshape(2, 2 * len(b), 4)   # block i: columns 2i, 2i + 1
    want = block_straight_np(img)
    got = channels(out)[..., :3]
    assert np.array_equal(got, want[0]), "alpha-weighted block colour"
    assert (got[20000:20500] == 0).all()
    assert np.array_equal(got[20500:21000], one[:, 0, :3])
    n = len(b) - 5000
    assert np.array_equal(out[n:], avg[n:]), "four opaque pixels: export_avg4"


@pytest.mark.parametrize("bits", [8, 10])
@pytest.mark.parametrize("e", [0, 1, 2, 3], ids=[ENCODINGS[e] for e in range(4)])
def test_bounds_against_float64_of_the_exact_straight_colour(shim, e, bits):
    err = np.zeros(3)
    shim.t_bounds(e, bits, err.ctypes.data)
    assert (err <= np.array(BOUND[e, bits])).all(), (ENCODINGS[e], bits, err)
    assert (err > np.array(BOUND[e, bits]) - 0.0002).all(), err        # the maxima DESIGN 4.19 records, to 4 places


# ---- the kernels' walks into sentinel buffers ------------------------------------------------------------------------------------
def layout(fmt, w, h, pad, gap=64):
    """(pitch, Cb offset, Cb to Cr distance, total) of a sentinel buffer: `pad` bytes past every row, `gap` past each plane"""
    if fmt in (RGBA_S, BGRA_S):
        pitch = (4 * w + pad + 15) // 16 * 16
        return pitch, 0, 0, pitch * h + gap
    row = 2 * w if fmt == YUVA444P10 else w
    pitch = (row + pad + 31) // 32 * 32
    cb_off = pitch * h + gap
    cr = ((pitch // 2) * (h // 2) if fmt == YUVA420P else pitch * h) + gap
    return pitch, cb_off, cr, cb_off + 2 * cr + pitch * h + gap


def planes_of(buf, fmt, w, h, pitch, cb_off, cr):
    written = np.zeros(buf.size, bool)

    def plane(off, rows, p, nbytes, dt):
        idx = off + np.arange(rows)[:, None] * p + np.arange(nbytes)[None, :]
        written[idx] = True
        return np.ascontiguousarray(buf[idx]).view(dt)

    if fmt in (RGBA_S, BGRA_S):
        return plane(0, h, pitch, 4 * w, np.uint8).reshape(h, w, 4), written
    if fmt == YUVA444P10:
        return tuple(plane(o, h, pitch, 2 * w, np.uint16) for o in (0, cb_off, cb_off + cr, cb_off + 2 * cr)), written
    return (plane(0, h, pitch, w, np.uint8), plane(cb_off, h // 2, pitch // 2, w // 2, np.uint8),
            plane(cb_off + cr, h // 2, pitch // 2, w // 2, np.uint8), plane(cb_off + 2 * cr, h, pitch, w, np.uint8)), written


def walk(L, frame, fmt, e, bg=(0, 0, 0), native=True, marks=None, rows=0, pad=32):
    h, w = frame.shape[:2]
    pitch, cb_off, cr, total = layout(fmt, w, h, pad)
    buf = np.full(total, SENTINEL, np.uint8)
    fb = np.ascontiguousarray(frame).view(np.uint32).reshape(h, w)
    m = None if marks is None else np.ascontiguousarray(marks, np.uint32)
    L.t_walk(e, fb.ctypes.data, w, h, None if m is None else m.ctypes.data, rows, fmt, int(not native), int(native),
             int(pack(*bg[:3])), buf.ctypes.data, pitch, buf.ctypes.data + cb_off, cr)
    planes, written = planes_of(buf, fmt, w, h, pitch, cb_off, cr)
    assert (buf[~written] == SENTINEL).all(), "written outside the planes"
    return planes


def scaled_img(frame, size, crop, native, bg):
    h, w = frame.shape[:2]
    x, y, cw, ch = crop or (0, 0, w, h)
    img = frame[::-1][y:y + ch, x:x + cw].astype(np.int64)
    return area_np(img if native else over_np(img, bg, False), size)


def scaled(L, img, fmt, e, pad=48):
    oh, ow = img.shape[:2]
    pitch, cb_off, cr, total = layout(fmt, ow, oh, pad)
    buf = np.full(total, SENTINEL, np.uint8)
    px = words(img)
    L.t_scaled_walk(e, px.ctypes.data, ow, oh, fmt, buf.ctypes.data, pitch, buf.ctypes.data + cb_off, cr)
    planes, written = planes_of(buf, fmt, ow, oh, pitch, cb_off, cr)
    assert (buf[~written] == SENTINEL).all(), "written outside the planes"
    return planes


def np_name(fmt):
    return {RGBA_S: "rgba", BGRA_S: "bgra", YUVA420P: "yuva420p", YUVA444P10: "yuva444p10"}[fmt]


def same(a, b):
    if isinstance(b, tuple):
        return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))
    return np.array_equal(a, b)


def graph_like(rng, h, w):
    """premultiplied pixels, some zero rows, and unassociated ones (c > a) as Graph stores them"""
    f = premultiplied(rng, (h, w))
    f[: h // 3] = 0
    f[h // 2, ::3] = rng.integers(0, 256, (len(range(0, w, 3)), 4))
    return f


@pytest.mark.parametrize("w,h", [(128, 64), (130, 32), (66, 10), (2, 2), (390, 8), (98, 34), (6, 4), (258, 2), (134, 6)])
@pytest.mark.parametrize("fmt,e", FMT_E)
def test_walk_equals_the_restatement(shim, w, h, fmt, e):
    rng = np.random.default_rng(w * 1000 + h + fmt + 10 * e)
    for native in (True, False):
        frame = graph_like(rng, h, w)
        bg = (17, 240, 66)
        assert same(walk(shim, frame, fmt, e, bg, native), frame_alpha_np(frame, np_name(fmt), e, native)), native
    if fmt != YUVA420P:                                                 # odd heights and widths
        frame = graph_like(rng, h + 1, w + 1)
        assert same(walk(shim, frame, fmt, e), frame_alpha_np(frame, np_name(fmt), e))


@pytest.mark.parametrize("w,h,rows", [(256, 40, 8), (300, 34, 5), (128, 64, 64), (134, 18, 1), (64, 30, 540), (302, 34, 7)])
@pytest.mark.parametrize("fmt", [YUVA420P, YUVA444P10, RGBA_S])
def test_marks_skip_rows_without_reading_them(shim, w, h, rows, fmt):
    rows = min(rows, h)
    rng = np.random.default_rng(w * h + rows + fmt)
    for garbage in (False, True):
        frame, clean, marks = marked_frame(rng, w, h, rows, garbage)
        for e in ((0, 3) if fmt != RGBA_S else (0,)):
            aware = walk(shim, frame, fmt, e, (40, 50, 60), marks=marks, rows=rows)
            assert same(aware, frame_alpha_np(clean, np_name(fmt), e)), (garbage, e)


@pytest.mark.parametrize("e", [0, 1, 2, 3])
def test_zero_constants_are_transparent_black(shim, e):
    out = (C.c_uint32 * 4)()
    y0 = 0 if e & 1 else 16
    shim.t_zero(e, YUVA420P, 0, 1, 0x4280f0, out)
    assert list(out) == [y0 * 0x01010101, 128 * 0x0101, 128 * 0x0101, 0]
    shim.t_zero(e, YUVA444P10, 0, 1, 0x4280f0, out)
    assert list(out) == [(4 * y0) * 0x10001, 512 * 0x10001, 512 * 0x10001, 0]
    shim.t_zero(e, YUVA420P, 1, 0, 0x4280f0, out)                     # any other opacity: opaque black
    assert list(out) == [y0 * 0x01010101, 128 * 0x0101, 128 * 0x0101, 0xffffffff]
    shim.t_zero(0, RGBA_S, 0, 1, 0x4280f0, out)
    assert out[0] == 0
    shim.t_zero(0, BGRA_S, 1, 0, 0x4280f0, out)
    assert out[0] == 0xff000000


@pytest.mark.parametrize("fmt,e", FMT_E)
def test_scaled_walk_is_the_format_on_the_scaled_image(shim, fmt, e):
    rng = np.random.default_rng(60 + e + fmt)
    w, h = 300, 170
    frame = graph_like(rng, h, w)
    bg = (30, 60, 200)
    sizes = [((100, 56), None), ((64, 32), (10, 20, 200, 100)), ((34, 18), None), ((2, 2), None), ((38, 8), (3, 5, 101, 47))]
    if fmt != YUVA420P:
        sizes += [((37, 9), None), ((1, 1), None)]
    for native in (True, False):
        for size, crop in sizes:
            img = scaled_img(frame, size, crop, native, bg)
            assert same(scaled(shim, img, fmt, e), scaled_alpha_np(frame, np_name(fmt), size, crop, e, native, bg)), (size, crop)
    # the whole frame at its own size is the whole-frame walk
    assert same(scaled(shim, scaled_img(frame, (w, h), None, True, bg), fmt, e), walk(shim, frame, fmt, e, bg))


# ---- identities --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("e", [0, 1, 2, 3])
def test_identities_with_the_opaque_exports(shim, e):
    """any other opacity than native: YUVA420P is I420 with A = 255, YUVA444P10 is YUV444P10 with A = 1023, straight RGBA
    is EXPORT_OVER's RGBA; an all-opaque frame under native opacity gives the same"""
    from tests.export_422_np import _coder
    rng = np.random.default_rng(90 + e)
    bg = (9, 99, 199)
    for frame, native in ((premultiplied(rng, (10, 130)), False), (rng.integers(0, 256, (6, 66, 4), dtype=np.uint8), False)):
        opaque = rng.integers(0, 256, frame.shape, dtype=np.uint8)
        opaque[..., 3] = 255
        for f, nat in ((frame, native), (opaque, True)):
            comp = over_np(f[::-1], bg, nat)
            y, cb, cr, a = walk(shim, f, YUVA444P10, e, bg, nat)
            assert same((y, cb, cr), p10_np(comp, "yuv444p10", e)) and (a == 1023).all()
            y, cb, cr, a = walk(shim, f, YUVA420P, e, bg, nat)
            ky, kcb, kcr, yoff, coff, code, dot = _coder(e, 8)
            hh, ww = comp.shape[:2]
            avg = (comp[..., :3].reshape(hh // 2, 2, ww // 2, 2, 3).sum(axis=(1, 3)) + 2) >> 2
            assert np.array_equal(y, code(dot(ky, comp) + (yoff << 16) + (1 << 15), 16))
            assert np.array_equal(cb, code(dot(kcb, avg) + (coff << 16) + (1 << 15), 16))
            assert np.array_equal(cr, code(dot(kcr, avg) + (coff << 16) + (1 << 15), 16)) and (a == 255).all()
            if e == 0:
                assert np.array_equal(walk(shim, f, RGBA_S, 0, bg, nat), comp.astype(np.uint8))


# ---- refusals, byte counts and launches through the fake runtime --------------------------------------------------------------------
def test_predicates_and_kernel_choice(shim):
    out = (C.c_longlong * 9)()
    for fmt, want_ in ((YUVA420P, [1, 1, 1, 1, 1, 1, 64 * 8, 0, 0]), (YUVA444P10, [1, 1, 1, 1, 0, 1, 128 * 16, 0, 0]),
                       (RGBA_S, [0, 1, 0, 0, 0, 0, 0, 1, 0]), (BGRA_S, [0, 1, 0, 0, 0, 0, 0, 1, 0]), (RGBA, [0] * 9)):
        shim.t_predicates(fmt, 128, 16, out)
        assert list(out) == want_, (fmt, list(out))
    assert shim.t_kernel_format(RGBA, STRAIGHT) == RGBA_S and shim.t_kernel_format(BGRA, STRAIGHT) == BGRA_S
    assert shim.t_kernel_format(YUVA420P, 0x300) == YUVA420P and shim.t_kernel_format(RGBA, OVER) == RGBA
    pick = lambda f, e: shim.t_ladder_kernel((C.c_int * len(f))(*f), (C.c_int * len(e))(*e), len(f))
    assert pick([NV12, RGBA], [0, 0]) == 0 and pick([I420, NV12], [0, 0]) == 1 and pick([NV12], [1]) == 2
    assert pick([YUV444P10], [0]) == 3 and pick([10, NV12], [0, 0]) == 4
    for f in ([YUVA420P], [NV12, YUVA444P10], [RGBA_S], [10, BGRA_S, YUV444P10], [YUVA420P, NV12, 12]):
        assert pick(f, [0] * len(f)) == 5 and pick(f, [3] * len(f)) == 5, f


def test_refusals_byte_counts_and_launches(fake):
    L = fake
    L.fake_fail_at(-1)
    r, odd_h, odd_w = renderer(L, 64, 32), renderer(L, 66, 33), renderer(L, 63, 32)
    buf, buf2 = device_buf(L), device_buf(L)
    s = np.zeros(1, np.int32)
    one, uv = (C.c_void_p * 1)(buf.value), (C.c_void_p * 1)(buf2.value)

    def frames(h, d):
        return call(L, L.glava_b200_export_frames, h, s.ctypes.data, 1, one, C.byref(d), None, None)

    def scaled_call(h, d, size, dst_uv=None):
        return call(L, L.glava_b200_export_scaled, h, s.ctypes.data, 1, one, dst_uv, C.byref(d), C.byref(scale_of(size)), None, None)

    taken = [(r, YUVA420P, 64, 0, 0), (r, YUVA444P10, 128, 0, 0), (r, YUVA420P, 96, 48 * 16 + 16, 0x300),
             (r, YUVA444P10, 128, 128 * 40, 0x100), (odd_h, YUVA444P10, 144, 0, 0x200), (odd_w, RGBA, 256, 0, STRAIGHT),
             (odd_h, BGRA, 272, 0, STRAIGHT)]
    for h, fmt, pitch, uvo, flags in taken:
        rc, msg, trace, launched = frames(h, desc_of(fmt, pitch, flags, uv=uvo))
        assert rc == 0 and launched == 1 and len(memcpys(trace)) == 1, (fmt, pitch, flags, msg)
    refused = [  # (renderer, desc, what)
        (r, desc_of(RGBA, 256, STRAIGHT | OVER), "EXPORT_STRAIGHT and EXPORT_OVER exclude each other"),
        (r, desc_of(BGRA, 256, STRAIGHT | OVER), "EXPORT_STRAIGHT and EXPORT_OVER exclude each other"),
        (r, desc_of(NV12, 64, STRAIGHT), "EXPORT_STRAIGHT is for RGBA and BGRA, not NV12"),
        (r, desc_of(I420, 64, STRAIGHT), "EXPORT_STRAIGHT is for RGBA and BGRA, not I420"),
        (r, desc_of(YUVA420P, 64, STRAIGHT), "EXPORT_STRAIGHT is for RGBA and BGRA, not YUVA420P"),
        (r, desc_of(YUVA444P10, 128, STRAIGHT), "not YUVA444P10"),
        (r, desc_of(YUVA420P, 64, OVER), "YUVA420P is never composited"),
        (r, desc_of(YUVA444P10, 128, OVER), "YUVA444P10 is never composited"),
        (odd_h, desc_of(YUVA420P, 96), "YUVA420P needs an even width and height, the frame is 66x33"),
        (odd_w, desc_of(YUVA420P, 64), "YUVA420P needs an even width and height, the frame is 63x32"),
        (r, desc_of(YUVA420P, 80), "YUVA420P pitch 80 must be a multiple of 32"),
        (r, desc_of(YUVA420P, 32), "at least 64"),
        (r, desc_of(YUVA444P10, 112), "at least 128"),
        (r, desc_of(YUVA444P10, 136), "multiple of 16"),
        (r, desc_of(YUVA420P, 64, uv=8), "YUVA420P uv_offset 8 (Cb plane to Cr plane)"),
        (r, desc_of(YUVA420P, 64, uv=32 * 15), "one chroma plane, 512 bytes"),
        (r, desc_of(YUVA444P10, 128, uv=128 * 32 - 16), "one chroma plane, 4096 bytes"),
        (r, desc_of(RGBA, 256, 0x2), "unknown flags 0x2"),
        (r, desc_of(RGBA, 256, 0x400 | STRAIGHT), "unknown flags 0x404"),
        (r, desc_of(13, 256), "unknown format 13"),
        (r, desc_of(16, 256), "unknown format 16"),
    ]
    for h, d, what in refused:
        rc, msg, trace, launched = frames(h, d)
        assert rc != 0 and "glava_b200_export_frames" in msg and what in msg, (what, msg)
        assert trace == "" and launched == 0, what
    # the scaled export: YUVA420P needs an even output, the others take any; dst_uv for YUVA, not for straight RGBA
    rc, msg, trace, launched = scaled_call(r, desc_of(YUVA420P, 64), (16, 7))
    assert rc != 0 and "YUVA420P needs an even width and height, the output is 16x7" in msg and launched == 0, msg
    for d, size in ((desc_of(YUVA444P10, 64), (15, 7)), (desc_of(RGBA, 64, STRAIGHT), (15, 7)), (desc_of(YUVA420P, 32), (16, 8))):
        rc, msg, _, launched = scaled_call(r, d, size)
        assert rc == 0 and launched == 1, (d.format, msg)
    rc, msg, _, launched = scaled_call(r, desc_of(YUVA444P10, 64), (16, 7), uv)
    assert rc == 0 and launched == 1, msg
    rc, msg, trace, launched = scaled_call(r, desc_of(BGRA, 64, STRAIGHT), (16, 7), uv)
    assert rc != 0 and "BGRA has no chroma plane" in msg and trace == "" and launched == 0, msg
    rc, msg, trace, launched = scaled_call(r, desc_of(RGBA, 64, STRAIGHT | OVER), (16, 8))
    assert rc != 0 and "glava_b200_export_scaled" in msg and "exclude each other" in msg and launched == 0, msg
    # the overlay refuses the new formats and the flag by name
    for fmt, name in ((YUVA420P, "YUVA420P"), (YUVA444P10, "YUVA444P10")):
        rc, msg, trace, launched = call(L, L.glava_b200_overlay_frames, r, s.ctypes.data, 1, one, None,
                                        C.byref(desc_of(fmt, 128)), None, None)
        assert rc != 0 and f"format {name}: the overlay takes RGBA, BGRA or NV12" in msg and launched == 0, msg
    rc, msg, trace, launched = call(L, L.glava_b200_overlay_frames, r, s.ctypes.data, 1, one, None,
                                    C.byref(desc_of(RGBA, 256, STRAIGHT)), None, None)
    assert rc != 0 and "EXPORT_STRAIGHT is for the exports" in msg and trace == "" and launched == 0, msg
    # ladder rungs: checked as their scaled exports; the zero A word reaches the kernel's arguments
    three = (C.c_void_p * 3)(buf.value, buf.value, buf.value)
    pairs = [(desc_of(YUVA420P, 64, 0x100), scale_of((64, 32))), (desc_of(RGBA, 64, STRAIGHT), scale_of((16, 8))),
             (desc_of(NV12, 32), scale_of((16, 8)))]
    rc, msg, _, launched = call(L, L.glava_b200_export_ladder, r, s.ctypes.data, 1, rungs_of(pairs), 3, three, None, None, None)
    assert rc == 0 and launched == 1, msg
    lad = np.zeros(5 * 8, np.int64)
    L.formats_fake_ladder(lad.ctypes.data)
    assert lad[0] == 32 * 16 and lad[1:4].tolist() == [0, 128 * 0x0101, 128 * 0x0101] and lad[4] == 0, lad[:10]
    rc, msg, _, launched = call(L, L.glava_b200_export_ladder, r, s.ctypes.data, 1,
                                rungs_of([(desc_of(YUVA420P, 64, OVER), scale_of((16, 8)))]), 1, three, None, None, None)
    assert rc != 0 and "rung 0" in msg and "never composited" in msg and launched == 0, msg
    rc, msg, _, launched = call(L, L.glava_b200_export_ladder, r, s.ctypes.data, 1, rungs_of(pairs), 3, three,
                                (C.c_void_p * 3)(buf2.value, buf2.value, None), None, None)
    assert rc != 0 and "rung 1: dst_uv[1] is for NV12 only" in msg and launched == 0, msg
    # byte counts: pitch * h + twice the Cb to Cr distance + pitch * h
    n = C.c_size_t()
    for d, want_ in ((desc_of(YUVA420P, 64), 64 * 32 + 2 * 32 * 16 + 64 * 32), (desc_of(YUVA420P, 64, uv=4096), 64 * 32 * 2 + 2 * 4096),
                     (desc_of(YUVA444P10, 128), 4 * 128 * 32), (desc_of(RGBA, 256, STRAIGHT), 256 * 32)):
        assert L.glava_b200_export_bytes(r, C.byref(d), C.byref(n)) == 0 and n.value == want_, (d.format, n.value, want_)
    assert L.glava_b200_export_scaled_bytes(r, C.byref(desc_of(YUVA444P10, 64)), C.byref(scale_of((16, 7))), C.byref(n)) == 0
    assert n.value == 4 * 64 * 7
    assert L.glava_b200_export_bytes(r, C.byref(desc_of(YUVA420P, 64, OVER)), C.byref(n)) != 0
    for h in (r, odd_h, odd_w):
        L.glava_b200_destroy(h)
    L.cudaFree(buf); L.cudaFree(buf2)
