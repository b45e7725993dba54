"""Planar 10-bit export, YUV420P10 and YUV444P10 (DESIGN 4.16), on the host: the per-pixel 4:4:4 chroma of export_core.h over
every colour and encoding (equal to P010's chroma of a 2x2 block of the pixel, within the float64 bounds of DESIGN 4.15), a
host walk of export_p10_kernel's and export_scaled_p10_kernel's loops checked bit for bit against a numpy restatement
with sentinel bytes around and between every plane, the identities with P010, and the refusals and enqueued work of the
export calls through capi.cu, export.cpp and export_ladder.cpp built against tests/fakecuda's runtime."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from tests.export_fake import desc_of
from tests.test_export_core import CSRC, marked_frame, over_np, pack, premultiplied
from tests.test_export_formats_core import call, device_buf, memcpys, renderer
from tests.test_export_formats_core import fake  # noqa: F401 (the fake-runtime fixture)
from tests.test_export_ladder_core import rungs_of, scale_of
from tests.test_export_matrix_core import BOUND, ENCODINGS, coef_py, float_codes
from tests.test_export_scaled_core import SHIM as SCALED_SHIM
from tests.test_export_scaled_core import area_np

RGBA, NV12, I420, YUV444, P010, YUV420P10, YUV444P10 = 0, 2, 4, 5, 6, 7, 8
NAMES = {YUV420P10: "yuv420p10", YUV444P10: "yuv444p10"}
SENTINEL = 0xA5

# t_scaled (test_export_scaled_core) is export_scaled_kernel's walk; its RGBA leg with EXPORT_OVER gives scaled_px, the
# 8-bit scaled image the planar 10-bit items convert
SHIM = SCALED_SHIM + r"""
template <int E> static void px(const uint32_t* c, size_t n, uint16_t* y, uint16_t* cb, uint16_t* cr, uint16_t* bcb, uint16_t* bcr) {
    for (size_t i = 0; i < n; ++i) {
        const uint32_t uv = export_cbcr10_px<E>(c[i]), blk = export_cbcr10<E>(export_sum4(c[i], c[i], c[i], c[i]));
        y[i] = (uint16_t) export_y10<E>(c[i]); cb[i] = uv & 0xffffu; cr[i] = uv >> 16; bcb[i] = blk & 0xffffu; bcr[i] = blk >> 16;
    }
}
static void put(uint8_t* p, const uint32_t* v, int n) {       // the first n uint16 samples of the words v[]
    for (int k = 0; k < n; ++k) { const uint16_t s = (uint16_t) (v[k >> 1] >> (16 * (k & 1))); memcpy(p + 2 * k, &s, 2); }
}
// one slot [h][w] -> the planes, as export_p10_kernel walks it (p10_item): row pairs, 128-pixel strips, a quad per lane
template <int E> static void walk(const uint32_t* fb, int w, int h, const uint32_t* marks, int rows, int format, int native,
                                  uint32_t bg, uint8_t* dst, size_t pitch, uint8_t* cb, size_t cr) {
    const ExportFmt f = { format, 1, native, bg };
    const ExportZero z = export_zero10<E>(f);
    const int strips = (w + 127) >> 7;
    for (int j = 0; j < (h + 1) / 2; ++j)
        for (int strip = 0; strip < strips; ++strip)
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
                const size_t o = (size_t) (2 * j) * pitch + 2 * (size_t) x;
                if (format == GLAVA_B200_EXPORT_YUV444P10) {
                    for (int r = 0; r < 2 && (r == 0 || y1 >= 0); ++r) {
                        uint32_t y[2] = { z.y, z.y }, u[2] = { z.u, z.u }, v[2] = { z.v, z.v };
                        if (q[r][0] | q[r][1] | q[r][2] | q[r][3]) export_444p10_quad<E>(f, q[r], y, u, v);
                        put(dst + o + r * pitch, y, n); put(cb + o + r * pitch, u, n); put(cb + cr + o + r * pitch, v, n);
                    }
                } else {
                    uint32_t yt[2] = { z.y, z.y }, yb[2] = { z.y, z.y }, u = z.u, v = z.v;
                    if (q[0][0] | q[0][1] | q[0][2] | q[0][3] | q[1][0] | q[1][1] | q[1][2] | q[1][3]) export_i010_quad<E>(f, q[0], q[1], yt, yb, &u, &v);
                    put(dst + o, yt, n); put(dst + o + pitch, yb, n);
                    uint8_t* pu = cb + (size_t) j * (pitch / 2) + x;
                    put(pu, &u, n / 2); put(pu + cr, &v, n / 2);
                }
            }
}
// the scaled image img [out_h][out_w] (scaled_px of each output pixel) -> the planes, as export_scaled_p10_kernel walks it
// (scaled_p10_item): units of one output row (YUV420P10: a row pair), runs of 32 lanes, the 2x2 chroma from lane + 1
template <int E> static void scaled(const uint32_t* img, int out_w, int out_h, int format, uint8_t* dst, size_t pitch, uint8_t* cb, size_t cr) {
    const bool pairs = format == GLAVA_B200_EXPORT_YUV420P10;
    const int units = pairs ? out_h / 2 : out_h, runs = (out_w + 31) / 32;
    auto at = [&](int Y, int X) { return X < out_w ? img[(size_t) Y * out_w + X] : 0u; };
    auto put1 = [](uint8_t* p, uint32_t v) { const uint16_t s = (uint16_t) v; memcpy(p, &s, 2); };
    for (int u = 0; u < units; ++u)
        for (int run = 0; run < runs; ++run)
            for (int lane = 0; lane < 32 && run * 32 + lane < out_w; ++lane) {
                const int X = run * 32 + lane;
                if (!pairs) {
                    const uint32_t c = at(u, X), uv = export_cbcr10_px<E>(c);
                    const size_t o = (size_t) u * pitch + 2 * (size_t) X;
                    put1(dst + o, export_y10<E>(c)); put1(cb + o, uv); put1(cb + cr + o, uv >> 16);
                    continue;
                }
                const uint32_t top = at(2 * u, X), bot = at(2 * u + 1, X);
                put1(dst + (size_t) (2 * u) * pitch + 2 * X, export_y10<E>(top));
                put1(dst + (size_t) (2 * u + 1) * pitch + 2 * X, export_y10<E>(bot));
                if (!(lane & 1)) {
                    const uint32_t uv = export_cbcr10<E>(export_sum4(top, at(2 * u, X + 1), bot, at(2 * u + 1, X + 1)));
                    uint8_t* pu = cb + (size_t) u * (pitch / 2) + X;
                    put1(pu, uv); put1(pu + cr, uv >> 16);
                }
            }
}
template <int E> static void zero10(int format, int native, uint32_t bg, uint32_t* out) {
    const ExportFmt f = { format, 1, native, bg };
    const ExportZero z = export_zero10<E>(f);
    out[0] = z.y; out[1] = z.u; out[2] = z.v;
}
#define DISPATCH(fn, ...) switch (e) { case 1: fn<1>(__VA_ARGS__); break; case 2: fn<2>(__VA_ARGS__); break; \
                                       case 3: fn<3>(__VA_ARGS__); break; default: fn<0>(__VA_ARGS__); }
extern "C" void t_p10_px(int e, const uint32_t* c, size_t n, uint16_t* y, uint16_t* cb, uint16_t* cr, uint16_t* bcb, uint16_t* bcr) {
    DISPATCH(px, c, n, y, cb, cr, bcb, bcr)
}
extern "C" void t_p10_walk(int e, const uint32_t* fb, int w, int h, const uint32_t* marks, int rows, int format, int native,
                           uint32_t bg, uint8_t* dst, size_t pitch, uint8_t* cb, size_t cr) {
    DISPATCH(walk, fb, w, h, marks, rows, format, native, bg, dst, pitch, cb, cr)
}
extern "C" void t_p10_scaled(int e, const uint32_t* img, int out_w, int out_h, int format, uint8_t* dst, size_t pitch, uint8_t* cb, size_t cr) {
    DISPATCH(scaled, img, out_w, out_h, format, dst, pitch, cb, cr)
}
extern "C" void t_p10_zero(int e, int format, int native, uint32_t bg, uint32_t* out) { DISPATCH(zero10, format, native, bg, out) }
// what the host checks see: export_p10 / export_ycbcr / export_420 / export_planar, and export_planes' plane
extern "C" void t_p10_predicates(int format, size_t pitch, int h, long long* out) {
    out[0] = export_yuv(format); out[1] = export_p10(format); out[2] = export_ycbcr(format); out[3] = export_420(format);
    out[4] = export_planar(format); out[5] = (long long) export_planes(format, pitch, 0, h).plane;
}
"""


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("export_p10_core")
    src, so = d / "shim.cpp", d / "shim.so"
    src.write_text(SHIM)
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I", CSRC,
                    "-include", "cstring", "-include", "algorithm", "-o", str(so), str(src)], check=True)
    L = C.CDLL(str(so))
    vp, sz, i32, u32 = C.c_void_p, C.c_size_t, C.c_int, C.c_uint32
    L.t_p10_px.argtypes = [i32, vp, sz, vp, vp, vp, vp, vp]
    L.t_p10_walk.argtypes = [i32, vp, i32, i32, vp, i32, i32, i32, u32, vp, sz, vp, sz]
    L.t_p10_scaled.argtypes = [i32, vp, i32, i32, i32, vp, sz, vp, sz]
    L.t_p10_zero.argtypes = [i32, i32, i32, u32, vp]
    L.t_p10_predicates.argtypes = [i32, sz, i32, vp]
    L.t_scaled.argtypes = [vp, i32, i32, vp, i32, i32, i32, i32, u32] + [i32] * 6 + [vp, vp, sz]
    return L


# ---- numpy restatement -------------------------------------------------------------------------------------------------------
def p10_np(c, fmt, e):
    """a composited top-down image c [h][w][>= 3] in encoding e -> (Y, Cb, Cr) uint16 planes of yuv420p10le / yuv444p10le:
    Y the 10-bit code per pixel; 4:2:0 chroma from the exact 2x2 block sums (shift 18), 4:4:4 chroma per pixel at 10 bits"""
    c = np.asarray(c, np.int64)
    h, w = c.shape[:2]
    ky, kcb, kcr, yoff, coff, top, full = coef_py(e, 10)
    code = (lambda acc, sh: np.minimum(acc >> sh, top)) if full else (lambda acc, sh: acc >> sh)
    dot = lambda k, v: k[0] * v[..., 0] + k[1] * v[..., 1] + k[2] * v[..., 2]
    y = code(dot(ky, c) + (yoff << 16) + (1 << 15), 16)
    if fmt == "yuv420p10":
        s = c[..., :3].reshape(h // 2, 2, w // 2, 2, 3).sum(axis=(1, 3))
        cb, cr = code(dot(kcb, s) + (coff << 18) + (1 << 17), 18), code(dot(kcr, s) + (coff << 18) + (1 << 17), 18)
    else:
        cb, cr = code(dot(kcb, c) + (coff << 16) + (1 << 15), 16), code(dot(kcr, c) + (coff << 16) + (1 << 15), 16)
    return y.astype(np.uint16), cb.astype(np.uint16), cr.astype(np.uint16)


def p010_np(c, e):
    """P010 of the same image: [h * 3 / 2][w] uint16, codes << 6, Y rows then interleaved (Cb, Cr) rows"""
    c = np.asarray(c, np.int64)
    h, w = c.shape[:2]
    ky, kcb, kcr, yoff, coff, top, full = coef_py(e, 10)
    code = (lambda acc, sh: np.minimum(acc >> sh, top)) if full else (lambda acc, sh: acc >> sh)
    dot = lambda k, v: k[0] * v[..., 0] + k[1] * v[..., 1] + k[2] * v[..., 2]
    y = code(dot(ky, c) + (yoff << 16) + (1 << 15), 16)
    s = c[..., :3].reshape(h // 2, 2, w // 2, 2, 3).sum(axis=(1, 3))
    cb, cr = code(dot(kcb, s) + (coff << 18) + (1 << 17), 18), code(dot(kcr, s) + (coff << 18) + (1 << 17), 18)
    return (np.concatenate([y, np.stack([cb, cr], axis=-1).reshape(h // 2, w)]) << 6).astype(np.uint16)


def planes_of(buf, fmt, w, h, pitch, cb_off, cr):
    """the three planes of a destination buffer (uint8) read with linesizes pitch and pitch / 2 (4:2:0) as ffmpeg reads
    yuv420p10le, and the mask of every byte they cover"""
    cw, ch, cp = (w // 2, h // 2, pitch // 2) if fmt == YUV420P10 else (w, h, pitch)
    written = np.zeros(buf.size, bool)

    def plane(off, nrows, p, nsamples):
        idx = off + np.arange(nrows)[:, None] * p + np.arange(2 * nsamples)[None, :]
        written[idx] = True
        return np.ascontiguousarray(buf[idx]).view(np.uint16)

    return (plane(0, h, pitch, w), plane(cb_off, ch, cp, cw), plane(cb_off + cr, ch, cp, cw)), written


def layout(fmt, w, h, pad, gap=64, uv_gap=None):
    """(pitch, Cb offset, Cb to Cr distance, total bytes) of a sentinel buffer: `pad` bytes past every row, `gap` bytes
    between planes"""
    pitch = (2 * w + pad + 31) // 32 * 32
    cp, ch = (pitch // 2, h // 2) if fmt == YUV420P10 else (pitch, h)
    cb_off = pitch * h + gap
    cr = cp * ch + (gap if uv_gap is None else uv_gap)
    return pitch, cb_off, cr, cb_off + cr + cp * ch + gap


def walk(L, frame, fmt, e, bg=(0, 0, 0), native=True, marks=None, rows=0, pad=32):
    """t_p10_walk into one sentinel buffer -> (Y, Cb, Cr), after checking that nothing outside the planes was written"""
    h, w = frame.shape[:2]
    pitch, cb_off, cr, total = layout(fmt, w, h, pad)
    buf = np.full(total, SENTINEL, np.uint8)
    fb = np.ascontiguousarray(frame).view(np.uint32).reshape(h, w)
    m = None if marks is None else np.ascontiguousarray(marks, np.uint32)
    L.t_p10_walk(e, fb.ctypes.data, w, h, None if m is None else m.ctypes.data, rows, fmt, int(native), int(pack(*bg[:3])),
                 buf.ctypes.data, pitch, buf.ctypes.data + cb_off, cr)
    planes, written = planes_of(buf, fmt, w, h, pitch, cb_off, cr)
    assert (buf[~written] == SENTINEL).all(), "written outside the planes"
    return planes


def scaled(L, frame, fmt, e, size, crop=None, bg=(0, 0, 0), native=True, marks=None, rows=0, pad=48):
    """export_scaled_kernel's walk (t_scaled, RGBA over the background: scaled_px) then t_p10_scaled, into sentinels"""
    h, w = frame.shape[:2]
    ow, oh = size
    x, y, cw, ch = crop or (0, 0, w, h)
    img = np.zeros((oh, ow * 4), np.uint8)
    fb = np.ascontiguousarray(frame).view(np.uint32).reshape(h, w)
    m = None if marks is None else np.ascontiguousarray(marks, np.uint32)
    L.t_scaled(fb.ctypes.data, w, h, None if m is None else m.ctypes.data, rows, RGBA, 1, int(native), int(pack(*bg[:3])),
               x, y, cw, ch, ow, oh, img.ctypes.data, None, ow * 4)
    pitch, cb_off, cr, total = layout(fmt, ow, oh, pad)
    buf = np.full(total, SENTINEL, np.uint8)
    L.t_p10_scaled(e, img.ctypes.data, ow, oh, fmt, buf.ctypes.data, pitch, buf.ctypes.data + cb_off, cr)
    planes, written = planes_of(buf, fmt, ow, oh, pitch, cb_off, cr)
    assert (buf[~written] == SENTINEL).all(), "written outside the planes"
    return planes


def same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


# ---- the per-pixel 4:4:4 chroma over every colour ----------------------------------------------------------------------------
@pytest.mark.parametrize("e", [0, 1, 2, 3], ids=[ENCODINGS[e] for e in range(4)])
def test_444_chroma_of_every_colour(shim, e):
    """all 2^24 colours: export_cbcr10_px is P010's chroma of the 2x2 block of that pixel, within the per-pixel 10-bit
    float64 bounds of DESIGN 4.15; greys are 512, and Y is the 10-bit code"""
    c = np.arange(1 << 24, dtype=np.uint32)
    y, cb, cr, bcb, bcr = (np.empty(c.shape, np.uint16) for _ in range(5))
    shim.t_p10_px(e, c.ctypes.data, c.size, y.ctypes.data, cb.ctypes.data, cr.ctypes.data, bcb.ctypes.data, bcr.ctypes.data)
    assert np.array_equal(cb, bcb) and np.array_equal(cr, bcr)
    del bcb, bcr
    fy, fcb, fcr = float_codes(c, e, 10)
    errs = [float(np.abs(got.astype(np.float64) - want).max()) for got, want in ((y, fy), (cb, fcb), (cr, fcr))]
    assert max(errs) <= BOUND, (ENCODINGS[e], errs)
    grey = np.arange(256, dtype=np.uint32) * 0x010101
    assert (cb[grey] == 512).all() and (cr[grey] == 512).all()
    assert y[0] == (0 if e & 1 else 64)


def test_the_restatement_is_p010_without_the_shift():
    rng = np.random.default_rng(1)
    c = rng.integers(0, 256, (6, 10, 4))
    for e in range(4):
        y, cb, cr = p10_np(c, "yuv420p10", e)
        p = p010_np(c, e)
        assert np.array_equal(y, p[:6] >> 6) and np.array_equal(cb, p[6:, 0::2] >> 6) and np.array_equal(cr, p[6:, 1::2] >> 6)
        assert np.array_equal(p10_np(c, "yuv444p10", e)[0], y)


def test_predicates_and_plane_sizes(shim):
    """the existing kernels' export_yuv does not name the new formats; the host predicates do"""
    out = (C.c_longlong * 6)()
    for fmt, want in ((YUV420P10, [0, 1, 1, 1, 1, 64 * 8]), (YUV444P10, [0, 1, 1, 0, 1, 128 * 16]),
                      (I420, [1, 0, 1, 1, 1, 64 * 8]), (P010, [1, 0, 1, 1, 0, 0]), (RGBA, [0, 0, 0, 0, 0, 0])):
        shim.t_p10_predicates(fmt, 128, 16, out)
        assert list(out) == want, (fmt, list(out))


@pytest.mark.parametrize("e", [0, 1, 2, 3])
def test_zero_quad_constants(shim, e):
    out = (C.c_uint32 * 3)()
    for bg in (0x000000, 0xffffff, 0x4280f0):
        for native in (0, 1):
            c = np.array([[[bg & 255, (bg >> 8) & 255, bg >> 16, 255]]]) if native else np.zeros((1, 1, 4), np.int64)
            y, cb, cr = (int(v[0, 0]) for v in p10_np(c, "yuv444p10", e))
            for fmt in (YUV420P10, YUV444P10):
                shim.t_p10_zero(e, fmt, native, bg, out)
                assert list(out) == [y * 0x10001, cb * 0x10001, cr * 0x10001], (fmt, bg, native)


# ---- the kernels' walks ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w,h", [(128, 64), (130, 30), (66, 10), (4, 2), (390, 8), (97, 33), (5, 3), (259, 1), (7, 4), (134, 6)])
@pytest.mark.parametrize("fmt", [YUV420P10, YUV444P10])
@pytest.mark.parametrize("e", [0, 1, 2, 3])
def test_walk_equals_the_restatement(shim, w, h, fmt, e):
    if fmt == YUV420P10 and (w | h) & 1:
        w, h = w + (w & 1), h + (h & 1)
    rng = np.random.default_rng(w * 1000 + h + fmt + 10 * e)
    for native in (True, False):
        frame = premultiplied(rng, (h, w)) if native else rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
        frame[: h // 3] = 0                                            # zero quads take the constants
        bg = (17, 240, 66)
        assert same(walk(shim, frame, fmt, e, bg, native), p10_np(over_np(frame[::-1], bg, native), NAMES[fmt], e)), native


def test_tails_cover_every_width_residue(shim):
    """w % 4 == 2 for YUV420P10 (the last two pixels of a row) and every w % 4 for YUV444P10 (sample by sample)"""
    rng = np.random.default_rng(3)
    for fmt, widths in ((YUV420P10, (2, 6, 130, 258)), (YUV444P10, (1, 2, 3, 5, 129, 130, 131))):
        for w in widths:
            frame = rng.integers(0, 256, (4, w, 4), dtype=np.uint8)
            assert same(walk(shim, frame, fmt, 2, (5, 6, 7), False), p10_np(over_np(frame[::-1], (5, 6, 7), False), NAMES[fmt], 2))


@pytest.mark.parametrize("w,h,rows", [(256, 40, 8), (300, 34, 5), (128, 64, 64), (134, 18, 1), (64, 30, 540), (301, 33, 7)])
@pytest.mark.parametrize("fmt", [YUV420P10, YUV444P10])
def test_marks_skip_rows_without_reading_them(shim, w, h, rows, fmt):
    if fmt == YUV420P10 and (w | h) & 1:
        w, h = w - (w & 1), h - (h & 1)
    rows = min(rows, h)
    rng = np.random.default_rng(w * h + rows + fmt)
    for garbage in (False, True):
        frame, clean, marks = marked_frame(rng, w, h, rows, garbage)
        for e in (0, 3):
            aware = walk(shim, frame, fmt, e, (40, 50, 60), marks=marks, rows=rows)
            assert same(aware, p10_np(over_np(clean[::-1], (40, 50, 60), True), NAMES[fmt], e)), (garbage, e)
            assert same(aware, walk(shim, clean, fmt, e, (40, 50, 60))), (garbage, e)


@pytest.mark.parametrize("e", [0, 1, 2, 3])
def test_identities_with_p010(shim, e):
    """YUV420P10 is P010 deinterleaved and >> 6; YUV444P10's Y is the same Y and its chroma is P010's of a 2x2 block of
    each pixel (a frame of 2x2-replicated pixels exports the same chroma in both)"""
    rng = np.random.default_rng(40 + e)
    w, h = 130, 22
    frame = premultiplied(rng, (h, w))
    bg = (9, 99, 199)
    comp = over_np(frame[::-1], bg, True)
    y, cb, cr = walk(shim, frame, YUV420P10, e, bg)
    p = p010_np(comp, e)
    assert np.array_equal(y, p[:h] >> 6) and np.array_equal(cb, p[h:, 0::2] >> 6) and np.array_equal(cr, p[h:, 1::2] >> 6)
    y4, cb4, cr4 = walk(shim, frame, YUV444P10, e, bg)
    assert np.array_equal(y4, y)
    small = premultiplied(rng, (h // 2, w // 2))
    big = small.repeat(2, axis=0).repeat(2, axis=1)
    _, cb2, cr2 = walk(shim, big, YUV420P10, e, bg)
    _, cb4, cr4 = walk(shim, small, YUV444P10, e, bg)
    assert np.array_equal(cb4, cb2) and np.array_equal(cr4, cr2)
    if not e & 1:                                                     # limited range: greys 512, black Y 64
        grey = np.full((4, 8, 4), 0x80, np.uint8); grey[..., 3] = 255
        for fmt in (YUV420P10, YUV444P10):
            gy, gcb, gcr = walk(shim, grey, fmt, e, native=False)
            assert (gcb == 512).all() and (gcr == 512).all()
            assert (walk(shim, np.zeros((4, 8, 4), np.uint8), fmt, e)[0] == 64).all()
    else:
        assert (walk(shim, np.zeros((4, 8, 4), np.uint8), YUV420P10, e)[0] == 0).all()


@pytest.mark.parametrize("fmt", [YUV420P10, YUV444P10])
@pytest.mark.parametrize("e", [0, 1, 2, 3])
def test_scaled_walk_is_the_format_on_the_scaled_image(shim, fmt, e):
    rng = np.random.default_rng(60 + e + fmt)
    w, h = 300, 170
    frame = premultiplied(rng, (h, w))
    bg = (30, 60, 200)
    cases = [((100, 56), None), ((64, 30), (10, 20, 200, 100)), ((34, 18), None), ((300, 170), None)]
    if fmt == YUV444P10:
        cases += [((37, 19), None), ((1, 1), None), ((33, 7), (3, 5, 101, 47))]
    for size, crop in cases:
        x, y, cw, ch = crop or (0, 0, w, h)
        img = area_np(over_np(frame[::-1][y:y + ch, x:x + cw].astype(np.int64), bg, True), size)
        assert same(scaled(shim, frame, fmt, e, size, crop, bg), p10_np(img, NAMES[fmt], e)), (size, crop)
    # the whole frame at its own size is the whole-frame walk, with and without marks
    assert same(scaled(shim, frame, fmt, e, (w, h), None, bg), walk(shim, frame, fmt, e, bg))
    dirty, clean, marks = marked_frame(rng, w, h, 8, True)
    assert same(scaled(shim, dirty, fmt, e, (100, 56), None, bg, marks=marks, rows=8), scaled(shim, clean, fmt, e, (100, 56), None, bg))


# ---- refusals and enqueued work through the fake runtime (test_export_formats_core's `fake` library) ----------------------
def test_refusals_and_byte_counts(fake):
    L = fake
    L.fake_fail_at(-1)
    r, odd = renderer(L, 64, 32), renderer(L, 63, 31)
    buf, buf2 = device_buf(L), device_buf(L)
    s = np.zeros(1, np.int32)
    one, uv = (C.c_void_p * 1)(buf.value), (C.c_void_p * 1)(buf2.value)

    def frames(h, d):
        return call(L, L.glava_b200_export_frames, h, s.ctypes.data, 1, one, C.byref(d), None, None)

    def scaled_call(h, d, size, dst_uv=None):
        return call(L, L.glava_b200_export_scaled, h, s.ctypes.data, 1, one, dst_uv, C.byref(d), C.byref(scale_of(size)), None, None)

    for fmt, pitch, *uvo in [(YUV420P10, 128), (YUV444P10, 128), (YUV420P10, 160, 80 * 16 + 48), (YUV444P10, 128, 128 * 33)]:
        for flags in (0, 0x100, 0x200, 0x300):
            rc, msg, trace, launched = frames(r, desc_of(fmt, pitch, flags, uv=uvo[0] if uvo else 0))
            assert rc == 0 and launched == 1 and len(memcpys(trace)) == 1, (fmt, flags, msg)
    rc, msg, _, launched = frames(odd, desc_of(YUV444P10, 128))
    assert rc == 0 and launched == 1, msg                             # 4:4:4 takes odd sizes
    refused = [  # (renderer, desc, what)
        (odd, desc_of(YUV420P10, 128), "YUV420P10 needs an even width and height, the frame is 63x31"),
        (r, desc_of(YUV420P10, 144), "YUV420P10 pitch 144 must be a multiple of 32"),
        (r, desc_of(YUV420P10, 96), "at least 128"),
        (r, desc_of(YUV444P10, 112), "at least 128"),
        (odd, desc_of(YUV444P10, 112), "at least 126"),
        (r, desc_of(YUV444P10, 136), "multiple of 16"),
        (r, desc_of(YUV420P10, 128, uv=8), "YUV420P10 uv_offset 8 (Cb plane to Cr plane)"),
        (r, desc_of(YUV420P10, 128, uv=64 * 15), "one chroma plane, 1024 bytes"),
        (r, desc_of(YUV444P10, 128, uv=128 * 31), "YUV444P10 uv_offset 3968 (Cb plane to Cr plane)"),
        (r, desc_of(YUV444P10, 128, uv=128 * 32 + 8), "must be a multiple of 16"),
        (r, desc_of(9, 256), "unknown format 9"),
    ]
    for h, d, what in refused:
        rc, msg, trace, launched = frames(h, d)
        assert rc != 0 and "glava_b200_export_frames" in msg and what in msg, (what, msg)
        assert trace == "" and launched == 0, what
    # the scaled export: odd output sizes, dst_uv legal for both
    rc, msg, trace, launched = scaled_call(r, desc_of(YUV420P10, 32), (15, 8))
    assert rc != 0 and "YUV420P10 needs an even width and height, the output is 15x8" in msg and launched == 0, msg
    rc, msg, _, launched = scaled_call(r, desc_of(YUV444P10, 32), (15, 7))
    assert rc == 0 and launched == 1, msg
    for fmt, pitch in ((YUV420P10, 32), (YUV444P10, 32)):
        rc, msg, _, launched = scaled_call(r, desc_of(fmt, pitch), (16, 8), uv)
        assert rc == 0 and launched == 1, (fmt, msg)
    rc, msg, trace, launched = scaled_call(r, desc_of(YUV420P10, 16), (16, 8), uv)
    assert rc != 0 and "at least 32" in msg and trace == "" and launched == 0, msg
    # the overlay keeps its three formats and names the new ones
    for fmt, name in ((YUV420P10, "YUV420P10"), (YUV444P10, "YUV444P10")):
        for flags in (0, 0x100):
            rc, msg, trace, launched = call(L, L.glava_b200_overlay_frames, r, s.ctypes.data, 1, one, None,
                                            C.byref(desc_of(fmt, 128, flags)), None, None)
            assert rc != 0 and f"format {name}: the overlay takes RGBA, BGRA or NV12" in msg and "unknown" not in msg, msg
            assert trace == "" and launched == 0
    # a ladder rung in a new format is checked as its scaled export; dst_uv entries are legal for it
    pairs = [(desc_of(YUV420P10, 128), scale_of((64, 32))), (desc_of(RGBA, 64), scale_of((16, 8))),
             (desc_of(YUV444P10, 32, 0x300), scale_of((15, 9)))]
    three = (C.c_void_p * 3)(buf.value, buf.value, buf.value)
    rc, msg, _, launched = call(L, L.glava_b200_export_ladder, r, s.ctypes.data, 1, rungs_of(pairs), 3, three,
                                (C.c_void_p * 3)(buf2.value, None, buf2.value), None, None)
    assert rc == 0 and launched == 1, msg
    rc, msg, _, launched = call(L, L.glava_b200_export_ladder, r, s.ctypes.data, 1,
                                rungs_of([(desc_of(YUV420P10, 48), scale_of((16, 8)))]), 1, three, None, None, None)
    assert rc != 0 and "rung 0: YUV420P10 pitch 48" in msg and launched == 0, msg
    # byte counts: pitch * h + the Cb to Cr distance + one chroma plane
    n = C.c_size_t()
    for d, want in ((desc_of(YUV420P10, 128), 128 * 32 + 2 * 64 * 16), (desc_of(YUV420P10, 128, uv=4096), 128 * 32 + 4096 + 64 * 16),
                    (desc_of(YUV444P10, 128), 3 * 128 * 32), (desc_of(YUV444P10, 128, uv=8192), 128 * 32 + 8192 + 128 * 32)):
        assert L.glava_b200_export_bytes(r, C.byref(d), C.byref(n)) == 0 and n.value == want, (d.format, n.value, want)
    assert L.glava_b200_export_scaled_bytes(r, C.byref(desc_of(YUV420P10, 32)), C.byref(scale_of((16, 8))), C.byref(n)) == 0
    assert n.value == 32 * 8 + 2 * 16 * 4
    assert L.glava_b200_export_scaled_bytes(r, C.byref(desc_of(YUV444P10, 32)), C.byref(scale_of((15, 7))), C.byref(n)) == 0
    assert n.value == 3 * 32 * 7
    assert L.glava_b200_export_bytes(odd, C.byref(desc_of(YUV420P10, 128)), C.byref(n)) != 0
    assert L.glava_b200_export_bytes(odd, C.byref(desc_of(YUV444P10, 128)), C.byref(n)) == 0 and n.value == 3 * 128 * 31
    for h in (r, odd):
        L.glava_b200_destroy(h)
    L.cudaFree(buf); L.cudaFree(buf2)


def test_one_copy_one_launch_and_the_plane_offsets(fake):
    L = fake
    L.fake_fail_at(-1)
    r = renderer(L, 64, 32)
    buf = device_buf(L)
    s = np.zeros(3, np.int32)
    dst = (C.c_void_p * 6)(*[buf.value] * 6)
    pcm = np.zeros((2, 1024), np.float32)
    assert L.glava_b200_update(r, pcm.ctypes.data, pcm.ctypes.data, 1024, 1) == 0
    got = (C.c_longlong * 3)()
    for fmt, pitch, uvo, cr in ((YUV420P10, 32, 0, 16 * 4), (YUV420P10, 64, 4096, 4096), (YUV444P10, 32, 0, 32 * 8)):
        rc, msg, trace, launched = call(L, L.glava_b200_export_scaled, r, s.ctypes.data, 3, dst, None, C.byref(desc_of(fmt, pitch, uv=uvo)),
                                        C.byref(scale_of((16, 8))), None, None)
        assert rc == 0 and launched == 1 and memcpys(trace) == [3 * 24], (fmt, msg, trace)
        L.formats_fake_scaled(got)
        assert list(got) == [fmt, 1, cr], (fmt, list(got))
    pairs = [(desc_of(NV12, 64), scale_of((64, 32))), (desc_of(YUV420P10, 128, 0x100), scale_of((64, 32))),
             (desc_of(YUV444P10, 32, uv=512), scale_of((15, 9))), (desc_of(P010, 128), scale_of((64, 32)))]
    rc, msg, trace, launched = call(L, L.glava_b200_export_ladder, r, s.ctypes.data, 1, rungs_of(pairs), 4, dst, None, None, None)
    assert rc == 0 and launched == 1 and memcpys(trace)[-1] == 4 * 24, (msg, trace)
    lad = (C.c_longlong * (5 * 8))()
    L.formats_fake_ladder(lad)
    assert [lad[5 * j] for j in range(4)] == [0, 64 * 16, 512, 0]
    assert [lad[5 * j + 4] for j in range(4)] == [1, 1, 1, 1]          # every YUV rung composites
    # the zero constants are the background (black) as LSB-aligned codes: full range Y 0, limited range Y 64, chroma 512
    assert lad[5 + 1] == 0 and lad[5 + 2] == 512 * 0x10001 and lad[5 + 3] == 512 * 0x10001
    assert lad[10 + 1] == 64 * 0x10001 and lad[10 + 2] == 512 * 0x10001
    L.glava_b200_destroy(r)
    L.cudaFree(buf)
