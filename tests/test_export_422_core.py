"""4:2:2 export and overlay, YUV422P, YUV422P10 and UYVY (DESIGN 4.18), on the host: the pair chroma of export_core.h over
every per-channel pair sum (511^3) and encoding against float64, host walks of export_422_kernel's and
export_scaled_422_kernel's loops and of the overlay's row422 body checked bit for bit against the numpy restatement of
tests/export_422_np.py with sentinel bytes around and between every plane, the identities with the library's own I420 and
YUV420P10 walks of the row-doubled frame, and the refusals, byte counts and launches of the export calls through capi.cu,
export.cpp and export_ladder.cpp built against tests/fakecuda's runtime (the overlay's C-ABI refusals and geometry are
tests/test_overlay_422_core.py's)."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from tests.export_422_np import NAMES, export422_np, overlay422_np, planar_of, uyvy_of
from tests.export_fake import desc_of
from tests.test_export_core import CSRC, marked_frame, over_np, pack, premultiplied
from tests.test_export_formats_core import call, device_buf, memcpys, renderer
from tests.test_export_formats_core import fake  # noqa: F401 (the fake-runtime fixture)
from tests.test_export_ladder_core import rungs_of, scale_of
from tests.test_export_matrix_core import ENCODINGS
from tests.test_export_p10_core import SHIM as P10_SHIM
from tests.test_export_p10_core import p10_np
from tests.test_export_p10_core import walk as p10_walk
from tests.test_export_scaled_core import area_np

RGBA, NV12, I420, P010, YUV420P10, YUV444P10 = 0, 2, 4, 6, 7, 8
YUV422P, YUV422P10, UYVY = 10, 11, 12
SENTINEL = 0xA5
# the largest distance from the float64 formula on the exact pair mean over all 511^3 pair sums, per (encoding, bits), as
# DESIGN 4.18 records it: 8 bits the byte average's rounding, as NV12 has it; 10 bits P010's exact-sum chroma
PAIR_BOUND = {(0, 8): 0.7217, (1, 8): 0.7511, (2, 8): 0.7217, (3, 8): 0.7501,
              (0, 10): 0.5027, (1, 10): 0.5018, (2, 10): 0.5023, (3, 10): 0.5017}

# test_export_p10_core's shim (t_scaled, the 8-bit scaled image, and the planar 10-bit walk) plus the 4:2:2 walks
SHIM = P10_SHIM + r"""
static void put(uint8_t* p, uint32_t v, int n) { memcpy(p, &v, n); }     // the first n bytes of v, little-endian
// as export_kernels.cu row_422: the quad q at x of output row r
template <int E> static void row422(const ExportFmt& f, int fmt, const uint32_t q[4], uint8_t* dst, uint8_t* cb, size_t cr,
                                    size_t pitch, int r, int x, bool full, const ExportZero& z) {
    const bool any = (q[0] | q[1] | q[2] | q[3]) != 0u;
    if (fmt == GLAVA_B200_EXPORT_UYVY) {
        uint32_t w[2] = { z.y, z.y };
        if (any) { uint32_t y; const uint32_t uv = export_422_quad<E>(f, q, &y); export_uyvy_words(y, uv, w); }
        uint8_t* p = dst + (size_t) r * pitch + 2 * (size_t) x;
        put(p, w[0], 4); if (full) put(p + 4, w[1], 4);
    } else if (fmt == GLAVA_B200_EXPORT_YUV422P) {
        uint32_t y = z.y, u = z.u, v = z.v;
        if (any) { const uint32_t uv = export_422_quad<E>(f, q, &y); u = export_cb_pair(uv); v = export_cr_pair(uv); }
        uint8_t* pu = cb + (size_t) r * (pitch >> 1) + (x >> 1);
        put(dst + (size_t) r * pitch + x, y, full ? 4 : 2); put(pu, u, full ? 2 : 1); put(pu + cr, v, full ? 2 : 1);
    } else {
        uint32_t y[2] = { z.y, z.y }, u = z.u, v = z.v;
        if (any) export_422p10_quad<E>(f, q, y, &u, &v);
        uint8_t* py = dst + (size_t) r * pitch + 2 * (size_t) x;
        uint8_t* pu = cb + (size_t) r * (pitch >> 1) + x;
        put(py, y[0], 4); if (full) put(py + 4, y[1], 4);
        put(pu, u, full ? 4 : 2); put(pu + cr, v, full ? 4 : 2);
    }
}
// one slot [h][w] -> the planes, as export_422_kernel walks it (item_422): row pairs, 128-pixel strips, a quad per lane
template <int E> static void walk422(const uint32_t* fb, int w, int h, const uint32_t* marks, int rows, int format, int native,
                                     uint32_t bg, uint8_t* dst, size_t pitch, uint8_t* cb, size_t cr) {
    const ExportFmt f = { format, 1, native, bg };
    const ExportZero z = export_zero422<E>(f);
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
                const bool full = x + 4 <= w;
                row422<E>(f, format, q[0], dst, cb, cr, pitch, 2 * j, x, full, z);
                if (y1 >= 0) row422<E>(f, format, q[1], dst, cb, cr, pitch, 2 * j + 1, x, full, z);
            }
}
// the scaled image img [out_h][out_w] -> the planes, as export_scaled_422_kernel walks it (scaled_422_item): one output row
// per unit, runs of 32 lanes, the pair's right pixel from lane + 1
template <int E> static void scaled422(const uint32_t* img, int out_w, int out_h, int format, uint8_t* dst, size_t pitch, uint8_t* cb, size_t cr) {
    auto at = [&](int Y, int X) { return X < out_w ? img[(size_t) Y * out_w + X] : 0u; };
    for (int u = 0; u < out_h; ++u)
        for (int run = 0; run < (out_w + 31) / 32; ++run)
            for (int lane = 0; lane < 32 && run * 32 + lane < out_w; ++lane) {
                const int X = run * 32 + lane;
                const uint32_t px = at(u, X), px1 = at(u, X + 1);
                if (format == GLAVA_B200_EXPORT_UYVY) {
                    if (!(lane & 1)) {
                        const uint32_t uv = export_cbcr<E>(export_avg4(px, px1, px, px1));
                        put(dst + (size_t) u * pitch + 2 * (size_t) X, (uv & 0xffu) | (export_y<E>(px) << 8) | ((uv & 0xff00u) << 8) | (export_y<E>(px1) << 24), 4);
                    }
                } else if (format == GLAVA_B200_EXPORT_YUV422P) {
                    put(dst + (size_t) u * pitch + X, export_y<E>(px), 1);
                    if (!(lane & 1)) {
                        const uint32_t uv = export_cbcr<E>(export_avg4(px, px1, px, px1));
                        uint8_t* pu = cb + (size_t) u * (pitch / 2) + (X >> 1);
                        put(pu, uv, 1); put(pu + cr, uv >> 8, 1);
                    }
                } else {
                    put(dst + (size_t) u * pitch + 2 * (size_t) X, export_y10<E>(px), 2);
                    if (!(lane & 1)) {
                        const uint32_t uv = export_cbcr10<E>(export_sum4(px, px1, px, px1));
                        uint8_t* pu = cb + (size_t) u * (pitch / 2) + X;
                        put(pu, uv, 2); put(pu + cr, uv >> 16, 2);
                    }
                }
            }
}
template <int E> static void zero422(int format, int native, uint32_t bg, uint32_t* out) {
    const ExportFmt f = { format, 1, native, bg };
    const ExportZero z = export_zero422<E>(f);
    out[0] = z.y; out[1] = z.u; out[2] = z.v;
}
// every per-channel pair sum t = a + b (0..510): the largest distance of the pair chroma from float64 on the mean t / 2
template <int E> static void sweep(int bits, double* err) {
    const double kr = E & 2 ? 0.299 : 0.2126, kb = E & 2 ? 0.114 : 0.0722, kg = 1 - kr - kb;
    const bool full = E & 1;
    const double top = bits == 10 ? 1023 : 255, cs = full ? top / 255 : (bits == 10 ? 896.0 : 224.0) / 255, coff = bits == 10 ? 512 : 128;
    double e0 = 0, e1 = 0;
    for (uint32_t tr = 0; tr <= 510; ++tr)
        for (uint32_t tg = 0; tg <= 510; ++tg)
            for (uint32_t tb = 0; tb <= 510; ++tb) {
                uint32_t c;
                if (bits == 10) {
                    c = export_cbcr10<E>((2 * tr) | ((2 * tg) << 10) | ((2 * tb) << 20));
                } else {
                    const uint32_t a = (tr + 1) >> 1, b = tr >> 1, g0 = (tg + 1) >> 1, g1 = tg >> 1, b0 = (tb + 1) >> 1, b1 = tb >> 1;
                    c = export_cbcr<E>(export_avg4(a | (g0 << 8) | (b0 << 16), b | (g1 << 8) | (b1 << 16), a | (g0 << 8) | (b0 << 16),
                                                   b | (g1 << 8) | (b1 << 16)));
                    c = (c & 255u) | ((c >> 8) << 16);
                }
                const double r = tr / 2.0, g = tg / 2.0, b = tb / 2.0, yp = kr * r + kg * g + kb * b;
                double fcb = coff + cs * (b - yp) / (2 * (1 - kb)), fcr = coff + cs * (r - yp) / (2 * (1 - kr));
                fcb = fcb > top ? top : fcb; fcr = fcr > top ? top : fcr;
                const double d0 = std::fabs((double) (c & 0xffffu) - fcb), d1 = std::fabs((double) (c >> 16) - fcr);
                e0 = d0 > e0 ? d0 : e0; e1 = d1 > e1 ? d1 : e1;
            }
    err[0] = e0; err[1] = e1;
}
// as export_kernels.cu OverlayPlanesBody::row422, over a top-down image img [h][w] (stored pixels) and the planes
template <int E> static void over422(const uint32_t* img, int w, int h, int format, int native, uint8_t* dst, size_t pitch,
                                     uint8_t* cb, uint8_t* crp, size_t cpitch) {
    const ExportFmt f = { format, 1, 0, 0u };
    for (int r = 0; r < h; ++r)
        for (int x = 0; x < w; x += 4) {
            uint32_t q[4];
            for (int k = 0; k < 4; ++k) q[k] = x + k < w ? img[(size_t) r * w + x + k] : 0u;
            if (native && (q[0] | q[1] | q[2] | q[3]) == 0u) continue;
            const bool full = x + 4 <= w;
            if (format == GLAVA_B200_EXPORT_UYVY) {
                uint8_t* p = dst + (size_t) r * pitch + 2 * (size_t) x;
                uint32_t wd[2] = { 0u, 0u }, y, uv;
                memcpy(wd, p, full ? 8 : 4);
                if (native) { export_uyvy_split(wd, &y, &uv); overlay_422_quad<E>(q, &y, &uv); }
                else uv = export_422_quad<E>(f, q, &y);
                export_uyvy_words(y, uv, wd);
                memcpy(p, wd, full ? 8 : 4);
            } else if (format == GLAVA_B200_EXPORT_YUV422P) {
                uint8_t *py = dst + (size_t) r * pitch + x, *pu = cb + (size_t) r * cpitch + x / 2, *pv = crp + (size_t) r * cpitch + x / 2;
                uint32_t y = 0, u = 0, v = 0;
                memcpy(&y, py, full ? 4 : 2); memcpy(&u, pu, full ? 2 : 1); memcpy(&v, pv, full ? 2 : 1);
                if (native) {
                    uint32_t uv = (u & 0xffu) | ((v & 0xffu) << 8) | ((u & 0xff00u) << 8) | ((v & 0xff00u) << 16);
                    overlay_422_quad<E>(q, &y, &uv);
                    u = export_cb_pair(uv); v = export_cr_pair(uv);
                } else {
                    const uint32_t uv = export_422_quad<E>(f, q, &y);
                    u = export_cb_pair(uv); v = export_cr_pair(uv);
                }
                memcpy(py, &y, full ? 4 : 2); memcpy(pu, &u, full ? 2 : 1); memcpy(pv, &v, full ? 2 : 1);
            } else {
                uint8_t *py = dst + (size_t) r * pitch + 2 * (size_t) x, *pu = cb + (size_t) r * cpitch + x, *pv = crp + (size_t) r * cpitch + x;
                uint32_t y[2] = { 0u, 0u }, u = 0, v = 0;
                memcpy(y, py, full ? 8 : 4); memcpy(&u, pu, full ? 4 : 2); memcpy(&v, pv, full ? 4 : 2);
                if (native) overlay_422p10_quad<E>(q, y, &u, &v);
                else export_422p10_quad<E>(f, q, y, &u, &v);
                memcpy(py, y, full ? 8 : 4); memcpy(pu, &u, full ? 4 : 2); memcpy(pv, &v, full ? 4 : 2);
            }
        }
}
// I420 as export_yuv_kernel walks it (export_kernels.cu yuv_item's I420 branch under encoding E): row pairs, 128-pixel
// strips, export_nv12_quad<E> split into the Cb and Cr pairs, export_zero<E> for all-zero quads
template <int E> static void i420walk(const uint32_t* fb, int w, int h, int native, uint32_t bg, uint8_t* dst, size_t pitch,
                                      uint8_t* cb, size_t cr) {
    const ExportFmt f = { GLAVA_B200_EXPORT_I420, 1, native, bg };
    const ExportZero z = export_zero<E>(f);
    for (int j = 0; j < h / 2; ++j)
        for (int x = 0; x < w; x += 4) {
            uint32_t q[2][4];
            for (int r = 0; r < 2; ++r)
                for (int k = 0; k < 4; ++k) q[r][k] = x + k < w ? fb[(size_t) (h - 1 - 2 * j - r) * w + x + k] : 0u;
            const bool full = x + 4 <= w;
            uint32_t yt = z.y, yb = z.y, u = z.u, v = z.v;
            if (q[0][0] | q[0][1] | q[0][2] | q[0][3] | q[1][0] | q[1][1] | q[1][2] | q[1][3]) {
                const uint32_t uv = export_nv12_quad<E>(f, q[0], q[1], &yt, &yb);
                u = export_cb_pair(uv); v = export_cr_pair(uv);
            }
            put(dst + (size_t) (2 * j) * pitch + x, yt, full ? 4 : 2); put(dst + (size_t) (2 * j + 1) * pitch + x, yb, full ? 4 : 2);
            uint8_t* pu = cb + (size_t) j * (pitch / 2) + x / 2;
            put(pu, u, full ? 2 : 1); put(pu + cr, v, full ? 2 : 1);
        }
}
extern "C" void t_i420_walk(int e, const uint32_t* fb, int w, int h, int native, uint32_t bg, uint8_t* dst, size_t pitch, uint8_t* cb,
                            size_t cr) {
    DISPATCH(i420walk, fb, w, h, native, bg, dst, pitch, cb, cr)
}
extern "C" void t_422_walk(int e, const uint32_t* fb, int w, int h, const uint32_t* marks, int rows, int format, int native,
                           uint32_t bg, uint8_t* dst, size_t pitch, uint8_t* cb, size_t cr) {
    DISPATCH(walk422, fb, w, h, marks, rows, format, native, bg, dst, pitch, cb, cr)
}
extern "C" void t_422_scaled(int e, const uint32_t* img, int out_w, int out_h, int format, uint8_t* dst, size_t pitch, uint8_t* cb, size_t cr) {
    DISPATCH(scaled422, img, out_w, out_h, format, dst, pitch, cb, cr)
}
extern "C" void t_422_zero(int e, int format, int native, uint32_t bg, uint32_t* out) { DISPATCH(zero422, format, native, bg, out) }
extern "C" void t_422_sweep(int e, int bits, double* err) { DISPATCH(sweep, bits, err) }
extern "C" void t_422_over(int e, const uint32_t* img, int w, int h, int format, int native, uint8_t* dst, size_t pitch, uint8_t* cb,
                           uint8_t* cr, size_t cpitch) {
    DISPATCH(over422, img, w, h, format, native, dst, pitch, cb, cr, cpitch)
}
extern "C" void t_422_predicates(int format, size_t pitch, int h, long long* out) {
    out[0] = export_yuv(format); out[1] = export_p10(format); out[2] = export_422(format); out[3] = export_ycbcr(format);
    out[4] = export_chroma_planes(format); out[5] = export_420(format); out[6] = export_planar(format);
    out[7] = (long long) export_planes(format, pitch, 0, h).plane;
}
extern "C" int t_ladder_kernel(const int* format, const int* enc, int n) { return ladder_kernel(format, enc, n); }
"""


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("export_422_core")
    src, so = d / "shim.cpp", d / "shim.so"
    src.write_text(SHIM)
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I", CSRC,
                    "-include", "cstring", "-include", "algorithm", "-include", "cmath", "-o", str(so), str(src)], check=True)
    L = C.CDLL(str(so))
    vp, sz, i32, u32 = C.c_void_p, C.c_size_t, C.c_int, C.c_uint32
    L.t_p10_walk.argtypes = [i32, vp, i32, i32, vp, i32, i32, i32, u32, vp, sz, vp, sz]
    L.t_422_walk.argtypes = [i32, vp, i32, i32, vp, i32, i32, i32, u32, vp, sz, vp, sz]
    L.t_422_scaled.argtypes = [i32, vp, i32, i32, i32, vp, sz, vp, sz]
    L.t_422_zero.argtypes = [i32, i32, i32, u32, vp]
    L.t_422_sweep.argtypes = [i32, i32, vp]
    L.t_422_over.argtypes = [i32, vp, i32, i32, i32, i32, vp, sz, vp, vp, sz]
    L.t_422_predicates.argtypes = [i32, sz, i32, vp]
    L.t_i420_walk.argtypes = [i32, vp, i32, i32, i32, u32, vp, sz, vp, sz]
    L.t_ladder_kernel.argtypes = [vp, vp, i32]
    L.t_scaled.argtypes = [vp, i32, i32, vp, i32, i32, i32, i32, u32] + [i32] * 6 + [vp, vp, sz]
    return L


# ---- the walks into sentinel buffers ---------------------------------------------------------------------------------------------
def layout(fmt, w, h, pad, gap=64):
    """(pitch, Cb offset, Cb to Cr distance, total bytes) of a sentinel buffer: `pad` bytes past every row, `gap` bytes
    between planes (UYVY: one plane)"""
    row = 2 * w if fmt in (YUV422P10, UYVY) else w
    pitch = (row + pad + 31) // 32 * 32
    if fmt == UYVY:
        return pitch, 0, 0, pitch * h + gap
    cb_off = pitch * h + gap
    cr = (pitch // 2) * h + gap
    return pitch, cb_off, cr, cb_off + cr + (pitch // 2) * h + gap


def planes_of(buf, fmt, w, h, pitch, cb_off, cr):
    """the planes of a destination buffer (uint8), read with linesizes pitch and pitch / 2 as ffmpeg reads yuv422p /
    yuv422p10le (UYVY: one plane at pitch), and the mask of every byte they cover"""
    written = np.zeros(buf.size, bool)
    sb = 2 if fmt == YUV422P10 else 1

    def plane(off, p, nbytes):
        idx = off + np.arange(h)[:, None] * p + np.arange(nbytes)[None, :]
        written[idx] = True
        v = np.ascontiguousarray(buf[idx])
        return v.view(np.uint16) if sb == 2 else v

    if fmt == UYVY:
        return plane(0, pitch, 2 * w), written
    return (plane(0, pitch, w * sb), plane(cb_off, pitch // 2, w // 2 * sb), plane(cb_off + cr, pitch // 2, w // 2 * sb)), written


def walk(L, frame, fmt, e, bg=(0, 0, 0), native=True, marks=None, rows=0, pad=32):
    h, w = frame.shape[:2]
    pitch, cb_off, cr, total = layout(fmt, w, h, pad)
    buf = np.full(total, SENTINEL, np.uint8)
    fb = np.ascontiguousarray(frame).view(np.uint32).reshape(h, w)
    m = None if marks is None else np.ascontiguousarray(marks, np.uint32)
    L.t_422_walk(e, fb.ctypes.data, w, h, None if m is None else m.ctypes.data, rows, fmt, int(native), int(pack(*bg[:3])),
                 buf.ctypes.data, pitch, buf.ctypes.data + cb_off, cr)
    planes, written = planes_of(buf, fmt, w, h, pitch, cb_off, cr)
    assert (buf[~written] == SENTINEL).all(), "written outside the planes"
    return planes


def scaled(L, frame, fmt, e, size, crop=None, bg=(0, 0, 0), native=True, marks=None, rows=0, pad=48):
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
    L.t_422_scaled(e, img.ctypes.data, ow, oh, fmt, buf.ctypes.data, pitch, buf.ctypes.data + cb_off, cr)
    planes, written = planes_of(buf, fmt, ow, oh, pitch, cb_off, cr)
    assert (buf[~written] == SENTINEL).all(), "written outside the planes"
    return planes


def same(a, b):
    if isinstance(b, tuple):
        return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))
    return np.array_equal(a, b)


def want(frame, fmt, e, bg, native):
    return export422_np(over_np(frame[::-1], bg, native), NAMES[fmt], e)


# ---- arithmetic ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [8, 10])
@pytest.mark.parametrize("e", [0, 1, 2, 3], ids=[ENCODINGS[e] for e in range(4)])
def test_pair_chroma_of_every_pair_sum(shim, e, bits):
    """all 511^3 per-channel pair sums: the pair chroma within PAIR_BOUND of float64 on the exact pair mean (8 bits: the
    byte average rounds half up, as NV12's 2x2 average does; 10 bits: the exact sums, as P010)"""
    err = np.zeros(2)
    shim.t_422_sweep(e, bits, err.ctypes.data)
    assert err.max() <= PAIR_BOUND[e, bits], (ENCODINGS[e], bits, err)
    assert err.max() > PAIR_BOUND[e, bits] - 0.0002, err             # the maximum recorded in DESIGN 4.18, to 4 places


def test_the_restatement_against_i420_and_yuv420p10_of_the_doubled_image():
    rng = np.random.default_rng(1)
    c = rng.integers(0, 256, (7, 10, 4))
    c2 = c.repeat(2, axis=0)
    for e in range(4):
        y, cb, cr = export422_np(c, "yuv422p10", e)
        y2, cb2, cr2 = p10_np(c2, "yuv420p10", e)
        assert np.array_equal(y, y2[0::2]) and np.array_equal(cb, cb2) and np.array_equal(cr, cr2)
        u = export422_np(c, "uyvy", e)
        assert same(planar_of(u), export422_np(c, "yuv422p", e)) and np.array_equal(uyvy_of(*planar_of(u)), u)


def test_predicates_plane_sizes_and_the_ladder_kernel(shim):
    out = (C.c_longlong * 8)()
    for fmt, want_ in ((YUV422P, [0, 0, 1, 1, 1, 0, 1, 64 * 16]), (YUV422P10, [0, 0, 1, 1, 1, 0, 1, 64 * 16]),
                       (UYVY, [0, 0, 1, 1, 0, 0, 0, 0]), (I420, [1, 0, 0, 1, 1, 1, 1, 64 * 8]), (RGBA, [0] * 8)):
        shim.t_422_predicates(fmt, 128, 16, out)
        assert list(out) == want_, (fmt, list(out))
    pick = lambda f, e: shim.t_ladder_kernel((C.c_int * len(f))(*f), (C.c_int * len(e))(*e), len(f))
    assert pick([NV12, RGBA], [0, 0]) == 0 and pick([I420, NV12], [0, 0]) == 1 and pick([NV12], [1]) == 2
    assert pick([YUV420P10, NV12], [0, 3]) == 3
    for f in ([UYVY], [NV12, YUV422P], [YUV420P10, YUV422P10, I420], [RGBA, UYVY]):
        assert pick(f, [0] * len(f)) == 4 and pick(f, [2] * len(f)) == 4, f


@pytest.mark.parametrize("e", [0, 1, 2, 3])
def test_zero_constants(shim, e):
    out = (C.c_uint32 * 3)()
    for bg in (0x000000, 0xffffff, 0x4280f0):
        for native in (0, 1):
            c = np.zeros((1, 2, 4), np.int64)
            if native:
                c[...] = [bg & 255, (bg >> 8) & 255, bg >> 16, 255]
            y, cb, cr = (int(v[0, 0]) for v in export422_np(c, "yuv422p", e))
            shim.t_422_zero(e, YUV422P, native, bg, out)
            assert list(out) == [y * 0x01010101, cb * 0x0101, cr * 0x0101]
            shim.t_422_zero(e, UYVY, native, bg, out)
            assert out[0] == cb | y << 8 | cr << 16 | y << 24
            y, cb, cr = (int(v[0, 0]) for v in export422_np(c, "yuv422p10", e))
            shim.t_422_zero(e, YUV422P10, native, bg, out)
            assert list(out) == [y * 0x10001, cb * 0x10001, cr * 0x10001]


# ---- the kernels' walks ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w,h", [(128, 64), (130, 31), (66, 10), (2, 1), (390, 8), (98, 33), (6, 3), (258, 1), (134, 7)])
@pytest.mark.parametrize("fmt", [YUV422P, YUV422P10, UYVY])
@pytest.mark.parametrize("e", [0, 1, 2, 3])
def test_walk_equals_the_restatement(shim, w, h, fmt, e):
    rng = np.random.default_rng(w * 1000 + h + fmt + 10 * e)
    for native in (True, False):
        frame = premultiplied(rng, (h, w)) if native else rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
        frame[: h // 3] = 0                                            # zero quads take the constants
        bg = (17, 240, 66)
        assert same(walk(shim, frame, fmt, e, bg, native), want(frame, fmt, e, bg, native)), native


@pytest.mark.parametrize("w,h,rows", [(256, 40, 8), (300, 34, 5), (128, 64, 64), (134, 17, 1), (64, 31, 540), (302, 33, 7)])
@pytest.mark.parametrize("fmt", [YUV422P, YUV422P10, UYVY])
def test_marks_skip_rows_without_reading_them(shim, w, h, rows, fmt):
    rows = min(rows, h)
    rng = np.random.default_rng(w * h + rows + fmt)
    for garbage in (False, True):
        frame, clean, marks = marked_frame(rng, w, h, rows, garbage)
        for e in (0, 3):
            aware = walk(shim, frame, fmt, e, (40, 50, 60), marks=marks, rows=rows)
            assert same(aware, want(clean, fmt, e, (40, 50, 60), True)), (garbage, e)
            assert same(aware, walk(shim, clean, fmt, e, (40, 50, 60))), (garbage, e)


@pytest.mark.parametrize("e", [0, 1, 2, 3])
def test_identities_with_the_row_doubled_frame(shim, e):
    """F2 = F with every row doubled: YUV422P of F is I420 of F2 (its Y rows 2r, its chroma row r), YUV422P10 of F is
    YUV420P10 of F2 likewise, each against the library's own 4:2:0 walk; UYVY is YUV422P interleaved; YUV422P10's Y is
    YUV420P10's Y"""
    rng = np.random.default_rng(40 + e)
    bg = (9, 99, 199)
    frames = (premultiplied(rng, (11, 130)), premultiplied(rng, (5, 256)), rng.integers(0, 256, (7, 66, 4), dtype=np.uint8),
              np.zeros((3, 6, 4), np.uint8), np.full((4, 2, 4), 255, np.uint8))
    for frame in frames:
        h, w = frame.shape[:2]
        f2 = frame.repeat(2, axis=0)
        for native in (True, False):
            y, cb, cr = walk(shim, frame, YUV422P10, e, bg, native)
            y2, cb2, cr2 = p10_walk(shim, f2, YUV420P10, e, bg, native)
            assert np.array_equal(y, y2[0::2]) and np.array_equal(cb, cb2) and np.array_equal(cr, cr2), native
            p = walk(shim, frame, YUV422P, e, bg, native)
            i420 = i420_walk(shim, f2, e, bg, native)
            assert np.array_equal(p[0], i420[0][0::2]) and np.array_equal(p[1], i420[1]) and np.array_equal(p[2], i420[2]), native
            assert same(planar_of(walk(shim, frame, UYVY, e, bg, native)), p)
            if h % 2 == 0:
                assert np.array_equal(y, p10_walk(shim, frame, YUV420P10, e, bg, native)[0])
                assert np.array_equal(p[0], i420_walk(shim, frame, e, bg, native)[0])


def i420_walk(L, frame, e, bg, native, pad=32, gap=64):
    """t_i420_walk (the library's I420 arithmetic) into one sentinel buffer -> (Y, Cb, Cr), nothing written outside them"""
    h, w = frame.shape[:2]
    pitch = (w + pad + 31) // 32 * 32
    cb_off, cr = pitch * h + gap, (pitch // 2) * (h // 2) + gap
    buf = np.full(cb_off + 2 * cr, SENTINEL, np.uint8)
    fb = np.ascontiguousarray(frame).view(np.uint32).reshape(h, w)
    L.t_i420_walk(e, fb.ctypes.data, w, h, int(native), int(pack(*bg[:3])), buf.ctypes.data, pitch, buf.ctypes.data + cb_off, cr)
    written = np.zeros(buf.size, bool)

    def plane(off, rows, p, nbytes):
        idx = off + np.arange(rows)[:, None] * p + np.arange(nbytes)[None, :]
        written[idx] = True
        return buf[idx]

    planes = (plane(0, h, pitch, w), plane(cb_off, h // 2, pitch // 2, w // 2), plane(cb_off + cr, h // 2, pitch // 2, w // 2))
    assert (buf[~written] == SENTINEL).all(), "written outside the planes"
    return planes


@pytest.mark.parametrize("fmt", [YUV422P, YUV422P10, UYVY])
@pytest.mark.parametrize("e", [0, 1, 2, 3])
def test_scaled_walk_is_the_format_on_the_scaled_image(shim, fmt, e):
    rng = np.random.default_rng(60 + e + fmt)
    w, h = 300, 170
    frame = premultiplied(rng, (h, w))
    bg = (30, 60, 200)
    for size, crop in [((100, 56), None), ((64, 31), (10, 20, 200, 100)), ((34, 17), None), ((2, 1), None), ((38, 7), (3, 5, 101, 47))]:
        x, y, cw, ch = crop or (0, 0, w, h)
        img = area_np(over_np(frame[::-1][y:y + ch, x:x + cw].astype(np.int64), bg, True), size)
        assert same(scaled(shim, frame, fmt, e, size, crop, bg), export422_np(img, NAMES[fmt], e)), (size, crop)
    assert same(scaled(shim, frame, fmt, e, (w, h), None, bg), walk(shim, frame, fmt, e, bg))
    dirty, clean, marks = marked_frame(rng, w, h, 8, True)
    assert same(scaled(shim, dirty, fmt, e, (100, 57), None, bg, marks=marks, rows=8), scaled(shim, clean, fmt, e, (100, 57), None, bg))


# ---- the overlay's row422 body ----------------------------------------------------------------------------------------------
def over(L, frame, planes, fmt, e, native):
    """t_422_over onto copies of planes ((Y, Cb, Cr) or (UYVY,)), each embedded in a sentinel buffer with padded rows"""
    h, w = frame.shape[:2]
    img = np.ascontiguousarray(frame[::-1]).view(np.uint32).reshape(h, w)
    bufs, ptrs, pitches = [], [], []
    for p in planes:
        b = p.view(np.uint8)
        pitch = (b.shape[1] + 40 + 15) // 16 * 16
        buf = np.full((h, pitch), SENTINEL, np.uint8)
        buf[:, :b.shape[1]] = b
        bufs.append(buf); ptrs.append(buf.ctypes.data); pitches.append(pitch)
    if fmt == UYVY:
        ptrs += [None, None]; pitches.append(0)
    L.t_422_over(e, img.ctypes.data, w, h, fmt, int(native), ptrs[0], pitches[0], ptrs[1], ptrs[2], pitches[1])
    out = []
    for buf, p in zip(bufs, planes):
        nb = p.view(np.uint8).shape[1]
        assert (buf[:, nb:] == SENTINEL).all(), "written past the rectangle"
        out.append(np.ascontiguousarray(buf[:, :nb]).view(p.dtype))
    return out


def random_planes(rng, fmt, w, h):
    if fmt == UYVY:
        return [rng.integers(0, 256, (h, 2 * w), dtype=np.uint8)]
    dt, top = (np.uint16, 1 << 16) if fmt == YUV422P10 else (np.uint8, 256)
    return [rng.integers(0, top, (h, w), dtype=dt), rng.integers(0, top, (h, w // 2), dtype=dt), rng.integers(0, top, (h, w // 2), dtype=dt)]


@pytest.mark.parametrize("w,h", [(128, 8), (130, 5), (6, 3), (2, 1)])
@pytest.mark.parametrize("fmt", [YUV422P, YUV422P10, UYVY])
@pytest.mark.parametrize("e", [0, 1, 2, 3])
def test_overlay_equals_the_restatement(shim, w, h, fmt, e):
    """the blend against numpy, 10-bit samples with garbage in their padding bits, zero pixels and zero pairs leaving the
    picture's bytes (all 16 bits)"""
    rng = np.random.default_rng(w + 7 * h + fmt + 100 * e)
    for native in (True, False):
        frame = premultiplied(rng, (h, w))
        frame[:, 1::3] = 0                                             # lone zero pixels, zero pairs, zero quads
        frame[: h // 2, : w // 2] = 0
        before = random_planes(rng, fmt, w, h)
        got = over(shim, frame, before, fmt, e, native)
        assert same(tuple(got), tuple(overlay422_np(frame, before, NAMES[fmt], e, native))), native


@pytest.mark.parametrize("fmt", [YUV422P, YUV422P10, UYVY])
@pytest.mark.parametrize("e", [0, 1, 2, 3])
def test_overlay_identities(shim, fmt, e):
    """an all-zero frame leaves the picture; an opaque frame, and any frame under another opacity, gives export_frames'
    bytes; YUV422P10's blend of F is YUV420P10's blend of F2 (overlay_planes_np) on the doubled picture"""
    rng = np.random.default_rng(90 + e + fmt)
    w, h = 130, 6
    before = random_planes(rng, fmt, w, h)
    assert same(tuple(over(shim, np.zeros((h, w, 4), np.uint8), before, fmt, e, True)), tuple(before))
    frame = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    frame[..., 3] = 255
    exp = export422_np(over_np(frame[::-1], (0, 0, 0), True), NAMES[fmt], e)
    exp = (exp,) if fmt == UYVY else exp
    assert same(tuple(over(shim, frame, before, fmt, e, True)), exp)
    frame = premultiplied(rng, (h, w))
    exp = export422_np(over_np(frame[::-1], (0, 0, 0), False), NAMES[fmt], e)
    exp = (exp,) if fmt == UYVY else exp
    assert same(tuple(over(shim, frame, before, fmt, e, False)), exp)
    if fmt == YUV422P10:
        from tests.overlay_planes_np import planes_np
        f2 = frame.repeat(2, axis=0)
        p2 = [before[0].repeat(2, axis=0), before[1], before[2]]
        a = over(shim, frame, before, fmt, e, True)
        b = planes_np(f2, p2, "yuv420p10", e, True)
        assert np.array_equal(a[0], b[0][0::2]) and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


# ---- refusals, byte counts and launches through the fake runtime ------------------------------------------------------------------
def test_refusals_byte_counts_and_launches(fake):
    L = fake
    L.fake_fail_at(-1)
    r, odd_h, odd_w = renderer(L, 64, 31), renderer(L, 66, 33), renderer(L, 63, 32)
    buf, buf2 = device_buf(L), device_buf(L)
    s = np.zeros(1, np.int32)
    one, uv = (C.c_void_p * 1)(buf.value), (C.c_void_p * 1)(buf2.value)

    def frames(h, d):
        return call(L, L.glava_b200_export_frames, h, s.ctypes.data, 1, one, C.byref(d), None, None)

    def scaled_call(h, d, size, dst_uv=None):
        return call(L, L.glava_b200_export_scaled, h, s.ctypes.data, 1, one, dst_uv, C.byref(d), C.byref(scale_of(size)), None, None)

    taken = [(r, YUV422P, 64, 0), (r, YUV422P10, 128, 0), (r, UYVY, 128, 0), (r, YUV422P, 96, 48 * 31 + 16),
             (r, YUV422P10, 128, 64 * 40), (odd_h, YUV422P, 96, 0), (odd_h, YUV422P10, 160, 0), (odd_h, UYVY, 144, 0)]
    for h, fmt, pitch, uvo in taken:                                   # 64x31 and 66x33: any height, w % 4 == 2
        for flags in (0, 0x100, 0x200, 0x300):
            rc, msg, trace, launched = frames(h, desc_of(fmt, pitch, flags, uv=uvo))
            assert rc == 0 and launched == 1 and len(memcpys(trace)) == 1, (fmt, pitch, flags, msg)
    refused = [  # (renderer, desc, what)
        (odd_w, desc_of(YUV422P, 64), "YUV422P needs an even width, the frame is 63x32"),
        (odd_w, desc_of(UYVY, 128), "UYVY needs an even width, the frame is 63x32"),
        (odd_w, desc_of(YUV422P10, 128), "YUV422P10 needs an even width"),
        (r, desc_of(YUV422P, 80), "YUV422P pitch 80 must be a multiple of 32"),
        (r, desc_of(YUV422P10, 144), "YUV422P10 pitch 144 must be a multiple of 32"),
        (r, desc_of(YUV422P10, 96), "at least 128"),
        (r, desc_of(UYVY, 112), "at least 128"),
        (r, desc_of(UYVY, 136), "multiple of 16"),
        (r, desc_of(YUV422P, 32), "at least 64"),
        (r, desc_of(YUV422P, 64, uv=8), "YUV422P uv_offset 8 (Cb plane to Cr plane)"),
        (r, desc_of(YUV422P, 64, uv=32 * 30), "one chroma plane, 992 bytes"),
        (r, desc_of(YUV422P10, 128, uv=64 * 31 + 8), "must be a multiple of 16"),
        (r, desc_of(UYVY, 128, uv=4096), "UYVY uv_offset 4096 must be 0"),
        (r, desc_of(3, 256), "unknown format 3"),
        (r, desc_of(9, 256), "unknown format 9"),
        (r, desc_of(13, 256), "unknown format 13"),
    ]
    for h, d, what in refused:
        rc, msg, trace, launched = frames(h, d)
        assert rc != 0 and "glava_b200_export_frames" in msg and what in msg, (what, msg)
        assert trace == "" and launched == 0, what
    # the scaled export: odd output widths refused, odd heights taken; dst_uv for the planar pair, not for UYVY
    rc, msg, trace, launched = scaled_call(r, desc_of(YUV422P10, 64), (15, 8))
    assert rc != 0 and "YUV422P10 needs an even width, the output is 15x8" in msg and launched == 0, msg
    for fmt, pitch in ((YUV422P, 32), (YUV422P10, 64), (UYVY, 32)):
        rc, msg, _, launched = scaled_call(r, desc_of(fmt, pitch), (16, 7))
        assert rc == 0 and launched == 1, (fmt, msg)
    for fmt, pitch in ((YUV422P, 32), (YUV422P10, 64)):
        rc, msg, _, launched = scaled_call(r, desc_of(fmt, pitch), (16, 7), uv)
        assert rc == 0 and launched == 1, (fmt, msg)
    rc, msg, trace, launched = scaled_call(r, desc_of(UYVY, 32), (16, 7), uv)
    assert rc != 0 and "UYVY has no chroma plane" in msg and trace == "" and launched == 0, msg
    # the overlay keeps its three formats and names the new ones
    for fmt, name in ((YUV422P, "YUV422P"), (YUV422P10, "YUV422P10"), (UYVY, "UYVY")):
        for flags in (0, 0x100):
            rc, msg, trace, launched = call(L, L.glava_b200_overlay_frames, r, s.ctypes.data, 1, one, None,
                                            C.byref(desc_of(fmt, 128, flags)), None, None)
            assert rc != 0 and f"format {name}: the overlay takes RGBA, BGRA or NV12" in msg and "unknown" not in msg, msg
            assert trace == "" and launched == 0
    # a ladder rung in a new format is checked as its scaled export; a dst_uv entry for a UYVY rung is refused
    three = (C.c_void_p * 3)(buf.value, buf.value, buf.value)
    pairs = [(desc_of(YUV422P10, 128), scale_of((64, 31))), (desc_of(RGBA, 64), scale_of((16, 8))),
             (desc_of(UYVY, 32, 0x300), scale_of((16, 9)))]
    rc, msg, _, launched = call(L, L.glava_b200_export_ladder, r, s.ctypes.data, 1, rungs_of(pairs), 3, three,
                                (C.c_void_p * 3)(buf2.value, None, None), None, None)
    assert rc == 0 and launched == 1, msg
    rc, msg, _, launched = call(L, L.glava_b200_export_ladder, r, s.ctypes.data, 1, rungs_of(pairs), 3, three,
                                (C.c_void_p * 3)(buf2.value, None, buf2.value), None, None)
    assert rc != 0 and "rung 2: dst_uv[2] is for NV12 only" in msg and launched == 0, msg
    rc, msg, _, launched = call(L, L.glava_b200_export_ladder, r, s.ctypes.data, 1,
                                rungs_of([(desc_of(YUV422P, 48), scale_of((16, 8)))]), 1, three, None, None, None)
    assert rc != 0 and "rung 0: YUV422P pitch 48" in msg and launched == 0, msg
    # byte counts: pitch * h + the Cb to Cr distance + one chroma plane; UYVY pitch * h
    n = C.c_size_t()
    for d, want_ in ((desc_of(YUV422P, 64), 64 * 31 + 2 * 32 * 31), (desc_of(YUV422P, 64, uv=4096), 64 * 31 + 4096 + 32 * 31),
                     (desc_of(YUV422P10, 128), 128 * 31 + 2 * 64 * 31), (desc_of(UYVY, 128), 128 * 31)):
        assert L.glava_b200_export_bytes(r, C.byref(d), C.byref(n)) == 0 and n.value == want_, (d.format, n.value, want_)
    assert L.glava_b200_export_scaled_bytes(r, C.byref(desc_of(YUV422P10, 64)), C.byref(scale_of((16, 7))), C.byref(n)) == 0
    assert n.value == 64 * 7 + 2 * 32 * 7
    assert L.glava_b200_export_scaled_bytes(r, C.byref(desc_of(UYVY, 32)), C.byref(scale_of((16, 7))), C.byref(n)) == 0
    assert n.value == 32 * 7
    assert L.glava_b200_export_bytes(odd_w, C.byref(desc_of(UYVY, 128)), C.byref(n)) != 0
    for h in (r, odd_h, odd_w):
        L.glava_b200_destroy(h)
    L.cudaFree(buf); L.cudaFree(buf2)
