"""A g++ build of export_core.h's BT.2020 HDR arithmetic (DESIGN 4.22) for the host and GPU tests: per-pixel codes, block
chroma, the linearisation table, the overlay blend, and host walks that lay whole pictures out plane by plane as the kernels
do, so that device bytes can be held to the host build bit for bit."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from tests.test_export_core import CSRC

P010, YUV420P10, YUV444P10, YUV422P10 = 6, 7, 8, 11
HDR_FORMATS = {P010: "p010", YUV420P10: "yuv420p10", YUV444P10: "yuv444p10", YUV422P10: "yuv422p10"}

SHIM = r"""
#include "export_core.h"
using namespace glb;
#define BOTH(name, params, args) \
    extern "C" void name params { if (E == GLB_ENC_PQ) name##_t<GLB_ENC_PQ> args; else name##_t<GLB_ENC_HLG> args; }

extern "C" float hdr_lin_c(int v) { return hdr_lin((uint32_t) v); }
// per pixel: Y, Cb, Cr codes and the unrounded values
template <int E> static void codes_t(const uint32_t* c, size_t n, uint16_t* y, uint16_t* cb, uint16_t* cr, float* f) {
    for (size_t i = 0; i < n; ++i) {
        const uint32_t uv = export_cbcr10_px<E>(c[i]);
        y[i] = (uint16_t) export_y10<E>(c[i]); cb[i] = uv & 0xffffu; cr[i] = uv >> 16;
        if (f) { const HdrRgb e = hdr_rgb<E>(c[i]); f[3 * i] = hdr_yf(e); f[3 * i + 1] = hdr_cbf(e); f[3 * i + 2] = hdr_crf(e); }
    }
}
BOTH(codes, (int E, const uint32_t* c, size_t n, uint16_t* y, uint16_t* cb, uint16_t* cr, float* f), (c, n, y, cb, cr, f))
// chroma of 2x2 blocks q[4 i .. 4 i + 3] (a, b top row)
template <int E> static void blocks_t(const uint32_t* q, size_t n, uint16_t* cb, uint16_t* cr) {
    for (size_t i = 0; i < n; ++i) {
        const uint32_t uv = export_block10<E>(q[4 * i], q[4 * i + 1], q[4 * i + 2], q[4 * i + 3]);
        cb[i] = uv & 0xffffu; cr[i] = uv >> 16;
    }
}
BOTH(blocks, (int E, const uint32_t* q, size_t n, uint16_t* cb, uint16_t* cr), (q, n, cb, cr))
// overlay primitives: Y of px[i] over yd[i]; chroma of the block q[4 i ..] over (cbd, crd)[i]
template <int E> static void over_t(const uint32_t* px, const uint16_t* yd, size_t n, const uint32_t* q, const uint16_t* cd,
                                    size_t nb, uint16_t* y, uint16_t* cb, uint16_t* cr) {
    for (size_t i = 0; i < n; ++i) y[i] = (uint16_t) hdr_over_y(hdr_px<E>(px[i]), yd[i]);
    for (size_t i = 0; i < nb; ++i) {
        const uint32_t uv = hdr_over_cbcr(hdr_px<E>(q[4 * i]), hdr_px<E>(q[4 * i + 1]), hdr_px<E>(q[4 * i + 2]), hdr_px<E>(q[4 * i + 3]),
                                          cd[2 * i], cd[2 * i + 1]);
        cb[i] = uv & 0xffffu; cr[i] = uv >> 16;
    }
}
BOTH(over, (int E, const uint32_t* px, const uint16_t* yd, size_t n, const uint32_t* q, const uint16_t* cd, size_t nb, uint16_t* y,
            uint16_t* cb, uint16_t* cr), (px, yd, n, q, cd, nb, y, cb, cr))

// A whole picture, top-down composited pixels img[h][w] -> the planes of `format` (uint16 samples; P010 y << 6 and
// interleaved CbCr << 6), every sample the per-pixel / per-block host function
template <int E> static void planes_t(int format, const uint32_t* img, int w, int h, uint16_t* y, uint16_t* cb, uint16_t* cr) {
    for (int r = 0; r < h; ++r)
        for (int x = 0; x < w; ++x) {
            const uint32_t v = export_y10<E>(img[(size_t) r * w + x]);
            y[(size_t) r * w + x] = (uint16_t) (format == GLAVA_B200_EXPORT_P010 ? v << 6 : v);
        }
    if (format == GLAVA_B200_EXPORT_YUV444P10) {
        for (size_t i = 0; i < (size_t) w * h; ++i) { const uint32_t uv = export_cbcr10_px<E>(img[i]); cb[i] = uv & 0xffffu; cr[i] = uv >> 16; }
        return;
    }
    const bool c420 = format != GLAVA_B200_EXPORT_YUV422P10;
    for (int r = 0; r < (c420 ? h / 2 : h); ++r)
        for (int x = 0; x < w / 2; ++x) {
            const uint32_t* t = img + (size_t) (c420 ? 2 * r : r) * w + 2 * x;
            const uint32_t* b = c420 ? t + w : t;
            const uint32_t uv = export_block10<E>(t[0], t[1], b[0], b[1]);
            const size_t o = (size_t) r * (w / 2) + x;
            if (format == GLAVA_B200_EXPORT_P010) { cb[2 * o] = (uint16_t) ((uv & 0xffffu) << 6); cb[2 * o + 1] = (uint16_t) ((uv >> 16) << 6); }
            else { cb[o] = uv & 0xffffu; cr[o] = uv >> 16; }
        }
}
BOTH(planes, (int E, int format, const uint32_t* img, int w, int h, uint16_t* y, uint16_t* cb, uint16_t* cr), (format, img, w, h, y, cb, cr))

// The native overlay of top-down stored pixels px[h][w] (w a multiple of 4) onto planes held as uint16 samples (P010: Y and
// the interleaved CbCr plane in y / cb), walked in the kernels' quads through the overlay quad functions
template <int E> static void overlay_t(int format, const uint32_t* px, int w, int h, uint16_t* y, uint16_t* cb, uint16_t* cr) {
    auto word = [](const uint16_t* p) { return (uint32_t) p[0] | ((uint32_t) p[1] << 16); };
    auto put = [](uint16_t* p, uint32_t v) { p[0] = (uint16_t) v; p[1] = (uint16_t) (v >> 16); };
    const int cw = format == GLAVA_B200_EXPORT_YUV444P10 ? w : w / 2;
    for (int r = 0; r < h; r += (format == GLAVA_B200_EXPORT_P010 || format == GLAVA_B200_EXPORT_YUV420P10) ? 2 : 1)
        for (int x = 0; x < w; x += 4) {
            const uint32_t* q = px + (size_t) r * w + x;
            uint16_t* py = y + (size_t) r * w + x;
            if (format == GLAVA_B200_EXPORT_YUV444P10) {
                uint32_t yy[2] = { word(py), word(py + 2) }, u[2], v[2];
                uint16_t* pu = cb + (size_t) r * cw + x; uint16_t* pv = cr + (size_t) r * cw + x;
                u[0] = word(pu); u[1] = word(pu + 2); v[0] = word(pv); v[1] = word(pv + 2);
                overlay_444p10_quad<E>(q, yy, u, v);
                put(py, yy[0]); put(py + 2, yy[1]); put(pu, u[0]); put(pu + 2, u[1]); put(pv, v[0]); put(pv + 2, v[1]);
            } else if (format == GLAVA_B200_EXPORT_YUV422P10) {
                uint32_t yy[2] = { word(py), word(py + 2) };
                uint16_t* pu = cb + (size_t) r * cw + x / 2; uint16_t* pv = cr + (size_t) r * cw + x / 2;
                uint32_t u = word(pu), v = word(pv);
                overlay_422p10_quad<E>(q, yy, &u, &v);
                put(py, yy[0]); put(py + 2, yy[1]); put(pu, u); put(pv, v);
            } else {
                const bool msb = format == GLAVA_B200_EXPORT_P010;
                uint32_t yt[2] = { word(py), word(py + 2) }, yb[2] = { word(py + w), word(py + w + 2) }, uv[2];
                uint16_t* pu = msb ? cb + (size_t) (r / 2) * w + x : cb + (size_t) (r / 2) * cw + x / 2;
                uint16_t* pv = cr + (size_t) (r / 2) * cw + x / 2;
                if (msb) { uv[0] = word(pu); uv[1] = word(pu + 2); overlay_p10_quad<E, true>(q, q + w, yt, yb, uv); put(pu, uv[0]); put(pu + 2, uv[1]); }
                else { uv[0] = word(pu); uv[1] = word(pv); overlay_p10_quad<E, false>(q, q + w, yt, yb, uv); put(pu, uv[0]); put(pv, uv[1]); }
                put(py, yt[0]); put(py + 2, yt[1]); put(py + w, yb[0]); put(py + w + 2, yb[1]);
            }
        }
}
BOTH(overlay, (int E, int format, const uint32_t* px, int w, int h, uint16_t* y, uint16_t* cb, uint16_t* cr), (format, px, w, h, y, cb, cr))
"""

_LIB = None


def lib():
    """the shim, built once per process"""
    global _LIB
    if _LIB is None:
        d = tempfile.mkdtemp(prefix="glava_hdr_shim_")
        src, so = os.path.join(d, "hdr.cpp"), os.path.join(d, "libhdr.so")
        with open(src, "w") as f:
            f.write(SHIM)
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I", CSRC,
                        "-I", os.path.join(CSRC, "..", "..", "include"), "-o", so, src], check=True)
        _LIB = C.CDLL(so)
        _LIB.hdr_lin_c.restype = C.c_float
        _LIB.hdr_lin_c.argtypes = [C.c_int]
    return _LIB


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def codes(e, c, with_float=False):
    """per-pixel (Y, Cb, Cr) codes of uint32 triples c (and the unrounded float32 [n, 3])"""
    c = np.ascontiguousarray(c, np.uint32).reshape(-1)
    y, cb, cr = (np.empty(c.size, np.uint16) for _ in range(3))
    f = np.empty((c.size, 3), np.float32) if with_float else None
    lib().codes(e, _p(c), C.c_size_t(c.size), _p(y), _p(cb), _p(cr), _p(f))
    return (y, cb, cr, f) if with_float else (y, cb, cr)


def blocks(e, q):
    """chroma codes of blocks q [n, 4] (top-left, top-right, bottom-left, bottom-right)"""
    q = np.ascontiguousarray(q, np.uint32)
    cb, cr = np.empty(q.shape[0], np.uint16), np.empty(q.shape[0], np.uint16)
    lib().blocks(e, _p(q), C.c_size_t(q.shape[0]), _p(cb), _p(cr))
    return cb, cr


def over(e, px, yd, q, cd):
    """overlay Y of px [n] over yd [n]; chroma of blocks q [m, 4] over cd [m, 2]"""
    px, yd = np.ascontiguousarray(px, np.uint32), np.ascontiguousarray(yd, np.uint16)
    q, cd = np.ascontiguousarray(q, np.uint32), np.ascontiguousarray(cd, np.uint16)
    y = np.empty(px.size, np.uint16)
    cb, cr = np.empty(q.shape[0], np.uint16), np.empty(q.shape[0], np.uint16)
    lib().over(e, _p(px), _p(yd), C.c_size_t(px.size), _p(q), _p(cd), C.c_size_t(q.shape[0]), _p(y), _p(cb), _p(cr))
    return y, cb, cr


def chroma_shape(fmt, w, h):
    """(rows, cols) of one chroma plane in samples (P010: the interleaved plane)"""
    return {P010: (h // 2, w), YUV420P10: (h // 2, w // 2), YUV444P10: (h, w), YUV422P10: (h, w // 2)}[fmt]


def planes(e, fmt, img):
    """the expected planes of top-down composited pixels img [h, w] (uint32): (Y, Cb, Cr) uint16 arrays, P010 (Y, CbCr)"""
    img = np.ascontiguousarray(img, np.uint32)
    h, w = img.shape
    y = np.empty((h, w), np.uint16)
    cb, cr = np.zeros(chroma_shape(fmt, w, h), np.uint16), np.zeros(chroma_shape(fmt, w, h), np.uint16)
    lib().planes(e, fmt, _p(img), w, h, _p(y), _p(cb), _p(cr))
    return (y, cb) if fmt == P010 else (y, cb, cr)


def overlay(e, fmt, px, pl):
    """the native overlay of top-down stored pixels px [h, w] (uint32) onto copies of the planes pl (uint16 arrays as
    planes() lays them out); returns the new planes"""
    px = np.ascontiguousarray(px, np.uint32)
    h, w = px.shape
    y = np.ascontiguousarray(pl[0], np.uint16).copy()
    cb = np.ascontiguousarray(pl[1], np.uint16).copy()
    cr = np.ascontiguousarray(pl[2], np.uint16).copy() if len(pl) > 2 else np.zeros(1, np.uint16)
    lib().overlay(e, fmt, _p(px), w, h, _p(y), _p(cb), _p(cr))
    return (y, cb) if fmt == P010 else (y, cb, cr)


def pack(rgba):
    """[..., 4] uint8 -> uint32 0xAABBGGRR"""
    a = np.asarray(rgba).astype(np.uint32)
    return a[..., 0] | (a[..., 1] << 8) | (a[..., 2] << 16) | (a[..., 3] << 24)
