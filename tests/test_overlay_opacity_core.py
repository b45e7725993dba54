"""The overlay at a per-entry opacity (glava_b200_overlay_frames_opacity / glava_b200_overlay_planes_opacity, DESIGN 4.20) on
the host: export_core.h fade_px exhaustively over (c, K) with its identities; every native blend helper at K = 255 and K = 0;
the measured float64 bounds of the faded composite per format and encoding; a g++ walk of the fade kernels' items
(overlay_walk driving OverlayFadeBody: band items under live marks, row-pair items under stale or absent marks and under
any other opacity) for every overlay format bit for bit against the plain overlay's numpy restatements applied to the
pre-scaled frame, over sentinel-filled planes; and the refusals, list sizes and launches of the two calls through capi.cu,
export.cpp and overlay_planes.cpp built against the fake runtime of tests/fakecuda."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from tests import export_fake, fakecuda
from tests.export_422_np import overlay422_np
from tests.export_fake import desc_of
from tests.overlay_planes_np import planes_np
from tests.test_export_core import BGRA, CSRC, NV12, RGBA, marked_frame, pack, premultiplied
from tests.test_export_matrix_core import kr_kb
from tests.test_overlay_core import mul_norm8_np, overlay_np
from tests.test_overlay_planes_core import PLANES_STUBS

I420, YUV444, P010, YUV420P10, YUV444P10, YUV422P, YUV422P10, UYVY = 4, 5, 6, 7, 8, 10, 11, 12
NAME = {NV12: "nv12", I420: "i420", YUV444: "yuv444", P010: "p010", YUV420P10: "yuv420p10", YUV444P10: "yuv444p10",
        YUV422P: "yuv422p", YUV422P10: "yuv422p10", UYVY: "uyvy"}
C420 = (NV12, I420, P010, YUV420P10)
WIDE = (P010, YUV420P10, YUV444P10, YUV422P10)
K_SET = (0, 1, 37, 128, 254, 255)

SHIM = r"""
#include "export_core.h"
#include <algorithm>
#include <cstring>
using namespace glb;
extern "C" void t_fade_px(const uint32_t* px, const uint32_t* k, size_t n, uint32_t* out) {
    for (size_t i = 0; i < n; ++i) out[i] = fade_px(px[i], k[i]);
}
extern "C" void t_fade_opaque(const uint32_t* px, const uint32_t* k, size_t n, uint32_t* out) {
    for (size_t i = 0; i < n; ++i) out[i] = fade_opaque(px[i], k[i]);
}
extern "C" void t_overlay_px(const uint32_t* px, const uint32_t* d, size_t n, uint32_t* out) {
    for (size_t i = 0; i < n; ++i) out[i] = overlay_px(px[i], d[i]);
}
template <int E> static void y8(const uint32_t* px, const uint32_t* yd, size_t n, uint32_t* out) {
    for (size_t i = 0; i < n; ++i) out[i] = overlay_y<E>(px[i], yd[i]);
}
template <int E> static void c8(const uint32_t* m, const uint32_t* uvd, size_t n, uint32_t* out) {
    for (size_t i = 0; i < n; ++i) out[i] = overlay_cbcr<E>(m[i], uvd[i]);
}
template <int E> static void y10(const uint32_t* px, const uint32_t* yd, size_t n, uint32_t* out) {
    for (size_t i = 0; i < n; ++i) out[i] = overlay_y10<E>(px[i], yd[i]);
}
template <int E> static void c10(const uint32_t* s, const uint32_t* sa, const uint32_t* vd, size_t n, uint32_t* out) {
    for (size_t i = 0; i < n; ++i) out[i] = overlay_cbcr10<E>(s[i], sa[i], vd[i] & 0xffffu, vd[i] >> 16);
}

// ---- the fade kernels' walk: overlay_walk over OverlayFadeBody, restated with memcpy for the device's loads and stores --------
struct Walk {
    const uint32_t* fb; int w, h; const uint32_t* marks; int rows, fmt, native; uint32_t k;
    uint8_t *p0, *p1, *p2; size_t P, CP;
    static bool any(const uint32_t* q, int n) { for (int i = 0; i < n; ++i) if (q[i]) return true; return false; }
    uint32_t ld(const uint8_t* p, int n) const { uint32_t v = 0u; memcpy(&v, p, n); return v; }
    void ld2(const uint8_t* p, uint32_t v[2], int n) const { v[0] = v[1] = 0u; memcpy(v, p, n); }
    template <int E> void row(int r, int x, const uint32_t q[4]) const {     // native: the scaled quad onto output row r
        if (!any(q, 4)) return;
        const int n = std::min(4, w - x), nf = x + 4 <= w ? 4 : 2;
        if (fmt == GLAVA_B200_EXPORT_RGBA || fmt == GLAVA_B200_EXPORT_BGRA) {
            for (int i = 0; i < n; ++i) {
                uint8_t* d = p0 + r * P + 4 * (size_t) (x + i);
                uint32_t v = ld(d, 4);
                v = overlay_px(fmt == GLAVA_B200_EXPORT_BGRA ? export_swap_rb(q[i]) : q[i], v);
                memcpy(d, &v, 4);
            }
        } else if (fmt == GLAVA_B200_EXPORT_YUV444) {
            uint8_t *py = p0 + r * P + x, *pu = p1 + r * CP + x, *pv = p2 + r * CP + x;
            uint32_t y = ld(py, n), u = ld(pu, n), v = ld(pv, n);
            overlay_444_quad<E>(q, &y, &u, &v);
            memcpy(py, &y, n); memcpy(pu, &u, n); memcpy(pv, &v, n);
        } else if (fmt == GLAVA_B200_EXPORT_YUV444P10) {
            uint8_t *py = p0 + r * P + 2 * x, *pu = p1 + r * CP + 2 * x, *pv = p2 + r * CP + 2 * x;
            uint32_t y[2], u[2], v[2];
            ld2(py, y, 2 * n); ld2(pu, u, 2 * n); ld2(pv, v, 2 * n);
            overlay_444p10_quad<E>(q, y, u, v);
            memcpy(py, y, 2 * n); memcpy(pu, u, 2 * n); memcpy(pv, v, 2 * n);
        } else if (fmt == GLAVA_B200_EXPORT_YUV422P) {
            uint8_t *py = p0 + r * P + x, *pu = p1 + r * CP + x / 2, *pv = p2 + r * CP + x / 2;
            uint32_t y = ld(py, nf), u = ld(pu, nf / 2), v = ld(pv, nf / 2);
            uint32_t uv = (u & 0xffu) | ((v & 0xffu) << 8) | ((u & 0xff00u) << 8) | ((v & 0xff00u) << 16);
            overlay_422_quad<E>(q, &y, &uv);
            u = export_cb_pair(uv); v = export_cr_pair(uv);
            memcpy(py, &y, nf); memcpy(pu, &u, nf / 2); memcpy(pv, &v, nf / 2);
        } else if (fmt == GLAVA_B200_EXPORT_YUV422P10) {
            uint8_t *py = p0 + r * P + 2 * x, *pu = p1 + r * CP + x, *pv = p2 + r * CP + x;
            uint32_t y[2], u = ld(pu, nf), v = ld(pv, nf);
            ld2(py, y, 2 * nf);
            overlay_422p10_quad<E>(q, y, &u, &v);
            memcpy(py, y, 2 * nf); memcpy(pu, &u, nf); memcpy(pv, &v, nf);
        } else {                                                            // UYVY
            uint8_t* p = p0 + r * P + 2 * x;
            uint32_t wd[2], y, uv;
            ld2(p, wd, 2 * nf);
            export_uyvy_split(wd, &y, &uv);
            overlay_422_quad<E>(q, &y, &uv);
            export_uyvy_words(y, uv, wd);
            memcpy(p, wd, 2 * nf);
        }
    }
    template <int E> void pair(int j, int x, const uint32_t t[4], const uint32_t b[4]) const {   // native: rows 2j, 2j + 1
        uint32_t all[8];
        for (int i = 0; i < 4; ++i) { all[i] = t[i]; all[4 + i] = b[i]; }
        if (!any(all, 8)) return;
        const int n = x + 4 <= w ? 4 : 2;
        uint8_t* r0 = p0 + (size_t) (2 * j) * P;
        uint8_t* cj = p1 + (size_t) j * CP;
        if (fmt == GLAVA_B200_EXPORT_NV12) {
            uint32_t yt = ld(r0 + x, n), yb = ld(r0 + P + x, n), c = ld(cj + x, n);
            overlay_nv12_quad<E>(t, b, &yt, &yb, &c);
            memcpy(r0 + x, &yt, n); memcpy(r0 + P + x, &yb, n); memcpy(cj + x, &c, n);
        } else if (fmt == GLAVA_B200_EXPORT_I420) {
            uint8_t *pu = cj + x / 2, *pv = p2 + (size_t) j * CP + x / 2;
            uint32_t yt = ld(r0 + x, n), yb = ld(r0 + P + x, n), u = ld(pu, n / 2), v = ld(pv, n / 2);
            overlay_i420_quad<E>(t, b, &yt, &yb, &u, &v);
            memcpy(r0 + x, &yt, n); memcpy(r0 + P + x, &yb, n); memcpy(pu, &u, n / 2); memcpy(pv, &v, n / 2);
        } else {
            const bool msb = fmt == GLAVA_B200_EXPORT_P010;
            uint8_t *py = r0 + 2 * x, *pu = msb ? cj + 2 * x : cj + x, *pv = msb ? nullptr : p2 + (size_t) j * CP + x;
            uint32_t yt[2], yb[2], uv[2] = { 0u, 0u };
            ld2(py, yt, 2 * n); ld2(py + P, yb, 2 * n);
            if (msb) ld2(pu, uv, 2 * n);
            else { uv[0] = ld(pu, n); uv[1] = ld(pv, n); }
            if (msb) overlay_p10_quad<E, true>(t, b, yt, yb, uv);
            else overlay_p10_quad<E, false>(t, b, yt, yb, uv);
            memcpy(py, yt, 2 * n); memcpy(py + P, yb, 2 * n);
            if (msb) memcpy(pu, uv, 2 * n);
            else { memcpy(pu, &uv[0], n); memcpy(pv, &uv[1], n); }
        }
    }
    template <int E> void run(bool band) const {
        const bool pairs = fmt == GLAVA_B200_EXPORT_NV12 || fmt == GLAVA_B200_EXPORT_I420 || fmt == GLAVA_B200_EXPORT_P010 ||
                           fmt == GLAVA_B200_EXPORT_YUV420P10;
        const int strips = (w + 127) >> 7;
        auto mark = [&](int y, int s) { return marks[export_mark_index(0, w, h, rows, y, s)]; };
        auto load = [&](int y, int x, uint32_t q[4]) { for (int i = 0; i < 4; ++i) q[i] = x + i < w ? fb[(size_t) y * w + x + i] : 0u; };
        auto scale = [&](bool nat, const uint32_t q[4], uint32_t s[4]) { for (int i = 0; i < 4; ++i) s[i] = nat ? fade_px(q[i], k) : fade_opaque(q[i], k); };
        const int R = band ? rows : 2;
        for (int u = 0; u < (h + R - 1) / R; ++u)
            for (int strip = 0; strip < strips; ++strip)
                for (int lane = 0; lane < 32; ++lane) {
                    const int x = strip * 128 + lane * 4;
                    if (x >= w) continue;
                    uint32_t top[4] = { 0u, 0u, 0u, 0u }, bot[4] = { 0u, 0u, 0u, 0u }, st[4], sb[4];
                    if (band) {
                        const int b0 = u * rows, b1 = std::min(b0 + rows, h);
                        const uint32_t m = mark(b0, strip);
                        const int lo = std::max((int) (m & 0xffffu), b0), hi = std::min((int) (m >> 16), b1);
                        if (lo >= hi) continue;
                        if (!pairs) {
                            for (int y = lo; y < hi; ++y) { load(y, x, top); scale(true, top, st); row<E>(h - 1 - y, x, st); }
                            continue;
                        }
                        int ja, jb;
                        const uint32_t below = overlay_band_pairs(h, b0, lo, hi, &ja, &jb) ? mark(b0 - 1, strip) : 0u;
                        if (overlay_top_straddles(h, b1, ja) && export_row_read(mark(b1, strip), b1)) ++ja;
                        for (int j = ja; j < jb; ++j) {
                            const int y0 = h - 1 - 2 * j, y1 = y0 - 1;
                            uint32_t t[4] = { 0u, 0u, 0u, 0u }, b[4] = { 0u, 0u, 0u, 0u };
                            if (y0 >= lo && y0 < hi) load(y0, x, t);
                            if (y1 >= b0 ? y1 >= lo && y1 < hi : export_row_read(below, y1)) load(y1, x, b);
                            scale(true, t, st); scale(true, b, sb);
                            pair<E>(j, x, st, sb);
                        }
                        continue;
                    }
                    const int y0 = h - 1 - 2 * u, y1 = y0 - 1;
                    if (!marks || export_row_read(mark(y0, strip), y0)) load(y0, x, top);
                    if (y1 >= 0 && (!marks || export_row_read(mark(y1, strip), y1))) load(y1, x, bot);
                    scale(native, top, st); scale(native, bot, sb);
                    if (pairs) pair<E>(u, x, st, sb);
                    else { row<E>(2 * u, x, st); if (y1 >= 0) row<E>(2 * u + 1, x, sb); }
                }
    }
};
extern "C" void t_fade_walk(const uint32_t* fb, int w, int h, const uint32_t* marks, int rows, int fmt, int e, int native, int band,
                            uint32_t k, uint8_t* p0, uint8_t* p1, uint8_t* p2, size_t P, size_t CP) {
    const Walk W = { fb, w, h, marks, rows, fmt, native, k, p0, p1, p2, P, CP };
    if (e == 0) W.run<0>(band); else if (e == 1) W.run<1>(band); else if (e == 2) W.run<2>(band); else W.run<3>(band);
}
"""
for _n, _args, _call in (("y8", "const uint32_t* a, const uint32_t* b, size_t n, uint32_t* out", "y8<E>(a, b, n, out)"),
                         ("c8", "const uint32_t* a, const uint32_t* b, size_t n, uint32_t* out", "c8<E>(a, b, n, out)"),
                         ("y10", "const uint32_t* a, const uint32_t* b, size_t n, uint32_t* out", "y10<E>(a, b, n, out)"),
                         ("c10", "const uint32_t* a, const uint32_t* b, const uint32_t* c, size_t n, uint32_t* out",
                          "c10<E>(a, b, c, n, out)")):
    SHIM += f'extern "C" void t_{_n}(int e, {_args}) {{\n'
    SHIM += "".join(f"    if (e == {E}) {{ constexpr int E = {E}; {_call}; }}\n" for E in range(4)) + "}\n"


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("overlay_opacity_core")
    src, so = d / "shim.cpp", d / "shim.so"
    src.write_text(SHIM)
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I", CSRC,
                    "-I", CSRC + "/../../include", "-include", "cstdint", "-include", "cstddef", "-o", str(so), str(src)], check=True)
    L = C.CDLL(str(so))
    vp, i32, sz = C.c_void_p, C.c_int, C.c_size_t
    L.t_fade_walk.argtypes = [vp, i32, i32, vp, i32, i32, i32, i32, i32, C.c_uint32, vp, vp, vp, sz, sz]
    return L


def call(fn, *arrays, e=None):
    arrays = [np.ascontiguousarray(a, np.uint32) for a in arrays]
    out = np.zeros(arrays[0].size, np.uint32)
    head = [C.c_int(e)] if e is not None else []
    fn(*head, *[C.c_void_p(a.ctypes.data) for a in arrays], C.c_size_t(out.size), C.c_void_p(out.ctypes.data))
    return out


def fade_np(frame, k, native):
    """the pixels the fade composites: every channel of the stored pixel (alpha 255 under any other opacity) times K / 255
    in the unorm8 product; frame [..., 4] uint8, k a scalar"""
    c = frame.astype(np.int64)
    if not native:
        c = c.copy()
        c[..., 3] = 255
    return mul_norm8_np(c, int(k)).astype(np.uint8)


# ---- fade_px --------------------------------------------------------------------------------------------------------------------
def test_fade_px_every_channel_and_opacity(shim):
    """all 2^16 (x, K) pairs in each channel position; the identities K = 255 and K = 0; c <= a is kept; fade_opaque is
    fade_px of the pixel with alpha 255"""
    x, k = (v.reshape(-1).astype(np.uint32) for v in np.meshgrid(np.arange(256), np.arange(256), indexing="ij"))
    want = mul_norm8_np(x.astype(np.int64), k.astype(np.int64))
    assert np.array_equal(want, np.floor(x.astype(np.float64) * k / 255 + 0.5))        # the unorm8 product is round(x K / 255)
    for ch in range(4):
        got = call(shim.t_fade_px, x << (8 * ch), k)
        assert np.array_equal(got, want.astype(np.uint32) << (8 * ch)), ch
    rng = np.random.default_rng(1)
    P = premultiplied(rng, (1 << 16,)).astype(np.uint32)
    px = pack(P[:, 0], P[:, 1], P[:, 2], P[:, 3])
    assert np.array_equal(call(shim.t_fade_px, px, np.full(px.size, 255)), px)
    assert not call(shim.t_fade_px, px, np.zeros(px.size)).any()
    kk = rng.integers(0, 256, px.size)
    f = call(shim.t_fade_px, px, kk)
    assert all(((f >> (8 * c)) & 255 <= f >> 24).all() for c in range(3))              # still premultiplied
    assert np.array_equal(call(shim.t_fade_opaque, px, kk), call(shim.t_fade_px, px | 0xFF000000, kk))
    assert np.array_equal(call(shim.t_fade_opaque, px, np.full(px.size, 255)), px | 0xFF000000)


@pytest.mark.parametrize("e", range(4))
def test_every_blend_helper_at_full_and_zero_opacity(shim, e):
    """K = 255 feeds every native blend the pixel itself, K = 0 a zero pixel, which leaves every destination as it was"""
    rng = np.random.default_rng(40 + e)
    P = premultiplied(rng, (1 << 14,)).astype(np.uint32)
    px = pack(P[:, 0], P[:, 1], P[:, 2], P[:, 3])
    full = call(shim.t_fade_px, px, np.full(px.size, 255))
    zero = call(shim.t_fade_px, px, np.zeros(px.size))
    d = rng.integers(0, 1 << 32, px.size, dtype=np.uint64).astype(np.uint32)
    d8, d16 = d & 0xFFFF, d & 0x3FF03FF
    assert np.array_equal(call(shim.t_overlay_px, full, d), call(shim.t_overlay_px, px, d))
    assert np.array_equal(call(shim.t_overlay_px, zero, d), d)
    assert np.array_equal(call(shim.t_y8, full, d & 255, e=e), call(shim.t_y8, px, d & 255, e=e))
    assert np.array_equal(call(shim.t_y8, zero, d & 255, e=e), d & 255)
    assert np.array_equal(call(shim.t_c8, zero, d8, e=e), d8)
    assert np.array_equal(call(shim.t_y10, zero, d & 1023, e=e), d & 1023)
    assert np.array_equal(call(shim.t_c10, zero, zero, d16, e=e), d16)


# ---- float64 bounds -------------------------------------------------------------------------------------------------------------
# The bound of each blend against float64 of c K / 255 + D (1 - a K / 255^2), in code values of the output, per encoding
# (DESIGN 4.20).  RGBA is exact (every c <= a, K and D); the Y'CbCr ones are the maxima over the 2^20 seeded samples of
# test_ycbcr_bounds_against_float64, pinned to 1e-4.  At 10 bits the 8-bit rounding of the faded colour and alpha is
# worth four 10-bit codes per 8-bit step, so those bounds are about four times the 8-bit ones.
BOUND_RGBA = 1.4922
BOUND_Y8 = (1.3140, 1.3903, 1.2868, 1.3934)
BOUND_C8 = (1.1109, 1.1652, 1.1000, 1.1466)
BOUND_Y10 = (3.7981, 4.4115, 3.6937, 4.2429)
BOUND_C10 = (3.0739, 3.1510, 3.0189, 3.3374)


def float_ycc(e, bits, c, al, VD, what):
    """float64 composite code of colour c [..., 3] (already times K / 255, premultiplied) at coverage al over codes VD"""
    kr, kb = kr_kb(e)
    full = bool(e & 1)
    top = 1023 if bits == 10 else 255
    ys = top / 255 if full else (876 if bits == 10 else 219) / 255
    cs = top / 255 if full else (896 if bits == 10 else 224) / 255
    yoff = 0 if full else (64 if bits == 10 else 16)
    coff = 512 if bits == 10 else 128
    r, g, b = c[..., 0], c[..., 1], c[..., 2]
    yp = kr * r + (1 - kr - kb) * g + kb * b
    if what == "y":
        v = yoff * al + ys * yp
    elif what == "cb":
        v = coff * al + cs * (b - yp) / (2 * (1 - kb))
    else:
        v = coff * al + cs * (r - yp) / (2 * (1 - kr))
    return np.clip(v + (1 - al) * VD, 0, top)


def sample_fade(rng, n):
    P = premultiplied(rng, (n,)).astype(np.int64)
    P[::5, :3] = P[::5, 3:4]                                                 # colour at alpha
    k = rng.integers(1, 255, n)
    k[::7] = 128
    return P, k


def test_rgba_bound_against_float64():
    """exact over every (c <= a, K, D): the error is e1(c, K) + g(a, K, D), e1 = mul_norm8(c, K) - c K / 255 and g =
    mul_norm8(D, 255 - mul_norm8(a, K)) - D (1 - a K / 255^2), and no sum passes 255 (c' <= a'), so its extremes are the
    extremes of e1 over c <= a plus those of g over D"""
    x = np.arange(256)
    c, K = np.meshgrid(x, x, indexing="ij")
    e1 = mul_norm8_np(c, K) - c * K / 255.0
    hi1, lo1 = np.maximum.accumulate(e1, axis=0), np.minimum.accumulate(e1, axis=0)   # [a, K]: over c <= a
    worst = 0.0
    D = x[:, None]
    for a in range(256):
        g = mul_norm8_np(D, 255 - mul_norm8_np(a, x)[None, :]) - D * (1 - a * x[None, :] / 255.0 ** 2)   # [D, K]
        worst = max(worst, (hi1[a] + g.max(axis=0)).max(), -(lo1[a] + g.min(axis=0)).min())
    assert abs(worst - BOUND_RGBA) < 1e-4, worst


@pytest.mark.parametrize("e", range(4))
def test_ycbcr_bounds_against_float64(shim, e):
    """Y and per-pixel chroma (YUV 4:4:4) at 8 and 10 bits; 4:2:0 / 4:2:2 chroma adds only the plain overlay's block
    average to these (DESIGN 4.17, 4.18)"""
    rng = np.random.default_rng(100 + e)
    P, k = sample_fade(rng, 1 << 20)
    px = pack(P[:, 0], P[:, 1], P[:, 2], P[:, 3])
    f = call(shim.t_fade_px, px, k)
    c, al = P[:, :3] * k[:, None] / 255, P[:, 3] * k / 255 ** 2
    v8 = rng.integers(0, 256, (px.size, 2))
    v10 = rng.integers(0, 1024, (px.size, 2))
    y8 = call(shim.t_y8, f, v8[:, 0], e=e)
    c8 = call(shim.t_c8, f, v8[:, 0] | (v8[:, 1] << 8), e=e)
    y10 = call(shim.t_y10, f, v10[:, 0], e=e)
    fi = np.stack([(f >> (8 * ch)) & 255 for ch in range(4)], 1).astype(np.int64)
    s = 4 * fi
    c10 = call(shim.t_c10, s[:, 0] | (s[:, 1] << 10) | (s[:, 2] << 20), s[:, 3], v10[:, 0] | (v10[:, 1] << 16), e=e)
    worst = lambda got, *want: max(np.abs(g - w).max() for g, w in zip(got, want))
    errs = (worst([y8], float_ycc(e, 8, c, al, v8[:, 0], "y")),
            worst([c8 & 255, c8 >> 8], float_ycc(e, 8, c, al, v8[:, 0], "cb"), float_ycc(e, 8, c, al, v8[:, 1], "cr")),
            worst([y10], float_ycc(e, 10, c, al, v10[:, 0], "y")),
            worst([c10 & 0xFFFF, c10 >> 16], float_ycc(e, 10, c, al, v10[:, 0], "cb"), float_ycc(e, 10, c, al, v10[:, 1], "cr")))
    for err, bound in zip(errs, (BOUND_Y8[e], BOUND_C8[e], BOUND_Y10[e], BOUND_C10[e])):
        assert abs(err - bound) < 1e-4, (errs, e)


# ---- the kernels' walk ----------------------------------------------------------------------------------------------------------
def plane_shapes(fmt, w, h):
    """[(rows, row bytes)] of the rectangle's planes"""
    if fmt in (RGBA, BGRA):
        return [(h, 4 * w)]
    if fmt == UYVY:
        return [(h, 2 * w)]
    sb = 2 if fmt in WIDE else 1
    luma = (h, sb * w)
    if fmt in (NV12, P010):
        return [luma, (h // 2, sb * w)]
    cw = w // 2 if fmt in (I420, YUV420P10, YUV422P, YUV422P10) else w
    ch = h // 2 if fmt in C420 else h
    return [luma, (ch, sb * cw), (ch, sb * cw)]


def walk(L, frame, planes, fmt, e, k, native, marks=None, rows=0, band=False, off=16, pad=32):
    """run the walk onto copies of `planes` (byte arrays [rows, row bytes]) placed `off` bytes into sentinel-filled rows;
    checks the sentinels and returns the rectangle's planes"""
    h, w = frame.shape[:2]
    bufs, ptrs, pitches = [], [], []
    for p in planes:
        pitch = (off + p.shape[1] + pad + 15) // 16 * 16
        b = np.full((p.shape[0] + 2, pitch), 0xA5, np.uint8)
        b[1:-1, off:off + p.shape[1]] = p
        bufs.append(b)
        ptrs.append(b.ctypes.data + pitch + off)
        pitches.append(pitch)
    before = [b.copy() for b in bufs]
    ptrs += [None] * (3 - len(ptrs))
    fb = np.ascontiguousarray(frame).view(np.uint32).reshape(h, w)
    m = None if marks is None else np.ascontiguousarray(marks, np.uint32)
    L.t_fade_walk(fb.ctypes.data, w, h, None if m is None else m.ctypes.data, rows, fmt, e, int(native), int(band), int(k),
                  *ptrs, pitches[0], pitches[1] if len(pitches) > 1 else 0)
    out = []
    for b, b0, p in zip(bufs, before, planes):
        inside = np.zeros(b.shape, bool)
        inside[1:-1, off:off + p.shape[1]] = True
        assert np.array_equal(b[~inside], b0[~inside]), "written outside the rectangle"
        out.append(b[1:-1, off:off + p.shape[1]].copy())
    return out


def restated(frame, planes, fmt, e, k, native):
    """the plain overlay's restatement applied to the pre-scaled frame (native blend), on byte planes"""
    f = fade_np(frame, k, native)
    h, w = frame.shape[:2]
    if fmt in (RGBA, BGRA):
        return [overlay_np(f, planes[0].reshape(h, w, 4), fmt, True).reshape(planes[0].shape)]
    wide = fmt in WIDE
    view = [p.view(np.uint16) if wide else p for p in planes]
    if fmt in (YUV422P, YUV422P10, UYVY):
        if fmt == UYVY:
            return [overlay422_np(f, (planes[0],), "uyvy", e, True)[0]]
        got = overlay422_np(f, tuple(view), NAME[fmt], e, True)
    else:
        if fmt == P010:
            view = [view[0], view[1]]
        got = planes_np(f, view, NAME[fmt], e, True)
    return [np.ascontiguousarray(g).view(np.uint8).reshape(p.shape) for g, p in zip(got, planes)]


def random_planes(rng, fmt, w, h):
    return [rng.integers(0, 256, s, dtype=np.uint8) for s in plane_shapes(fmt, w, h)]


FORMATS = (RGBA, BGRA, NV12, I420, YUV444, P010, YUV420P10, YUV444P10, YUV422P, YUV422P10, UYVY)


def fits(fmt, w, h):
    return not ((fmt in C420 and (w | h) & 1) or (fmt in (YUV422P, YUV422P10, UYVY) and w & 1))


@pytest.mark.parametrize("w,h", [(128, 64), (132, 30), (66, 10), (97, 7), (4, 2), (258, 5)])
@pytest.mark.parametrize("native", [True, False])
def test_walk_without_marks_equals_the_restatement(shim, w, h, native):
    rng = np.random.default_rng(w * 31 + h)
    frame = premultiplied(rng, (h, w)) if native else rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    frame[rng.random((h, w)) < 0.4] = 0
    frame[: h // 3] = 0
    for fmt in FORMATS:
        if not fits(fmt, w, h):
            continue
        for e in ((0,) if fmt in (RGBA, BGRA) else range(4)):
            planes = random_planes(rng, fmt, w, h)
            for k in K_SET:
                got = walk(shim, frame, planes, fmt, e, k, native)
                want = restated(frame, planes, fmt, e, k, native)
                for g, wnt in zip(got, want):
                    assert np.array_equal(g, wnt), (fmt, e, k)
                if k == 0:
                    assert all(np.array_equal(g, p) for g, p in zip(got, planes))


@pytest.mark.parametrize("w,h,rows", [(256, 40, 8), (300, 34, 5), (132, 18, 1), (98, 36, 7), (130, 24, 3), (66, 20, 9)])
def test_mark_aware_walks_equal_the_restatement(shim, w, h, rows):
    """band items under live marks, row-pair items under the same marks, over garbage in the rows the marks skip, odd
    band heights included; under any other opacity every row of the rectangle is written"""
    rows = min(rows, h)
    rng = np.random.default_rng(w * h + rows)
    for fmt in FORMATS:
        if not fits(fmt, w, h):
            continue
        for garbage in (False, True):
            frame, clean, marks = marked_frame(rng, w, h, rows, garbage)
            e = int(rng.integers(0, 4)) if fmt not in (RGBA, BGRA) else 0
            planes = random_planes(rng, fmt, w, h)
            for k in (1, 128, 254):
                want = restated(clean, planes, fmt, e, k, True)
                for band in (True, False):
                    got = walk(shim, frame, planes, fmt, e, k, True, marks=marks, rows=rows, band=band)
                    assert all(np.array_equal(g, x) for g, x in zip(got, want)), (fmt, garbage, band, k)
                if not garbage:
                    got = walk(shim, frame, planes, fmt, e, k, False, marks=marks, rows=rows)
                    want = restated(clean, planes, fmt, e, k, False)
                    assert all(np.array_equal(g, x) for g, x in zip(got, want)), (fmt, "opaque", k)


def test_opaque_full_opacity_is_the_export_restatement(shim):
    """under any other opacity K = 255 blends the opaque pixel, which is the plain call's bytes (overlay_np / planes_np
    of the export)"""
    rng = np.random.default_rng(70)
    w, h = 132, 18
    frame = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    for fmt in FORMATS:
        planes = random_planes(rng, fmt, w, h)
        got = walk(shim, frame, planes, fmt, 0, 255, False)
        if fmt in (RGBA, BGRA):
            want = [overlay_np(frame, planes[0].reshape(h, w, 4), fmt, False).reshape(planes[0].shape)]
        elif fmt in (YUV422P, YUV422P10, UYVY):
            wide = fmt in WIDE
            src = (planes[0],) if fmt == UYVY else tuple(p.view(np.uint16) if wide else p for p in planes)
            want = [np.ascontiguousarray(g).view(np.uint8).reshape(p.shape)
                    for g, p in zip(overlay422_np(frame, src, NAME[fmt], 0, False), planes)]
        else:
            wide = fmt in WIDE
            want = [np.ascontiguousarray(g).view(np.uint8).reshape(p.shape)
                    for g, p in zip(planes_np(frame, [p.view(np.uint16) if wide else p for p in planes], NAME[fmt], 0, False),
                                    planes)]
        assert all(np.array_equal(g, x) for g, x in zip(got, want)), fmt


# ---- the fake runtime -----------------------------------------------------------------------------------------------------------
FADE_STUBS = r"""
extern "C" void fade_fake_last(long* out) {
    out[0] = g_overlay.count; out[1] = g_overlay.fade; out[2] = g_overlay.band; out[3] = g_pl.count; out[4] = g_pl.fade;
}
"""


@pytest.fixture(scope="module")
def fake():
    inc = fakecuda.cuda_include()
    if inc is None:
        pytest.skip("no CUDA toolkit headers")
    from glava_b200.api import Export, OverlayPlanesDesc, Params, Picture
    out = tempfile.mkdtemp(prefix="glava_fade_fake_")
    src, so = os.path.join(out, "fade_fake.cpp"), os.path.join(out, "libfade_fake.so")
    with open(src, "w") as f:
        f.write("#include <vector>\n" + export_fake.STUBS + PLANES_STUBS + FADE_STUBS)
    subprocess.run(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I", inc,
                    "-I", fakecuda.CSRC, "-x", "c++", "-include", "cuda_runtime.h", "-o", so,
                    *[os.path.join(fakecuda.CSRC, f) for f in ("capi.cu", "export.cpp", "overlay_planes.cpp", "config.cpp")],
                    os.path.join(fakecuda.HERE, "fakecuda.cpp"), src, "-lpthread", "-Wl,-Bsymbolic"], check=True)
    L = C.CDLL(so)
    shutil.rmtree(out)
    vp, i32, P = C.c_void_p, C.c_int, C.POINTER(Params)
    sig = {
        "glava_b200_default_params": (i32, [P, C.c_char_p]), "glava_b200_new": (vp, [P, i32, i32]),
        "glava_b200_destroy": (None, [vp]), "glava_b200_last_error": (C.c_char_p, []), "glava_b200_set_abort_hook": (None, [vp]),
        "glava_b200_update": (i32, [vp, vp, vp, C.c_size_t, i32]),
        "glava_b200_overlay_frames_opacity": (i32, [vp, vp, i32, vp, vp, C.POINTER(Export), vp, vp, vp]),
        "glava_b200_overlay_planes_opacity": (i32, [vp, vp, i32, C.POINTER(Picture), C.POINTER(OverlayPlanesDesc), vp, vp, vp]),
        "cudaMalloc": (i32, [C.POINTER(vp), C.c_size_t]), "cudaEventCreate": (i32, [C.POINTER(vp)]),
        "cudaEventDestroy": (i32, [vp]), "fake_trace": (C.c_char_p, []),
        "export_fake_device": (None, [vp, C.c_size_t]), "export_fake_launches": (C.c_long, []),
        "planes_fake_launches": (C.c_long, []), "fade_fake_last": (None, [vp]),
        "glava_b200_framebuffer_device": (vp, [vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = res, args
    L._quiet = C.CFUNCTYPE(None, C.c_char_p)(lambda msg: None)
    L.glava_b200_set_abort_hook(C.cast(L._quiet, vp))
    return L


def _renderer(L, w=64, h=32, batch=2):
    from glava_b200.api import Params
    p = Params()
    assert L.glava_b200_default_params(C.byref(p), b"bars") == 0
    p.n, p.w, p.h = 1024, w, h
    r = L.glava_b200_new(C.byref(p), batch, 0)
    assert r, L.glava_b200_last_error()
    return C.c_void_p(r)


def _device(L, nbytes=1 << 18):
    b = C.c_void_p()
    assert L.cudaMalloc(C.byref(b), nbytes) == 0
    L.export_fake_device(b, nbytes)
    return b.value + (-b.value) % 256


def _frames(L, r, streams, dsts, d, opacity, uvs=None, after=None, done=None):
    s = np.asarray(streams, np.int32)
    arr = (C.c_void_p * max(len(dsts), 1))(*dsts)
    uv = None if uvs is None else (C.c_void_p * max(len(uvs), 1))(*uvs)
    k = None if opacity is None else np.ascontiguousarray(opacity, np.uint8)
    n0 = L.export_fake_launches()
    L.fake_trace_begin()
    rc = L.glava_b200_overlay_frames_opacity(r, s.ctypes.data if len(streams) else None, len(streams), arr, uv, C.byref(d),
                                             None if k is None else k.ctypes.data, after, done)
    L.fake_trace_end()
    return rc, L.glava_b200_last_error().decode(), L.fake_trace().decode(), L.export_fake_launches() - n0


def _planes(L, r, streams, pics, fmt, pitch, cpitch, opacity, flags=0, after=None, done=None):
    from glava_b200.api import OverlayPlanesDesc, Picture
    s = np.asarray(streams, np.int32)
    arr = (Picture * max(len(pics), 1))()
    for i, p in enumerate(pics):
        arr[i].plane = (C.c_void_p * 3)(*p)
    d = OverlayPlanesDesc()
    d.format, d.flags, d.pitch, d.chroma_pitch = fmt, flags, pitch, cpitch
    k = None if opacity is None else np.ascontiguousarray(opacity, np.uint8)
    n0 = L.planes_fake_launches()
    L.fake_trace_begin()
    rc = L.glava_b200_overlay_planes_opacity(r, s.ctypes.data if len(streams) else None, len(streams), arr, C.byref(d),
                                             None if k is None else k.ctypes.data, after, done)
    L.fake_trace_end()
    return rc, L.glava_b200_last_error().decode(), L.fake_trace().decode(), L.planes_fake_launches() - n0


def test_refusals_name_the_opacity_calls_and_enqueue_nothing(fake):
    """the plain calls' refusals, over every entry (K = 0 ones included), named after the _opacity call"""
    L = fake
    r = _renderer(L)
    b = _device(L)
    cases = [
        ([0], [b], desc_of(3, 256), [0], "unknown format"),
        ([0], [b], desc_of(RGBA, 240), [128], "pitch"),
        ([0, 1], [b, b], desc_of(RGBA, 1024), [0, 0], "overlaps"),                 # every entry checked, K = 0 too
        ([0, 1], [b, b + 240], desc_of(RGBA, 1024), [255, 0], "overlaps"),
        ([2], [b], desc_of(RGBA, 256), [0], "out of range"),
        ([0], [b + 8], desc_of(RGBA, 256), [0], "aligned"),
        ([], [], desc_of(RGBA, 256), [], "count"),
        ([0], [b], desc_of(I420, 256), [7], "overlay takes"),
    ]
    for streams, dsts, d, k, what in cases:
        rc, msg, trace, n = _frames(L, r, streams, dsts, d, k)
        assert rc != 0 and "glava_b200_overlay_frames_opacity" in msg and what in msg, (what, msg)
        assert trace == "" and n == 0, (what, trace)
    i420 = (b, b + 4096, b + 8192)
    pcases = [
        ([0], [i420], RGBA, 64, 32, [0], "overlay_frames"),
        ([0], [i420], I420, 72, 32, [128], "pitch"),
        ([0, 1], [i420, i420], I420, 64, 32, [0, 0], "overlaps"),
        ([0], [(b, b + 4096, 0)], YUV444, 64, 64, [0], "null"),
        ([2], [i420], I420, 64, 32, [3], "out of range"),
    ]
    for streams, pics, fmt, P_, CP, k, what in pcases:
        rc, msg, trace, n = _planes(L, r, streams, pics, fmt, P_, CP, k)
        assert rc != 0 and "glava_b200_overlay_planes_opacity" in msg and what in msg, (what, msg)
        assert trace == "" and n == 0, (what, trace)
    L.glava_b200_destroy(r)


def test_lists_choose_plain_fade_or_no_kernel(fake):
    """NULL and all-255 lists launch the plain kernel with every entry; a mixed list one fade kernel behind one list copy
    of the entries whose K is not 0; an all-zero list no copy and no kernel, with after / done still on the raster stream"""
    L = fake
    r = _renderer(L, w=64, h=32)
    b = _device(L)
    a, d = C.c_void_p(), C.c_void_p()
    assert L.cudaEventCreate(C.byref(a)) == 0 and L.cudaEventCreate(C.byref(d)) == 0
    last = np.zeros(5, np.int64)
    dsts = [b, b + 256, b + 512]
    for fmt, pic, P_, CP in ((I420, lambda i: (b + 64 * i, b + 8192 + 32 * i, b + 16384 + 32 * i), 256, 128),
                             (None, None, 1024, 0)):
        for k, fade, kept in ((None, 0, 3), ([255, 255, 255], 0, 3), ([255, 0, 128], 1, 2), ([1, 2, 3], 1, 3),
                              ([0, 0, 0], None, 0)):
            if fmt is None:
                rc, msg, trace, n = _frames(L, r, [0, 1, 1], dsts, desc_of(RGBA, 1024), k, after=a, done=d)
                entry = 24
            else:
                rc, msg, trace, n = _planes(L, r, [0, 1, 1], [pic(i) for i in range(3)], fmt, P_, CP, k, after=a, done=d)
                entry = 32
            assert rc == 0, msg
            kinds = [x.split()[0] for x in trace.splitlines()]
            L.fade_fake_last(last.ctypes.data)
            if kept == 0:
                assert n == 0 and kinds[-2:] == ["wait", "record"] and "memcpy" not in kinds, trace
                continue
            assert n == 1 and kinds[-4:] == ["wait", "memcpy", "record", "record"], trace
            assert f"H2D {kept * entry} " in trace, (trace, kept)
            count, fflag = (last[0], last[1]) if fmt is None else (last[3], last[4])
            assert (count, fflag) == (kept, fade), (fmt, k, list(last))
    # after a raster pass bars keeps marks: native fades take band items
    pcm = np.zeros((2, 1024), np.float32)
    assert L.glava_b200_update(r, pcm.ctypes.data, pcm.ctypes.data, 1024, 1) == 0
    rc, msg, trace, n = _frames(L, r, [0], [b], desc_of(RGBA, 256), [128])
    L.fade_fake_last(last.ctypes.data)
    assert rc == 0 and n == 1 and list(last[:3]) == [1, 1, 1], (msg, list(last))
    L.cudaEventDestroy(a); L.cudaEventDestroy(d)
    L.glava_b200_destroy(r)


def test_python_opacity_argument():
    from glava_b200.api import _FrameExport
    op = _FrameExport._opacity
    assert op(None, 3) is None
    assert list(op(0.5, 3)) == [128, 128, 128]
    assert list(op([0.0, 1.0, 0.999, 0.002, 0.5 / 255], 5)) == [0, 255, 255, 1, 1]
    assert list(op(np.linspace(0, 1, 256), 256)) == list(range(256))
    for bad in ([0.5, float("nan")], [1.01, 0.5], [-0.1, 0.5], [0.5], [[0.5, 0.5]]):
        with pytest.raises(ValueError):
            op(bad, 2)
    with pytest.raises(ValueError):
        op(float("nan"), 2)
