"""The Y'CbCr encodings of the exports (DESIGN 4.15) on the host: export_core.h's construction of the coefficient sets against
today's BT.709 literals and a Python restatement, every colour and every P010 block sum of each set against float64, the
overlay's blend per set, and the refusals and enqueued work of the colour flags through capi.cu, export.cpp and
export_ladder.cpp built against tests/fakecuda's runtime (tests/export_fake.py's stubs plus recorders of the encoding)."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from tests import export_fake, fakecuda
from tests.export_fake import desc_of
from tests.test_export_core import CSRC, pack
from tests.test_export_ladder_core import LADDER_STUBS, _ladder, scale_of
from tests.test_overlay_core import _overlay, cbcr_np, premult_colours, y_np

RGBA, BGRA, NV12, I420, YUV444, P010 = 0, 1, 2, 4, 5, 6
FULL, BT601 = 0x100, 0x200
ENCODINGS = {0: "bt709 limited", 1: "bt709 full", 2: "bt601 limited", 3: "bt601 full"}
# The float64 bound of every code: 0.5 for the final rounding plus what the 2^16-scaled coefficients add, at most 255 * 1.5 /
# 2^16 = 0.0058.  Measured over all 2^24 colours and all P010 block sums, the largest is 0.50339 (BT.601 limited, 10-bit Y;
# BT.709 limited's largest is 0.50289); DESIGN 4.15 lists each set and depth
BOUND = 0.504

SHIM = r"""
#include "export_core.h"
using namespace glb;
template <int E> static void px8(const uint32_t* px, size_t n, uint8_t* y, uint8_t* cb, uint8_t* cr) {
    for (size_t i = 0; i < n; ++i) { const uint32_t c = export_cbcr<E>(px[i]); y[i] = (uint8_t) export_y<E>(px[i]); cb[i] = c & 255u; cr[i] = c >> 8; }
}
template <int E> static void px10(const uint32_t* px, size_t n, uint16_t* y, uint16_t* cb, uint16_t* cr) {
    for (size_t i = 0; i < n; ++i) {
        const uint32_t c = export_cbcr10<E>(export_sum4(px[i], px[i], px[i], px[i]));
        y[i] = (uint16_t) export_y10<E>(px[i]); cb[i] = c & 0xffffu; cr[i] = c >> 16;
    }
}
// every block sum (Sr, Sg, Sb) in 0..1020 against float64: the largest error of Cb and Cr, and the greys whose chroma is not 512
template <int E> static long sweep10(double* err) {
    constexpr YuvCoef S = yuv_enc(E, 10);
    const double kr = E & 2 ? 0.299 : 0.2126, kb = E & 2 ? 0.114 : 0.0722, kg = 1 - kr - kb;
    const double cs = S.full ? 1023.0 / 255 : 896.0 / 255;
    double ecb = 0, ecr = 0;
    long bad = 0;
    for (int sr = 0; sr <= 1020; ++sr)
        for (int sg = 0; sg <= 1020; ++sg)
            for (int sb = 0; sb <= 1020; ++sb) {
                const uint32_t v = export_cbcr10<E>((uint32_t) sr | ((uint32_t) sg << 10) | ((uint32_t) sb << 20));
                const double yp = (kr * sr + kg * sg + kb * sb) / 4;
                const double fcb = std::fmin(1023.0, 512 + cs * (sb / 4.0 - yp) / (2 * (1 - kb)));
                const double fcr = std::fmin(1023.0, 512 + cs * (sr / 4.0 - yp) / (2 * (1 - kr)));
                const double a = std::fabs((double) (v & 0xffffu) - fcb), b = std::fabs((double) (v >> 16) - fcr);
                if (a > ecb) ecb = a;
                if (b > ecr) ecr = b;
                if (sr == sg && sg == sb && v != (512u | (512u << 16))) ++bad;
            }
    err[0] = ecb; err[1] = ecr;
    return bad;
}
template <int E> static void ov_y(const uint32_t* px, const uint8_t* yd, size_t n, uint8_t* out) {
    for (size_t i = 0; i < n; ++i) out[i] = (uint8_t) overlay_y<E>(px[i], yd[i]);
}
template <int E> static void ov_cbcr(const uint32_t* m, const uint16_t* uvd, size_t n, uint16_t* out) {
    for (size_t i = 0; i < n; ++i) out[i] = (uint16_t) overlay_cbcr<E>(m[i], uvd[i]);
}
template <int E> static void zero(int format, int native, uint32_t bg, uint32_t* out) {
    const ExportFmt f = { format, 1, native, bg };
    const ExportZero z = export_zero<E>(f);
    out[0] = z.y; out[1] = z.u; out[2] = z.v;
}
#define DISPATCH(fn, ...) switch (e) { case 1: fn<1>(__VA_ARGS__); break; case 2: fn<2>(__VA_ARGS__); break; \
                                       case 3: fn<3>(__VA_ARGS__); break; default: fn<0>(__VA_ARGS__); }
extern "C" void t_px8(int e, const uint32_t* px, size_t n, uint8_t* y, uint8_t* cb, uint8_t* cr) { DISPATCH(px8, px, n, y, cb, cr) }
extern "C" void t_px10(int e, const uint32_t* px, size_t n, uint16_t* y, uint16_t* cb, uint16_t* cr) { DISPATCH(px10, px, n, y, cb, cr) }
extern "C" long t_sweep10(int e, double* err) {
    switch (e) { case 1: return sweep10<1>(err); case 2: return sweep10<2>(err); case 3: return sweep10<3>(err); default: return sweep10<0>(err); }
}
extern "C" void t_ov_y(int e, const uint32_t* px, const uint8_t* yd, size_t n, uint8_t* out) { DISPATCH(ov_y, px, yd, n, out) }
extern "C" void t_ov_cbcr(int e, const uint32_t* m, const uint16_t* uvd, size_t n, uint16_t* out) { DISPATCH(ov_cbcr, m, uvd, n, out) }
extern "C" void t_zero(int e, int format, int native, uint32_t bg, uint32_t* out) { DISPATCH(zero, format, native, bg, out) }
// the set of encoding e at 8 or 10 bits: Y R G B, Cb R G B, Cr R G B, Y offset, C offset, top code, full
extern "C" void t_set(int e, int bits, int* out) {
    const YuvCoef s = yuv_enc(e, bits);
    const int v[13] = { s.yr, s.yg, s.yb, s.cbr, s.cbg, s.cbb, s.crr, s.crg, s.crb, s.yoff, s.coff, s.top, (int) s.full };
    for (int k = 0; k < 13; ++k) out[k] = v[k];
}
extern "C" void t_literals(int* out) {
    const int v[18] = { GLB_Y_R, GLB_Y_G, GLB_Y_B, GLB_CB_R, GLB_CB_G, GLB_CB_B, GLB_CR_R, GLB_CR_G, GLB_CR_B,
                        GLB_Y10_R, GLB_Y10_G, GLB_Y10_B, GLB_CB10_R, GLB_CB10_G, GLB_CB10_B, GLB_CR10_R, GLB_CR10_G, GLB_CR10_B };
    for (int k = 0; k < 18; ++k) out[k] = v[k];
}
"""


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("export_matrix_core")
    src, so = d / "shim.cpp", d / "shim.so"
    src.write_text(SHIM)
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I", CSRC,
                    "-include", "cstring", "-include", "cmath", "-o", str(so), str(src)], check=True)
    L = C.CDLL(str(so))
    vp, sz, i32, u32 = C.c_void_p, C.c_size_t, C.c_int, C.c_uint32
    L.t_px8.argtypes = L.t_px10.argtypes = [i32, vp, sz, vp, vp, vp]
    L.t_sweep10.argtypes, L.t_sweep10.restype = [i32, vp], C.c_long
    L.t_ov_y.argtypes = L.t_ov_cbcr.argtypes = [i32, vp, vp, sz, vp]
    L.t_zero.argtypes = [i32, i32, i32, u32, vp]
    L.t_set.argtypes = [i32, i32, vp]
    L.t_literals.argtypes = [vp]
    return L


# ---- the construction ------------------------------------------------------------------------------------------------------
def kr_kb(e):
    return (0.299, 0.114) if e & 2 else (0.2126, 0.0722)


def coef_py(e, bits):
    """the construction restated: Y, Cb, Cr rows (R, G, B), Y offset, C offset, top code, full"""
    kr, kb = kr_kb(e)
    kg = 1 - kr - kb
    full = bool(e & 1)
    top = 1023 if bits == 10 else 255
    ys = top / 255 if full else (876 if bits == 10 else 219) / 255
    cs = top / 255 if full else (896 if bits == 10 else 224) / 255
    s = 65536
    rnd = lambda x: int(np.sign(x) * np.floor(abs(x) + 0.5))
    y = [rnd(k * ys * s) for k in (kr, kg, kb)]
    cb = [rnd(-kr / (2 * (1 - kb)) * cs * s), rnd(-kg / (2 * (1 - kb)) * cs * s)]
    cr = [rnd(-kg / (2 * (1 - kr)) * cs * s), rnd(-kb / (2 * (1 - kr)) * cs * s)]
    return (y, [cb[0], cb[1], -(cb[0] + cb[1])], [-(cr[0] + cr[1]), cr[0], cr[1]], 0 if full else (64 if bits == 10 else 16),
            512 if bits == 10 else 128, top, full)


def coef_c(L, e, bits):
    out = (C.c_int * 13)()
    L.t_set(e, bits, out)
    v = list(out)
    return v[0:3], v[3:6], v[6:9], v[9], v[10], v[11], bool(v[12])


def test_the_construction_gives_todays_bt709_literals_exactly(shim):
    lit = (C.c_int * 18)()
    shim.t_literals(lit)
    lit = list(lit)
    for bits, k in ((8, 0), (10, 9)):
        y, cb, cr, yoff, coff, top, full = coef_c(shim, 0, bits)
        assert y + cb + cr == lit[k:k + 9], bits
        assert (yoff, coff, top, full) == ((16, 128, 255, False) if bits == 8 else (64, 512, 1023, False))


@pytest.mark.parametrize("bits", [8, 10])
@pytest.mark.parametrize("e", [0, 1, 2, 3])
def test_every_set_is_the_restated_construction(shim, e, bits):
    got = coef_c(shim, e, bits)
    assert got == coef_py(e, bits), (ENCODINGS[e], bits)
    y, cb, cr = got[:3]
    assert sum(cb) == 0 and sum(cr) == 0                               # greys have no chroma


def test_the_jfif_set_is_the_familiar_one(shim):
    """BT.601 full range at 8 bits is JFIF's Y'CbCr: libjpeg's 16-bit fixed point Y row 19595, 38470, 7471"""
    y, cb, cr, yoff, coff, top, full = coef_c(shim, 3, 8)
    assert y == [19595, 38470, 7471] and (yoff, coff, full) == (0, 128, True)


# ---- every colour ------------------------------------------------------------------------------------------------------------
def float_codes(c, e, bits):
    kr, kb = kr_kb(e)
    full = bool(e & 1)
    r, g, b = (c & 255).astype(np.float64), ((c >> 8) & 255).astype(np.float64), (c >> 16).astype(np.float64)
    top = 1023 if bits == 10 else 255
    ys = top / 255 if full else (876 if bits == 10 else 219) / 255
    cs = top / 255 if full else (896 if bits == 10 else 224) / 255
    yoff = 0 if full else (64 if bits == 10 else 16)
    coff = 512 if bits == 10 else 128
    yp = kr * r + (1 - kr - kb) * g + kb * b
    clamp = lambda v: np.clip(v, 0, top)
    return (clamp(yoff + ys * yp), clamp(coff + cs * (b - yp) / (2 * (1 - kb))), clamp(coff + cs * (r - yp) / (2 * (1 - kr))))


@pytest.mark.parametrize("bits", [8, 10])
@pytest.mark.parametrize("e", [1, 2, 3])
def test_every_colour_within_its_bound(shim, e, bits):
    """all 2^24 colours: each code within BOUND of the clamped float64 formula; grey has Cb = Cr = 128 (512); black and white
    are (16, 235) / (64, 940) in limited range and (0, 255) / (0, 1023) in full range"""
    c = np.arange(1 << 24, dtype=np.uint32)
    dt = np.uint16 if bits == 10 else np.uint8
    y, cb, cr = (np.empty(c.shape, dt) for _ in range(3))
    (shim.t_px10 if bits == 10 else shim.t_px8)(e, c.ctypes.data, c.size, y.ctypes.data, cb.ctypes.data, cr.ctypes.data)
    fy, fcb, fcr = float_codes(c, e, bits)
    errs = [float(np.abs(got.astype(np.float64) - want).max()) for got, want in ((y, fy), (cb, fcb), (cr, fcr))]
    assert max(errs) <= BOUND, (ENCODINGS[e], bits, errs)
    mid = 512 if bits == 10 else 128
    grey = np.arange(256, dtype=np.uint32) * 0x010101
    assert (cb[grey] == mid).all() and (cr[grey] == mid).all() and (np.diff(y[grey].astype(int)) >= 0).all()
    black, white = (0, 0) if e & 1 else ((16, 235) if bits == 8 else (64, 940))
    if e & 1:
        white = 1023 if bits == 10 else 255
    assert (y[0], cb[0], cr[0]) == (black, mid, mid)
    assert (y[(1 << 24) - 1], cb[(1 << 24) - 1], cr[(1 << 24) - 1]) == (white, mid, mid)
    if e & 1:                                                          # blue's Cb and red's Cr reach the top code
        top = 1023 if bits == 10 else 255
        assert cb[0xff0000] == top and cr[0x0000ff] == top


@pytest.mark.parametrize("e", [1, 2, 3])
def test_p010_chroma_of_every_block_sum(shim, e):
    """all 1021^3 (Sr, Sg, Sb) sums per set: every grey sum is (512, 512), the codes within BOUND of float64, and the
    accumulators in [0, 2^31)"""
    err = np.zeros(2)
    assert shim.t_sweep10(e, err.ctypes.data) == 0
    assert err.max() <= BOUND, (ENCODINGS[e], err)
    _, cb, cr, _, coff, _, _ = coef_py(e, 10)
    for k in (cb, cr):
        lo = sum(min(0, v) for v in k) * 1020 + (coff << 18)
        hi = sum(max(0, v) for v in k) * 1020 + (coff << 18) + (1 << 17)
        assert 0 <= lo and hi < 1 << 31


def test_every_accumulator_stays_in_range():
    """8 and 10 bits per pixel, every set: the extreme sums of each row over 0..255, offset and rounding included"""
    for e in range(4):
        for bits in (8, 10):
            y, cb, cr, yoff, coff, _, _ = coef_py(e, bits)
            for k, off in ((y, yoff), (cb, coff), (cr, coff)):
                assert 0 <= sum(min(0, v) for v in k) * 255 + (off << 16)
                assert sum(max(0, v) for v in k) * 255 + (off << 16) + (1 << 15) < 1 << 31


@pytest.mark.parametrize("e", [0, 1, 2, 3])
def test_zero_quad_constants(shim, e):
    """export_zero per set: what a zero pixel becomes over a background, as the per-pixel arithmetic gives it"""
    out = (C.c_uint32 * 3)()
    for bg in (0x000000, 0xffffff, 0x4280f0):
        for native in (0, 1):
            c = np.array([0 if native == 0 else bg], np.uint32)      # the composite of a zero pixel
            y8, cb8, cr8 = (np.empty(1, np.uint8) for _ in range(3))
            shim.t_px8(e, c.ctypes.data, 1, y8.ctypes.data, cb8.ctypes.data, cr8.ctypes.data)
            shim.t_zero(e, YUV444, native, bg, out)
            assert list(out) == [int(y8[0]) * 0x01010101, int(cb8[0]) * 0x01010101, int(cr8[0]) * 0x01010101]
            shim.t_zero(e, I420, native, bg, out)
            assert list(out) == [int(y8[0]) * 0x01010101, int(cb8[0]) * 0x0101, int(cr8[0]) * 0x0101]
            y10, cb10, cr10 = (np.empty(1, np.uint16) for _ in range(3))
            shim.t_px10(e, c.ctypes.data, 1, y10.ctypes.data, cb10.ctypes.data, cr10.ctypes.data)
            shim.t_zero(e, P010, native, bg, out)
            assert out[0] == (int(y10[0]) << 6) * 0x10001 and out[1] == (int(cb10[0]) << 6) | (int(cr10[0]) << 22)


# ---- the overlay per set -------------------------------------------------------------------------------------------------------
def call(fn, e, dt, *arrays):
    arrays = [np.ascontiguousarray(a) for a in arrays]
    out = np.empty(arrays[0].shape[0], dt)
    fn(e, *[a.ctypes.data for a in arrays], arrays[0].shape[0], out.ctypes.data)
    return out


def overlay_float(e, P, VD, chroma):
    """the float64 composite of premultiplied P (alpha included) over destination codes VD: Y or (Cb, Cr)"""
    kr, kb = kr_kb(e)
    full = bool(e & 1)
    ys, cs = (1.0, 1.0) if full else (219 / 255, 224 / 255)
    r, g, b, al = P[:, 0], P[:, 1], P[:, 2], P[:, 3] / 255.0
    yp = kr * r + (1 - kr - kb) * g + kb * b
    if not chroma:
        return np.clip((0 if full else 16) * al + ys * yp + (1 - al) * VD, 0, 255)
    return (np.clip(128 * al + cs * (b - yp) / (2 * (1 - kb)) + (1 - al) * VD[:, 0], 0, 255),
            np.clip(128 * al + cs * (r - yp) / (2 * (1 - kr)) + (1 - al) * VD[:, 1], 0, 255))


def overlay_int_np(e, P, VD, chroma):
    """the integer blend restated with the set's coefficients and offsets"""
    y, cb, cr, yoff, coff, _, _ = coef_py(e, 8)
    al = P[:, 3].astype(np.int64)
    frac = lambda off, vd: (((off * al + (255 - al) * vd) << 16) + 127) // 255
    dot = lambda k: k[0] * P[:, 0] + k[1] * P[:, 1] + k[2] * P[:, 2]
    if not chroma:
        return np.clip((dot(y) + frac(yoff, VD) + (1 << 15)) >> 16, 0, 255)
    return (np.clip((dot(cb) + frac(coff, VD[:, 0]) + (1 << 15)) >> 16, 0, 255),
            np.clip((dot(cr) + frac(coff, VD[:, 1]) + (1 << 15)) >> 16, 0, 255))


def test_the_restated_overlay_is_todays_for_bt709_limited():
    rng = np.random.default_rng(7)
    P = premult_colours(rng, np.arange(256), 4)
    VD = rng.integers(0, 256, P.shape[0])
    assert np.array_equal(overlay_int_np(0, P, VD, False), y_np(P, VD))
    UV = rng.integers(0, 256, (P.shape[0], 2))
    cb, cr = cbcr_np(P, UV[:, 0], UV[:, 1])
    got = overlay_int_np(0, P, UV, True)
    assert np.array_equal(got[0], cb) and np.array_equal(got[1], cr)


@pytest.mark.parametrize("e", [1, 2, 3])
def test_overlay_y_and_cbcr_every_alpha_and_destination(shim, e):
    """every (alpha, destination code) for sampled premultiplied colours: equal to the integer restatement and within 0.502
    of the clamped float64 composite"""
    rng = np.random.default_rng(10 + e)
    px = premult_colours(rng, np.arange(256), 12)
    P, VD = np.repeat(px, 256, axis=0), np.tile(np.arange(256), px.shape[0])
    got = call(shim.t_ov_y, e, np.uint8, pack(P[:, 0], P[:, 1], P[:, 2], P[:, 3]), VD.astype(np.uint8)).astype(np.int64)
    assert np.array_equal(got, overlay_int_np(e, P, VD, False))
    err_y = np.abs(got - overlay_float(e, P, VD, False)).max()
    UV = np.stack([VD, rng.integers(0, 256, VD.size)], axis=1)
    got = call(shim.t_ov_cbcr, e, np.uint16, pack(P[:, 0], P[:, 1], P[:, 2], P[:, 3]),
               (UV[:, 0] | (UV[:, 1] << 8)).astype(np.uint16)).astype(np.int64)
    cb, cr = overlay_int_np(e, P, UV, True)
    assert np.array_equal(got & 255, cb) and np.array_equal(got >> 8, cr)
    fcb, fcr = overlay_float(e, P, UV, True)
    err_c = max(np.abs((got & 255) - fcb).max(), np.abs((got >> 8) - fcr).max())
    assert err_y <= 0.502 and err_c <= 0.502, (ENCODINGS[e], err_y, err_c)


@pytest.mark.parametrize("e", [1, 2, 3])
def test_overlay_endpoints_per_set(shim, e):
    """a zero pixel returns the destination code; an opaque pixel (block) gives the export's code"""
    v = np.arange(256)
    zero = np.zeros(256, np.uint32)
    assert np.array_equal(call(shim.t_ov_y, e, np.uint8, zero, v.astype(np.uint8)), v)
    uv = (v[:, None] | (v[None, :] << 8)).reshape(-1).astype(np.uint16)
    assert np.array_equal(call(shim.t_ov_cbcr, e, np.uint16, np.zeros(uv.size, np.uint32), uv), uv)
    c = np.arange(1 << 24, dtype=np.uint32)[::5] | np.uint32(0xff000000)
    y0, cb0, cr0 = (np.empty(c.shape, np.uint8) for _ in range(3))
    shim.t_px8(e, c.ctypes.data, c.size, y0.ctypes.data, cb0.ctypes.data, cr0.ctypes.data)
    rng = np.random.default_rng(20 + e)
    assert np.array_equal(call(shim.t_ov_y, e, np.uint8, c, rng.integers(0, 256, c.size).astype(np.uint8)), y0)
    got = call(shim.t_ov_cbcr, e, np.uint16, c, rng.integers(0, 1 << 16, c.size).astype(np.uint16))
    assert np.array_equal(got & 255, cb0) and np.array_equal(got >> 8, cr0)


# ---- refusals and enqueued work through the fake runtime -----------------------------------------------------------------
MATRIX_STUBS = r"""
// the encoding the last scaled export, overlay and ladder (per rung) reached their launchers with
extern "C" void matrix_fake_enc(int* out) {
    out[0] = g_scaled.enc; out[1] = g_overlay.enc;
    for (int j = 0; j < GLAVA_B200_LADDER_MAX; ++j) out[2 + j] = g_ladder.rung[j].enc;
}
"""


@pytest.fixture(scope="module")
def fake():
    """export_fake's stubs and the ladder launcher over capi.cu, export.cpp, export_ladder.cpp and config.cpp"""
    inc = fakecuda.cuda_include()
    if inc is None:
        pytest.skip("no CUDA toolkit headers")
    from glava_b200.api import Export, ExportScale, Params
    out = tempfile.mkdtemp(prefix="glava_matrix_fake_")
    src, so = os.path.join(out, "matrix_fake.cpp"), os.path.join(out, "libmatrix_fake.so")
    with open(src, "w") as f:
        f.write(export_fake.STUBS + LADDER_STUBS + MATRIX_STUBS)
    subprocess.run(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I", inc,
                    "-I", fakecuda.CSRC, "-x", "c++", "-include", "cuda_runtime.h", "-o", so,
                    *[os.path.join(fakecuda.CSRC, f) for f in ("capi.cu", "export.cpp", "export_ladder.cpp", "config.cpp")],
                    os.path.join(fakecuda.HERE, "fakecuda.cpp"), src, "-lpthread", "-Wl,-Bsymbolic"], check=True)
    L = C.CDLL(so)
    shutil.rmtree(out)                                                # stays mapped
    vp, i32, P, E, S = C.c_void_p, C.c_int, C.POINTER(Params), C.POINTER(Export), C.POINTER(ExportScale)
    sig = {
        "glava_b200_default_params": (i32, [P, C.c_char_p]), "glava_b200_new": (vp, [P, i32, i32]),
        "glava_b200_destroy": (None, [vp]), "glava_b200_update": (i32, [vp, vp, vp, C.c_size_t, i32]),
        "glava_b200_last_error": (C.c_char_p, []), "glava_b200_set_abort_hook": (None, [vp]),
        "glava_b200_export_frames": (i32, [vp, vp, i32, vp, E, vp, vp]),
        "glava_b200_export_bytes": (i32, [vp, E, C.POINTER(C.c_size_t)]),
        "glava_b200_export_scaled": (i32, [vp, vp, i32, vp, vp, E, S, vp, vp]),
        "glava_b200_export_scaled_bytes": (i32, [vp, E, S, C.POINTER(C.c_size_t)]),
        "glava_b200_overlay_frames": (i32, [vp, vp, i32, vp, vp, E, vp, vp]),
        "glava_b200_export_ladder": (i32, [vp, vp, i32, vp, i32, vp, vp, vp, vp]),
        "cudaMalloc": (i32, [C.POINTER(vp), C.c_size_t]), "cudaFree": (i32, [vp]),
        "fake_trace": (C.c_char_p, []), "fake_fail_at": (None, [C.c_long]),
        "export_fake_device": (None, [vp, C.c_size_t]), "export_fake_forget": (None, [vp]),
        "export_fake_launches": (C.c_long, []), "ladder_fake_launches": (C.c_long, []), "matrix_fake_enc": (None, [vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = res, args
    L._quiet = C.CFUNCTYPE(None, C.c_char_p)(lambda msg: None)
    L.glava_b200_set_abort_hook(C.cast(L._quiet, vp))

    def renderer(module="bars", batch=2, **kw):
        p = Params()
        assert L.glava_b200_default_params(C.byref(p), module.encode()) == 0
        for k, v in kw.items():
            setattr(p, k, v)
        h = L.glava_b200_new(C.byref(p), batch, 0)
        assert h, L.glava_b200_last_error()
        return C.c_void_p(h), p

    def device_buf(nbytes=1 << 16):
        b = C.c_void_p()
        assert L.cudaMalloc(C.byref(b), nbytes) == 0
        L.export_fake_device(b, nbytes)
        return b

    L.renderer, L.device_buf = renderer, device_buf
    return L


def encs(L):
    out = (C.c_int * 10)()
    L.matrix_fake_enc(out)
    return list(out)


def _call(L, fn, *args):
    n0 = L.export_fake_launches()
    L.fake_trace_begin()
    rc = fn(*args)
    L.fake_trace_end()
    return rc, L.glava_b200_last_error().decode(), L.fake_trace().decode(), L.export_fake_launches() - n0


def test_colour_bits_are_refused_on_rgba_and_bgra_naming_the_function(fake):
    L = fake
    L.fake_fail_at(-1)
    h, p = L.renderer(n=1024, w=64, h=32)
    buf = L.device_buf()
    s = np.zeros(1, np.int32)
    dst = (C.c_void_p * 1)(buf.value)
    sc = scale_of((32, 16))
    for fmt, name in ((RGBA, "RGBA"), (BGRA, "BGRA")):
        for flags in (FULL, BT601, FULL | BT601, FULL | 1):
            d = desc_of(fmt, 256, flags=flags)
            calls = [("glava_b200_export_frames", lambda: L.glava_b200_export_frames(h, s.ctypes.data, 1, dst, C.byref(d), None, None)),
                     ("glava_b200_export_scaled", lambda: L.glava_b200_export_scaled(h, s.ctypes.data, 1, dst, None, C.byref(d),
                                                                                     C.byref(sc), None, None)),
                     ("glava_b200_overlay_frames", lambda: L.glava_b200_overlay_frames(h, s.ctypes.data, 1, dst, None, C.byref(d),
                                                                                       None, None))]
            for who, fn in calls:
                rc, msg, trace, launched = _call(L, fn)
                assert rc != 0 and msg.startswith(who) and name in msg and "no matrix or range" in msg, (who, flags, msg)
                assert trace == "" and launched == 0
            n = C.c_size_t()
            assert L.glava_b200_export_bytes(h, C.byref(d), C.byref(n)) != 0
            assert "glava_b200_export_bytes" in L.glava_b200_last_error().decode()
            rc, msg, trace, launched = _ladder(L, h, [0], [(d, sc)], [buf.value])
            assert rc != 0 and "glava_b200_export_ladder: rung 0:" in msg and "no matrix or range" in msg, msg
            assert trace == "" and launched == 0
    # bit 0x2 stays an unknown flag for every format, with or without the colour bits
    for fmt in (RGBA, NV12, I420, YUV444, P010):
        for extra in (0, FULL, BT601):
            d = desc_of(fmt, 256, flags=2 | extra)
            rc, msg, trace, launched = _call(L, lambda: L.glava_b200_export_frames(h, s.ctypes.data, 1, dst, C.byref(d), None, None))
            assert rc != 0 and "unknown flags" in msg and launched == 0, (fmt, extra, msg)
        d = desc_of(fmt, 256, flags=0x400)
        rc, msg, _, _ = _call(L, lambda: L.glava_b200_export_frames(h, s.ctypes.data, 1, dst, C.byref(d), None, None))
        assert rc != 0 and "unknown flags" in msg
    L.glava_b200_destroy(h)
    L.cudaFree(buf)


def test_every_yuv_format_takes_the_bits_and_the_byte_counts_do_not_change(fake):
    L = fake
    L.fake_fail_at(-1)
    h, p = L.renderer(n=1024, w=64, h=32)
    buf = L.device_buf(1 << 18)
    s = np.zeros(1, np.int32)
    dst = (C.c_void_p * 1)(buf.value)
    sc = scale_of((32, 16))
    for fmt, pitch in ((NV12, 64), (I420, 64), (YUV444, 64), (P010, 128)):
        base, base_s = C.c_size_t(), C.c_size_t()
        assert L.glava_b200_export_bytes(h, C.byref(desc_of(fmt, pitch)), C.byref(base)) == 0
        assert L.glava_b200_export_scaled_bytes(h, C.byref(desc_of(fmt, pitch)), C.byref(sc), C.byref(base_s)) == 0
        for flags, e in ((FULL, 1), (BT601, 2), (FULL | BT601, 3), (FULL | BT601 | 1, 3)):
            d = desc_of(fmt, pitch, flags=flags)
            n, n_s = C.c_size_t(), C.c_size_t()
            assert L.glava_b200_export_bytes(h, C.byref(d), C.byref(n)) == 0 and n.value == base.value
            assert L.glava_b200_export_scaled_bytes(h, C.byref(d), C.byref(sc), C.byref(n_s)) == 0 and n_s.value == base_s.value
            rc, msg, trace, launched = _call(L, lambda: L.glava_b200_export_frames(h, s.ctypes.data, 1, dst, C.byref(d), None, None))
            assert rc == 0 and launched == 1, msg
            assert [x.split()[0] for x in trace.splitlines()].count("memcpy") == 1
            rc, msg, trace, launched = _call(L, lambda: L.glava_b200_export_scaled(h, s.ctypes.data, 1, dst, None, C.byref(d),
                                                                                   C.byref(sc), None, None))
            assert rc == 0 and launched == 1 and encs(L)[0] == e, msg
    L.glava_b200_destroy(h)
    L.cudaFree(buf)


def test_the_overlay_takes_the_bits_on_nv12_only(fake):
    L = fake
    L.fake_fail_at(-1)
    h, p = L.renderer(n=1024, w=64, h=32)
    buf = L.device_buf()
    s = np.zeros(1, np.int32)
    dst = (C.c_void_p * 1)(buf.value)
    for flags, e in ((0, 0), (FULL, 1), (BT601, 2), (FULL | BT601, 3)):
        d = desc_of(NV12, 64, flags=flags)
        rc, msg, trace, launched = _overlay(L, h, [0], [buf.value], d)
        assert rc == 0 and launched == 1 and encs(L)[1] == e, msg
        rc, msg, trace, launched = _overlay(L, h, [0], [buf.value], desc_of(NV12, 64, flags=flags | 1))
        assert rc != 0 and "takes none" in msg and launched == 0, msg
    for fmt, name in ((I420, "I420"), (YUV444, "YUV444"), (P010, "P010")):   # refused by name, as without the bits
        rc, msg, trace, launched = _overlay(L, h, [0], [buf.value], desc_of(fmt, 128, flags=FULL))
        assert rc != 0 and name in msg and "the overlay takes RGBA, BGRA or NV12" in msg and launched == 0, msg
    L.glava_b200_destroy(h)
    L.cudaFree(buf)


def test_a_ladder_mixing_encodings_is_one_copy_and_one_launch(fake):
    L = fake
    L.fake_fail_at(-1)
    h, p = L.renderer(n=1024, w=64, h=32)
    bufs = [L.device_buf(1 << 16) for _ in range(6)]
    pairs = [(desc_of(NV12, 64), scale_of((64, 32))), (desc_of(NV12, 32, flags=FULL | BT601), scale_of((32, 16))),
             (desc_of(I420, 64, flags=BT601), scale_of((64, 32))), (desc_of(P010, 64, flags=FULL), scale_of((16, 8))),
             (desc_of(YUV444, 32, flags=FULL | BT601), scale_of((16, 8))), (desc_of(RGBA, 256, flags=1), scale_of((32, 16)))]
    dsts = [b.value for b in bufs] * 2
    n0 = L.ladder_fake_launches()
    rc, msg, trace, launched = _ladder(L, h, [0, 1], pairs, dsts)
    assert rc == 0 and launched == 1 and L.ladder_fake_launches() - n0 == 1, msg
    kinds = [x.split()[0] for x in trace.splitlines()]
    assert kinds.count("memcpy") <= 2 and kinds.count("memcpy") >= 1, trace         # the list (and the schedule, once)
    assert encs(L)[2:8] == [0, 3, 2, 1, 3, 0]
    rc, msg, trace, launched = _ladder(L, h, [0, 1], pairs, dsts)                    # same geometry: the list copy alone
    assert rc == 0 and launched == 1 and [x.split()[0] for x in trace.splitlines()].count("memcpy") == 1, trace
    L.glava_b200_destroy(h)
    for b in bufs:
        L.cudaFree(b)


def test_python_matrix_names_and_flags():
    import glava_b200 as g
    from glava_b200.api import _export_desc
    assert (g.EXPORT_FULL_RANGE, g.EXPORT_BT601) == (0x100, 0x200)
    assert _export_desc("nv12", False, (0, 0, 0)).flags == 0
    assert _export_desc("p010", False, (0, 0, 0), "bt601", True).flags == 0x300
    assert _export_desc("i420", False, (0, 0, 0), "bt709", True).flags == 0x100
    assert _export_desc("rgba", True, (0, 0, 0), "bt601").flags == 0x201                 # the library refuses it
    with pytest.raises(ValueError, match="matrix"):
        _export_desc("nv12", False, (0, 0, 0), "bt2020")
