"""I420, YUV 4:4:4 and P010 export (DESIGN 4.14) on the host: the arithmetic of export_core.h through a g++ shim (the 10-bit
coefficients over every colour and every block sum against float64), a host walk of export_yuv_kernel's loop (row pairs,
128-pixel strips, quads, the dirty-row marks, the zero-quad constants, the tails) checked bit for bit against numpy
restatements with sentinel bytes around every plane, the identities with NV12, and the refusals and enqueued work of the
export calls through capi.cu, export.cpp and export_ladder.cpp built against tests/fakecuda's runtime."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from tests import export_fake, fakecuda
from tests.export_fake import desc_of
from tests.test_export_core import BGRA, CSRC, NV12, RGBA, bt709_fixed, export, marked_frame, over_np, pack, premultiplied
from tests.test_export_ladder_core import LADDER_STUBS, rungs_of, scale_of

I420, YUV444, P010 = 4, 5, 6
NAMES = {I420: "i420", YUV444: "yuv444", P010: "p010"}
Y10, CB10, CR10 = (47864, 161017, 16255), (-26383, -88755, 115138), (115137, -104580, -10557)
SENTINEL = 0xA5

SHIM = r"""
#include "export_core.h"
using namespace glb;
extern "C" void t_p010_px(const uint32_t* px, size_t n, uint16_t* y, uint16_t* cb, uint16_t* cr) {
    for (size_t i = 0; i < n; ++i) {
        const uint32_t c = export_cbcr10(export_sum4(px[i], px[i], px[i], px[i]));
        y[i] = (uint16_t) export_y10(px[i]); cb[i] = c & 0xffffu; cr[i] = c >> 16;
    }
}
// every block sum (Sr, Sg, Sb) in 0..1020 against float64: the largest error of Cb and Cr, and the greys whose chroma is not 512
extern "C" long t_cbcr10_sweep(double* err) {
    const double kr = 0.2126, kb = 0.0722, kg = 1 - kr - kb;
    double ecb = 0, ecr = 0;
    long bad = 0;
    for (int sr = 0; sr <= 1020; ++sr)
        for (int sg = 0; sg <= 1020; ++sg)
            for (int sb = 0; sb <= 1020; ++sb) {
                const uint32_t v = export_cbcr10((uint32_t) sr | ((uint32_t) sg << 10) | ((uint32_t) sb << 20));
                const double yp = (kr * sr + kg * sg + kb * sb) / 4;
                const double fcb = 512 + 896.0 / 255 * (sb / 4.0 - yp) / (2 * (1 - kb));
                const double fcr = 512 + 896.0 / 255 * (sr / 4.0 - yp) / (2 * (1 - kr));
                const double a = std::fabs((double) (v & 0xffffu) - fcb), b = std::fabs((double) (v >> 16) - fcr);
                if (a > ecb) ecb = a;
                if (b > ecr) ecr = b;
                if (sr == sg && sg == sb && v != (512u | (512u << 16))) ++bad;
            }
    err[0] = ecb; err[1] = ecr;
    return bad;
}
static void put(uint8_t* p, uint64_t v, int nbytes) { for (int k = 0; k < nbytes; ++k) p[k] = (uint8_t) (v >> (8 * k)); }
// one slot [h][w] -> the planes, as export_yuv_kernel walks it (yuv_item); marks: the slot's [h][strips] words or null.
// cb: the chroma plane (I420 / YUV444: Cb, Cr `cr` bytes further; P010: CbCr)
extern "C" void t_export_yuv(const uint32_t* fb, int w, int h, const uint32_t* marks, int rows, int format, int native,
                             uint32_t bg, uint8_t* dst, size_t pitch, uint8_t* cb, size_t cr) {
    const ExportFmt f = { format, 1, native, bg };
    const ExportZero z = export_zero(f);
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
                const bool any = (q[0][0] | q[0][1] | q[0][2] | q[0][3] | q[1][0] | q[1][1] | q[1][2] | q[1][3]) != 0u;
                if (format == GLAVA_B200_EXPORT_YUV444) {
                    const int n = full ? 4 : w - x;
                    for (int r = 0; r < 2 && (r == 0 || y1 >= 0); ++r) {
                        uint32_t y = z.y, u = z.u, v = z.v;
                        if (q[r][0] | q[r][1] | q[r][2] | q[r][3]) export_444_quad(f, q[r], &y, &u, &v);
                        const size_t o = (size_t) (2 * j + r) * pitch + x;
                        put(dst + o, y, n); put(cb + o, u, n); put(cb + cr + o, v, n);
                    }
                } else if (format == GLAVA_B200_EXPORT_I420) {
                    uint32_t yt = z.y, yb = z.y, u = z.u, v = z.v;
                    if (any) { const uint32_t uv = export_nv12_quad(f, q[0], q[1], &yt, &yb); u = export_cb_pair(uv); v = export_cr_pair(uv); }
                    const int n = full ? 4 : 2;
                    put(dst + (size_t) (2 * j) * pitch + x, yt, n); put(dst + (size_t) (2 * j + 1) * pitch + x, yb, n);
                    uint8_t* pu = cb + (size_t) j * (pitch / 2) + x / 2;
                    put(pu, u, n / 2); put(pu + cr, v, n / 2);
                } else {
                    uint32_t yt[2] = { z.y, z.y }, yb[2] = { z.y, z.y }, uv[2] = { z.u, z.u };
                    if (any) export_p010_quad(f, q[0], q[1], yt, yb, uv);
                    const int n = full ? 8 : 4;
                    put(dst + (size_t) (2 * j) * pitch + 2 * x, yt[0] | ((uint64_t) yt[1] << 32), n);
                    put(dst + (size_t) (2 * j + 1) * pitch + 2 * x, yb[0] | ((uint64_t) yb[1] << 32), n);
                    put(cb + (size_t) j * pitch + 2 * x, uv[0] | ((uint64_t) uv[1] << 32), n);
                }
            }
}
"""


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("export_formats_core")
    src, so = d / "shim.cpp", d / "shim.so"
    src.write_text(SHIM)
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I", CSRC,
                    "-include", "cstring", "-include", "cmath", "-o", str(so), str(src)], check=True)
    L = C.CDLL(str(so))
    vp, sz, i32, u32 = C.c_void_p, C.c_size_t, C.c_int, C.c_uint32
    L.t_p010_px.argtypes = [vp, sz, vp, vp, vp]
    L.t_cbcr10_sweep.argtypes = [vp]
    L.t_cbcr10_sweep.restype = C.c_long
    L.t_export_yuv.argtypes = [vp, i32, i32, vp, i32, i32, i32, u32, vp, sz, vp, sz]
    return L


# ---- numpy restatements --------------------------------------------------------------------------------------------------
def yuv_np(c, fmt):
    """a composited top-down image c [h][w][>= 3] -> I420 / YUV444: (Y, Cb, Cr) uint8 planes; P010: [h * 3 / 2][w] uint16"""
    c = np.asarray(c, np.int64)
    h, w = c.shape[:2]
    ky, kcb, kcr = bt709_fixed()
    dot = lambda k, v: k[0] * v[..., 0] + k[1] * v[..., 1] + k[2] * v[..., 2]
    if fmt == "p010":
        y = (dot(Y10, c) + (64 << 16) + (1 << 15)) >> 16
        s = c[..., :3].reshape(h // 2, 2, w // 2, 2, 3).sum(axis=(1, 3))   # exact block sums
        cb = (dot(CB10, s) + (512 << 18) + (1 << 17)) >> 18
        cr = (dot(CR10, s) + (512 << 18) + (1 << 17)) >> 18
        return (np.concatenate([y, np.stack([cb, cr], axis=-1).reshape(h // 2, w)]) << 6).astype(np.uint16)
    y = ((dot(ky, c) + (16 << 16) + (1 << 15)) >> 16).astype(np.uint8)
    if fmt == "i420":
        c = (c[..., :3].reshape(h // 2, 2, w // 2, 2, 3).sum(axis=(1, 3)) + 2) >> 2
    cb = (dot(kcb, c) + (128 << 16) + (1 << 15)) >> 16
    cr = (dot(kcr, c) + (128 << 16) + (1 << 15)) >> 16
    return y, cb.astype(np.uint8), cr.astype(np.uint8)


def frame_np(frame, fmt, bg, native):
    """the expected export of one framebuffer slot ([h][w][4], row 0 = bottom)"""
    return yuv_np(over_np(frame[::-1], bg, native), fmt)


def export_yuv(L, frame, fmt, bg=(0, 0, 0), native=True, marks=None, rows=0, pad=32):
    """t_export_yuv into one buffer holding the planes with `pad` sentinel bytes past every row and a gap between planes;
    -> the planes as yuv_np returns them, after checking that no sentinel byte was written"""
    h, w = frame.shape[:2]
    row = w * 2 if fmt == P010 else w
    pitch = (row + pad + 31) // 32 * 32
    cw, ch, cp = (w // 2, h // 2, pitch // 2) if fmt == I420 else (w, h, pitch)
    gap = 64
    y_bytes = pitch * h
    cb_off = y_bytes + gap
    cr = (cp * ch + gap) if fmt != P010 else 0
    total = cb_off + (pitch * (h // 2) if fmt == P010 else cr + cp * ch) + gap
    buf = np.full(total, SENTINEL, np.uint8)
    fb = np.ascontiguousarray(frame).view(np.uint32).reshape(h, w)
    m = None if marks is None else np.ascontiguousarray(marks, np.uint32)
    L.t_export_yuv(fb.ctypes.data, w, h, None if m is None else m.ctypes.data, rows, fmt, int(native), int(pack(*bg[:3])),
                   buf.ctypes.data, pitch, buf.ctypes.data + cb_off, cr)
    written = np.zeros(total, bool)

    def plane(off, nrows, p, nbytes):
        idx = off + np.arange(nrows)[:, None] * p + np.arange(nbytes)[None, :]
        written[idx] = True
        return buf[idx]

    y = plane(0, h, pitch, row)
    if fmt == P010:
        uv = plane(cb_off, h // 2, pitch, row)
        assert (buf[~written] == SENTINEL).all(), "written outside the planes"
        return np.concatenate([y, uv]).view(np.uint16)
    cb, crp = plane(cb_off, ch, cp, cw), plane(cb_off + cr, ch, cp, cw)
    assert (buf[~written] == SENTINEL).all(), "written outside the planes"
    return y, cb, crp


def same(got, want):
    if isinstance(want, tuple):
        return all(np.array_equal(a, b) for a, b in zip(got, want))
    return np.array_equal(got, want)


# ---- 10-bit arithmetic -----------------------------------------------------------------------------------------------------
def test_p010_every_colour_within_half_a_code_value(shim):
    c = np.arange(1 << 24, dtype=np.uint32)
    y, cb, cr = (np.empty(c.shape, np.uint16) for _ in range(3))
    shim.t_p010_px(c.ctypes.data, c.size, y.ctypes.data, cb.ctypes.data, cr.ctypes.data)
    r, g, b = (c & 255).astype(np.float64), ((c >> 8) & 255).astype(np.float64), (c >> 16).astype(np.float64)
    kr, kb = 0.2126, 0.0722
    yp = kr * r + (1 - kr - kb) * g + kb * b
    fy = 64 + 876 / 255 * yp
    fcb = 512 + 896 / 255 * (b - yp) / (2 * (1 - kb))
    fcr = 512 + 896 / 255 * (r - yp) / (2 * (1 - kr))
    for got, want, bound in ((y, fy, 0.503), (cb, fcb, 0.503), (cr, fcr, 0.503)):
        assert np.abs(got.astype(np.float64) - want).max() <= bound
    assert (y[0], cb[0], cr[0]) == (64, 512, 512)
    white = (1 << 24) - 1
    assert (y[white], cb[white], cr[white]) == (940, 512, 512)
    grey = np.arange(256, dtype=np.uint32) * 0x010101
    assert (cb[grey] == 512).all() and (cr[grey] == 512).all() and (np.diff(y[grey].astype(int)) > 0).all()


def test_p010_coefficients_are_the_construction():
    kr, kb = 0.2126, 0.0722
    kg = 1 - kr - kb
    s = 65536
    assert Y10 == tuple(round(k * 876 / 255 * s) for k in (kr, kg, kb))
    cb = [round(-kr / (2 * (1 - kb)) * 896 / 255 * s), round(-kg / (2 * (1 - kb)) * 896 / 255 * s)]
    cr = [round(-kg / (2 * (1 - kr)) * 896 / 255 * s), round(-kb / (2 * (1 - kr)) * 896 / 255 * s)]
    assert CB10 == (cb[0], cb[1], -(cb[0] + cb[1])) and CR10 == (-(cr[0] + cr[1]), cr[0], cr[1])


def test_p010_chroma_of_every_block_sum(shim):
    """all 1021^3 (Sr, Sg, Sb) sums: the accumulators stay in [0, 2^31) and the codes near float64"""
    err = np.zeros(2)
    assert shim.t_cbcr10_sweep(err.ctypes.data) == 0                  # every grey sum is (512, 512)
    assert err[0] <= 0.503 and err[1] <= 0.503, err
    for k in (CB10, CR10):                                             # extreme accumulators over the sum range
        lo = sum(min(0, v) for v in k) * 1020 + (512 << 18)
        hi = sum(max(0, v) for v in k) * 1020 + (512 << 18) + (1 << 17)
        assert 0 <= lo and hi < 1 << 31


# ---- the kernel's walk -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w,h", [(128, 64), (132, 30), (66, 10), (4, 2), (390, 8), (97, 33), (5, 3), (257, 1)])
@pytest.mark.parametrize("fmt", [I420, YUV444, P010])
@pytest.mark.parametrize("native", [True, False])
def test_walk_equals_the_restatement(shim, w, h, fmt, native):
    if fmt != YUV444 and (w | h) & 1:
        w, h = w + (w & 1), h + (h & 1)
    rng = np.random.default_rng(w * 1000 + h + fmt)
    frame = premultiplied(rng, (h, w)) if native else rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    bg = (17, 240, 66)
    assert same(export_yuv(shim, frame, fmt, bg, native), frame_np(frame, NAMES[fmt], bg, native))


@pytest.mark.parametrize("w,h,rows", [(256, 40, 8), (300, 34, 5), (128, 64, 64), (134, 18, 1), (64, 30, 540), (301, 33, 7)])
@pytest.mark.parametrize("fmt", [I420, YUV444, P010])
def test_marks_skip_rows_without_reading_them(shim, w, h, rows, fmt):
    if fmt != YUV444 and (w | h) & 1:
        w, h = w - (w & 1), h - (h & 1)
    rows = min(rows, h)
    rng = np.random.default_rng(w * h + rows + fmt)
    for garbage in (False, True):
        frame, clean, marks = marked_frame(rng, w, h, rows, garbage)
        aware = export_yuv(shim, frame, fmt, (40, 50, 60), marks=marks, rows=rows)
        assert same(aware, frame_np(clean, NAMES[fmt], (40, 50, 60), True)), garbage
        assert same(aware, export_yuv(shim, clean, fmt, (40, 50, 60))), garbage


@pytest.fixture(scope="module")
def plain(tmp_path_factory):
    """test_export_core's shim, whose walk is export_kernel's (NV12)"""
    from tests.test_export_core import SHIM as PLAIN
    d = tmp_path_factory.mktemp("export_formats_plain")
    src, so = d / "shim.cpp", d / "shim.so"
    src.write_text(PLAIN)
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I", CSRC,
                    "-include", "cstring", "-o", str(so), str(src)], check=True)
    L = C.CDLL(str(so))
    vp, sz, i32, u32 = C.c_void_p, C.c_size_t, C.c_int, C.c_uint32
    L.t_export.argtypes = [vp, i32, i32, vp, i32, i32, i32, i32, u32, vp, sz, sz]
    return L


@pytest.mark.parametrize("w,h", [(128, 64), (66, 10), (390, 8)])
@pytest.mark.parametrize("native", [True, False])
def test_i420_is_deinterleaved_nv12_and_yuv444_y_is_nv12_y(shim, plain, w, h, native):
    rng = np.random.default_rng(w + h)
    frame = premultiplied(rng, (h, w)) if native else rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    bg = (9, 99, 199)
    nv12 = export(plain, frame, NV12, bg=bg, native=native)
    y, cb, cr = export_yuv(shim, frame, I420, bg, native)
    assert np.array_equal(y, nv12[:h]) and np.array_equal(cb, nv12[h:, 0::2]) and np.array_equal(cr, nv12[h:, 1::2])
    assert np.array_equal(export_yuv(shim, frame, YUV444, bg, native)[0], nv12[:h])


# ---- refusals and enqueued work through the fake runtime -----------------------------------------------------------------
FORMAT_STUBS = r"""
extern "C" void formats_fake_scaled(long long* out) { out[0] = g_scaled.format; out[1] = g_scaled.over; out[2] = (long long) g_scaled.cr_offset; }
extern "C" void formats_fake_ladder(long long* out) {
    for (int j = 0; j < GLAVA_B200_LADDER_MAX; ++j) {
        out[5 * j] = (long long) g_ladder.yuv[j].cr_offset; out[5 * j + 1] = g_ladder.yuv[j].zy; out[5 * j + 2] = g_ladder.yuv[j].zu;
        out[5 * j + 3] = g_ladder.yuv[j].zv; out[5 * j + 4] = g_ladder.rung[j].over;
    }
}
"""


@pytest.fixture(scope="module")
def fake():
    """capi.cu, export.cpp, export_ladder.cpp and config.cpp with tests/export_fake.py's stubs and the ladder's launcher"""
    inc = fakecuda.cuda_include()
    if inc is None:
        pytest.skip("no CUDA toolkit headers")
    from glava_b200.api import Export, ExportScale, Params
    out = tempfile.mkdtemp(prefix="glava_formats_fake_")
    src, so = os.path.join(out, "formats_fake.cpp"), os.path.join(out, "libformats_fake.so")
    with open(src, "w") as f:
        f.write(export_fake.STUBS + LADDER_STUBS + FORMAT_STUBS)
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
        "export_fake_launches": (C.c_long, []), "formats_fake_scaled": (None, [vp]), "formats_fake_ladder": (None, [vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = res, args
    L._quiet = C.CFUNCTYPE(None, C.c_char_p)(lambda msg: None)
    L.glava_b200_set_abort_hook(C.cast(L._quiet, vp))
    return L


def renderer(L, w, h, batch=2):
    from glava_b200.api import Params
    p = Params()
    assert L.glava_b200_default_params(C.byref(p), b"bars") == 0
    p.n, p.w, p.h = 1024, w, h
    r = L.glava_b200_new(C.byref(p), batch, 0)
    assert r, L.glava_b200_last_error()
    return C.c_void_p(r)


def device_buf(L, nbytes=1 << 18):
    b = C.c_void_p()
    assert L.cudaMalloc(C.byref(b), nbytes) == 0
    L.export_fake_device(b, nbytes)
    return b


def call(L, fn, *args):
    """-> (rc, message, trace, launches) of one export call"""
    n0 = L.export_fake_launches()
    L.fake_trace_begin()
    rc = fn(*args)
    L.fake_trace_end()
    return rc, L.glava_b200_last_error().decode(), L.fake_trace().decode(), L.export_fake_launches() - n0


def memcpys(trace):
    return [int(x.split()[-2]) for x in trace.splitlines() if x.split()[0] == "memcpy"]


def test_refusals_and_byte_counts(fake):
    L = fake
    L.fake_fail_at(-1)
    r, odd = renderer(L, 64, 32), renderer(L, 63, 31)
    buf, buf2 = device_buf(L), device_buf(L)
    s = np.zeros(1, np.int32)
    one, uv = (C.c_void_p * 1)(buf.value), (C.c_void_p * 1)(buf2.value)

    def frames(h, d):
        return call(L, L.glava_b200_export_frames, h, s.ctypes.data, 1, one, C.byref(d), None, None)

    def scaled(h, d, size, dst_uv=None):
        return call(L, L.glava_b200_export_scaled, h, s.ctypes.data, 1, one, dst_uv, C.byref(d), C.byref(scale_of(size)), None, None)

    ok = [(I420, 64), (YUV444, 64), (P010, 128), (I420, 96, 48 * 16 + 64), (YUV444, 80, 80 * 32), (P010, 128, 128 * 40)]
    for fmt, pitch, *uvo in ok:
        rc, msg, trace, launched = frames(r, desc_of(fmt, pitch, uv=uvo[0] if uvo else 0))
        assert rc == 0 and launched == 1, (fmt, msg)
        assert len(memcpys(trace)) == 1, trace
    rc, msg, _, launched = frames(odd, desc_of(YUV444, 64))
    assert rc == 0 and launched == 1, msg                             # 4:4:4 takes odd sizes
    refused = [  # (renderer, desc, what)
        (r, desc_of(3, 256), "unknown format 3"),
        (odd, desc_of(I420, 64), "I420 needs an even width and height"),
        (odd, desc_of(P010, 128), "P010 needs an even width and height"),
        (r, desc_of(I420, 80), "I420 pitch 80 must be a multiple of 32"),
        (r, desc_of(I420, 32), "at least 64"),
        (r, desc_of(P010, 112), "at least 128"),
        (r, desc_of(YUV444, 48), "at least 64"),
        (r, desc_of(I420, 64, uv=8), "uv_offset 8 (Cb plane to Cr plane)"),
        (r, desc_of(I420, 64, uv=16 * 15), "one chroma plane, 512 bytes"),
        (r, desc_of(YUV444, 64, uv=64 * 31), "one chroma plane, 2048 bytes"),
        (r, desc_of(P010, 128, uv=8), "at least pitch * h"),
        (r, desc_of(P010, 128, uv=128 * 16), "at least pitch * h"),
    ]
    for h, d, what in refused:
        rc, msg, trace, launched = frames(h, d)
        assert rc != 0 and "glava_b200_export_frames" in msg and what in msg, (what, msg)
        assert trace == "" and launched == 0, what
    # the scaled export: odd output sizes, dst_uv legal for every YUV format and refused for RGBA
    for fmt, pitch in ((I420, 32), (P010, 32)):
        rc, msg, trace, launched = scaled(r, desc_of(fmt, pitch), (15, 8))
        assert rc != 0 and "needs an even width and height, the output is 15x8" in msg and launched == 0, msg
    rc, msg, _, launched = scaled(r, desc_of(YUV444, 16), (15, 7))
    assert rc == 0 and launched == 1, msg
    for fmt, pitch in ((I420, 32), (YUV444, 16), (P010, 32), (NV12, 16)):
        rc, msg, _, launched = scaled(r, desc_of(fmt, pitch), (16, 8), uv)
        assert rc == 0 and launched == 1, (fmt, msg)
    rc, msg, trace, launched = scaled(r, desc_of(RGBA, 64), (16, 8), uv)
    assert rc != 0 and "NV12 only" in msg and trace == "" and launched == 0, msg
    # the overlay keeps its three formats and names the others
    for fmt, name in ((I420, "I420"), (YUV444, "YUV444"), (P010, "P010")):
        rc, msg, trace, launched = call(L, L.glava_b200_overlay_frames, r, s.ctypes.data, 1, one, None, C.byref(desc_of(fmt, 128)),
                                        None, None)
        assert rc != 0 and f"format {name}: the overlay takes RGBA, BGRA or NV12" in msg and "unknown" not in msg, msg
        assert trace == "" and launched == 0
    rc, msg, _, _ = call(L, L.glava_b200_overlay_frames, r, s.ctypes.data, 1, one, None, C.byref(desc_of(3, 256)), None, None)
    assert rc != 0 and "unknown format 3" in msg
    # a ladder rung in a new format is checked as its scaled export; dst_uv entries are legal for it
    pairs = [(desc_of(I420, 64), scale_of((64, 32))), (desc_of(RGBA, 64), scale_of((16, 8)))]
    two = (C.c_void_p * 2)(buf.value, buf.value)
    rc, msg, _, launched = call(L, L.glava_b200_export_ladder, r, s.ctypes.data, 1, rungs_of(pairs), 2, two,
                                (C.c_void_p * 2)(buf2.value, None), None, None)
    assert rc == 0 and launched == 1, msg
    rc, msg, _, launched = call(L, L.glava_b200_export_ladder, r, s.ctypes.data, 1, rungs_of([(desc_of(I420, 48), scale_of((16, 8)))]),
                                1, two, None, None, None)
    assert rc != 0 and "rung 0: I420 pitch 48" in msg and launched == 0, msg
    # byte counts
    n = C.c_size_t()
    for d, want in ((desc_of(I420, 64), 64 * 32 + 2 * 32 * 16), (desc_of(I420, 64, uv=1024), 64 * 32 + 1024 + 32 * 16),
                    (desc_of(YUV444, 64), 3 * 64 * 32), (desc_of(YUV444, 64, uv=4096), 64 * 32 + 4096 + 64 * 32),
                    (desc_of(P010, 128), 128 * 48), (desc_of(P010, 128, uv=8192), 8192 + 128 * 16)):
        assert L.glava_b200_export_bytes(r, C.byref(d), C.byref(n)) == 0 and n.value == want, (d.format, n.value, want)
    assert L.glava_b200_export_scaled_bytes(r, C.byref(desc_of(I420, 32)), C.byref(scale_of((16, 8))), C.byref(n)) == 0
    assert n.value == 32 * 8 + 2 * 16 * 4
    assert L.glava_b200_export_bytes(odd, C.byref(desc_of(P010, 128)), C.byref(n)) != 0
    assert L.glava_b200_export_bytes(r, C.byref(desc_of(3, 256)), C.byref(n)) != 0
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
    for fmt, pitch, uvo, cr in ((I420, 32, 0, 16 * 4), (I420, 64, 4096, 4096), (YUV444, 16, 0, 16 * 8), (P010, 32, 0, 0)):
        rc, msg, trace, launched = call(L, L.glava_b200_export_scaled, r, s.ctypes.data, 3, dst, None, C.byref(desc_of(fmt, pitch, uv=uvo)),
                                        C.byref(scale_of((16, 8))), None, None)
        assert rc == 0 and launched == 1 and memcpys(trace) == [3 * 24], (fmt, msg, trace)
        L.formats_fake_scaled(got)
        assert list(got) == [fmt, 1, cr], (fmt, list(got))
    pairs = [(desc_of(NV12, 64), scale_of((64, 32))), (desc_of(P010, 128), scale_of((64, 32))),
             (desc_of(I420, 32), scale_of((32, 16))), (desc_of(YUV444, 16, uv=512), scale_of((15, 9)))]
    rc, msg, trace, launched = call(L, L.glava_b200_export_ladder, r, s.ctypes.data, 1, rungs_of(pairs), 4, dst, None, None, None)
    assert rc == 0 and launched == 1 and memcpys(trace)[-1] == 4 * 24, (msg, trace)
    lad = (C.c_longlong * (5 * 8))()
    L.formats_fake_ladder(lad)
    assert [lad[5 * j] for j in range(4)] == [0, 0, 16 * 8, 512]
    assert [lad[5 * j + 4] for j in range(4)] == [1, 1, 1, 1]          # every YUV rung composites
    # P010's zero constants: the background (black) as 10-bit codes << 6, Y twice and (Cb, Cr)
    assert lad[5 + 1] == (64 << 6) | (64 << 22) and lad[5 + 2] == (512 << 6) | (512 << 22)
    L.glava_b200_destroy(r)
    L.cudaFree(buf)
