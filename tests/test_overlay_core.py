"""The overlay (DESIGN 4.12) on the host: the arithmetic of export_core.h (overlay_px, overlay_y, overlay_cbcr, overlay_avg4)
through a g++ shim against numpy restatements, exhaustively where the space allows, with the float64 bound of the Y'CbCr
blend and the identities that tie the overlay to the export; a g++ walk of overlay_kernel's loops (band items under the
dirty-row marks, row-pair items otherwise) bit for bit against the restatement over sentinel-filled images; the overlap
test against brute force; and the refusals and enqueued work of glava_b200_overlay_frames through capi.cu and export.cpp
built against the fake runtime of tests/fakecuda (tests/export_fake.py)."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from tests import export_fake
from tests.export_fake import desc_of
from tests.test_export_core import SHIM as PLAIN_SHIM
from tests.test_export_core import BGRA, CSRC, NV12, RGBA, bt709_fixed, export, marked_frame, nv12_np, over_np, pack, premultiplied

SHIM = PLAIN_SHIM + r"""
extern "C" void t_overlay_px(const uint32_t* px, const uint32_t* d, size_t n, uint32_t* out) {
    for (size_t i = 0; i < n; ++i) out[i] = overlay_px(px[i], d[i]);
}
extern "C" void t_overlay_y(const uint32_t* px, const uint8_t* yd, size_t n, uint8_t* out) {
    for (size_t i = 0; i < n; ++i) out[i] = (uint8_t) overlay_y(px[i], yd[i]);
}
extern "C" void t_overlay_cbcr(const uint32_t* m, const uint16_t* uvd, size_t n, uint16_t* out) {
    for (size_t i = 0; i < n; ++i) out[i] = (uint16_t) overlay_cbcr(m[i], uvd[i]);
}
extern "C" void t_overlay_avg4(const uint32_t* q, size_t n, uint32_t* out) {
    for (size_t i = 0; i < n; ++i) out[i] = overlay_avg4(q[4 * i], q[4 * i + 1], q[4 * i + 2], q[4 * i + 3]);
}
// one slot [h][w] of RGBA8 words composited onto the rectangle at dst (Y or RGBA rows) / dst_uv, as overlay_kernel walks it:
// band = 1 (native, marks): one item per (band, strip); else one per (row pair, strip), marks (or null) checked per row
extern "C" void t_overlay(const uint32_t* fb, int w, int h, const uint32_t* marks, int rows, int format, int native, int band,
                          uint8_t* dst, uint8_t* dst_uv, size_t pitch) {
    const ExportFmt f = { format, 1, 0, 0u };
    const bool nv12 = format == GLAVA_B200_EXPORT_NV12, bgra = format == GLAVA_B200_EXPORT_BGRA;
    const int strips = (w + 127) >> 7;
    auto mark = [&](int y, int strip) { return marks[export_mark_index(0, w, h, rows, y, strip)]; };
    auto load = [&](int y, int x, uint32_t q[4]) { for (int k = 0; k < 4; ++k) q[k] = x + k < w ? fb[(size_t) y * w + x + k] : 0u; };
    auto rgba = [&](uint8_t* row, int x, const uint32_t in[4]) {
        if ((in[0] | in[1] | in[2] | in[3]) == 0u) return;
        for (int k = 0; k < 4 && x + k < w; ++k) {
            uint32_t d;
            memcpy(&d, row + 4 * (x + k), 4);
            d = overlay_px(bgra ? export_swap_rb(in[k]) : in[k], d);
            memcpy(row + 4 * (x + k), &d, 4);
        }
    };
    auto nv = [&](bool nat, uint8_t* r0, uint8_t* uv, int x, const uint32_t top[4], const uint32_t bot[4]) {
        const int n = x + 4 <= w ? 4 : 2;
        uint32_t yt = 0u, yb = 0u, c = 0u;
        if (nat) {
            if ((top[0] | top[1] | top[2] | top[3] | bot[0] | bot[1] | bot[2] | bot[3]) == 0u) return;
            memcpy(&yt, r0 + x, n); memcpy(&yb, r0 + pitch + x, n); memcpy(&c, uv + x, n);
            overlay_nv12_quad(top, bot, &yt, &yb, &c);
        } else {
            c = export_nv12_quad(f, top, bot, &yt, &yb);
        }
        memcpy(r0 + x, &yt, n); memcpy(r0 + pitch + x, &yb, n); memcpy(uv + x, &c, n);
    };
    if (band) {
        for (int u = 0; u < (h + rows - 1) / rows; ++u)
            for (int strip = 0; strip < strips; ++strip)
                for (int lane = 0; lane < 32; ++lane) {
                    const int x = strip * 128 + lane * 4;
                    if (x >= w) continue;
                    const int b0 = u * rows, b1 = std::min(b0 + rows, h);
                    const uint32_t m = mark(b0, strip);
                    const int lo = std::max((int) (m & 0xffffu), b0), hi = std::min((int) (m >> 16), b1);
                    if (lo >= hi) continue;
                    if (!nv12) {
                        for (int y = lo; y < hi; ++y) {
                            uint32_t q[4];
                            load(y, x, q);
                            rgba(dst + (size_t) (h - 1 - y) * pitch, x, q);
                        }
                        continue;
                    }
                    int ja, jb;
                    const uint32_t below = overlay_band_pairs(h, b0, lo, hi, &ja, &jb) ? mark(b0 - 1, strip) : 0u;
                    if (overlay_top_straddles(h, b1, ja) && export_row_read(mark(b1, strip), b1)) ++ja;
                    for (int j = ja; j < jb; ++j) {
                        const int y0 = h - 1 - 2 * j, y1 = y0 - 1;
                        uint32_t top[4] = { 0u, 0u, 0u, 0u }, bot[4] = { 0u, 0u, 0u, 0u };
                        if (y0 >= lo && y0 < hi) load(y0, x, top);
                        if (y1 >= b0 ? y1 >= lo && y1 < hi : export_row_read(below, y1)) load(y1, x, bot);
                        nv(true, dst + (size_t) (2 * j) * pitch, dst_uv + (size_t) j * pitch, x, top, bot);
                    }
                }
        return;
    }
    for (int j = 0; j < (h + 1) / 2; ++j)
        for (int strip = 0; strip < strips; ++strip)
            for (int lane = 0; lane < 32; ++lane) {
                const int x = strip * 128 + lane * 4;
                if (x >= w) continue;
                const int y0 = h - 1 - 2 * j, y1 = y0 - 1;
                uint32_t top[4] = { 0u, 0u, 0u, 0u }, bot[4] = { 0u, 0u, 0u, 0u };
                if (!marks || export_row_read(mark(y0, strip), y0)) load(y0, x, top);
                if (y1 >= 0 && (!marks || export_row_read(mark(y1, strip), y1))) load(y1, x, bot);
                uint8_t* r0 = dst + (size_t) (2 * j) * pitch;
                if (nv12) {
                    nv(native, r0, dst_uv + (size_t) j * pitch, x, top, bot);
                } else if (native) {
                    rgba(r0, x, top);
                    if (y1 >= 0) rgba(r0 + pitch, x, bot);
                } else {
                    for (int r = 0; r < 2 && (r == 0 || y1 >= 0); ++r)
                        for (int k = 0; k < 4 && x + k < w; ++k) {
                            const uint32_t v = export_px(f, r ? bot[k] : top[k]);
                            memcpy(r0 + (size_t) r * pitch + (size_t) (x + k) * 4, &v, 4);
                        }
                }
            }
}
"""


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("overlay_core")
    src, so = d / "shim.cpp", d / "shim.so"
    src.write_text(SHIM)
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I", CSRC,
                    "-include", "cstring", "-include", "algorithm", "-o", str(so), str(src)], check=True)
    L = C.CDLL(str(so))
    vp, sz, i32, u32 = C.c_void_p, C.c_size_t, C.c_int, C.c_uint32
    L.t_overlay_px.argtypes = [vp, vp, sz, vp]
    L.t_overlay_y.argtypes = [vp, vp, sz, vp]
    L.t_overlay_cbcr.argtypes = [vp, vp, sz, vp]
    L.t_overlay_avg4.argtypes = [vp, sz, vp]
    L.t_overlay.argtypes = [vp, i32, i32, vp, i32, i32, i32, i32, vp, vp, sz]
    L.t_export.argtypes = [vp, i32, i32, vp, i32, i32, i32, i32, u32, vp, sz, sz]
    L.t_ycbcr.argtypes = [vp, sz, vp, vp, vp]
    return L


def call(fn, out_dtype, *arrays):
    arrays = [np.ascontiguousarray(a) for a in arrays]
    out = np.empty(arrays[0].shape[:1] if arrays[0].ndim == 1 else arrays[0].shape[:-1], out_dtype)
    n = out.shape[0]
    fn(*[a.ctypes.data for a in arrays], n, out.ctypes.data)
    return out


# ---- numpy restatement ---------------------------------------------------------------------------------------------------
def mul_norm8_np(x, y):
    return (2 * x * y + 255) // 510


def frac_np(off, a, vd):
    return ((off * a + (255 - a) * vd) * 65536 + 127) // 255


def y_np(c, yd):
    """c [..., 4] stored pixels, yd [...]: the overlay Y byte"""
    ky, _, _ = bt709_fixed()
    dot = ky[0] * c[..., 0] + ky[1] * c[..., 1] + ky[2] * c[..., 2]
    return np.clip((dot + frac_np(16, c[..., 3], yd) + (1 << 15)) >> 16, 0, 255)


def cbcr_np(m, cbd, crd):
    """m [..., 4] block averages (alpha included): the overlay (Cb, Cr)"""
    _, kcb, kcr = bt709_fixed()
    a = m[..., 3]
    dot = lambda k: k[0] * m[..., 0] + k[1] * m[..., 1] + k[2] * m[..., 2]
    cb = np.clip((dot(kcb) + frac_np(128, a, cbd) + (1 << 15)) >> 16, 0, 255)
    cr = np.clip((dot(kcr) + frac_np(128, a, crd) + (1 << 15)) >> 16, 0, 255)
    return cb, cr


def overlay_np(frame, rect, fmt, native):
    """frame: read-back [h][w][4] (row 0 = bottom); rect: the destination rectangle's bytes before the call (RGBA / BGRA
    [h][w][4], NV12 [h * 3 / 2][w]) -> its bytes after"""
    h, w = frame.shape[:2]
    if not native:
        if fmt == NV12:
            return nv12_np(frame, (0, 0, 0), False)
        out = over_np(frame[::-1], (0, 0, 0), False).astype(np.uint8)
        return out[..., [2, 1, 0, 3]] if fmt == BGRA else out
    c = frame[::-1].astype(np.int64)
    if fmt != NV12:
        if fmt == BGRA:
            c = c[..., [2, 1, 0, 3]]
        d = rect.astype(np.int64)
        return np.minimum(255, c + mul_norm8_np(d, 255 - c[..., 3:4])).astype(np.uint8)
    y = y_np(c, rect[:h].astype(np.int64))
    avg = (c.reshape(h // 2, 2, w // 2, 2, 4).sum(axis=(1, 3)) + 2) >> 2
    uvd = rect[h:].astype(np.int64).reshape(h // 2, w // 2, 2)
    cb, cr = cbcr_np(avg, uvd[..., 0], uvd[..., 1])
    return np.concatenate([y, np.stack([cb, cr], axis=-1).reshape(h // 2, w)]).astype(np.uint8)


# ---- arithmetic --------------------------------------------------------------------------------------------------------------
def test_rgba_overlay_every_channel_alpha_and_destination(shim):
    """all 2^24 (c, a, D): c in R, G and B, D in all four channels"""
    c, a, d = (v.reshape(-1).astype(np.uint32) for v in np.meshgrid(np.arange(256), np.arange(256), np.arange(256), indexing="ij"))
    out = call(shim.t_overlay_px, np.uint32, pack(c, c, c, a), pack(d, d, d, d))
    ci, ai, di = c.astype(np.int64), a.astype(np.int64), d.astype(np.int64)
    want_c = np.minimum(255, ci + mul_norm8_np(di, 255 - ai))
    want_a = np.minimum(255, ai + mul_norm8_np(di, 255 - ai))
    for k in range(3):
        assert np.array_equal((out >> (8 * k)) & 255, want_c), k
    assert np.array_equal(out >> 24, want_a)
    assert np.array_equal(out[(c == 0) & (a == 0)], pack(d, d, d, d)[(c == 0) & (a == 0)])   # zero leaves D


def premult_colours(rng, a, n):
    """n random premultiplied (r, g, b) per alpha value in a, with the extremes 0 and a included"""
    a = np.repeat(a, n)
    rgb = (rng.random((a.size, 3)) * (a[:, None] + 1)).astype(np.int64)
    rgb = np.minimum(rgb, a[:, None])
    rgb[::n] = 0
    rgb[1::n] = a[1::n, None]
    return np.concatenate([rgb, a[:, None]], axis=1)


def test_nv12_y_every_alpha_and_destination_with_its_float_bound(shim):
    """overlay_y over every (a, Y_D) for sampled premultiplied colours: equal to the integer restatement, and within 0.51 code
    values of the float64 composite 16 a / 255 + 219 / 255 (Kr r + Kg g + Kb b) + (1 - a / 255) Y_D: 0.5008 on this sample
    (the final rounding, the 16-bit coefficients and the floor of the T term)"""
    rng = np.random.default_rng(1)
    px = premult_colours(rng, np.arange(256), 24)                   # [256 * 24][4]
    yd = np.arange(256)
    P, YD = np.repeat(px, 256, axis=0), np.tile(yd, px.shape[0])
    got = call(shim.t_overlay_y, np.uint8, pack(P[:, 0], P[:, 1], P[:, 2], P[:, 3]), YD.astype(np.uint8)).astype(np.int64)
    assert np.array_equal(got, y_np(P, YD))
    kr, kb = 0.2126, 0.0722
    al = P[:, 3] / 255.0
    fy = 16 * al + 219 / 255 * (kr * P[:, 0] + (1 - kr - kb) * P[:, 1] + kb * P[:, 2]) + (1 - al) * YD
    err = np.abs(got - fy).max()
    assert err <= 0.501, err


def test_nv12_cbcr_every_alpha_and_destination_with_its_float_bound(shim):
    rng = np.random.default_rng(2)
    m = premult_colours(rng, np.arange(256), 12)
    d = rng.integers(0, 256, (256, 2))
    d[0], d[1], d[2] = (0, 0), (255, 255), (128, 128)
    M, D = np.repeat(m, 256, axis=0), np.tile(d, (m.shape[0], 1))
    got = call(shim.t_overlay_cbcr, np.uint16, pack(M[:, 0], M[:, 1], M[:, 2], M[:, 3]),
               (D[:, 0] | (D[:, 1] << 8)).astype(np.uint16)).astype(np.int64)
    cb, cr = cbcr_np(M, D[:, 0], D[:, 1])
    assert np.array_equal(got & 255, cb) and np.array_equal(got >> 8, cr)
    # every (a, Cb_D) for one colour per alpha: the T term alone
    M2 = np.repeat(premult_colours(rng, np.arange(256), 1), 256, axis=0)
    V = np.tile(np.arange(256), 256)
    got2 = call(shim.t_overlay_cbcr, np.uint16, pack(M2[:, 0], M2[:, 1], M2[:, 2], M2[:, 3]), (V | (V << 8)).astype(np.uint16))
    cb2, cr2 = cbcr_np(M2, V, V)
    assert np.array_equal(got2.astype(np.int64) & 255, cb2) and np.array_equal(got2.astype(np.int64) >> 8, cr2)
    kr, kb = 0.2126, 0.0722
    r, g, b, al = M[:, 0], M[:, 1], M[:, 2], M[:, 3] / 255.0
    yp = kr * r + (1 - kr - kb) * g + kb * b
    fcb = 128 * al + 224 / 255 * (b - yp) / (2 * (1 - kb)) + (1 - al) * D[:, 0]
    fcr = 128 * al + 224 / 255 * (r - yp) / (2 * (1 - kr)) + (1 - al) * D[:, 1]
    err = max(np.abs((got & 255) - fcb).max(), np.abs((got >> 8) - fcr).max())
    assert err <= 0.502, err                                        # 0.5015 measured


def test_avg4_is_the_export_average_with_alpha(shim):
    rng = np.random.default_rng(3)
    q = rng.integers(0, 1 << 32, (4096, 4), dtype=np.uint64).astype(np.uint32)
    got = call(shim.t_overlay_avg4, np.uint32, q)
    b = q.view(np.uint8).reshape(4096, 4, 4).astype(np.int64)
    want = ((b.sum(axis=1) + 2) >> 2).astype(np.uint8)
    assert np.array_equal(got.view(np.uint8).reshape(4096, 4), want)


def test_endpoint_identities(shim):
    """a zero pixel leaves every Y / CbCr byte; an opaque pixel gives export_y, an opaque block export_cbcr of export_avg4"""
    v = np.arange(256)
    zero = np.zeros(256, np.uint32)
    assert np.array_equal(call(shim.t_overlay_y, np.uint8, zero, v.astype(np.uint8)), v)
    uv = (v[:, None] | (v[None, :] << 8)).reshape(-1).astype(np.uint16)
    assert np.array_equal(call(shim.t_overlay_cbcr, np.uint16, np.zeros(uv.size, np.uint32), uv), uv)
    c = np.arange(1 << 24, dtype=np.uint32)[::7] | np.uint32(0xff000000)
    y0, cb0, cr0 = (np.empty(c.shape, np.uint8) for _ in range(3))
    shim.t_ycbcr(c.ctypes.data, c.size, y0.ctypes.data, cb0.ctypes.data, cr0.ctypes.data)
    rng = np.random.default_rng(4)
    yd = rng.integers(0, 256, c.size).astype(np.uint8)
    assert np.array_equal(call(shim.t_overlay_y, np.uint8, c, yd), y0)
    uvd = rng.integers(0, 1 << 16, c.size).astype(np.uint16)
    got = call(shim.t_overlay_cbcr, np.uint16, c, uvd)
    assert np.array_equal(got & 255, cb0) and np.array_equal(got >> 8, cr0)


@pytest.mark.parametrize("fmt", [RGBA, BGRA])
def test_rgba_onto_an_opaque_colour_is_the_composited_export(shim, fmt):
    rng = np.random.default_rng(5)
    h, w = 30, 132
    frame = premultiplied(rng, (h, w))
    frame[rng.random((h, w)) < 0.3] = 0
    for bg in ((0, 0, 0), (255, 255, 255), (17, 240, 66)):
        img = np.empty((h, w, 4), np.uint8)
        img[:] = (*bg, 255) if fmt == RGBA else (bg[2], bg[1], bg[0], 255)
        got = overlay(shim, frame, img, fmt, True)
        assert np.array_equal(got, export(shim, frame, fmt, over=True, bg=bg).reshape(h, w, 4)), bg


def test_nv12_opaque_frames_give_the_export(shim):
    rng = np.random.default_rng(6)
    h, w = 16, 132
    frame = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    frame[..., 3] = 255
    img = rng.integers(0, 256, (h * 3 // 2, w), dtype=np.uint8)
    assert np.array_equal(overlay(shim, frame, img, NV12, True), export(shim, frame, NV12))


# ---- the kernel's walk -------------------------------------------------------------------------------------------------------
def overlay(L, frame, img, fmt, native, marks=None, rows=0, band=False, pad=32, off=16):
    """composite `frame` onto a copy of `img` (the rectangle's bytes) placed `off` bytes into sentinel-filled rows of
    `pad` extra bytes, with NV12 chroma rows in a separate area; checks the sentinels and returns the rectangle"""
    h, w = frame.shape[:2]
    nv12 = fmt == NV12
    row = w if nv12 else w * 4
    pitch = (off + row + pad + 15) // 16 * 16
    yrows = h
    buf = np.full((yrows + 2 + (h // 2 if nv12 else 0) + 2, pitch), 0xA5, np.uint8)
    ybase, uvbase = 1, yrows + 3
    rect = img.reshape(h * 3 // 2 if nv12 else h, row)
    buf[ybase:ybase + h, off:off + row] = rect[:h]
    if nv12:
        buf[uvbase:uvbase + h // 2, off:off + row] = rect[h:]
    before = buf.copy()
    fb = np.ascontiguousarray(frame).view(np.uint32).reshape(h, w)
    m = None if marks is None else np.ascontiguousarray(marks, np.uint32)
    L.t_overlay(fb.ctypes.data, w, h, None if m is None else m.ctypes.data, rows, fmt, int(native), int(band),
                buf.ctypes.data + ybase * pitch + off, buf.ctypes.data + uvbase * pitch + off, pitch)
    inside = np.zeros(buf.shape, bool)
    inside[ybase:ybase + h, off:off + row] = True
    if nv12:
        inside[uvbase:uvbase + h // 2, off:off + row] = True
    assert np.array_equal(buf[~inside], before[~inside]), "written outside the rectangle"
    out = buf[ybase:ybase + h, off:off + row]
    if nv12:
        out = np.concatenate([out, buf[uvbase:uvbase + h // 2, off:off + row]])
    return out.reshape(img.shape)


def random_image(rng, fmt, w, h):
    return rng.integers(0, 256, (h * 3 // 2, w) if fmt == NV12 else (h, w, 4), dtype=np.uint8)


@pytest.mark.parametrize("w,h", [(128, 64), (132, 30), (66, 10), (4, 2), (390, 8), (97, 7), (257, 1)])
@pytest.mark.parametrize("native", [True, False])
def test_walk_without_marks_equals_the_restatement(shim, w, h, native):
    rng = np.random.default_rng(w * 100 + h)
    frame = premultiplied(rng, (h, w)) if native else rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    frame[rng.random((h, w)) < 0.4] = 0
    frame[: h // 3] = 0                                              # whole zero rows
    for fmt in (RGBA, BGRA, NV12):
        if fmt == NV12 and (w | h) & 1:
            continue
        img = random_image(rng, fmt, w, h)
        got = overlay(shim, frame, img, fmt, native)
        assert np.array_equal(got, overlay_np(frame, img, fmt, native)), fmt
        if native:                                                   # where the frame is zero the image is untouched
            top = frame[::-1]
            if fmt != NV12:
                z = (top == 0).all(axis=-1)
                assert np.array_equal(got[z], img[z])


@pytest.mark.parametrize("w,h,rows", [(256, 40, 8), (300, 34, 5), (128, 64, 64), (132, 18, 1), (64, 30, 540), (98, 36, 7),
                                      (130, 24, 3), (66, 20, 9)])
@pytest.mark.parametrize("fmt", [RGBA, BGRA, NV12])
def test_mark_aware_walks_equal_the_restatement(shim, w, h, rows, fmt):
    """band items and row-pair items under marks, over garbage in the rows the marks skip, odd band heights included
    (NV12 row pairs that straddle a band edge)"""
    rows = min(rows, h)
    rng = np.random.default_rng(w * h + rows + 7 * fmt)
    for garbage in (False, True):
        frame, clean, marks = marked_frame(rng, w, h, rows, garbage)
        img = random_image(rng, fmt, w, h)
        want = overlay_np(clean, img, fmt, True)
        for band in (True, False):
            got = overlay(shim, frame, img, fmt, True, marks=marks, rows=rows, band=band)
            assert np.array_equal(got, want), (garbage, band)
        if not garbage:                                              # any other opacity: the export's bytes
            got = overlay(shim, frame, img, fmt, False, marks=marks, rows=rows)
            assert np.array_equal(got, overlay_np(clean, img, fmt, False))


def test_band_walk_straddling_pairs_with_every_mark_pattern(shim):
    """bands of 3 rows on a 12-row NV12 frame: every combination of marked intervals in neighbouring bands, so every
    straddling pair is blended exactly once"""
    w, h, rows = 8, 12, 3
    rng = np.random.default_rng(9)
    frame = premultiplied(rng, (h, w))
    frame[..., 3] = np.maximum(frame[..., 3], 1)
    img = random_image(rng, NV12, w, h)
    intervals = [(0, 0), (0, 1), (0, 3), (1, 2), (2, 3), (1, 3)]
    for trial in range(300):
        marks = np.zeros((h, 1), np.uint32)
        clean = frame.copy()
        keep = np.zeros(h, bool)
        for b0 in range(0, h, rows):
            lo, hi = intervals[rng.integers(len(intervals))]
            if lo < hi:
                marks[b0, 0] = (b0 + lo) | ((b0 + hi) << 16)
                keep[b0 + lo:b0 + hi] = True
        clean[~keep] = 0
        got = overlay(shim, clean, img, NV12, True, marks=marks, rows=rows, band=True)
        assert np.array_equal(got, overlay_np(clean, img, NV12, True)), trial


# ---- the overlap test ----------------------------------------------------------------------------------------------------------
def brute_overlap(rects, P, B):
    spans = set()
    for (p, n) in rects:
        for k in range(n):
            for b in range(p + k * P, p + k * P + B):
                if b in spans:
                    return True
                spans.add(b)
    return False


def brute_meets(rects, P, B, f0, f1):
    return any(p + k * P < f1 and p + k * P + B > f0 for p, n in rects for k in range(n))


@pytest.fixture(scope="module")
def fake():
    L = export_fake.lib()
    if L is None:
        pytest.skip("no CUDA toolkit headers")
    return L


def test_overlap_test_equals_brute_force(fake):
    rng = np.random.default_rng(10)
    base = 1 << 20
    for trial in range(3000):
        w = int(rng.integers(1, 5)) * 2
        h = int(rng.integers(1, 4)) * 2
        nv12 = bool(rng.random() < 0.5)
        B = w if nv12 else 4 * w
        P = B + int(rng.integers(0, 4)) * 16 if rng.random() < 0.8 else B
        P = (P + 15) // 16 * 16
        count = int(rng.integers(1, 5))
        span = P * (3 * h + 4)
        dst = [base + int(rng.integers(0, span // 16)) * 16 for _ in range(count)]
        uv = [base + int(rng.integers(0, span // 16)) * 16 for _ in range(count)] if nv12 else None
        rects = [(p, h) for p in dst] + ([(p, h // 2) for p in uv] if nv12 else [])
        f0 = base + int(rng.integers(0, span))
        f1 = f0 + int(rng.integers(1, 3 * P))
        d = (C.c_size_t * count)(*dst)
        u = (C.c_size_t * count)(*uv) if nv12 else None
        rc = fake.t_geometry(w, h, count, d, u, P, f0, f1 - f0)
        want = brute_overlap(rects, P, B) or brute_meets(rects, P, B, f0, f1)
        assert (rc != 0) == want, (trial, w, h, nv12, P, dst, uv, f0, f1)
        if rc == 0:
            continue
        msg = fake.glava_b200_last_error().decode()
        assert "t_geometry" in msg and ("framebuffer" in msg) == brute_meets(rects, P, B, f0, f1), msg   # checked first


def test_a_mosaic_of_1024_tiles_checks_fast(fake):
    """32 x 32 NV12 tiles of 128 x 72 in one 4096 x 2304 image: accepted, and sorted by address the check stays far
    from quadratic"""
    import time
    P, th, tw, H = 4096, 72, 128, 2304
    base = 1 << 32
    dst = [base + (i // 32) * th * P + (i % 32) * tw for i in range(1024)]
    uv = [base + (H + (i // 32) * th // 2) * P + (i % 32) * tw for i in range(1024)]
    d, u = (C.c_size_t * 1024)(*dst), (C.c_size_t * 1024)(*uv)
    t = time.perf_counter()
    assert fake.t_geometry(tw, th, 1024, d, u, P, 1 << 20, 4096) == 0
    assert time.perf_counter() - t < 0.05
    dst[700] = dst[699] + 16                                         # one tile shifted onto its neighbour
    assert fake.t_geometry(tw, th, 1024, (C.c_size_t * 1024)(*dst), u, P, 1 << 20, 4096) != 0
    assert "entry 699" in fake.glava_b200_last_error().decode()


def _overlay(L, h, streams, dsts, d, uvs=None, after=None, done=None):
    s = np.asarray(streams, np.int32)
    arr = (C.c_void_p * max(len(dsts), 1))(*dsts)
    uv = None if uvs is None else (C.c_void_p * max(len(uvs), 1))(*uvs)
    n0 = L.export_fake_launches()
    L.fake_trace_begin()
    rc = L.glava_b200_overlay_frames(h, s.ctypes.data, len(streams), arr, uv, C.byref(d), after, done)
    L.fake_trace_end()
    return rc, L.glava_b200_last_error().decode(), L.fake_trace().decode(), L.export_fake_launches() - n0


def test_refusals_name_the_function_and_enqueue_nothing(fake):
    L = fake
    L.fake_fail_at(-1)
    h, p = L.renderer(n=1024, w=64, h=32)                              # frame 64 x 32
    buf, buf2 = L.device_buf(1 << 18), L.device_buf()
    host = np.zeros(1 << 16, np.uint8)
    aligned_host = host.ctypes.data + (-host.ctypes.data) % 16
    b = buf.value
    # two RGBA rectangles side by side in a 1024-byte pitch, one stream twice
    rc, msg, trace, launched = _overlay(L, h, [0, 1, 1], [b, b + 256, b + 512], desc_of(RGBA, 1024))
    assert rc == 0 and launched == 1, msg
    last = (C.c_int * 4)()
    L.overlay_fake_last(last)
    assert list(last) == [3, 0, 1, RGBA]                              # no marks before the first pass: row-pair items
    rc, msg, trace, launched = _overlay(L, h, [0, 1], [b, b + 64], desc_of(NV12, 128), uvs=[b + 128 * 32, b + 128 * 32 + 64])
    assert rc == 0 and launched == 1, msg
    rc, msg, trace, launched = _overlay(L, h, [0], [b], desc_of(NV12, 64))              # chroma at pitch * h
    assert rc == 0 and launched == 1, msg
    fbp = L.glava_b200_framebuffer_device(h)
    L.export_fake_device(fbp, 2 * 64 * 32 * 4)
    cases = [
        ([0], [b], desc_of(3, 256), None, "unknown format"),
        ([0], [b], desc_of(RGBA, 256, flags=1), None, "takes none"),
        ([0], [b], desc_of(RGBA, 256, flags=2), None, "unknown flags"),
        ([0], [b], desc_of(RGBA, 240), None, "pitch"),
        ([0], [b], desc_of(RGBA, 264), None, "pitch"),
        ([0], [b], desc_of(NV12, 64, uv=8), None, "uv_offset"),
        ([0], [b], desc_of(NV12, 64, uv=64 * 16), None, "uv_offset"),
        ([0], [b], desc_of(RGBA, 256), [b2 := buf2.value], "NV12 only"),
        ([0], [b], desc_of(NV12, 64), [b2 + 8], "dst_uv[0]"),
        ([0], [b], desc_of(NV12, 64), [None], "dst_uv[0]"),
        ([0], [b], desc_of(NV12, 64), [aligned_host], "dst_uv[0] = "),
        ([0], [b + 8], desc_of(RGBA, 256), None, "aligned"),
        ([0], [None], desc_of(RGBA, 256), None, "null"),
        ([0], [aligned_host], desc_of(RGBA, 256), None, "not device memory"),
        ([2], [b], desc_of(RGBA, 256), None, "out of range"),
        ([-1], [b], desc_of(RGBA, 256), None, "out of range"),
        ([], [], desc_of(RGBA, 256), None, "count"),
        ([0, 1], [b, b], desc_of(RGBA, 1024), None, "overlaps"),                    # the same rectangle twice
        ([0, 1], [b, b + 240], desc_of(RGBA, 1024), None, "overlaps"),              # 16 bytes shared per row
        ([0, 1], [b, b + 1024 * 31], desc_of(RGBA, 1024), None, "overlaps"),        # last row / first row
        ([0, 1], [b, b + 64], desc_of(NV12, 128), [b + 128 * 32, b + 128 * 32 + 48], "CbCr rectangle"),
        ([0, 1], [b, b + 64 * 40], desc_of(NV12, 64), None, "overlaps"),            # entry 1's luma on entry 0's chroma
        ([0], [fbp], desc_of(RGBA, 256), None, "framebuffer"),
        ([0], [b], desc_of(NV12, 64), [fbp], "framebuffer"),
    ]
    for streams, dsts, d, uvs, what in cases:
        rc, msg, trace, launched = _overlay(L, h, streams, dsts, d, uvs)
        assert rc != 0, what
        assert "glava_b200_overlay_frames" in msg and what in msg, (msg, what)
        assert trace == "" and launched == 0, (what, trace)
    h2, _ = L.renderer(n=1024, w=64, h=31)
    rc, msg, trace, launched = _overlay(L, h2, [0], [b], desc_of(NV12, 64))
    assert rc != 0 and "even" in msg and trace == "" and launched == 0
    L.glava_b200_destroy(h2)
    q = p.__class__.from_buffer_copy(bytes(p))
    q.smooth_factor = 0.03 if p.smooth_factor != 0.03 else 0.02
    L.fake_fail_at(0)
    assert L.glava_b200_reconfigure(h, C.byref(q)) != 0
    L.fake_fail_at(-1)
    rc, msg, trace, launched = _overlay(L, h, [0], [b], desc_of(RGBA, 256))
    assert rc != 0 and "glava_b200_overlay_frames" in msg and "no tables" in msg and trace == "" and launched == 0
    L.glava_b200_destroy(h)
    assert L.cudaFree(buf) == 0 and L.cudaFree(buf2) == 0


def test_one_copy_one_launch_on_the_raster_stream(fake):
    """wait for `after`, the list copy, its event, the kernel, `done`, all on the raster stream; band items once a pass has
    kept marks; the list buffers are the export's and live until the renderer is destroyed"""
    L = fake
    L.fake_fail_at(-1)
    live0 = [L.fake_live(k) for k in range(4)]
    h, p = L.renderer(n=1024, w=64, h=32)
    buf = L.device_buf()
    a, d = C.c_void_p(), C.c_void_p()
    assert L.cudaEventCreate(C.byref(a)) == 0 and L.cudaEventCreate(C.byref(d)) == 0
    pcm = np.zeros((2, 1024), np.float32)
    assert L.glava_b200_update(h, pcm.ctypes.data, pcm.ctypes.data, 1024, 1) == 0
    last = (C.c_int * 4)()
    for rep in range(6):                                              # past the four list buffers
        rc, msg, trace, launched = _overlay(L, h, [rep % 2], [buf.value], desc_of(NV12, 64), None, a, d)
        assert rc == 0 and launched == 1, msg
        lines = [x.split() for x in trace.splitlines()]
        kinds = [x[0] for x in lines]
        assert kinds[-4:] == ["wait", "memcpy", "record", "record"], trace
        assert len({lines[-4][1], lines[-3][-1], lines[-2][-1], lines[-1][-1]}) == 1, trace
        L.overlay_fake_last(last)
        assert list(last)[:3] == [1, 1, 1]                            # bars keeps marks: band items under native opacity
        dst = (C.c_void_p * 1)(buf.value)
        s = np.zeros(1, np.int32)
        assert L.glava_b200_export_frames(h, s.ctypes.data, 1, dst, C.byref(desc_of(RGBA, 256)), None, None) == 0
    L.glava_b200_destroy(h)
    L.cudaEventDestroy(a); L.cudaEventDestroy(d); L.cudaFree(buf)
    assert [L.fake_live(k) for k in range(4)] == live0
