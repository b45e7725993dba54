"""Frame export (DESIGN 4.10) on the host: the pixel arithmetic of export_core.h through a g++ shim, and the refusals and
enqueued work of glava_b200_export_frames / _export_bytes through capi.cu and export.cpp built against the fake runtime of
tests/fakecuda (tests/export_fake.py).

The shim's t_export walks one framebuffer slot the way export_kernels.cu does (row pairs, 128-pixel strips, quads, the
dirty-row marks deciding which rows are read) with the same core functions, so the layout and the mark logic are checked
here against independent numpy restatements, bit for bit."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import export_fake
from tests.export_fake import desc_of

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "glava_b200", "csrc")
RGBA, BGRA, NV12, OVER = 0, 1, 2, 1

SHIM = r"""
#include "export_core.h"
using namespace glb;
extern "C" void t_ycbcr(const uint32_t* px, size_t n, uint8_t* y, uint8_t* cb, uint8_t* cr) {
    for (size_t i = 0; i < n; ++i) { const uint32_t c = export_cbcr(px[i]); y[i] = (uint8_t) export_y(px[i]); cb[i] = c & 255u; cr[i] = c >> 8; }
}
extern "C" void t_px(const uint32_t* px, size_t n, int format, int over, int native, uint32_t bg, uint32_t* out) {
    const ExportFmt f = { format, over, native, bg };
    for (size_t i = 0; i < n; ++i) out[i] = export_px(f, px[i]);
}
// one slot [h][w] of RGBA8 words -> dst, as export_kernel walks it; marks: the slot's [h][strips] words or null
extern "C" void t_export(const uint32_t* fb, int w, int h, const uint32_t* marks, int rows, int format, int over, int native,
                         uint32_t bg, uint8_t* dst, size_t pitch, size_t uv_offset) {
    const ExportFmt f = { format, format == GLAVA_B200_EXPORT_NV12 || over, native, bg };
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
                uint8_t* r0 = dst + (size_t) (2 * j) * pitch;
                if (format == GLAVA_B200_EXPORT_NV12) {
                    uint32_t yt, yb;
                    const uint32_t uv = export_nv12_quad(f, q[0], q[1], &yt, &yb);
                    const int n = x + 4 <= w ? 4 : 2;
                    for (int k = 0; k < n; ++k) {
                        r0[x + k] = (uint8_t) (yt >> (8 * k)); r0[pitch + x + k] = (uint8_t) (yb >> (8 * k));
                        dst[uv_offset + (size_t) j * pitch + x + k] = (uint8_t) (uv >> (8 * k));
                    }
                } else {
                    for (int r = 0; r < 2 && (r == 0 || y1 >= 0); ++r)
                        for (int k = 0; k < 4 && x + k < w; ++k) {
                            const uint32_t v = export_px(f, q[r][k]);
                            memcpy(r0 + (size_t) r * pitch + (size_t) (x + k) * 4, &v, 4);
                        }
                }
            }
}
"""


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("export_core")
    src, so = d / "shim.cpp", d / "shim.so"
    src.write_text(SHIM)
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I", CSRC,
                    "-include", "cstring", "-o", str(so), str(src)], check=True)
    L = C.CDLL(str(so))
    vp, sz, i32, u32 = C.c_void_p, C.c_size_t, C.c_int, C.c_uint32
    L.t_ycbcr.argtypes = [vp, sz, vp, vp, vp]
    L.t_px.argtypes = [vp, sz, i32, i32, i32, u32, vp]
    L.t_export.argtypes = [vp, i32, i32, vp, i32, i32, i32, i32, u32, vp, sz, sz]
    return L


def ycbcr(L, px):
    px = np.ascontiguousarray(px, np.uint32)
    y, cb, cr = (np.empty(px.shape, np.uint8) for _ in range(3))
    L.t_ycbcr(px.ctypes.data, px.size, y.ctypes.data, cb.ctypes.data, cr.ctypes.data)
    return y, cb, cr


def pack(r, g, b, a=0):
    return (np.asarray(r, np.uint32) | (np.asarray(g, np.uint32) << 8) | (np.asarray(b, np.uint32) << 16)
            | (np.asarray(a, np.uint32) << 24))


# ---- numpy restatements --------------------------------------------------------------------------------------------------
def over_np(frame, bg, native):
    """[..., 4] uint8 -> composited [..., 4]: c + round_half_up(bg * (255 - a) / 255), saturated; alpha 255"""
    out = frame.astype(np.int64).copy()
    if native:
        ia = 255 - out[..., 3:4]
        out[..., :3] = np.minimum(255, out[..., :3] + (2 * np.asarray(bg[:3], np.int64) * ia + 255) // 510)
    out[..., 3] = 255
    return out


def bt709_fixed():
    """the 16-bit coefficients from the formula: Y rows scaled by 219/255, chroma by 224/255, grey-exact chroma"""
    kr, kb = 0.2126, 0.0722
    kg = 1 - kr - kb
    s = 65536
    y = [round(k * 219 / 255 * s) for k in (kr, kg, kb)]
    cb = [round(-kr / (2 * (1 - kb)) * 224 / 255 * s), round(-kg / (2 * (1 - kb)) * 224 / 255 * s)]
    cr = [round(-kg / (2 * (1 - kr)) * 224 / 255 * s), round(-kb / (2 * (1 - kr)) * 224 / 255 * s)]
    return y, [cb[0], cb[1], -(cb[0] + cb[1])], [-(cr[0] + cr[1]), cr[0], cr[1]]


def nv12_np(frame, bg, native):
    """[h][w][4] bottom-up framebuffer slot -> NV12 bytes [h * 3 / 2][w] (tight pitch)"""
    h, w = frame.shape[:2]
    c = over_np(frame[::-1], bg, native)
    ky, kcb, kcr = bt709_fixed()
    dot = lambda k, v: k[0] * v[..., 0] + k[1] * v[..., 1] + k[2] * v[..., 2]
    y = (dot(ky, c) + (16 << 16) + (1 << 15)) >> 16
    blk = c[..., :3].reshape(h // 2, 2, w // 2, 2, 3).sum(axis=(1, 3))
    avg = (blk + 2) >> 2
    cb = (dot(kcb, avg) + (128 << 16) + (1 << 15)) >> 16
    cr = (dot(kcr, avg) + (128 << 16) + (1 << 15)) >> 16
    uv = np.stack([cb, cr], axis=-1).reshape(h // 2, w)
    return np.concatenate([y, uv]).astype(np.uint8)


def export(L, frame, fmt, over=False, native=True, bg=(0, 0, 0), marks=None, rows=0, pitch=None):
    h, w = frame.shape[:2]
    row = w if fmt == NV12 else w * 4
    pitch = pitch or (row + 15) // 16 * 16
    nrows = h * 3 // 2 if fmt == NV12 else h
    dst = np.full((nrows, pitch), 0xA5, np.uint8)
    fb = np.ascontiguousarray(frame).view(np.uint32).reshape(h, w)
    m = None if marks is None else np.ascontiguousarray(marks, np.uint32)
    L.t_export(fb.ctypes.data, w, h, None if m is None else m.ctypes.data, rows, fmt, int(over), int(native),
               int(pack(*bg[:3])), dst.ctypes.data, pitch, pitch * h)
    assert (dst[:, row:] == 0xA5).all(), "written past the row"
    return dst[:, :row]


def premultiplied(rng, shape):
    """random RGBA8 with c <= a (what setopacity "native" stores)"""
    a = rng.integers(0, 256, shape + (1,))
    c = (rng.random(shape + (3,)) * (a + 1)).astype(np.int64)
    return np.concatenate([np.minimum(c, a), a], axis=-1).astype(np.uint8)


# ---- BT.709 ---------------------------------------------------------------------------------------------------------------
def test_bt709_every_colour_within_one_code_value(shim):
    c = np.arange(1 << 24, dtype=np.uint32)
    y, cb, cr = ycbcr(shim, c)
    r, g, b = (c & 255).astype(np.float64), ((c >> 8) & 255).astype(np.float64), (c >> 16).astype(np.float64)
    kr, kb = 0.2126, 0.0722
    yp = kr * r + (1 - kr - kb) * g + kb * b
    fy = 16 + 219 / 255 * yp
    fcb = 128 + 224 / 255 * (b - yp) / (2 * (1 - kb))
    fcr = 128 + 224 / 255 * (r - yp) / (2 * (1 - kr))
    for got, want in ((y, fy), (cb, fcb), (cr, fcr)):
        assert np.abs(got.astype(np.float64) - want).max() <= 1.0
    # black, white, greys
    assert (y[0], cb[0], cr[0]) == (16, 128, 128)
    white = (1 << 24) - 1
    assert (y[white], cb[white], cr[white]) == (235, 128, 128)
    grey = np.arange(256, dtype=np.uint32) * 0x010101
    assert (cb[grey] == 128).all() and (cr[grey] == 128).all()
    assert (np.diff(y[grey].astype(int)) >= 0).all()


def test_bt709_matches_the_restated_coefficients(shim):
    rng = np.random.default_rng(3)
    frame = rng.integers(0, 256, (64, 96, 4), dtype=np.uint8)
    frame[..., 3] = 255
    assert np.array_equal(export(shim, frame, NV12), nv12_np(frame, (0, 0, 0), True))


# ---- composite -------------------------------------------------------------------------------------------------------------
def test_composite_every_premultiplied_pixel_and_background(shim):
    a, c = np.meshgrid(np.arange(256), np.arange(256), indexing="ij")
    keep = c <= a
    a, c = a[keep], c[keep]                                       # every (c, a) with c <= a
    # one call per background value, all (c, a) at once, in every channel
    pa = pack(c, c, c, a)
    for v in range(256):
        out = np.empty_like(pa)
        shim.t_px(pa.ctypes.data, pa.size, RGBA, 1, 1, int(pack(v, v, v)), out.ctypes.data)
        want = np.minimum(255, c + (2 * v * (255 - a) + 255) // 510)
        assert np.array_equal(out & 255, want) and np.array_equal((out >> 8) & 255, want)
        assert np.array_equal((out >> 16) & 255, want) and ((out >> 24) == 255).all(), v


def test_composite_per_channel_background_and_bgra(shim):
    rng = np.random.default_rng(5)
    frame = premultiplied(rng, (4096,))
    px = np.ascontiguousarray(frame).view(np.uint32).reshape(-1)
    bg = (200, 30, 99)
    out = np.empty_like(px)
    shim.t_px(px.ctypes.data, px.size, RGBA, 1, 1, int(pack(*bg)), out.ctypes.data)
    assert np.array_equal(out.view(np.uint8).reshape(-1, 4), over_np(frame, bg, True))
    shim.t_px(px.ctypes.data, px.size, BGRA, 1, 1, int(pack(*bg)), out.ctypes.data)
    assert np.array_equal(out.view(np.uint8).reshape(-1, 4), over_np(frame, bg, True)[:, [2, 1, 0, 3]])
    shim.t_px(px.ctypes.data, px.size, BGRA, 0, 1, int(pack(*bg)), out.ctypes.data)
    assert np.array_equal(out.view(np.uint8).reshape(-1, 4), frame[:, [2, 1, 0, 3]])


def test_non_native_frames_pass_through(shim):
    rng = np.random.default_rng(6)
    frame = rng.integers(0, 256, (4096, 4), dtype=np.uint8)      # any alpha: the window ignores it
    px = np.ascontiguousarray(frame).view(np.uint32).reshape(-1)
    out = np.empty_like(px)
    shim.t_px(px.ctypes.data, px.size, RGBA, 1, 0, int(pack(255, 255, 255)), out.ctypes.data)
    want = frame.copy(); want[:, 3] = 255
    assert np.array_equal(out.view(np.uint8).reshape(-1, 4), want)
    shim.t_px(px.ctypes.data, px.size, RGBA, 0, 0, 0, out.ctypes.data)
    assert np.array_equal(out, px)


# ---- layout: flip, RGBA / BGRA rows, NV12 planes ------------------------------------------------------------------------------
@pytest.mark.parametrize("w,h", [(128, 64), (132, 30), (66, 10), (4, 2), (390, 8)])
@pytest.mark.parametrize("native", [True, False])
def test_nv12_planes_and_chroma_average(shim, w, h, native):
    rng = np.random.default_rng(w * 1000 + h)
    frame = premultiplied(rng, (h, w)) if native else rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    bg = (17, 240, 66)
    assert np.array_equal(export(shim, frame, NV12, bg=bg, native=native), nv12_np(frame, bg, native))


@pytest.mark.parametrize("w,h", [(128, 64), (130, 7), (5, 3), (257, 1), (4, 1)])
@pytest.mark.parametrize("fmt", [RGBA, BGRA])
@pytest.mark.parametrize("over", [False, True])
def test_rgba_rows_are_top_down(shim, w, h, fmt, over):
    rng = np.random.default_rng(w + 7 * h)
    frame = premultiplied(rng, (h, w))
    bg = (9, 99, 199)
    want = over_np(frame, bg, True).astype(np.uint8) if over else frame
    want = want[::-1]
    if fmt == BGRA:
        want = want[..., [2, 1, 0, 3]]
    for pitch in (None, (w * 4 + 15) // 16 * 16 + 48):
        got = export(shim, frame, fmt, over=over, bg=bg, pitch=pitch)
        assert np.array_equal(got.reshape(h, w, 4), want)


# ---- mark-aware reads ------------------------------------------------------------------------------------------------------
def marked_frame(rng, w, h, rows, garbage):
    """a frame and its marks: per (band, strip) a random interval [lo, hi) of rows that may be non-zero; the other rows of
    the band are 0 (garbage=False) or random (garbage=True: memory the marks say is zero is not read)"""
    strips = (w + 127) // 128
    frame = premultiplied(rng, (h, w))
    marks = np.zeros((h, strips), np.uint32)
    zero = np.ones((h, w), bool)
    for y0 in range(0, h, rows):
        y1 = min(h, y0 + rows)
        for s in range(strips):
            lo, hi = sorted(rng.integers(y0, y1 + 1, 2))
            if rng.random() < 0.2:
                lo = hi = 0
            marks[y0, s] = lo | (hi << 16) if lo < hi else 0
            zero[lo:hi, s * 128:(s + 1) * 128] = False
    clean = frame.copy()
    clean[zero] = 0
    return (frame if garbage else clean), clean, marks


@pytest.mark.parametrize("w,h,rows", [(256, 40, 8), (300, 33, 5), (128, 64, 64), (132, 17, 1), (64, 30, 540)])
@pytest.mark.parametrize("fmt", [RGBA, BGRA, NV12])
def test_mark_aware_walk_equals_a_full_read(shim, w, h, rows, fmt):
    if fmt == NV12 and (w | h) & 1:
        h -= 1
    rows = min(rows, h)
    rng = np.random.default_rng(w * h + rows)
    for garbage in (False, True):
        frame, clean, marks = marked_frame(rng, w, h, rows, garbage)
        full = export(shim, clean, fmt, over=True, bg=(40, 50, 60))
        aware = export(shim, frame, fmt, over=True, bg=(40, 50, 60), marks=marks, rows=rows)
        assert np.array_equal(aware, full), garbage


# ---- refusals and enqueued work through the fake runtime -----------------------------------------------------------------
# capi.cu, export.cpp and config.cpp built with g++ against tests/fakecuda's runtime (tests/export_fake.py)
@pytest.fixture(scope="module")
def fake():
    L = export_fake.lib()
    if L is None:
        pytest.skip("no CUDA toolkit headers")
    return L


def _export(L, h, streams, dsts, d, after=None, done=None):
    s = np.asarray(streams, np.int32)
    arr = (C.c_void_p * max(len(dsts), 1))(*dsts)
    n0 = L.export_fake_launches()
    L.fake_trace_begin()
    rc = L.glava_b200_export_frames(h, s.ctypes.data, len(streams), arr, C.byref(d), after, done)
    L.fake_trace_end()
    return rc, L.glava_b200_last_error().decode(), L.fake_trace().decode(), L.export_fake_launches() - n0


def test_refusals_name_the_function_and_enqueue_nothing(fake):
    L = fake
    L.fake_fail_at(-1)
    h, p = L.renderer(n=1024, w=64, h=32)
    buf, buf2 = L.device_buf(), L.device_buf()
    host = np.zeros(1 << 16, np.uint8)
    aligned_host = host.ctypes.data + (-host.ctypes.data) % 16
    rc, msg, trace, launched = _export(L, h, [0, 1, 1], [buf.value, buf2.value, buf2.value], desc_of(RGBA, 256))
    assert rc == 0 and launched == 1, msg
    cases = [
        ([0], [buf.value], desc_of(3, 256), "unknown format"),
        ([0], [buf.value], desc_of(RGBA, 256, flags=2), "unknown flags"),
        ([0], [buf.value], desc_of(RGBA, 240), "pitch"),                      # short: w * 4 = 256
        ([0], [buf.value], desc_of(RGBA, 264), "pitch"),                      # not a multiple of 16
        ([0], [buf.value], desc_of(NV12, 64, uv=8), "uv_offset"),
        ([0], [buf.value], desc_of(NV12, 64, uv=64 * 16), "uv_offset"),       # inside the Y plane
        ([0], [buf.value + 8], desc_of(RGBA, 256), "aligned"),
        ([0], [None], desc_of(RGBA, 256), "null"),
        ([0], [aligned_host], desc_of(RGBA, 256), "not device memory"),
        ([2], [buf.value], desc_of(RGBA, 256), "out of range"),
        ([-1], [buf.value], desc_of(RGBA, 256), "out of range"),
        ([], [], desc_of(RGBA, 256), "count"),
    ]
    for streams, dsts, d, what in cases:
        rc, msg, trace, launched = _export(L, h, streams, dsts, d)
        assert rc != 0, what
        assert "glava_b200_export_frames" in msg and what in msg, (msg, what)
        assert trace == "" and launched == 0, (what, trace)
    # odd NV12 geometry
    h2, _ = L.renderer(n=1024, w=64, h=31)
    rc, msg, trace, launched = _export(L, h2, [0], [buf.value], desc_of(NV12, 64))
    assert rc != 0 and "even" in msg and trace == "" and launched == 0
    n = C.c_size_t()
    assert L.glava_b200_export_bytes(h2, C.byref(desc_of(NV12, 64)), C.byref(n)) != 0
    assert L.glava_b200_export_bytes(h2, C.byref(desc_of(RGBA, 256)), C.byref(n)) == 0 and n.value == 256 * 31
    assert L.glava_b200_export_bytes(h, C.byref(desc_of(NV12, 64)), C.byref(n)) == 0 and n.value == 64 * 48
    assert L.glava_b200_export_bytes(h, C.byref(desc_of(NV12, 64, uv=4096)), C.byref(n)) == 0 and n.value == 4096 + 64 * 16
    L.glava_b200_destroy(h2)
    # an unbuilt renderer (a failed rebuild) refuses like an update
    q = p.__class__.from_buffer_copy(bytes(p))
    q.smooth_factor = 0.03 if p.smooth_factor != 0.03 else 0.02
    L.fake_fail_at(0)
    assert L.glava_b200_reconfigure(h, C.byref(q)) != 0
    L.fake_fail_at(-1)
    rc, msg, trace, launched = _export(L, h, [0], [buf.value], desc_of(RGBA, 256))
    assert rc != 0 and "glava_b200_export_frames" in msg and "no tables" in msg and trace == "" and launched == 0
    L.glava_b200_destroy(h)
    assert L.cudaFree(buf) == 0 and L.cudaFree(buf2) == 0


def test_export_orders_on_the_raster_stream_and_releases_its_buffers(fake):
    """the enqueued work — wait for `after`, the list copy, its event, the kernel, `done` — on the raster stream; the list
    buffers live until the renderer is destroyed"""
    L = fake
    L.fake_fail_at(-1)
    live0 = [L.fake_live(k) for k in range(4)]
    h, p = L.renderer(n=1024, w=64, h=32)
    buf = L.device_buf()
    a, d = C.c_void_p(), C.c_void_p()
    assert L.cudaEventCreate(C.byref(a)) == 0 and L.cudaEventCreate(C.byref(d)) == 0
    pcm = np.zeros((2, 1024), np.float32)
    assert L.glava_b200_update(h, pcm.ctypes.data, pcm.ctypes.data, 1024, 1) == 0
    for rep in range(6):                                              # past the four list buffers
        rc, msg, trace, launched = _export(L, h, [rep % 2], [buf.value], desc_of(RGBA, 256), a, d)
        assert rc == 0 and launched == 1, msg
        lines = [x.split() for x in trace.splitlines()]
        kinds = [x[0] for x in lines]
        assert kinds[-4:] == ["wait", "memcpy", "record", "record"], trace
        assert len({lines[-4][1], lines[-3][-1], lines[-2][-1], lines[-1][-1]}) == 1, trace   # all on one stream
    L.glava_b200_destroy(h)
    L.cudaEventDestroy(a); L.cudaEventDestroy(d); L.cudaFree(buf)
    assert [L.fake_live(k) for k in range(4)] == live0
