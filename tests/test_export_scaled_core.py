"""Scaled and cropped export (DESIGN 4.11) on the host: the area average of export_core.h through a g++ shim that walks one
framebuffer slot the way export_scaled_kernel does (runs of 32 output columns, strip by strip, band by band of the
dirty-row marks, aligned quads), against an independent numpy restatement built from interval overlaps, bit for bit; the exactness of the
reciprocal division over its whole range; and the refusals and enqueued work of glava_b200_export_scaled through capi.cu
and export.cpp built against the fake runtime of tests/fakecuda (tests/export_fake.py)."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from tests import export_fake
from tests.export_fake import desc_of
from tests.test_export_core import SHIM as PLAIN_SHIM
from tests.test_export_core import BGRA, CSRC, NV12, RGBA, export, marked_frame, nv12_np, over_np, pack, premultiplied

# the plain export's shim (t_export) comes along, for the full-size comparison
SHIM = PLAIN_SHIM + r"""
extern "C" void t_span(int X, int n, int m, uint32_t* out) {
    const ExportSpan s = export_span(X, n, m);
    out[0] = s.first; out[1] = s.last; out[2] = s.w_first; out[3] = s.w_last;
}
extern "C" void t_recip(uint64_t d, uint64_t* mul, int* shift) { const ExportRecip r = export_recip(d); *mul = r.mul; *shift = r.shift; }
extern "C" uint64_t t_div(uint64_t x, uint64_t mul, int shift) { return export_div(x, { mul, shift }); }
// every d in [lo, hi]: export_recip's multiplier fits and x e < 2^(64 + shift) for the largest dividend x = 255 d + d / 2,
// which makes umulhi(x, mul) >> shift = floor(x / d) for every smaller x (export_core.h); returns the first d that fails, or 0
extern "C" uint64_t t_recip_proof(uint64_t lo, uint64_t hi) {
    for (uint64_t d = lo; d <= hi; ++d) {
        const ExportRecip r = export_recip(d);
        if (d == 1) { if (r.mul) return d; continue; }
        const unsigned __int128 k = (unsigned __int128) 1 << (64 + r.shift);
        const unsigned __int128 m = r.mul, e = m * d - k;       // mul * d >= 2^(64 + shift) by construction
        if (m * d < k || e >= d || (unsigned __int128) (255 * d + d / 2) * e >= k) return d;
    }
    return 0;
}
// one slot [h][w] of RGBA8 words -> dst (Y or RGBA rows) and dst_uv, as export_scaled_kernel walks it
extern "C" void t_scaled(const uint32_t* fb, int w, int h, const uint32_t* marks, int rows, int format, int over, int native,
                         uint32_t bg, int src_x, int src_y, int src_w, int src_h, int out_w, int out_h, uint8_t* dst,
                         uint8_t* dst_uv, size_t pitch) {
    const bool nv12 = format == GLAVA_B200_EXPORT_NV12;
    const ExportFmt f = { format, nv12 || over, native, bg };
    const uint32_t zc = f.over ? export_over(0u, f.bg, f.native) : 0u;
    const uint64_t d = (uint64_t) src_w * src_h;
    const ExportRecip rcp = export_recip(d);
    const int units = nv12 ? out_h / 2 : out_h, runs = (out_w + 31) / 32;
    for (int u = 0; u < units; ++u)
        for (int run = 0; run < runs; ++run) {
            uint32_t px[2][32];
            for (int r = 0; r < (nv12 ? 2 : 1); ++r)
                for (int lane = 0; lane < 32; ++lane) {
                    const int X = run * 32 + lane, Y = nv12 ? 2 * u + r : u;
                    if (X >= out_w) { px[r][lane] = 0; continue; }
                    const ExportSpan sx = export_span(X, src_w, out_w), sy = export_span(Y, src_h, out_h);
                    const int x0 = src_x + sx.first, x1 = src_x + sx.last;
                    const int yb = export_fb_row(h, src_y, sy.last), ye = export_fb_row(h, src_y, sy.first) + 1;
                    const int brows = marks ? rows : 0;
                    uint64_t acc[4] = { 0, 0, 0, 0 }, wsum = 0;
                    for (int strip = x0 >> 7, last = brows ? x1 >> 7 : strip; strip <= last; ++strip) {
                        const int qa = std::max(x0, strip << 7) & ~3, qb = brows ? std::min(x1, (strip << 7) + 127) : x1;
                        for (int y = yb; y < ye;) {
                            int ra, rb;
                            const uint32_t mark = brows ? marks[export_mark_index(0, w, h, brows, y, strip)] : 0u;
                            y = export_band_rows(y, ye, brows, mark, &ra, &rb);
                            for (int yy = ra; yy < rb; ++yy) {
                                uint32_t row[4] = { 0, 0, 0, 0 }, row_w = 0;
                                for (int qx = qa; qx <= qb; qx += 4)
                                    for (int k = 0; k < 4; ++k) {
                                        const int x = qx + k;
                                        if (x >= x0 && x <= x1) export_acc(f, fb[(size_t) yy * w + x], export_span_weight(sx, x - src_x, out_w), row, &row_w);
                                    }
                                export_fold(row, row_w, export_span_weight(sy, h - 1 - src_y - yy, out_h), acc, &wsum);
                            }
                        }
                    }
                    px[r][lane] = export_scaled_px(f, acc, wsum, d, rcp, zc);
                }
            for (int lane = 0; lane < 32 && run * 32 + lane < out_w; ++lane) {
                const int X = run * 32 + lane;
                if (nv12) {
                    dst[(size_t) (2 * u) * pitch + X] = (uint8_t) export_y(px[0][lane]);
                    dst[(size_t) (2 * u + 1) * pitch + X] = (uint8_t) export_y(px[1][lane]);
                    if (!(lane & 1)) {
                        const uint32_t uv = export_cbcr(export_avg4(px[0][lane], px[0][lane + 1], px[1][lane], px[1][lane + 1]));
                        dst_uv[(size_t) u * pitch + X] = (uint8_t) uv; dst_uv[(size_t) u * pitch + X + 1] = (uint8_t) (uv >> 8);
                    }
                } else {
                    const uint32_t v = format == GLAVA_B200_EXPORT_BGRA ? export_swap_rb(px[0][lane]) : px[0][lane];
                    memcpy(dst + (size_t) u * pitch + (size_t) X * 4, &v, 4);
                }
            }
        }
}
"""


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("export_scaled_core")
    src, so = d / "shim.cpp", d / "shim.so"
    src.write_text(SHIM)
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I", CSRC,
                    "-include", "cstring", "-include", "algorithm", "-o", str(so), str(src)], check=True)
    L = C.CDLL(str(so))
    vp, sz, i32, u32, u64 = C.c_void_p, C.c_size_t, C.c_int, C.c_uint32, C.c_uint64
    L.t_span.argtypes = [i32, i32, i32, vp]
    L.t_recip.argtypes = [u64, C.POINTER(u64), C.POINTER(i32)]
    L.t_div.argtypes, L.t_div.restype = [u64, u64, i32], u64
    L.t_recip_proof.argtypes, L.t_recip_proof.restype = [u64, u64], u64
    L.t_scaled.argtypes = [vp, i32, i32, vp, i32, i32, i32, i32, u32] + [i32] * 6 + [vp, vp, sz]
    L.t_export.argtypes = [vp, i32, i32, vp, i32, i32, i32, i32, u32, vp, sz, sz]
    return L


# ---- numpy restatement ---------------------------------------------------------------------------------------------------
def weights_np(n, m):
    """[m][n] integer overlaps of output interval [X n, (X + 1) n) and source interval [i m, (i + 1) m)"""
    X, i = np.arange(m)[:, None], np.arange(n)[None, :]
    return np.maximum(0, np.minimum((X + 1) * n, (i + 1) * m) - np.maximum(X * n, i * m)).astype(np.int64)


def area_np(img, size):
    """[h][w][c] integers -> [out_h][out_w][c]: (Wy img Wx^T + D / 2) // D.  Every partial sum is an integer below 2^53,
    so the float64 products are exact."""
    h, w = img.shape[:2]
    ow, oh = size
    wy, wx = weights_np(h, oh).astype(np.float64), weights_np(w, ow).astype(np.float64)
    c = img.shape[2]
    s = (wy @ img.reshape(h, w * c).astype(np.float64)).reshape(oh, w, c)
    s = np.matmul(wx, s).astype(np.int64)
    d = w * h
    return (s + d // 2) // d


def scaled_np(frame, fmt, over, bg, native, size, crop=None):
    """the expected scaled export of a read-back frame ([h][w][4], row 0 = bottom): RGBA / BGRA [oh][ow][4], NV12 bytes
    [oh * 3 / 2][ow]"""
    top = frame[::-1]
    x, y, cw, ch = crop or (0, 0, frame.shape[1], frame.shape[0])
    img = top[y:y + ch, x:x + cw].astype(np.int64)
    comp = over or fmt == NV12
    if comp:
        img = over_np(img, bg, native)
    avg = area_np(img, size)
    if comp:
        avg[..., 3] = 255
    avg = avg.astype(np.uint8)
    if fmt == NV12:
        return nv12_np(avg[::-1], bg, native)                      # composited, alpha 255: the composite is the identity
    return avg[..., [2, 1, 0, 3]] if fmt == BGRA else avg


def scaled_shim(L, frame, fmt, size, crop=None, over=False, native=True, bg=(0, 0, 0), marks=None, rows=0, pad=48):
    h, w = frame.shape[:2]
    ow, oh = size
    x, y, cw, ch = crop or (0, 0, w, h)
    row = ow if fmt == NV12 else ow * 4
    pitch = (row + 15) // 16 * 16 + pad
    nrows = oh * 3 // 2 if fmt == NV12 else oh
    dst = np.full((nrows, pitch), 0xA5, np.uint8)
    fb = np.ascontiguousarray(frame).view(np.uint32).reshape(h, w)
    m = None if marks is None else np.ascontiguousarray(marks, np.uint32)
    L.t_scaled(fb.ctypes.data, w, h, None if m is None else m.ctypes.data, rows, fmt, int(over), int(native), int(pack(*bg[:3])),
               x, y, cw, ch, ow, oh, dst.ctypes.data, dst.ctypes.data + pitch * oh, pitch)
    assert (dst[:, row:] == 0xA5).all(), "written past the row"
    return dst[:, :row]


def test_weights_are_interval_overlaps_and_sum_to_the_source(shim):
    out = np.zeros(4, np.uint32)
    for n, m in ((1920, 7), (97, 13), (1080, 1), (1920, 480), (2048, 2048), (16384, 3), (5, 5), (7, 6), (2048, 2047)):
        wx = weights_np(n, m)
        assert (wx.sum(axis=1) == n).all() and (wx.sum(axis=0) == m).all()
        for X in sorted({0, min(1, m - 1), m // 2, m - 1}):
            shim.t_span(X, n, m, out.ctypes.data)
            first, last, wf, wl = (int(v) for v in out)
            nz = np.nonzero(wx[X])[0]
            assert (first, last) == (nz[0], nz[-1]), (n, m, X)
            got = [wf if i == first else wl if i == last else m for i in range(first, last + 1)]
            assert got == list(wx[X, first:last + 1]), (n, m, X)


def test_reciprocal_division_is_exact_over_every_divisor(shim):
    """D = src_w * src_h <= 16384^2: for every D the multiplier fits 64 bits and the error bound holds for the largest
    dividend 255 D + D / 2, which proves umulhi(x, mul) >> shift = floor(x / D) for all smaller x (export_core.h)"""
    assert shim.t_recip_proof(1, 1 << 24) == 0
    for s in range(24, 28):                                      # the upper range: every D next to a power of two, in blocks
        lo = 1 << s
        assert shim.t_recip_proof(lo - 4096, lo + 4096) == 0
    assert shim.t_recip_proof((1 << 28) - (1 << 20), 1 << 28) == 0
    # the bound holds generally: e < D <= 2^(shift + 1) and x < 2^63 give x e < 2^(64 + shift)
    mul, shift = C.c_uint64(), C.c_int()
    rng = np.random.default_rng(0)
    for d in [2, 3, 5, 7, 1 << 14, (1 << 28) - 1, 16383 * 16384, 1920 * 1080] + list(rng.integers(2, 1 << 28, 200)):
        shim.t_recip(int(d), C.byref(mul), C.byref(shift))
        for q in (0, 1, 127, 254, 255):
            for x in (q * int(d), q * int(d) + int(d) // 2, q * int(d) + int(d) - 1):
                assert shim.t_div(x, mul.value, shift.value) == x // int(d), (d, x)


CASES = [  # (w, h, crop, size)
    (128, 64, None, (128, 64)),
    (128, 64, None, (32, 16)),
    (97, 63, None, (13, 7)),
    (97, 63, (5, 3, 90, 58), (30, 29)),
    (300, 33, (100, 2, 60, 30), (12, 10)),                       # straddles strips 0 / 1 / 2
    (390, 20, (120, 0, 140, 20), (7, 1)),
    (1920, 8, None, (7, 2)),
    (1080, 6, None, (1, 2)),
    (130, 10, (1, 1, 129, 9), (64, 4)),
]


@pytest.mark.parametrize("w,h,crop,size", CASES)
@pytest.mark.parametrize("native", [True, False])
def test_shim_walk_equals_the_restatement(shim, w, h, crop, size, native):
    rng = np.random.default_rng(w * 31 + h + size[0])
    frame = premultiplied(rng, (h, w)) if native else rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    frame[rng.random((h, w)) < 0.3] = 0                           # zero pixels take the constant path
    bg = (17, 240, 66)
    for fmt in (RGBA, BGRA, NV12):
        if fmt == NV12 and (size[0] | size[1]) & 1:
            continue
        for over in (False, True):
            got = scaled_shim(shim, frame, fmt, size, crop, over=over, native=native, bg=bg)
            want = scaled_np(frame, fmt, over, bg, native, size, crop)
            assert np.array_equal(got.reshape(want.shape), want), (fmt, over)


def test_full_size_equals_the_plain_export(shim):
    rng = np.random.default_rng(8)
    for w, h in ((132, 30), (66, 10), (128, 64), (97, 7)):
        frame = premultiplied(rng, (h, w))
        frame[rng.random((h, w)) < 0.3] = 0
        for fmt in (RGBA, BGRA, NV12):
            if fmt == NV12 and (w | h) & 1:
                continue
            for over in (False, True):
                got = scaled_shim(shim, frame, fmt, (w, h), over=over, bg=(9, 99, 199), pad=0)
                want = export(shim, frame, fmt, over=over, bg=(9, 99, 199))
                assert np.array_equal(got, want), (w, h, fmt, over)


def test_a_constant_frame_stays_constant(shim):
    for px in ((10, 20, 30, 40), (255, 255, 255, 255), (0, 0, 0, 0), (1, 0, 0, 1)):
        frame = np.empty((45, 101, 4), np.uint8)
        frame[:] = px
        for size in ((7, 3), (33, 45), (1, 1), (100, 44)):
            got = scaled_shim(shim, frame, RGBA, size)
            assert (got.reshape(size[1], size[0], 4) == px).all(), (px, size)


@pytest.mark.parametrize("w,h,rows,crop,size", [(256, 40, 8, None, (64, 10)), (300, 33, 5, (60, 3, 200, 30), (14, 6)),
                                                (132, 17, 1, None, (5, 3)), (128, 64, 64, (0, 10, 128, 40), (32, 20)),
                                                (390, 30, 540, (1, 0, 389, 30), (100, 30))])
@pytest.mark.parametrize("fmt", [RGBA, BGRA, NV12])
def test_marks_are_honoured_and_skipped_rows_never_read(shim, w, h, rows, crop, size, fmt):
    if fmt == NV12 and (size[0] | size[1]) & 1:
        size = (size[0] + 1, size[1] + 1)
    rows = min(rows, h)
    rng = np.random.default_rng(w * h + rows + fmt)
    for garbage in (False, True):
        frame, clean, marks = marked_frame(rng, w, h, rows, garbage)
        for over in (False, True):
            full = scaled_shim(shim, clean, fmt, size, crop, over=over, bg=(40, 50, 60))
            aware = scaled_shim(shim, frame, fmt, size, crop, over=over, bg=(40, 50, 60), marks=marks, rows=rows)
            assert np.array_equal(aware, full), (garbage, over)
            want = scaled_np(clean, fmt, over, (40, 50, 60), True, size, crop)
            assert np.array_equal(full.reshape(want.shape), want), over


# ---- refusals and enqueued work through the fake runtime -----------------------------------------------------------------
@pytest.fixture(scope="module")
def fake():
    L = export_fake.lib()
    if L is None:
        pytest.skip("no CUDA toolkit headers")
    return L


def scale_of(out, crop=(0, 0, 0, 0)):
    from glava_b200.api import ExportScale
    s = ExportScale()
    s.src_x, s.src_y, s.src_w, s.src_h = crop
    s.out_w, s.out_h = out
    return s


def _scaled(L, h, streams, dsts, d, sc, uvs=None, after=None, done=None):
    s = np.asarray(streams, np.int32)
    arr = (C.c_void_p * max(len(dsts), 1))(*dsts)
    uv = None if uvs is None else (C.c_void_p * max(len(uvs), 1))(*uvs)
    n0 = L.export_fake_launches()
    L.fake_trace_begin()
    rc = L.glava_b200_export_scaled(h, s.ctypes.data, len(streams), arr, uv, C.byref(d), sc if sc is None else C.byref(sc),
                                    after, done)
    L.fake_trace_end()
    return rc, L.glava_b200_last_error().decode(), L.fake_trace().decode(), L.export_fake_launches() - n0


def test_refusals_name_the_function_and_enqueue_nothing(fake):
    L = fake
    L.fake_fail_at(-1)
    h, p = L.renderer(n=1024, w=64, h=32)
    buf, buf2 = L.device_buf(), L.device_buf()
    host = np.zeros(1 << 16, np.uint8)
    aligned_host = host.ctypes.data + (-host.ctypes.data) % 16
    ok = scale_of((16, 8), (4, 2, 40, 20))
    rc, msg, trace, launched = _scaled(L, h, [0, 1, 1], [buf.value, buf2.value, buf2.value], desc_of(RGBA, 64), ok)
    assert rc == 0 and launched == 1, msg
    last = (C.c_int * 8)()
    L.export_fake_last(last)
    assert list(last) == [4, 2, 40, 20, 16, 8, 3, 0]
    rc, msg, trace, launched = _scaled(L, h, [0], [buf.value], desc_of(NV12, 16), ok, uvs=[buf2.value])
    assert rc == 0 and launched == 1, msg
    rc, msg, trace, launched = _scaled(L, h, [1], [buf.value], desc_of(RGBA, 256), scale_of((64, 32)))
    assert rc == 0 and launched == 1, msg                                           # the whole frame at its size
    L.export_fake_last(last)
    assert list(last)[:6] == [0, 0, 64, 32, 64, 32]
    cases = [
        ([0], [buf.value], desc_of(RGBA, 64), None, None, "null scale"),
        ([0], [buf.value], desc_of(3, 64), ok, None, "unknown format"),
        ([0], [buf.value], desc_of(RGBA, 64, flags=2), ok, None, "unknown flags"),
        ([0], [buf.value], desc_of(RGBA, 48), ok, None, "pitch"),                    # short: out_w * 4 = 64
        ([0], [buf.value], desc_of(RGBA, 72), ok, None, "pitch"),                    # not a multiple of 16
        ([0], [buf.value], desc_of(NV12, 16, uv=8), ok, None, "uv_offset"),
        ([0], [buf.value], desc_of(NV12, 16, uv=16 * 4), ok, None, "uv_offset"),     # inside the Y plane
        ([0], [buf.value], desc_of(RGBA, 64), scale_of((16, 8), (30, 0, 40, 20)), None, "leaves"),
        ([0], [buf.value], desc_of(RGBA, 64), scale_of((16, 8), (0, 20, 40, 20)), None, "leaves"),
        ([0], [buf.value], desc_of(RGBA, 64), scale_of((16, 8), (-1, 0, 40, 20)), None, "leaves"),
        ([0], [buf.value], desc_of(RGBA, 64), scale_of((16, 8), (0, 0, 40, 0)), None, "empty"),
        ([0], [buf.value], desc_of(RGBA, 64), scale_of((16, 8), (3, 0, 0, 0)), None, "empty"),
        ([0], [buf.value], desc_of(RGBA, 256), scale_of((41, 8), (0, 0, 40, 20)), None, "upscaling"),
        ([0], [buf.value], desc_of(RGBA, 256), scale_of((16, 21), (0, 0, 40, 20)), None, "upscaling"),
        ([0], [buf.value], desc_of(RGBA, 256), scale_of((0, 8)), None, "upscaling"),
        ([0], [buf.value], desc_of(NV12, 16), scale_of((15, 8)), None, "even"),
        ([0], [buf.value], desc_of(NV12, 16), scale_of((16, 7)), None, "even"),
        ([0], [buf.value], desc_of(RGBA, 64), ok, [buf2.value], "NV12 only"),
        ([0], [buf.value], desc_of(NV12, 16), ok, [buf2.value + 8], "dst_uv[0]"),
        ([0], [buf.value], desc_of(NV12, 16), ok, [None], "dst_uv[0]"),
        ([0], [buf.value], desc_of(NV12, 16), ok, [aligned_host], "dst_uv[0] = "),
        ([0], [buf.value + 8], desc_of(RGBA, 64), ok, None, "aligned"),
        ([0], [None], desc_of(RGBA, 64), ok, None, "null"),
        ([0], [aligned_host], desc_of(RGBA, 64), ok, None, "not device memory"),
        ([2], [buf.value], desc_of(RGBA, 64), ok, None, "out of range"),
        ([], [], desc_of(RGBA, 64), ok, None, "count"),
    ]
    for streams, dsts, d, sc, uvs, what in cases:
        rc, msg, trace, launched = _scaled(L, h, streams, dsts, d, sc, uvs)
        assert rc != 0, what
        assert "glava_b200_export_scaled" in msg and what in msg, (msg, what)
        assert trace == "" and launched == 0, (what, trace)
    n = C.c_size_t()
    assert L.glava_b200_export_scaled_bytes(h, C.byref(desc_of(NV12, 16)), C.byref(scale_of((15, 8))), C.byref(n)) != 0
    assert L.glava_b200_export_scaled_bytes(h, C.byref(desc_of(NV12, 16)), None, C.byref(n)) != 0
    assert L.glava_b200_export_scaled_bytes(h, C.byref(desc_of(RGBA, 64)), C.byref(ok), C.byref(n)) == 0 and n.value == 64 * 8
    assert L.glava_b200_export_scaled_bytes(h, C.byref(desc_of(NV12, 16)), C.byref(ok), C.byref(n)) == 0 and n.value == 16 * 12
    assert L.glava_b200_export_scaled_bytes(h, C.byref(desc_of(NV12, 16, uv=256)), C.byref(ok), C.byref(n)) == 0 and n.value == 256 + 16 * 4
    # an unbuilt renderer (a failed rebuild) refuses
    q = p.__class__.from_buffer_copy(bytes(p))
    q.smooth_factor = 0.03 if p.smooth_factor != 0.03 else 0.02
    L.fake_fail_at(0)
    assert L.glava_b200_reconfigure(h, C.byref(q)) != 0
    L.fake_fail_at(-1)
    rc, msg, trace, launched = _scaled(L, h, [0], [buf.value], desc_of(RGBA, 64), ok)
    assert rc != 0 and "glava_b200_export_scaled" in msg and "no tables" in msg and trace == "" and launched == 0
    L.glava_b200_destroy(h)
    assert L.cudaFree(buf) == 0 and L.cudaFree(buf2) == 0


def test_one_copy_one_launch_on_the_raster_stream_and_shared_list_buffers(fake):
    """wait for `after`, the list copy, its event, the kernel, `done`, all on the raster stream; scaled and plain exports
    share the four list buffers, which live until the renderer is destroyed"""
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
        rc, msg, trace, launched = _scaled(L, h, [rep % 2], [buf.value], desc_of(NV12, 16), scale_of((16, 8)), None, a, d)
        assert rc == 0 and launched == 1, msg
        lines = [x.split() for x in trace.splitlines()]
        kinds = [x[0] for x in lines]
        assert kinds[-4:] == ["wait", "memcpy", "record", "record"], trace
        assert len({lines[-4][1], lines[-3][-1], lines[-2][-1], lines[-1][-1]}) == 1, trace
        rc, msg, trace, launched = _scaled(L, h, [0, 1], [buf.value] * 2, desc_of(RGBA, 64), scale_of((16, 8)))
        assert rc == 0 and launched == 1 and [x.split()[0] for x in trace.splitlines()][-2:] == ["memcpy", "record"], trace
        dst = (C.c_void_p * 1)(buf.value)
        s = np.zeros(1, np.int32)
        assert L.glava_b200_export_frames(h, s.ctypes.data, 1, dst, C.byref(desc_of(RGBA, 256)), None, None) == 0
    live = [L.fake_live(k) for k in range(4)]
    long_list = 300                                                   # grows the shared buffers past 64 plain entries
    rc, msg, trace, launched = _scaled(L, h, [0] * long_list, [buf.value] * long_list, desc_of(RGBA, 64), scale_of((16, 8)))
    assert rc == 0 and launched == 1, msg
    assert [L.fake_live(k) for k in range(4)] == live                 # regrown, not added to
    L.glava_b200_destroy(h)
    L.cudaEventDestroy(a); L.cudaEventDestroy(d); L.cudaFree(buf)
    assert [L.fake_live(k) for k in range(4)] == live0
