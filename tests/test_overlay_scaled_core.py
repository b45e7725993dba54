"""The overlay of a downscaled, cropped frame (glava_b200_overlay_scaled, DESIGN 4.21) on the host: a g++ walk of
overlay_scaled_kernel's items (export_scaled_kernel's runs of 32 output columns, each lane's pixel the area average of
scaled_px restated with its mark-aware footprint reads, faded by K, lanes past out_w zero, the quad at X = 0 mod 4 gathered
from four lanes into the fade walk's native bodies of tests/test_overlay_opacity_core.py with the rectangle out_w wide,
memcpy loads and stores) for every format and encoding, bit for bit against the opacity overlay's numpy restatement
(overlay_np / planes_np / overlay422_np after mul_norm8_np) applied to scaled_np's S, over sentinel-filled planes and
pitch padding, under native and any other opacity, every K of K_SET, crops touching each edge, odd and tiny outputs,
extreme ratios and marks live, stale and absent; its refusals, list sizes, launches and kernel choice through capi.cu,
export.cpp, overlay_planes.cpp and overlay_scaled.cpp built against the fake runtime of tests/fakecuda; and the Python
argument rules of size= / crop=."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from tests import export_fake, fakecuda
from tests.test_export_core import BGRA, CSRC, NV12, RGBA, marked_frame, premultiplied
from tests.test_export_scaled_core import scaled_np
from tests.test_overlay_opacity_core import K_SET, SHIM as FADE_SHIM
from tests.test_overlay_opacity_core import FORMATS, fits, plane_shapes, random_planes, restated
from tests.test_overlay_planes_core import PLANES_STUBS

I420, YUV444, P010, YUV420P10, YUV444P10, YUV422P, YUV422P10, UYVY, YUVA420P = 4, 5, 6, 7, 8, 10, 11, 12, 14
EXPORT_OVER, EXPORT_STRAIGHT, EXPORT_FULL_RANGE = 0x1, 0x4, 0x100

# ---- the kernel's walk on the host -----------------------------------------------------------------------------------------
# overlay_scaled_kernel restated: per item (output row or 4:2:0 row pair u, run of 32 columns) every lane's pixel is
# scaled_px (export_scaled_core's t_scaled restates the same footprint walk), faded, zero past out_w; lanes 0 mod 4 take the
# quad of lanes lane .. lane + 3 (__shfl_down_sync) into the fade walk's row / pair bodies, whose w is out_w.
WALK_SHIM = FADE_SHIM + r"""
static uint32_t scaled_px_host(const uint32_t* fb, int w, int h, const uint32_t* marks, int rows, const ExportFmt& f, int src_x,
                               int src_y, int src_w, int src_h, int out_w, int out_h, int X, int Y, const ExportRecip& rcp,
                               uint32_t zc) {
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
    return export_scaled_px(f, acc, wsum, (uint64_t) src_w * (uint64_t) src_h, rcp, zc);
}
template <int E>
static void scaled_walk(const uint32_t* fb, int w, int h, const uint32_t* marks, int rows, int fmt, int native, uint32_t k,
                        int src_x, int src_y, int src_w, int src_h, int out_w, int out_h, uint8_t* p0, uint8_t* p1, uint8_t* p2,
                        size_t P, size_t CP) {
    const Walk W = { fb, out_w, out_h, nullptr, 0, fmt, 1, k, p0, p1, p2, P, CP };   // the bodies' view: the rectangle
    const ExportFmt f = { fmt, native ? 0 : 1, native, 0u };
    const uint32_t zc = native ? 0u : export_over(0u, 0u, 0);
    const ExportRecip rcp = export_recip((uint64_t) src_w * (uint64_t) src_h);
    const bool pairs = fmt == GLAVA_B200_EXPORT_NV12 || fmt == GLAVA_B200_EXPORT_I420 || fmt == GLAVA_B200_EXPORT_P010 ||
                       fmt == GLAVA_B200_EXPORT_YUV420P10;
    const int units = pairs ? out_h / 2 : out_h, runs = (out_w + 31) / 32;
    for (int u = 0; u < units; ++u)
        for (int run = 0; run < runs; ++run) {
            uint32_t px[2][32];
            for (int r = 0; r < (pairs ? 2 : 1); ++r)
                for (int lane = 0; lane < 32; ++lane) {
                    const int X = run * 32 + lane;
                    if (X >= out_w) { px[r][lane] = 0u; continue; }
                    const uint32_t v = scaled_px_host(fb, w, h, marks, rows, f, src_x, src_y, src_w, src_h, out_w, out_h, X,
                                                      pairs ? 2 * u + r : u, rcp, zc);
                    px[r][lane] = native ? fade_px(v, k) : fade_opaque(v, k);
                }
            for (int lane = 0; lane < 32; lane += 4) {
                const int X = run * 32 + lane;
                if (X >= out_w) continue;
                uint32_t t[4], b[4];
                for (int i = 0; i < 4; ++i) { t[i] = px[0][lane + i]; b[i] = px[1][lane + i]; }
                if (pairs) W.pair<E>(u, X, t, b);
                else W.row<E>(u, X, t);
            }
        }
}
extern "C" void t_scaled_walk(const uint32_t* fb, int w, int h, const uint32_t* marks, int rows, int fmt, int e, int native,
                              uint32_t k, int src_x, int src_y, int src_w, int src_h, int out_w, int out_h, uint8_t* p0, uint8_t* p1,
                              uint8_t* p2, size_t P, size_t CP) {
    auto go = [&](auto E) {
        scaled_walk<decltype(E)::value>(fb, w, h, marks, rows, fmt, native, k, src_x, src_y, src_w, src_h, out_w, out_h, p0, p1, p2, P, CP);
    };
    if (e == 0) go(std::integral_constant<int, 0>()); else if (e == 1) go(std::integral_constant<int, 1>());
    else if (e == 2) go(std::integral_constant<int, 2>()); else go(std::integral_constant<int, 3>());
}
"""


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("overlay_scaled_core")
    src, so = d / "shim.cpp", d / "shim.so"
    src.write_text(WALK_SHIM)
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I", CSRC,
                    "-I", CSRC + "/../../include", "-include", "cstdint", "-include", "cstddef", "-include", "type_traits",
                    "-o", str(so), str(src)], check=True)
    L = C.CDLL(str(so))
    vp, i32, sz = C.c_void_p, C.c_int, C.c_size_t
    L.t_scaled_walk.argtypes = [vp, i32, i32, vp, i32, i32, i32, i32, C.c_uint32] + [i32] * 6 + [vp, vp, vp, sz, sz]
    return L


def scaled_walk(L, frame, planes, fmt, e, k, native, size, crop, marks=None, rows=0, off=16, pad=32):
    """the walk onto copies of `planes` (byte arrays [rows, row bytes]) placed `off` bytes into sentinel-filled rows with a
    sentinel row above and below; checks the sentinels (pitch padding included) and returns the rectangle's planes"""
    h, w = frame.shape[:2]
    x, y, cw, ch = crop or (0, 0, w, h)
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
    L.t_scaled_walk(fb.ctypes.data, w, h, None if m is None else m.ctypes.data, rows, fmt, e, int(native), int(k), x, y, cw, ch,
                    size[0], size[1], *ptrs, pitches[0], pitches[1] if len(pitches) > 1 else 0)
    out = []
    for b, b0, p in zip(bufs, before, planes):
        inside = np.zeros(b.shape, bool)
        inside[1:-1, off:off + p.shape[1]] = True
        assert np.array_equal(b[~inside], b0[~inside]), "written outside the rectangle"
        out.append(b[1:-1, off:off + p.shape[1]].copy())
    return out


def scaled_restated(frame, planes, fmt, e, k, native, size, crop):
    """the opacity overlay's restatement applied to S, export_scaled's RGBA image of the frame (read-back order)"""
    S = np.ascontiguousarray(scaled_np(frame, RGBA, not native, (0, 0, 0), native, size, crop)[::-1])
    return restated(S, planes, fmt, e, k, native)


def same_planes(got, want, what):
    for p, (a, b) in enumerate(zip(got, want)):
        if not np.array_equal(a, b):
            bad = np.argwhere(a != b)
            raise AssertionError(f"{what}: plane {p} differs at {len(bad)} bytes, first {bad[0]}: {a[tuple(bad[0])]} != {b[tuple(bad[0])]}")


# frame sizes and (size, crop): crops touching each edge, odd and non-multiple-of-4 widths, 1- and 2-pixel outputs, extreme
# ratios, a footprint spanning 128-pixel strips
WALK_CASES = [
    ((98, 62), [((48, 30), None), ((33, 21), (0, 0, 70, 50)), ((30, 14), (28, 12, 70, 50)), ((2, 2), (96, 60, 2, 2)),
                ((1, 1), None), ((98, 1), None), ((1, 62), (97, 0, 1, 62)), ((6, 4), (40, 30, 58, 32)), ((13, 7), (85, 0, 13, 62))]),
    ((300, 34), [((3, 34), None), ((299, 2), (1, 0, 299, 34)), ((70, 9), (0, 25, 300, 9)), ((150, 17), (150, 17, 150, 17))]),
]


@pytest.mark.parametrize("native", [True, False], ids=["native", "blended"])
@pytest.mark.parametrize("case", range(len(WALK_CASES)))
def test_walk_equals_the_restatement_without_marks(shim, case, native):
    (w, h), rects = WALK_CASES[case]
    rng = np.random.default_rng(w * 7 + h + native)
    frame = premultiplied(rng, (h, w)) if native else rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    frame[rng.random((h, w)) < 0.4] = 0
    frame[: h // 3] = 0
    for size, crop in rects:
        for fmt in FORMATS:
            if not fits(fmt, *size):
                continue
            for e in ((0,) if fmt in (RGBA, BGRA) else range(4)):
                planes = random_planes(rng, fmt, *size)
                for k in K_SET:
                    got = scaled_walk(shim, frame, planes, fmt, e, k, native, size, crop)
                    same_planes(got, scaled_restated(frame, planes, fmt, e, k, native, size, crop), (fmt, e, k, size, crop))
                    if k == 0:
                        same_planes(got, planes, (fmt, e, "K = 0 leaves the picture"))


@pytest.mark.parametrize("w,h,rows", [(256, 40, 8), (300, 34, 5), (132, 18, 1), (98, 36, 7), (66, 20, 9)])
def test_mark_aware_walk_equals_the_restatement(shim, w, h, rows):
    """live marks over garbage in the rows they call empty (those rows are not read), stale marks (each band's whole height
    over the clean frame), and no marks give the clean frame's result, under native opacity; under any other opacity live
    marks over the clean frame"""
    rows = min(rows, h)
    rng = np.random.default_rng(w * h + rows)
    rects = [((w // 3, h // 3), None), ((w // 2 - 1, h // 2 | 1), (w // 4, 1, w // 2 + 3, h - 1)), ((2, 2), (w - 2, h - 2, 2, 2))]
    frame, clean, marks = marked_frame(rng, w, h, rows, True)
    stale = marks.copy()
    for y0 in range(0, h, rows):
        stale[y0, :] = y0 | (min(h, y0 + rows) << 16)
    for size, crop in rects:
        for fmt in FORMATS:
            if not fits(fmt, *size):
                continue
            e = int(rng.integers(0, 4)) if fmt not in (RGBA, BGRA) else 0
            planes = random_planes(rng, fmt, *size)
            for k in (1, 128, 255):
                want = scaled_restated(clean, planes, fmt, e, k, True, size, crop)
                for what, fr, m in (("live", frame, marks), ("stale", clean, stale), ("absent", clean, None)):
                    got = scaled_walk(shim, fr, planes, fmt, e, k, True, size, crop, marks=m, rows=rows)
                    same_planes(got, want, (fmt, e, k, size, crop, what))
                got = scaled_walk(shim, clean, planes, fmt, e, k, False, size, crop, marks=marks, rows=rows)
                same_planes(got, scaled_restated(clean, planes, fmt, e, k, False, size, crop), (fmt, e, k, size, crop, "opaque"))


def test_zero_frame_leaves_the_picture_and_opaque_full_strength_is_the_export(shim):
    """identity 3 (a zero frame under native opacity) and identity 2 (any other opacity at K = 255: the rectangle holds the
    export's bytes, restated by the plain overlay's numpy restatement of the opaque blend) on the walk"""
    rng = np.random.default_rng(11)
    zero = np.zeros((62, 98, 4), np.uint8)
    frame = rng.integers(0, 256, (62, 98, 4), dtype=np.uint8)
    for fmt in FORMATS:
        size, crop = (30, 14), (28, 12, 70, 50)
        planes = random_planes(rng, fmt, *size)
        for k in K_SET:
            same_planes(scaled_walk(shim, zero, planes, fmt, 0, k, True, size, crop), planes, (fmt, k, "zero frame"))
        S = np.ascontiguousarray(scaled_np(frame, RGBA, True, (0, 0, 0), False, size, crop)[::-1])
        # the plain overlay under any other opacity writes the export's bytes: restated() at K = 255 of an opaque frame
        want = restated(S, [rng.integers(0, 256, p.shape, dtype=np.uint8) for p in planes], fmt, 0, 255, False)
        same_planes(scaled_walk(shim, frame, planes, fmt, 0, 255, False, size, crop), want, (fmt, "opaque K = 255"))


SCALED_STUBS = r"""
static long g_scaled_ov = 0;
static glb::OverlayScaledArgs g_so;
extern "C" long scaled_fake_launches(void) { return g_scaled_ov; }
extern "C" void scaled_fake_last(long* out) {
    out[0] = g_so.count; out[1] = g_so.format; out[2] = g_so.native; out[3] = g_so.out_w; out[4] = g_so.out_h; out[5] = g_so.src_x;
    out[6] = g_so.src_y; out[7] = g_so.src_w; out[8] = g_so.src_h; out[9] = (long) g_so.pitch; out[10] = (long) g_so.chroma_pitch;
    out[11] = g_so.enc; out[12] = g_so.w; out[13] = g_so.h;
}
namespace glb {
int launch_overlay_scaled(const OverlayScaledArgs& a, void*) {
    ++g_scaled_ov; g_so = a;
    return a.fb && a.list && a.count > 0 && a.out_w > 0 && a.out_h > 0 && (!a.marks || a.mark_rows > 0) ? 0
                                                                                                      : fail(GLAVA_B200_EINVAL, "scaled overlay launch: bad arguments");
}
}
"""


@pytest.fixture(scope="module")
def fake():
    inc = fakecuda.cuda_include()
    if inc is None:
        pytest.skip("no CUDA toolkit headers")
    from glava_b200.api import ExportScale, OverlayPlanesDesc, Params, Picture
    out = tempfile.mkdtemp(prefix="glava_scaled_ov_fake_")
    src, so = os.path.join(out, "scaled_fake.cpp"), os.path.join(out, "libscaled_fake.so")
    with open(src, "w") as f:
        f.write("#include <vector>\n" + export_fake.STUBS + PLANES_STUBS + SCALED_STUBS)
    subprocess.run(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I", inc,
                    "-I", fakecuda.CSRC, "-x", "c++", "-include", "cuda_runtime.h", "-o", so,
                    *[os.path.join(fakecuda.CSRC, f) for f in ("capi.cu", "export.cpp", "overlay_planes.cpp", "overlay_scaled.cpp",
                                                               "config.cpp")],
                    os.path.join(fakecuda.HERE, "fakecuda.cpp"), src, "-lpthread", "-Wl,-Bsymbolic"], check=True)
    L = C.CDLL(so)
    shutil.rmtree(out)
    vp, i32, P = C.c_void_p, C.c_int, C.POINTER(Params)
    sig = {
        "glava_b200_default_params": (i32, [P, C.c_char_p]), "glava_b200_new": (vp, [P, i32, i32]),
        "glava_b200_destroy": (None, [vp]), "glava_b200_last_error": (C.c_char_p, []), "glava_b200_set_abort_hook": (None, [vp]),
        "glava_b200_update": (i32, [vp, vp, vp, C.c_size_t, i32]),
        "glava_b200_overlay_scaled": (i32, [vp, vp, i32, C.POINTER(Picture), C.POINTER(OverlayPlanesDesc), C.POINTER(ExportScale),
                                            vp, vp, vp]),
        "cudaMalloc": (i32, [C.POINTER(vp), C.c_size_t]), "cudaEventCreate": (i32, [C.POINTER(vp)]),
        "cudaEventDestroy": (i32, [vp]), "fake_trace": (C.c_char_p, []),
        "export_fake_device": (None, [vp, C.c_size_t]), "export_fake_launches": (C.c_long, []),
        "planes_fake_launches": (C.c_long, []), "scaled_fake_launches": (C.c_long, []), "scaled_fake_last": (None, [vp]),
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


def _scaled(L, r, streams, pics, fmt, pitch, cpitch, scale, opacity=None, flags=0, after=None, done=None):
    """-> (rc, message, trace, [export overlay, planes overlay, scaled overlay] launches) of one call"""
    from glava_b200.api import ExportScale, OverlayPlanesDesc, Picture
    s = np.asarray(streams, np.int32)
    arr = (Picture * max(len(pics), 1))()
    for i, p in enumerate(pics):
        arr[i].plane = (C.c_void_p * 3)(*p)
    d = OverlayPlanesDesc()
    d.format, d.flags, d.pitch, d.chroma_pitch = fmt, flags, pitch, cpitch
    sc = None
    if scale is not None:
        sc = ExportScale()
        sc.src_x, sc.src_y, sc.src_w, sc.src_h, sc.out_w, sc.out_h = scale
    k = None if opacity is None else np.ascontiguousarray(opacity, np.uint8)
    n0 = [L.export_fake_launches(), L.planes_fake_launches(), L.scaled_fake_launches()]
    L.fake_trace_begin()
    rc = L.glava_b200_overlay_scaled(r, s.ctypes.data if len(streams) else None, len(streams), arr, C.byref(d),
                                     None if sc is None else C.byref(sc), None if k is None else k.ctypes.data, after, done)
    L.fake_trace_end()
    n1 = [L.export_fake_launches(), L.planes_fake_launches(), L.scaled_fake_launches()]
    return rc, L.glava_b200_last_error().decode(), L.fake_trace().decode(), [b - a for a, b in zip(n0, n1)]


HALF = (0, 0, 0, 0, 32, 16)                                   # the whole 64 x 32 frame to 32 x 16


def test_refusals_name_the_call_and_enqueue_nothing(fake):
    L = fake
    r = _renderer(L)
    b = _device(L)
    fb = L.glava_b200_framebuffer_device(r)
    L.export_fake_device(fb, 64 * 32 * 4)                     # the framebuffer is device memory
    i420 = (b, b + 4096, b + 8192)
    cases = [
        # the rectangle, as export_scaled's
        ([0], [(b, 0, 0)], RGBA, 128, 0, None, None, 0, "null scale"),
        ([0], [(b, 0, 0)], RGBA, 128, 0, (0, 0, 0, 0, 65, 16), None, 0, "no upscaling"),
        ([0], [(b, 0, 0)], RGBA, 128, 0, (0, 0, 64, 16, 32, 17), None, 0, "no upscaling"),
        ([0], [(b, 0, 0)], RGBA, 128, 0, (40, 0, 32, 16, 16, 8), None, 0, "leaves"),
        ([0], [(b, 0, 0)], RGBA, 128, 0, (0, 20, 8, 16, 8, 8), None, 0, "leaves"),
        ([0], [(b, 0, 0)], RGBA, 128, 0, (0, 0, 0, 16, 8, 8), None, 0, "empty"),
        ([0], [(b, 0, 0)], RGBA, 128, 0, (0, 0, 0, 0, 0, 8), None, 0, "at least 1x1"),
        # flags and formats
        ([0], [(b, 0, 0)], RGBA, 128, 0, HALF, None, EXPORT_OVER, "flags"),
        ([0], [(b, 0, 0)], RGBA, 128, 0, HALF, None, EXPORT_STRAIGHT, "STRAIGHT"),
        ([0], [(b, 0, 0)], RGBA, 128, 0, HALF, None, EXPORT_FULL_RANGE, "no matrix or range"),
        ([0], [i420], I420, 32, 16, HALF, None, EXPORT_OVER, "flags"),
        ([0], [i420], YUVA420P, 32, 16, HALF, None, 0, "alpha plane"),
        ([0], [(b, 0, 0)], 3, 128, 0, HALF, None, 0, "unknown format"),
        # RGBA / BGRA: one plane
        ([0], [(b, b + 4096, 0)], BGRA, 128, 0, HALF, None, 0, "one packed plane"),
        ([0], [(b, 0, b + 4096)], RGBA, 128, 0, HALF, None, 0, "one packed plane"),
        ([0], [(b, 0, 0)], RGBA, 128, 16, HALF, None, 0, "chroma_pitch"),
        # overlay_planes' refusals against the output size
        ([0], [(b, 0, 0)], RGBA, 112, 0, HALF, None, 0, "pitch"),
        ([0], [i420], I420, 32, 16, (0, 0, 0, 0, 31, 16), None, 0, "even width and height"),
        ([0], [i420], I420, 32, 16, (0, 0, 0, 0, 32, 15), None, 0, "even width and height"),
        ([0], [(b, b + 4096, b + 8192)], YUV422P, 32, 16, (0, 0, 0, 0, 31, 15), None, 0, "even width"),
        ([0], [i420], I420, 32, 8, HALF, None, 0, "chroma_pitch"),
        ([0], [(b + 8, 0, 0)], RGBA, 128, 0, HALF, None, 0, "aligned"),
        ([0], [(0, 0, 0)], RGBA, 128, 0, HALF, None, 0, "null"),
        ([0], [(b, b + 4096, 0)], I420, 32, 16, HALF, None, 0, "null"),
        ([0], [(fb, 0, 0)], RGBA, 128, 0, HALF, None, 0, "framebuffer"),
        ([0, 1], [(b, 0, 0), (b + 64, 0, 0)], RGBA, 256, 0, HALF, [0, 0], 0, "overlaps"),        # every entry, K = 0 too
        ([0, 1], [(b, 0, 0), (b + 128, 0, 0)], RGBA, 256, 0, HALF, [255, 0], 0, None),           # side by side: accepted
        ([0], [(b, b + 256, b + 512)], I420, 32, 16, HALF, None, 0, "overlaps"),                 # luma against chroma
        ([2], [(b, 0, 0)], RGBA, 128, 0, HALF, None, 0, "out of range"),
        ([], [], RGBA, 128, 0, HALF, None, 0, "count"),
    ]
    for streams, pics, fmt, P_, CP, sc, k, flags, what in cases:
        rc, msg, trace, n = _scaled(L, r, streams, pics, fmt, P_, CP, sc, k, flags)
        if what is None:
            assert rc == 0, msg
            continue
        assert rc != 0 and "glava_b200_overlay_scaled" in msg and what in msg, (what, msg)
        assert trace == "" and n == [0, 0, 0], (what, trace, n)
    L.glava_b200_destroy(r)


def test_lists_launches_and_kernel_choice(fake):
    """K = 0 entries are dropped and K rides in the entry's pad word (32-byte entries, 255 without opacity); one list copy and
    one scaled-overlay launch; a list of only K = 0 entries copies and launches nothing but keeps after / done on the raster
    stream; the whole frame at its own size runs the plain overlays' host path and kernels"""
    L = fake
    r = _renderer(L, w=64, h=32)
    b = _device(L)
    a, d = C.c_void_p(), C.c_void_p()
    assert L.cudaEventCreate(C.byref(a)) == 0 and L.cudaEventCreate(C.byref(d)) == 0
    last = np.zeros(14, np.int64)
    rgba = [(b + 128 * i, 0, 0) for i in range(3)]
    i420 = [(b + 32 * i, b + 8192 + 16 * i, b + 16384 + 16 * i) for i in range(3)]
    for fmt, pics, P_, CP in ((RGBA, rgba, 512, 0), (BGRA, rgba, 512, 0), (I420, i420, 128, 64)):
        for k, kept in ((None, 3), ([255, 255, 255], 3), ([255, 0, 128], 2), ([1, 2, 3], 3), ([0, 0, 0], 0)):
            rc, msg, trace, n = _scaled(L, r, [0, 1, 1], pics, fmt, P_, CP, (3, 5, 60, 27, 30, 16), k, after=a, done=d)
            assert rc == 0, msg
            kinds = [x.split()[0] for x in trace.splitlines()]
            if kept == 0:
                assert n == [0, 0, 0] and kinds[-2:] == ["wait", "record"] and "memcpy" not in kinds, trace
                continue
            assert n == [0, 0, 1] and kinds[-4:] == ["wait", "memcpy", "record", "record"], trace
            assert f"H2D {kept * 32} " in trace, (trace, kept)
            L.scaled_fake_last(last.ctypes.data)
            assert list(last[:11]) == [kept, fmt, 1, 30, 16, 3, 5, 60, 27, P_, CP] and list(last[12:]) == [64, 32], list(last)
    # the whole frame at its own size (all-zero or explicit rectangle): the plain overlays' kernels, not the scaled one
    for sc in ((0, 0, 0, 0, 64, 32), (0, 0, 64, 32, 64, 32)):
        rc, msg, trace, n = _scaled(L, r, [0, 1], [(b, 0, 0), (b + 256, 0, 0)], RGBA, 512, 0, sc, [255, 128])
        assert rc == 0 and n == [1, 0, 0], (msg, n)
        rc, msg, trace, n = _scaled(L, r, [0, 1], [(b, b + 8192, b + 12288), (b + 64, b + 8192 + 32, b + 12288 + 32)], I420, 256,
                                    128, sc, None)
        assert rc == 0 and n == [0, 1, 0], (msg, n)
    # a crop at the frame's own size is not the whole frame
    rc, msg, trace, n = _scaled(L, r, [0], [(b, 0, 0)], RGBA, 512, 0, (0, 0, 64, 32, 63, 32))
    assert rc == 0 and n == [0, 0, 1], (msg, n)
    L.cudaEventDestroy(a); L.cudaEventDestroy(d)
    L.glava_b200_destroy(r)


def test_python_size_and_crop_arguments():
    from glava_b200.api import _FrameExport
    sc = _FrameExport._overlay_scale
    assert sc(None, None) == (None, None)
    size, s = sc((32, 18), None)
    assert size == (32, 18) and (s.src_x, s.src_y, s.src_w, s.src_h, s.out_w, s.out_h) == (0, 0, 0, 0, 32, 18)
    size, s = sc(None, (4, 6, 40, 20))
    assert size == (40, 20) and (s.src_x, s.src_y, s.src_w, s.src_h, s.out_w, s.out_h) == (4, 6, 40, 20, 40, 20)
    size, s = sc((10, 5), (4, 6, 40, 20))
    assert size == (10, 5) and (s.src_w, s.out_w, s.out_h) == (40, 10, 5)
    for bad_size, bad_crop in (((0, 5), None), ((5,), None), ((1, 2, 3), None), (None, (1, 2, 3)), ((4, -1), (0, 0, 8, 8))):
        with pytest.raises(ValueError):
            sc(bad_size, bad_crop)


def test_python_frames_pictures():
    """overlay_frames' destinations as the scaled call's pictures: RGBA one plane, NV12 Y and CbCr at one pitch"""
    from glava_b200.api import Export, _FrameExport
    d = Export()
    d.format, d.flags, d.pitch = NV12, 0x100, 4096
    pd, arr = _FrameExport._frames_pictures(d, [1024, 2048], [8192, 16384], 2)
    assert (pd.format, pd.flags, pd.pitch, pd.chroma_pitch) == (NV12, 0x100, 4096, 4096)
    assert [list(arr[i].plane) for i in range(2)] == [[1024, 8192, None], [2048, 16384, None]]
    d.format, d.flags = RGBA, 0
    pd, arr = _FrameExport._frames_pictures(d, [1024], None, 1)
    assert (pd.format, pd.chroma_pitch) == (RGBA, 0) and list(arr[0].plane) == [1024, None, None]
