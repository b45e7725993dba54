"""Frame export at the geometry limits on the host: the walks of tests/test_export_core.py (t_export),
tests/test_export_scaled_core.py (t_scaled), tests/test_export_formats_core.py (t_export_yuv) and tests/test_overlay_core.py
(t_overlay) at 4-pixel-wide frames, frames of 1, 2 or 3 rows, widths around the 128-pixel strip, and 16384 x 8 / 8 x 16384,
with random dirty-row marks over garbage rows, against the numpy restatements bit for bit and against a plain float64
statement of each operation within bounds derived from the per-pixel float64 proofs of those files.

The float64 reference lives here and tests/test_z_gpu_export_limits.py applies it to the device's output: the composite over
the background, BT.709 limited range at 8 or 10 bits, the exact area average (integer prefix sums, so no weight matrix and
no rounding before the final division) and the 2x2 chroma mean.

These walks compile export_core.h for the host, so export_div takes its unsigned __int128 branch here; the device branch
(__umul64hi) is exercised by tests/test_z_gpu_export_limits.py, whose 16384 x 16384 cases need the upper half of the
64-bit numerator."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from tests.test_export_core import BGRA, CSRC, NV12, RGBA, export, marked_frame, nv12_np, over_np, premultiplied
from tests.test_export_formats_core import I420, P010, YUV444, export_yuv, frame_np, same, yuv_np
from tests.test_export_scaled_core import SHIM as SCALED_SHIM
from tests.test_export_scaled_core import area_np, scaled_np, scaled_shim
from tests.test_export_formats_core import SHIM as FORMATS_SHIM
from tests.test_overlay_core import SHIM as OVERLAY_SHIM
from tests.test_overlay_core import overlay, overlay_np, random_image

KR, KB = 0.2126, 0.0722
KG = 1 - KR - KB
FMT_NAME = {RGBA: "rgba", BGRA: "bgra", NV12: "nv12", I420: "i420", YUV444: "yuv444", P010: "p010"}

# ---- float64 bounds -----------------------------------------------------------------------------------------------------
# The per-pixel proofs of the host tier, each over every input colour (or block sum): the 8-bit BT.709 codes are within one
# code value of the float64 formula (test_export_core.test_bt709_every_colour_within_one_code_value), the 10-bit ones within
# 0.503 (test_export_formats_core: every colour, every 2x2 block sum); the NV12 overlay's Y within 0.501 and (Cb, Cr)
# within 0.502 of the float64 blend of the integer pixel or block average (test_overlay_core).
BT709_8, BT709_10 = 1.0, 0.503
OVERLAY_Y, OVERLAY_C = 0.501, 0.502


def yuv_bounds(fmt, e):
    """(Y bound, chroma bound) of a format applied to an image each of whose channels is within e of the exact float64 one.
    The formula is Lipschitz in R, G, B with constant 219 / 255 (Y: Kr + Kg + Kb = 1), 224 / 255 (Cb, Cr: the coefficient
    magnitudes sum to 2 (1 - Kb) and 2 (1 - Kr), which the scale divides out); 876 / 255 and 896 / 255 at 10 bits.  NV12 and
    I420 average a 2x2 block as (s + 2) >> 2, half a code more; P010 takes the exact block sums."""
    if fmt == "p010":
        return BT709_10 + 876 / 255 * e, BT709_10 + 896 / 255 * e
    return BT709_8 + 219 / 255 * e, BT709_8 + 224 / 255 * (e + 0.5 if fmt in ("nv12", "i420") else e)


def composite_error(over, native):
    """how far an integer composite can be from the float64 one: native opacity rounds bg (255 - a) / 255 once (mul_norm8,
    half a code, and the clamp at 255 is 1-Lipschitz); any other opacity keeps the stored colour, exact"""
    return 0.5 if over and native else 0.0


# ---- the float64 reference ----------------------------------------------------------------------------------------------
def comp255(top, bg, native, over=True):
    """255 x the float64 composite of top-down pixels [h][w][4] over bg, as exact integers (int64 [h][w][4]): native opacity
    min(255, c + bg (255 - a) / 255) per channel, otherwise c; alpha 255.  over=False: the stored pixel, alpha included."""
    c = top.astype(np.int64) * 255
    if not over:
        return c
    if native:
        a = top[..., 3:4].astype(np.int64)
        c[..., :3] = np.minimum(255 * 255, c[..., :3] + np.asarray(bg[:3], np.int64) * (255 - a))
    c[..., 3] = 255 * 255
    return c


def f64_ycbcr(c, bits=8):
    """float64 BT.709 limited range of float64 R, G, B ([..., >= 3]): (Y, Cb, Cr)"""
    r, g, b = c[..., 0], c[..., 1], c[..., 2]
    yp = KR * r + KG * g + KB * b
    sy, sc, oy, oc = (219, 224, 16, 128) if bits == 8 else (876, 896, 64, 512)
    return oy + sy / 255 * yp, oc + sc / 255 * (b - yp) / (2 * (1 - KB)), oc + sc / 255 * (r - yp) / (2 * (1 - KR))


def f64_planes(c, fmt):
    """a float64 top-down image [h][w][>= 3] -> float64 (Y, Cb, Cr) planes of fmt: YUV444 per pixel, the others' chroma
    from the mean of each 2x2 block"""
    h, w = c.shape[:2]
    bits = 10 if fmt == "p010" else 8
    y, cb, cr = f64_ycbcr(c, bits)
    if fmt != "yuv444":
        m = c[..., :3].reshape(h // 2, 2, w // 2, 2, 3).mean(axis=(1, 3))
        _, cb, cr = f64_ycbcr(m, bits)
    return y, cb, cr


def _axis_sums(v, m):
    """v int64 [n][...] -> [m][...]: sum over i of overlap(output X, source i) v[i], output X covering [X n, (X + 1) n) and
    source i [i m, (i + 1) m), from the prefix sums: the integral of the step function up to T is m P[T // m] + (T % m) v[T // m]"""
    n = v.shape[0]
    P = np.concatenate([np.zeros((1,) + v.shape[1:], np.int64), np.cumsum(v, axis=0)])
    vz = np.concatenate([v, np.zeros((1,) + v.shape[1:], np.int64)])
    T = np.arange(m + 1, dtype=np.int64) * n
    q, r = T // m, (T % m).reshape((-1,) + (1,) * (v.ndim - 1))
    return np.diff(m * P[q] + r * vz[q], axis=0)


def area_sums(img, size):
    """img int64 [h][w][c] -> int64 [oh][ow][c]: the area-weighted sums, total weight D = w h per output pixel"""
    ow, oh = size
    out = []
    for k in range(img.shape[2]):                                   # per channel: a few hundred MB at 7680 x 4320
        v = _axis_sums(np.ascontiguousarray(img[..., k].T.astype(np.int64)), ow).T   # [h][ow]
        out.append(_axis_sums(np.ascontiguousarray(v), oh))
    return np.stack(out, axis=-1)


def area_int(img, size):
    """the exact integer area average (sum + D / 2) // D of area_np, from prefix sums instead of a weight matrix"""
    d = img.shape[0] * img.shape[1]
    return (area_sums(img, size) + d // 2) // d


def f64_area(c255, size):
    """the float64 area average of a 255-scaled image (comp255): every sum is an exact integer, one division at the end"""
    return area_sums(c255, size) / (255.0 * c255.shape[0] * c255.shape[1])


def scaled_exact(frame, fmt, over, bg, native, size, crop=None):
    """scaled_np / yuv_np of the scaled image with area_int in place of area_np: the same bytes at any size (no weight matrix)"""
    top = frame[::-1]
    x, y, cw, ch = crop or (0, 0, frame.shape[1], frame.shape[0])
    yuv = fmt in ("i420", "yuv444", "p010")
    comp = over or yuv or fmt == "nv12"
    img = top[y:y + ch, x:x + cw].astype(np.int64)
    if comp:
        img = over_np(img, bg, native)
    avg = area_int(img, size)
    if comp:
        avg[..., 3] = 255
    avg = avg.astype(np.uint8)
    if yuv:
        return yuv_np(avg, fmt)
    if fmt == "nv12":
        return nv12_np(avg[::-1], bg, native)
    return avg[..., [2, 1, 0, 3]] if fmt == "bgra" else avg


def planes_of(got, fmt, h):
    """an export's bytes -> float64 (Y, Cb, Cr): NV12 / P010 [h * 3 / 2][w] (P010 codes << 6), I420 / YUV444 a plane tuple"""
    if fmt in ("nv12", "p010"):
        g = np.asarray(got).astype(np.float64) / (64 if fmt == "p010" else 1)
        return g[:h], g[h:, 0::2], g[h:, 1::2]
    return tuple(np.asarray(p).astype(np.float64) for p in got)


def check_f64(got, fmt, c, e, what=""):
    """got: an export of fmt (RGBA / BGRA [h][w][4]); c: the exact float64 top-down image it states ([h][w][4], composited
    or not); e: how far the integer image the kernel formats can be from c, per channel.  Asserts every code within bound and
    returns the largest error seen."""
    h = c.shape[0]
    if fmt in ("rgba", "bgra"):
        g = np.asarray(got).reshape(c.shape).astype(np.float64)
        if fmt == "bgra":
            g = g[..., [2, 1, 0, 3]]
        err = np.abs(g - c).max()
        assert err <= e, (what, fmt, err, e)
        return err
    by, bc = yuv_bounds(fmt, e)
    worst = 0.0
    for k, (gp, wp) in enumerate(zip(planes_of(got, fmt, h), f64_planes(c, fmt))):
        err = np.abs(gp - wp).max()
        assert err <= (by if k == 0 else bc), (what, fmt, "YCbCr"[k] if k else "Y", err, by if k == 0 else bc)
        worst = max(worst, err)
    return worst


def f64_whole(frame, over, bg, native):
    """the float64 image a whole-frame export states: top-down, composited (over, or any YUV format) or as stored"""
    return comp255(frame[::-1], bg, native, over) / 255.0


def f64_scaled(frame, over, bg, native, size, crop=None):
    """the float64 image a scaled export states: the exact area average of the (composited) crop"""
    top = frame[::-1]
    x, y, cw, ch = crop or (0, 0, frame.shape[1], frame.shape[0])
    return f64_area(comp255(top[y:y + ch, x:x + cw], bg, native, over), size)


def f64_overlay(frame, rect, fmt, native):
    """the float64 overlay of a read-back frame onto a rectangle's bytes, and the bound per plane: RGBA / BGRA the "over"
    c + d (255 - a) / 255 in all four channels (mul_norm8 rounds once: 0.5); NV12 the affine blend in Y'CbCr, Y per pixel
    (0.501) and chroma from the exact 2x2 mean of the stored pixels, alpha included (0.502 for the integer mean, plus the
    half code of (s + 2) >> 2 in each channel through the blend's Lipschitz constants 224 / 255 in R, G, B and 128 / 255 in
    alpha).  Any other opacity: the export's bytes (composite exact, background black).
    -> (float64 expected, bounds) with expected [h][w][4] (RGBA / BGRA order of the destination) or NV12 planes"""
    h, w = frame.shape[:2]
    top = frame[::-1].astype(np.float64)
    if fmt != NV12:
        if not native:
            c = top.copy()
            c[..., 3] = 255
            return (c[..., [2, 1, 0, 3]] if fmt == BGRA else c), 0.0
        c = top[..., [2, 1, 0, 3]] if fmt == BGRA else top
        d = rect.astype(np.float64)
        return np.minimum(255, c + d * (255 - c[..., 3:4]) / 255), 0.5
    if not native:
        c = top.copy()
        return f64_planes(c, "nv12"), yuv_bounds("nv12", 0.0)
    a = top[..., 3] / 255
    yd = rect[:h].astype(np.float64)
    y = 16 * a + 219 / 255 * (KR * top[..., 0] + KG * top[..., 1] + KB * top[..., 2]) + (1 - a) * yd
    m = top.reshape(h // 2, 2, w // 2, 2, 4).mean(axis=(1, 3))
    am = m[..., 3] / 255
    uvd = rect[h:].astype(np.float64).reshape(h // 2, w // 2, 2)
    yp = KR * m[..., 0] + KG * m[..., 1] + KB * m[..., 2]
    cb = 128 * am + 224 / 255 * (m[..., 2] - yp) / (2 * (1 - KB)) + (1 - am) * uvd[..., 0]
    cr = 128 * am + 224 / 255 * (m[..., 0] - yp) / (2 * (1 - KR)) + (1 - am) * uvd[..., 1]
    return (y, cb, cr), (OVERLAY_Y, OVERLAY_C + 0.5 * (224 + 128) / 255)


def check_overlay_f64(got, frame, rect, fmt, native, what=""):
    want, bound = f64_overlay(frame, rect, fmt, native)
    h = frame.shape[0]
    if fmt != NV12:
        err = np.abs(np.asarray(got).astype(np.float64).reshape(want.shape) - want).max()
        assert err <= bound, (what, fmt, err, bound)
        return
    for k, (gp, wp) in enumerate(zip(planes_of(got, "nv12", h), want)):
        err = np.abs(gp - wp).max()
        assert err <= bound[k > 0], (what, "YCbCr"[k] if k else "Y", err, bound[k > 0])


# ---- shims -----------------------------------------------------------------------------------------------------------------
def _compile(tmp_path_factory, name, src_text):
    d = tmp_path_factory.mktemp(name)
    src, so = d / "shim.cpp", d / "shim.so"
    src.write_text(src_text)
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I", CSRC,
                    "-include", "cstring", "-include", "algorithm", "-include", "cmath", "-o", str(so), str(src)], check=True)
    return C.CDLL(str(so))


@pytest.fixture(scope="module")
def shims(tmp_path_factory):
    """(scaled: t_export and t_scaled, formats: t_export_yuv, overlay: t_overlay) with the argument types their files give"""
    vp, sz, i32, u32 = C.c_void_p, C.c_size_t, C.c_int, C.c_uint32
    s = _compile(tmp_path_factory, "limits_scaled", SCALED_SHIM)
    s.t_scaled.argtypes = [vp, i32, i32, vp, i32, i32, i32, i32, u32] + [i32] * 6 + [vp, vp, sz]
    s.t_export.argtypes = [vp, i32, i32, vp, i32, i32, i32, i32, u32, vp, sz, sz]
    f = _compile(tmp_path_factory, "limits_formats", FORMATS_SHIM)
    f.t_export_yuv.argtypes = [vp, i32, i32, vp, i32, i32, i32, u32, vp, sz, vp, sz]
    o = _compile(tmp_path_factory, "limits_overlay", OVERLAY_SHIM)
    o.t_overlay.argtypes = [vp, i32, i32, vp, i32, i32, i32, i32, vp, vp, sz]
    return s, f, o


# ---- the reference itself ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w,size", [(7, 5, (3, 2)), (64, 97, (13, 7)), (33, 300, (299, 32)), (8, 1920, (7, 2)),
                                      (40, 7919, (13, 3)), (16, 16384, (16383, 15)), (2, 4, (1, 1))])
def test_prefix_sum_area_equals_the_weight_matrix_restatement(h, w, size):
    """area_int (prefix sums) is area_np (interval-overlap weight matrices) bit for bit, and f64_area is their exact mean"""
    rng = np.random.default_rng(h * w)
    img = rng.integers(0, 256, (h, w, 4)).astype(np.int64)
    assert np.array_equal(area_int(img, size), area_np(img, size))
    exact = area_sums(img, size)
    assert (exact.sum(axis=(0, 1)) == img.sum(axis=(0, 1)) * size[0] * size[1]).all()   # every weight sums to D
    assert np.abs(f64_area(img * 255, size) * (h * w) - exact).max() < 1e-6 * exact.max()


def test_float64_reference_endpoints():
    """black, white and greys through the float64 BT.709 at both depths, and the composite's extremes"""
    c = np.array([[0, 0, 0], [255, 255, 255], [128, 128, 128]], np.float64)
    for bits, lo, hi, mid in ((8, 16, 235, 128), (10, 64, 940, 512)):
        y, cb, cr = f64_ycbcr(c, bits)
        assert np.allclose(y[:2], [lo, hi]) and np.allclose(cb, mid) and np.allclose(cr, mid)
    px = np.array([[[0, 0, 0, 0], [255, 255, 255, 255], [10, 20, 30, 40]]], np.uint8)
    got = comp255(px, (200, 100, 50), True) / 255
    assert np.allclose(got[0, 0, :3], [200, 100, 50]) and np.allclose(got[0, 1, :3], 255)
    assert np.allclose(got[0, 2, :3], np.array([10, 20, 30]) + np.array([200, 100, 50]) * 215 / 255)


# ---- the walks at the limits ---------------------------------------------------------------------------------------------------
TINY = [(w, h) for w in (4, 5, 6, 7, 8) for h in (1, 2, 3)]
STRIPS = [(w, h) for w in (127, 128, 129, 255, 257) for h in (1, 6)]
TALL = [(16384, 8), (8, 16384)]
GEOMETRIES = TINY + STRIPS + TALL


def _accepts(fmt, w, h):
    """4:2:0 needs an even width and height (refused by design otherwise)"""
    return fmt not in (NV12, I420, P010) or not (w | h) & 1


def _marks_for(rng, w, h):
    """a band height for the marks: 1, 7, the whole frame or a random one"""
    return int(rng.choice([1, 7, h, int(rng.integers(1, h + 1))])) if h > 1 else 1


def _frame(rng, w, h, native):
    frame = premultiplied(rng, (h, w)) if native else rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    frame[rng.random((h, w)) < 0.3] = 0
    return frame


@pytest.mark.parametrize("w,h", GEOMETRIES)
def test_whole_frame_walks_at_the_limits(shims, w, h):
    """t_export (RGBA / BGRA / NV12) and t_export_yuv (I420 / YUV444 / P010), with and without marks over garbage rows:
    the restatement bit for bit and float64 within the derived bounds"""
    s, f, _ = shims
    rng = np.random.default_rng(w * 7 + h)
    bg = (250, 17, 128)
    for native in (True, False):
        frame = _frame(rng, w, h, native)
        for fmt in (RGBA, BGRA, NV12, I420, YUV444, P010):
            if not _accepts(fmt, w, h):
                continue
            name = FMT_NAME[fmt]
            for over in ((False, True) if fmt in (RGBA, BGRA) else (True,)):
                if fmt in (I420, YUV444, P010):
                    got = export_yuv(f, frame, fmt, bg, native)
                    assert same(got, frame_np(frame, name, bg, native)), (name, native)
                else:
                    got = export(s, frame, fmt, over=over, native=native, bg=bg)
                    if fmt == NV12:
                        assert np.array_equal(got, nv12_np(frame, bg, native)), (name, native)
                    else:
                        got = got.reshape(h, w, 4)
                        want = (over_np(frame, bg, native).astype(np.uint8) if over else frame)[::-1]
                        assert np.array_equal(got, want[..., [2, 1, 0, 3]] if fmt == BGRA else want), (name, over, native)
                check_f64(got, name, f64_whole(frame, over, bg, native), composite_error(over, native), (w, h, native))
        # marks: the same exports from a frame whose unmarked rows hold garbage
        rows = _marks_for(rng, w, h)
        dirty, clean, marks = marked_frame(rng, w, h, rows, True)
        for fmt in (RGBA, NV12, I420, YUV444, P010):
            if not _accepts(fmt, w, h):
                continue
            if fmt in (I420, YUV444, P010):
                got = export_yuv(f, dirty, fmt, bg, marks=marks, rows=rows)
                assert same(got, frame_np(clean, FMT_NAME[fmt], bg, True)), (fmt, rows)
            else:
                got = export(s, dirty, fmt, over=True, bg=bg, marks=marks, rows=rows)
                assert np.array_equal(got, export(s, clean, fmt, over=True, bg=bg)), (fmt, rows)
                if fmt == RGBA:
                    got = got.reshape(h, w, 4)
            check_f64(got, FMT_NAME[fmt], f64_whole(clean, True, bg, True), 0.5, (w, h, rows))


def _scale_cases(w, h):
    """(size, crop): 1x1 of the whole frame, n -> n - 1 on both axes, a prime-ish ratio, 1x1 / 2x2 crops at the four corners,
    a crop touching the right and bottom edges, and a 1-pixel-wide full-height column shrunk to 1x1"""
    cases = [((1, 1), None), ((max(1, w - 1), max(1, h - 1)), None), ((max(1, w // 7), max(1, h // 3)), None),
             ((1, 1), (w - 1, h // 2, 1, h - h // 2)), ((1, 1), (w // 2, 0, 1, h))]
    for cw, ch in ((1, 1), (2, 2)):
        if cw <= w and ch <= h:
            cases += [((1, 1), (x, y, cw, ch)) for x in (0, w - cw) for y in (0, h - ch)]
    if w >= 3 and h >= 2:
        cases.append(((2, 1), (w - 3, h - 2, 3, 2)))
    return cases


@pytest.mark.parametrize("w,h", GEOMETRIES)
def test_scaled_walk_at_the_limits(shims, w, h):
    """t_scaled without and with marks over garbage: scaled_np and area_int bit for bit, float64 within bounds"""
    s, _, _ = shims
    rng = np.random.default_rng(w * 11 + h)
    bg = (250, 17, 128)
    frame = _frame(rng, w, h, True)
    rows = _marks_for(rng, w, h)
    dirty, clean, marks = marked_frame(rng, w, h, rows, True)
    for size, crop in _scale_cases(w, h):
        for fmt in (RGBA, BGRA, NV12):
            if fmt == NV12 and (size[0] | size[1]) & 1:
                continue
            name = FMT_NAME[fmt]
            for over in ((False, True) if fmt != NV12 else (True,)):
                got = scaled_shim(s, frame, fmt, size, crop, over=over, bg=bg)
                want = scaled_exact(frame, name, over, bg, True, size, crop)
                assert np.array_equal(got.reshape(want.shape), want), (name, size, crop, over)
                if size[0] * size[1] <= 4096 and w * h <= 1 << 17:
                    assert np.array_equal(want, scaled_np(frame, fmt, over, bg, True, size, crop)), (name, size, crop)
                check_f64(got.reshape(want.shape), name, f64_scaled(frame, over or fmt == NV12, bg, True, size, crop),
                          composite_error(over or fmt == NV12, True) + 0.5, (size, crop))
                aware = scaled_shim(s, dirty, fmt, size, crop, over=over, bg=bg, marks=marks, rows=rows)
                assert np.array_equal(aware, scaled_shim(s, clean, fmt, size, crop, over=over, bg=bg)), (name, size, crop, rows)


@pytest.mark.parametrize("w,h", [g for g in GEOMETRIES if not (g[0] | g[1]) & 1] + [(5, 3), (129, 1), (257, 6)])
def test_overlay_walk_at_the_limits(shims, w, h):
    """t_overlay, band and row-pair items, marks over garbage: overlay_np bit for bit, float64 within bounds; RGBA / BGRA
    at any size, NV12 at even sizes"""
    _, _, o = shims
    rng = np.random.default_rng(w * 13 + h)
    rows = _marks_for(rng, w, h)
    dirty, clean, marks = marked_frame(rng, w, h, rows, True)
    for fmt in (RGBA, BGRA, NV12):
        if fmt == NV12 and (w | h) & 1:
            continue
        img = random_image(rng, fmt, w, h)
        want = overlay_np(clean, img, fmt, True)
        for band in (True, False):
            got = overlay(o, dirty, img, fmt, True, marks=marks, rows=rows, band=band)
            assert np.array_equal(got, want), (fmt, band, rows)
        check_overlay_f64(want, clean, img, fmt, True, (w, h, fmt))
        other = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
        got = overlay(o, other, img, fmt, False)
        assert np.array_equal(got, overlay_np(other, img, fmt, False)), fmt
        check_overlay_f64(got, other, img, fmt, False, (w, h, fmt, "other opacity"))


def test_yuv_bounds_are_the_derivation():
    """the bounds are the per-pixel proofs plus the Lipschitz terms, not fitted numbers"""
    assert yuv_bounds("yuv444", 0.0) == (1.0, 1.0)
    assert yuv_bounds("nv12", 0.0) == (1.0, 1.0 + 224 / 255 * 0.5)
    assert yuv_bounds("p010", 0.5) == (0.503 + 876 / 510, 0.503 + 896 / 510)
    assert composite_error(True, True) == 0.5 and composite_error(True, False) == 0.0 and composite_error(False, True) == 0.0
