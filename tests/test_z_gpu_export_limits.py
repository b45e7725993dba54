"""-m gpu: every frame export at the geometry limits, checked two ways.  Each case renders real frames, exports them, reads
the same streams back and compares every output with the numpy restatements of the host tier bit for bit (whole frames in
row bands, scaled outputs through the prefix-sum area average that tests/test_export_limits_core.py proves equal to
area_np) and with the float64 statement of the operation in that file, within bounds derived from the host tier's
per-pixel proofs (tests/test_export_limits_core.py yuv_bounds).

Geometries: 7680 x 4320 (bars; radial under non-native opacity), 3840 x 2160 radial, 16384 x 256 and 256 x 16384; a uniform
16384 x 16384 frame (module `test`, #55000055 everywhere) shrunk to 1x1 / 2x2, cropped at its corners and edges and shrunk
by one pixel per axis, whose 64-bit area numerators need their upper half on the device (export_div's __umul64hi branch,
which the host tier cannot reach); 4..8 x 1..3 frames and widths around the 128-pixel strip; n -> n - 1 and prime ratios;
band heights 1, 7, the default and the frame height with live, stale and absent dirty-row marks; an 8K ladder; overlays at
8K and 16384 x 256.  Every destination sits in a sentinel-filled buffer whose untouched bytes are checked.  Refused by
design, so not exported: odd NV12 / I420 / P010 sizes and upscaling."""
import numpy as np
import pytest

import glava_b200 as g
from tests.test_export_core import BGRA, NV12, RGBA, nv12_np, over_np
from tests.test_export_formats_core import frame_np, same
from tests.test_export_limits_core import (_scale_cases, check_f64, check_overlay_f64, composite_error, f64_scaled, f64_whole,
                                           scaled_exact)
from tests.test_overlay_core import overlay_np

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
torch = pytest.importorskip("torch")

BG = (250, 240, 230)
FORMATS = ("rgba", "bgra", "nv12", "i420", "yuv444", "p010")
YUV = ("nv12", "i420", "yuv444", "p010")
OVERLAY = {"rgba": RGBA, "bgra": BGRA, "nv12": NV12}
SENTINEL = 0xA5
CHUNK = 512                                                        # rows per restatement band (even)
BIG = 1 << 22                # pixels past which the host restates one stream and whole frames in three row bands only


def feed(r, steps, seed=0, scale=0.3):
    rng = np.random.default_rng(seed)
    n = r.params.n
    for _ in range(steps):
        lb = (rng.standard_normal((r.batch, n)) * scale).astype(np.float32)
        rb = (rng.standard_normal((r.batch, n)) * scale).astype(np.float32)
        r.update(lb, rb, True)


def host(t):
    return tuple(x.cpu().numpy() for x in t) if isinstance(t, tuple) else t.cpu().numpy()


def entry(got, i):
    return tuple(x[i] for x in got) if isinstance(got, tuple) else got[i]


def accepts(fmt, w, h):
    """4:2:0 formats need an even width and height: odd sizes are refused by design"""
    return fmt not in ("nv12", "i420", "p010") or not (w | h) & 1


def padded_export(r, streams, fmt, size=None, crop=None, over=False, bg=BG):
    """an export into a sentinel-filled buffer 48+ bytes wider and two rows taller than the output; asserts that every byte
    outside the output's planes keeps the sentinel and returns the output on the host"""
    w, h = size or (r.params.w, r.params.h)
    rows, row_bytes, align = g.api._export_layout(fmt, w, h)
    pitch = (row_bytes + 48 + align - 1) // align * align
    base = torch.full((len(streams), rows + 2, pitch), SENTINEL, dtype=torch.uint8, device="cuda")
    out = base[:, :rows]
    if size is None:
        got = r.export_frames(streams, fmt, over=over, background=bg, out=out)
    else:
        got = r.export_scaled(streams, size, crop, fmt, over=over, background=bg, out=out)
    mask = torch.zeros_like(base)
    views = g.api._export_views(fmt, mask[:, :rows], w, h)
    for v in (views if isinstance(views, tuple) else (views,)):
        v.fill_(0x0101 if v.dtype == torch.uint16 else 1)
    assert bool((base[mask == 0] == SENTINEL).all()), ("written outside the output", fmt, size, crop)
    return host(g.api._export_views(fmt, out, w, h))


def whole_np(sub, fmt, over, bg, native):
    """the restatement of a whole-frame export of framebuffer rows `sub` (bottom-up)"""
    if fmt in ("rgba", "bgra"):
        out = (over_np(sub, bg, native).astype(np.uint8) if over else sub)[::-1]
        return out[..., [2, 1, 0, 3]] if fmt == "bgra" else out
    if fmt == "nv12":
        return nv12_np(sub, bg, native)
    return frame_np(sub, fmt, bg, native)


def rows_of(got, fmt, h, r0, r1):
    """output rows [r0, r1) of a whole-frame export (r0, r1 even for 4:2:0) with their chroma rows"""
    if fmt in ("rgba", "bgra"):
        return got[r0:r1]
    if fmt in ("nv12", "p010"):
        return np.concatenate([got[r0:r1], got[h + r0 // 2:h + r1 // 2]])
    if fmt == "i420":
        return got[0][r0:r1], got[1][r0 // 2:r1 // 2], got[2][r0 // 2:r1 // 2]
    return tuple(p[r0:r1] for p in got)


def check_whole(got, frame, fmt, over, bg, native, what=""):
    """one entry of a whole-frame export against the restatement and float64, band by band of CHUNK output rows"""
    h, w = frame.shape[:2]
    comp = over or fmt in YUV
    starts = list(range(0, h, CHUNK))
    if w * h > BIG:                                                # the top, the middle and the bottom band
        starts = sorted({starts[0], starts[len(starts) // 2], starts[-1]})
    for r0 in starts:
        r1 = min(h, r0 + CHUNK)
        sub = frame[h - r1:h - r0]
        part = rows_of(got, fmt, h, r0, r1)
        assert same(part, whole_np(sub, fmt, over, bg, native)), (what, fmt, over, r0)
        check_f64(part, fmt, f64_whole(sub, comp, bg, native), composite_error(comp, native), (what, fmt, r0))


def check_scaled(got, frame, fmt, over, bg, native, size, crop=None, what=""):
    comp = over or fmt in YUV
    assert same(got, scaled_exact(frame, fmt, over, bg, native, size, crop)), (what, fmt, over, size, crop)
    check_f64(got, fmt, f64_scaled(frame, comp, bg, native, size, crop), composite_error(comp, native) + 0.5,
              (what, fmt, size, crop))


def prime_at_most(n):
    for k in range(n, 1, -1):
        if all(k % d for d in range(2, int(k ** 0.5) + 1)):
            return k
    return 1


# ---- uniform 16384 x 16384: known answers, 64-bit numerators ------------------------------------------------------------------
def test_uniform_16384_square_known_answers(built):
    """module `test` renders #55000055 everywhere, so every export of every crop is the export of that one pixel.  Shrunk
    to 1x1 / 2x2 from an 8192 x 8192 corner and to 64 x 64 from the whole frame, the per-channel numerator channel * D + D / 2
    (D = 2^26, 2^28) passes 2^32 in every format family.  (A 1x1 output of the whole frame is one lane walking 2^28 pixels:
    correct, but minutes of a test's time.)"""
    p = g.default_params("test", n=1024, w=16384, h=16384)
    native = bool(p.premultiply_alpha)
    px = np.array([0x55, 0, 0, 0x55], np.uint8)
    tiny = np.broadcast_to(px, (4, 4, 4)).copy()                  # any uniform frame has the same exports
    high = set()
    with g.Renderer(p, batch=1) as r:
        feed(r, 1)
        cases = [(False, "rgba", (1, 1), 8192), (False, "nv12", (2, 2), 8192), (True, "bgra", (1, 1), 8192),
                 (True, "yuv444", (1, 1), 8192), (True, "i420", (2, 2), 8192), (True, "p010", (2, 2), 8192)]
        cases += [(over, fmt, (64, 64), 16384) for over in (False, True) for fmt in FORMATS]
        for over, fmt, size, side in cases:
            crop = (16384 - side, 16384 - side, side, side)            # the bottom-right corner, or the whole frame
            src = np.broadcast_to(px, (size[1], size[0], 4)).copy()    # uniform at the output's size: the same exports
            got = entry(padded_export(r, [0], fmt, size, crop, over, BG), 0)
            check_scaled(got, src, fmt, over, BG, native, size, what=("uniform", side))
            img = over_np(tiny, BG, native) if over or fmt in YUV else tiny.astype(np.int64)
            # every output pixel's weights sum to D = src_w * src_h: its numerator is about channel * D + D / 2
            D = side * side
            if int(img[..., :3].max()) * D + D // 2 >= 1 << 32:
                high.add("rgb" if fmt in ("rgba", "bgra") else "444" if fmt == "yuv444" else "420")
        assert high == {"rgb", "444", "420"}, high                  # the cases cannot go vacuous
        # crops: 1x1 and 2x2 at the four corners, touching the right and bottom edges, a 1-pixel column of full height
        crops = [(x, y, c, c) for c in (1, 2) for x in (0, 16384 - c) for y in (0, 16384 - c)]
        crops += [(16384 - 5001, 16384 - 3001, 5001, 3001), (16383, 0, 1, 16384), (8191, 0, 1, 16384), (0, 16383, 16384, 1)]
        for crop in crops:
            for fmt, over in (("rgba", False), ("bgra", True), ("yuv444", True)):
                got = entry(padded_export(r, [0], fmt, (1, 1), crop, over, BG), 0)
                assert same(got, scaled_exact(tiny, fmt, over, BG, native, (1, 1))), (fmt, crop)
            if crop[2] % 2 == 0 and crop[3] % 2 == 0:
                got = entry(padded_export(r, [0], "p010", (2, 2), crop, True, BG), 0)
                assert same(got, scaled_exact(tiny, "p010", True, BG, native, (2, 2))), crop
        # n -> n - 1 on both axes (every weight partial) and the whole frame: every output pixel is the one pixel's
        for fmt, size in (("rgba", (16383, 16383)), ("nv12", None), ("yuv444", (16383, 16383))):
            got = (r.export_frames([0], fmt, over=True, background=BG) if size is None
                   else r.export_scaled([0], size, None, fmt, over=True, background=BG))
            want = scaled_exact(tiny, fmt, True, BG, native, (2, 2))
            if fmt == "rgba":
                assert bool((got[0] == torch.from_numpy(want[0, 0]).cuda()).all())
            elif fmt == "nv12":
                assert bool((got[0, :16384] == int(want[0, 0])).all()) and bool((got[0, 16384:, 0::2] == int(want[2, 0])).all())
                assert bool((got[0, 16384:, 1::2] == int(want[2, 1])).all())
            else:
                for k in range(3):
                    assert bool((got[k][0] == int(want[k][0, 0])).all()), k
            del got
            torch.cuda.empty_cache()


# ---- wide and tall real frames ----------------------------------------------------------------------------------------------------
WIDE = [("bars", 7680, 4320, True), ("radial", 7680, 4320, False), ("radial", 3840, 2160, True), ("bars", 16384, 256, True),
        ("graph", 256, 16384, True)]


def renderer_params(module, w, h, native, n=2048):
    kw = {} if native else dict(premultiply_alpha=0, clear_color=[0.1, 0.2, 0.3, 1.0])
    return g.default_params(module, n=n, w=w, h=h, **kw)


@pytest.mark.parametrize("module,w,h,native", WIDE, ids=[f"{m}-{w}x{h}" + ("" if n else "-blended") for m, w, h, n in WIDE])
def test_wide_and_tall_frames(built, module, w, h, native):
    p = renderer_params(module, w, h, native)
    with g.Renderer(p, batch=2) as r:
        feed(r, 2, seed=w + h, scale=0.5)
        big = w * h > BIG
        streams = [1] if big else [1, 0]
        frames = [r.readback(s) for s in streams]
        assert frames[0].any() and (native or (frames[0].view(np.uint32) != 0).all())   # non-native: no pixel is zero
        for fmt in FORMATS:
            for over in ((True, False) if fmt in ("rgba", "bgra") else (True,)):
                got = padded_export(r, streams, fmt, over=over)
                for i in range(len(streams)):
                    check_whole(entry(got, i), frames[i], fmt, over, BG, native, (module, w, h, i))
        # n -> n - 1 (every weight partial) and prime ratios; past BIG over a corner region of about 2048 x 1024
        sw, sh = (min(w, 2048), min(h, 1024)) if big else (w, h)
        cw, ch = prime_at_most(sw - 3), prime_at_most(sh - 1)
        cases = [((sw - 1, sh - 1), (w - sw, h - sh, sw, sh), "rgba", True), ((13, 7), (w - cw, 1, cw, ch), "rgba", False),
                 ((sw // 2 & ~1, sh // 2 & ~1), (0, h - sh, sw, sh), "i420", True), ((64, 2), None, "p010", True),
                 ((13, 7), (1, h - ch, cw, ch), "yuv444", True), ((sw // 3 & ~1, sh // 3 & ~1), (w - sw, 0, sw, sh), "nv12", True)]
        cases += [((1, 1), crop, fmt, False) for (_, crop) in _scale_cases(w, h) if crop for fmt in ("bgra",)]
        for size, crop, fmt, over in cases:
            got = padded_export(r, streams, fmt, size, crop, over)
            for i in range(len(streams)):
                check_scaled(entry(got, i), frames[i], fmt, over, BG, native, size, crop, (module, w, h, i))


# ---- tiny frames and strip edges ----------------------------------------------------------------------------------------------------
SMALL = [(w, h) for w in (4, 5, 6, 7, 8) for h in (1, 2, 3)] + [(w, h) for w in (127, 128, 129, 255, 257) for h in (2, 7)]


@pytest.mark.parametrize("w,h", SMALL, ids=[f"{w}x{h}" for w, h in SMALL])
def test_tiny_frames_and_strip_edges(built, w, h):
    """every format that takes the size, whole and scaled, and the overlay, from three streams"""
    module = ("bars", "graph", "wave", "radial")[(w + h) % 4]
    native = (w + h) % 3 != 0
    p = renderer_params(module, w, h, native, n=1024)
    rng = np.random.default_rng(w * 31 + h)
    with g.Renderer(p, batch=3) as r:
        feed(r, 3, seed=w * h, scale=0.8)
        streams = [2, 0, 1]
        frames = [r.readback(s) for s in streams]
        for fmt in FORMATS:
            if not accepts(fmt, w, h):
                continue
            for over in ((True, False) if fmt in ("rgba", "bgra") else (True,)):
                got = padded_export(r, streams, fmt, over=over)
                for i in range(3):
                    check_whole(entry(got, i), frames[i], fmt, over, BG, native, (w, h, i))
        for size, crop in _scale_cases(w, h):
            for fmt in ("rgba", "bgra", "yuv444", "nv12", "p010"):
                if not accepts(fmt, *size):
                    continue
                over = fmt != "rgba"
                got = padded_export(r, streams, fmt, size, crop, over)
                for i in range(3):
                    check_scaled(entry(got, i), frames[i], fmt, over, BG, native, size, crop, (w, h, i))
        for fmt in ("rgba", "bgra", "nv12"):
            if not accepts(fmt, w, h):
                continue
            check_overlay(r, streams, frames, fmt, rng, pad=(16, 4))


def check_overlay(r, streams, frames, fmt, rng, pad=(0, 0)):
    """overlay onto random images `pad` pixels larger, the frame at (pad[0], pad[1] even): the restatement over the image
    bytes before the call, bit for bit, everything else untouched, and the float64 composite"""
    w, h = r.params.w, r.params.h
    native = bool(r.params.premultiply_alpha)
    W, H = w + pad[0], h + pad[1]
    x, y = pad[0], pad[1] & ~1
    nv12 = fmt == "nv12"
    row = W if nv12 else W * 4
    shape = (len(streams), H * 3 // 2 if nv12 else H, (row + 15) // 16 * 16)
    before = rng.integers(0, 256, shape, dtype=np.uint8)
    img = torch.from_numpy(before).cuda()[..., :row]
    if not nv12:
        img = img.unflatten(-1, (W, 4))
    r.overlay_frames(streams, img, [(x, y)] * len(streams), fmt)
    after = img.cpu().numpy()
    for i, frame in enumerate(frames):
        b = before[i][:, :row]
        b = b if nv12 else b.reshape(H, W, 4)
        if nv12:
            rect = np.concatenate([b[y:y + h, x:x + w], b[H + y // 2:H + (y + h) // 2, x:x + w]])
        else:
            rect = b[y:y + h, x:x + w]
        want = b.copy()
        o = overlay_np(frame, rect, OVERLAY[fmt], native)
        if nv12:
            want[y:y + h, x:x + w] = o[:h]
            want[H + y // 2:H + (y + h) // 2, x:x + w] = o[h:]
        else:
            want[y:y + h, x:x + w] = o
        assert np.array_equal(after[i], want), (fmt, i, w, h)
        check_overlay_f64(o, frame, rect, OVERLAY[fmt], native, (fmt, i, w, h))


# ---- dirty-row marks at band heights 1, 7, default and h -----------------------------------------------------------------------
MARKS = [(256, 16384), (7680, 4320)]


@pytest.mark.parametrize("w,h", MARKS, ids=[f"{w}x{h}" for w, h in MARKS])
def test_marks_at_every_band_height(built, w, h, monkeypatch):
    """bars with lazy smoothing: the band height changes between steps (marks stale for the pass after a change, live on
    the next), then a reconfigure to MIRROR_YX runs the generic kernel (no marks); whole, scaled, ladder and overlay exports
    at every step"""
    p = g.default_params("bars", n=2048, w=w, h=h)
    p.lazy_smooth = 1
    rng = np.random.default_rng(w)
    big = w * h > 1 << 24
    steps = [None, None, "7", "7", "1", "1", str(h), str(h), "mirror", None]
    rungs = [dict(size=None, fmt="i420"), dict(size=(w // 4 & ~1, h // 4 & ~1), fmt="p010", background=BG)]
    with g.Renderer(p, batch=2) as r:
        for step, rows in enumerate(steps):
            if rows == "mirror":
                monkeypatch.delenv("GLAVA_B200_ROWS", raising=False)
                q = r.params.copy(); q.bars_mirror_yx = 1
                r.reconfigure(q)
            elif rows is None:
                monkeypatch.delenv("GLAVA_B200_ROWS", raising=False)
                if r.params.bars_mirror_yx:
                    q = r.params.copy(); q.bars_mirror_yx = 0
                    r.reconfigure(q)
            else:
                monkeypatch.setenv("GLAVA_B200_ROWS", rows)
            feed(r, 1, seed=step, scale=0.05 + 0.2 * (step % 3))
            what = (w, h, step, rows)
            streams = [0]                                              # one stream: ten steps of host restatement
            frames = [r.readback(s) for s in streams]
            got = padded_export(r, streams, "rgba")
            for i, f in enumerate(frames):
                assert np.array_equal(got[i], f[::-1]), what                # as stored: exact
            for fmt in ("nv12",) if big else ("nv12", "yuv444"):
                got = padded_export(r, streams, fmt)
                for i, f in enumerate(frames):
                    check_whole(entry(got, i), f, fmt, True, BG, True, what)
            sw, sh = (2048, 1024) if big else (w, h)
            for size, crop, fmt in (((sw // 16 & ~1, sh // 16 & ~1), (0, h - sh, sw, sh), "nv12"),
                                    ((7, 5), (w - sw + 3, h - sh // 2, sw - 3, sh // 2), "rgba")):
                got = padded_export(r, streams, fmt, size, crop, True)
                for i, f in enumerate(frames):
                    check_scaled(entry(got, i), f, fmt, True, BG, True, size, crop, what)
            lad = r.export_ladder(streams, rungs)
            for j, rung in enumerate(rungs):
                kw = dict(background=rung.get("background", (0, 0, 0)))
                alone = (r.export_frames(streams, rung["fmt"], **kw) if rung["size"] is None
                         else r.export_scaled(streams, rung["size"], None, rung["fmt"], **kw))
                assert same(host(lad[j]), host(alone)), (what, j)
            lh = host(lad[0])
            for i, f in enumerate(frames):
                check_whole(entry(lh, i), f, "i420", True, (0, 0, 0), True, what)
                if not big:
                    check_scaled(entry(host(lad[1]), i), f, "p010", True, BG, True, rungs[1]["size"], None, what)
            if not big or step in (1, 8):                             # 8K: live marks (band items) and none
                for fmt in ("nv12",) if big else ("nv12", "rgba"):
                    check_overlay(r, streams, frames, fmt, rng)


# ---- the 8K ladder ------------------------------------------------------------------------------------------------------------
def test_ladder_at_8k_equals_its_rungs_and_float64(built):
    p = g.default_params("bars", n=4096, w=7680, h=4320)
    p.lazy_smooth = 1
    rungs = [dict(size=None, fmt="nv12"), dict(size=(3840, 2160), fmt="p010"), dict(size=(1920, 1080), fmt="i420"),
             dict(size=(2, 2), fmt="rgba", over=True, background=BG)]
    with g.Renderer(p, batch=2) as r:
        for step in range(2):                                          # the second pass with live marks
            feed(r, 1, seed=40 + step, scale=0.4)
        frames = [r.readback(1)]                                       # the host restates one of the two
        got = r.export_ladder([1, 0], rungs)
        for j, rung in enumerate(rungs):
            kw = dict(over=rung.get("over", False), background=rung.get("background", (0, 0, 0)))
            alone = (r.export_frames([1, 0], rung["fmt"], **kw) if rung["size"] is None
                     else r.export_scaled([1, 0], rung["size"], None, rung["fmt"], **kw))
            assert same(host(got[j]), host(alone)), j
            h_got = host(got[j])
            for i in range(len(frames)):
                e = entry(h_got, i)
                if rung["size"] is None:
                    check_whole(e, frames[i], rung["fmt"], True, kw["background"], True, ("ladder", j, i))
                else:
                    check_scaled(e, frames[i], rung["fmt"], kw["over"], kw["background"], True, rung["size"], None, ("ladder", j, i))


# ---- overlays at 8K and 16384 x 256 ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w,h", [(7680, 4320), (16384, 256)], ids=["7680x4320", "16384x256"])
def test_overlay_wide_frames(built, w, h):
    p = g.default_params("bars", n=4096, w=w, h=h)
    rng = np.random.default_rng(h)
    with g.Renderer(p, batch=2) as r:
        feed(r, 2, seed=h, scale=0.5)
        streams = [1] if w * h > BIG else [1, 0]
        frames = [r.readback(s) for s in streams]
        for fmt in ("rgba", "bgra", "nv12"):
            check_overlay(r, streams, frames, fmt, rng, pad=(16, 2) if h < 1024 else (0, 0))
