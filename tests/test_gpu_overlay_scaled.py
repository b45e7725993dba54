"""-m gpu: the overlay of a downscaled, cropped frame (glava_b200_overlay_scaled, DESIGN 4.21).  What a call leaves in the
caller's pictures must equal, bit for bit, the opacity overlay's numpy restatement (tests/test_overlay_opacity_core.py
restated) applied to S, the export_scaled RGBA image of the same stream (tests/test_export_scaled_core.py scaled_np: the
premultiplied area average under native opacity, EXPORT_OVER under any other) taken from glava_b200_readback at the same
point in call order, with every byte outside the rectangles untouched (row padding included): every module, every format
and encoding, native and any other opacity, K in {0, 1, 37, 128, 254, 255} and mixed lists, crops touching each edge, odd
and tiny outputs, picture-in-picture 1920x1080 -> 640x360 inside a 1080p picture, bars at 1080p under marks, the framebuffer
ring and styles, a 1024-entry list, after / done ordering, the sharded handle against one handle, and the identities: the
whole frame at its own size is the opacity overlay, any other opacity at K = 255 is export_scaled's bytes, a zero frame
under native opacity and K = 0 leave the picture alone."""
import numpy as np
import pytest

import glava_b200 as g
from tests.test_export_scaled_core import scaled_np
from tests.test_gpu_overlay_opacity import ENCS, FNAME, K_LIST, Picture, feed, fits, same
from tests.test_overlay_opacity_core import BGRA, FORMATS, I420, NAME, NV12, RGBA, YUV422P10, restated

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


def formats(w, h):
    """(format, through overlay_planes) of every format that takes a w x h rectangle"""
    return [(f, False) for f in (RGBA, BGRA, NV12) if fits(f, w, h)] + [(f, True) for f in FORMATS if f not in (RGBA, BGRA)
                                                                        and fits(f, w, h)]


def frames_arg(p):
    """Picture.frames_arg with the allocation's pitch kept on a one-row RGBA rectangle (a view of one row has no row stride)"""
    if p.fmt in (RGBA, BGRA):
        t = p.full[0]
        return torch.as_strided(t, (p.h, p.w, 4), (t.stride(0), 4, 1))
    return p.frames_arg()


def run(r, streams, fmt, pics, k, kw, planes, size, crop):
    op = None if k is None else [v / 255.0 for v in k]
    if not planes:
        r.overlay_frames(streams, [frames_arg(p) for p in pics], None, FNAME[fmt], opacity=op, size=size, crop=crop, **kw)
    else:
        r.overlay_planes(streams, [p.planes_arg() for p in pics], None, NAME[fmt], opacity=op, size=size, crop=crop, **kw)
    torch.cuda.synchronize()


def scaled_frame(r, s, size, crop):
    """S of stream s as a read-back frame (row 0 = bottom): export_scaled's RGBA pixels, EXPORT_OVER under any other opacity"""
    native = bool(r.params.premultiply_alpha)
    return np.ascontiguousarray(scaled_np(r.readback(int(s)), RGBA, not native, (0, 0, 0), native, size, crop)[::-1])


def expect(r, streams, pics, before, k, e, size, crop):
    native = bool(r.params.premultiply_alpha)
    out = [[a.copy() for a in b] for b in before]
    for i, s in enumerate(streams):
        rect = pics[i].rect_planes(out[i])
        kk = 255 if k is None else k[i]
        for dst, new in zip(rect, restated(scaled_frame(r, s, size, crop), [v.copy() for v in rect], pics[i].fmt, e, kk, native)):
            dst[...] = new
    return out


def check(r, streams, fmt, k, kw, e, planes, size, crop, seed=0, what=""):
    ow, oh = size
    pics = [Picture(fmt, ow, oh, seed + 17 * i) for i in range(len(streams))]
    before = [p.host() for p in pics]
    run(r, streams, fmt, pics, k, kw, planes, size, crop)
    want = expect(r, streams, pics, before, k, e, size, crop)
    for i, p in enumerate(pics):
        same(p.host(), want[i], (what, fmt, e, None if k is None else k[i], size, crop, i))


# rectangles of a 98 x 62 frame: crops touching each edge, odd and non-multiple-of-4 widths, 1- and 2-pixel outputs,
# extreme ratios
RECTS = [((48, 30), None), ((33, 21), (0, 0, 70, 50)), ((30, 14), (28, 12, 70, 50)), ((2, 2), (96, 60, 2, 2)),
         ((1, 1), None), ((98, 1), None), ((1, 62), (97, 0, 1, 62)), ((6, 4), (40, 30, 58, 32))]


@pytest.mark.parametrize("native", [True, False], ids=["native", "blended"])
@pytest.mark.parametrize("module", g.MODULES)
def test_every_module_format_encoding_and_opacity(built, module, native):
    kw0 = {} if native else dict(premultiply_alpha=0, clear_color=[0.1, 0.2, 0.3, 1.0])
    streams = [0, 1, 2, 0, 1, 2]
    p = g.default_params(module, n=1024, w=98, h=62, **kw0)
    with g.Renderer(p, batch=3) as r:
        feed(r, 3, seed=7)
        for j, (size, crop) in enumerate(RECTS):
            for fmt, planes in formats(*size):
                for kw, e in (ENCS if fmt not in (RGBA, BGRA) else ENCS[:1]):
                    if (j + e) % 2 and j > 1:                 # each rectangle meets every format, half of the encodings
                        continue
                    check(r, streams, fmt, K_LIST, kw, e, planes, size, crop, seed=j + e, what=module)   # mixed list
                    k = [K_LIST[(j + e + fmt) % 6]] * 3
                    check(r, streams[:3], fmt, k, kw, e, planes, size, crop, seed=j + 5, what=module)    # one K for all
            check(r, [2, 1], RGBA, None, {}, 0, False, size, crop, seed=j, what=module)                 # no opacity


# ---- identities ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("native", [True, False], ids=["native", "blended"])
def test_whole_frame_at_its_own_size_is_the_opacity_overlay(built, native):
    kw0 = {} if native else dict(premultiply_alpha=0)
    p = g.default_params("bars", n=1024, w=160, h=90, **kw0)
    with g.Renderer(p, batch=3) as r:
        feed(r, 3)
        for fmt, planes in formats(160, 90):
            for kw, e in (ENCS if fmt not in (RGBA, BGRA) else ENCS[:1]):
                for k, crop in ((None, None), ([255, 0, 128], (0, 0, 160, 90))):
                    a = [Picture(fmt, 160, 90, 9 + i) for i in range(3)]
                    b = [Picture(fmt, 160, 90, 9 + i) for i in range(3)]
                    run(r, [2, 0, 1], fmt, a, k, kw, planes, (160, 90), crop)
                    op = None if k is None else [v / 255.0 for v in k]
                    if planes:
                        r.overlay_planes([2, 0, 1], [x.planes_arg() for x in b], None, NAME[fmt], opacity=op, **kw)
                    else:
                        r.overlay_frames([2, 0, 1], [frames_arg(x) for x in b], None, FNAME[fmt], opacity=op, **kw)
                    torch.cuda.synchronize()
                    for x, y in zip(a, b):
                        same(x.host(), y.host(), (fmt, e, k, "whole frame"))


def bytes_of(t):
    """the bytes of one picture's planes (a tensor or a tuple of plane tensors), row by row, plane after plane"""
    planes = t if isinstance(t, (tuple, list)) else (t,)
    return np.concatenate([x.contiguous().view(torch.uint8).cpu().numpy().reshape(-1) for x in planes])


def test_any_other_opacity_at_full_strength_is_the_scaled_export(built):
    """identity 2 for every format and encoding: any other opacity at K = 255 leaves export_scaled's bytes of the format and
    encoding in the rectangle (RGBA / BGRA: EXPORT_OVER)"""
    p = g.default_params("radial", n=1024, w=160, h=90, premultiply_alpha=0)
    with g.Renderer(p, batch=2) as r:
        feed(r, 3)
        size, crop = (62, 40), (10, 6, 130, 80)
        for fmt, planes in formats(*size):
            name = FNAME[fmt] if not planes else NAME[fmt]
            for kw, e in (ENCS if fmt not in (RGBA, BGRA) else ENCS[:1]):
                pics = [Picture(fmt, *size, 3 + i) for i in range(2)]
                run(r, [1, 0], fmt, pics, [255, 255], kw, planes, size, crop)
                ex = r.export_scaled([1, 0], size, crop, fmt=name, over=fmt in (RGBA, BGRA), **kw)
                torch.cuda.synchronize()
                for i, pic in enumerate(pics):
                    want = bytes_of(tuple(x[i] for x in ex) if isinstance(ex, tuple) else ex[i])
                    assert np.array_equal(bytes_of(tuple(pic.views)), want), (fmt, e, i)


def test_zero_frame_and_zero_opacity_leave_the_picture(built):
    p = g.default_params("bars", n=1024, w=128, h=64)
    with g.Renderer(p, batch=2) as r:
        # the framebuffer is allocated zero-filled: before the first raster pass every frame is zero
        assert not any(r.readback(s).any() for s in (0, 1))
        for fmt, planes in formats(40, 20):
            pics = [Picture(fmt, 40, 20, i) for i in range(2)]
            before = [x.host() for x in pics]
            run(r, [0, 1], fmt, pics, [255, 128], {}, planes, (40, 20), (8, 4, 100, 50))
            for x, y in zip(pics, before):
                same(x.host(), y, (fmt, "zero frame"))
        feed(r, 3)
        assert r.readback(0).any()
        for fmt, planes in formats(40, 20):
            pics = [Picture(fmt, 40, 20, i) for i in range(2)]
            before = [x.host() for x in pics]
            run(r, [0, 1], fmt, pics, [0, 0], {}, planes, (40, 20), (8, 4, 100, 50))
            for x, y in zip(pics, before):
                same(x.host(), y, (fmt, "K = 0"))


# ---- picture-in-picture, marks, ring, styles ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("full_store", ["0", "1"], ids=["live", "stale"])
def test_bars_1080p_picture_in_picture_under_marks(built, full_store, monkeypatch):
    """1920 x 1080 -> 640 x 360 at an offset inside a 1080p picture, under the marks the last pass kept (GLAVA_B200_FULL_STORE:
    the pass stores every row and the marks still describe the frame); every byte outside the rectangle untouched"""
    monkeypatch.setenv("GLAVA_B200_FULL_STORE", full_store)
    p = g.default_params("bars", n=1024, w=1920, h=1080)
    W, H, (x, y), size = 1920, 1080, (1248, 688), (640, 360)
    rng = np.random.default_rng(3)
    with g.Renderer(p, batch=2) as r:
        feed(r, 2)
        for fmt, k in ((RGBA, 255), (NV12, 128), (BGRA, 37)):
            host0 = rng.integers(0, 256, (H, W, 4) if fmt != NV12 else (H * 3 // 2, W), dtype=np.uint8)
            img = torch.from_numpy(host0).cuda()
            r.overlay_frames([1], [img], [(x, y)], FNAME[fmt], opacity=[k / 255.0], size=size)
            torch.cuda.synchronize()
            want = host0.copy()
            if fmt == NV12:
                rect = [want[y:y + 360, x:x + 640], want[H + y // 2:H + (y + 360) // 2, x:x + 640]]
            else:
                rect = [want[y:y + 360, x:x + 640].reshape(360, 640 * 4)]
            for dst, new in zip(rect, restated(scaled_frame(r, 1, size, None), [v.copy() for v in rect], fmt, 0, k, True)):
                dst[...] = new.reshape(dst.shape)
            assert np.array_equal(img.cpu().numpy(), want), fmt
        for fmt in (I420, YUV422P10):
            check(r, [1, 0], fmt, [128, 255], {}, 0, True, size, None, what="1080p")
            check(r, [0, 1], fmt, [37, 254], {}, 0, True, (480, 270), (320, 180, 1280, 720), what="1080p crop")


@pytest.mark.parametrize("slots", [1, 3])
def test_framebuffer_ring_and_styles(built, slots):
    p = g.default_params("graph", n=1024, w=128, h=64, fb_slots=slots)
    with g.Renderer(p, batch=5) as r:
        r.set_stream_styles([1, 4], [{"amplify": 500, "fg": "#ff8000"}, {"fg": (0.1, 0.9, 0.2, 1.0), "bg": (0.3, 0.3, 0.3, 0.5)}])
        feed(r, 3)
        for fmt, planes in formats(50, 24):
            check(r, [4, 0, 4, 1, 3], fmt, [1, 254, 0, 128, 200], {}, 0, planes, (50, 24), (3, 5, 120, 55), what=("ring", slots))


def test_a_list_of_1024_entries(built):
    """1024 16 x 8 thumbnails of 64 x 32 frames in one RGBA picture and one NV12 picture, each at its own opacity"""
    tw, th = 16, 8
    p = g.default_params("bars", n=1024, w=64, h=32)
    rng = np.random.default_rng(5)
    with g.Renderer(p, batch=64) as r:
        feed(r, 3)
        streams = [int(s) for s in rng.integers(0, 64, 1024)]
        k = [int(v) for v in rng.integers(0, 256, 1024)]
        at = [((i % 32) * tw, (i // 32) * th) for i in range(1024)]
        S = {s: scaled_frame(r, s, (tw, th), None) for s in set(streams)}
        for fmt in (RGBA, NV12):
            W, H = 32 * tw, 32 * th
            host0 = rng.integers(0, 256, (H, W, 4) if fmt == RGBA else (H * 3 // 2, W), dtype=np.uint8)
            img = torch.from_numpy(host0).cuda()
            r.overlay_frames(streams, [img] * 1024, at, FNAME[fmt], opacity=[v / 255.0 for v in k], size=(tw, th))
            torch.cuda.synchronize()
            want = host0.copy()
            for i, s in enumerate(streams):
                x, y = at[i]
                if fmt == RGBA:
                    rect = [want[y:y + th, x:x + tw]]
                    src = [rect[0].reshape(th, tw * 4).copy()]
                else:
                    rect = [want[y:y + th, x:x + tw], want[H + y // 2:H + (y + th) // 2, x:x + tw]]
                    src = [v.copy() for v in rect]
                for dst, new in zip(rect, restated(S[s], src, fmt, 0, k[i], True)):
                    dst[...] = new.reshape(dst.shape)
            assert np.array_equal(img.cpu().numpy(), want), fmt


# ---- ordering, refusals, sharding ------------------------------------------------------------------------------------------------
def test_after_and_done_events_order_a_side_stream(built):
    p = g.default_params("bars", n=1024, w=128, h=64)
    with g.Renderer(p, batch=2) as r:
        feed(r, 2)
        for opacity in ([1.0], [0.5], [0.0]):
            side = torch.cuda.Stream()
            with torch.cuda.stream(side):
                pic = (torch.zeros((32, 64), dtype=torch.uint8, device="cuda"),
                       torch.zeros((16, 32), dtype=torch.uint8, device="cuda"), torch.zeros((16, 32), dtype=torch.uint8, device="cuda"))
                pic[0].fill_(40)
                after, done = torch.cuda.Event(), torch.cuda.Event()
                after.record(side)
            r.overlay_planes([1], [pic], None, "i420", after=after, done=done, opacity=opacity, size=(64, 32))
            side.wait_event(done)
            side.synchronize()
            before = [np.full((32, 64), 40, np.uint8), np.zeros((16, 32), np.uint8), np.zeros((16, 32), np.uint8)]
            want = restated(scaled_frame(r, 1, (64, 32), None), before, I420, 0, int(opacity[0] * 255 + 0.5), True)
            for t, x in zip(pic, want):
                assert np.array_equal(t.cpu().numpy(), x), opacity


def test_python_and_library_refusals(built):
    p = g.default_params("bars", n=1024, w=64, h=32)
    with g.Renderer(p, batch=2) as r:
        feed(r, 1)
        img = torch.zeros((16, 32, 4), dtype=torch.uint8, device="cuda")
        with pytest.raises(ValueError, match="leaves"):
            r.overlay_frames([0], [img], None, "rgba", size=(40, 16))
        with pytest.raises(g.GlavaError, match="overlay_scaled.*upscaling"):
            r.overlay_frames([0], [img], None, "rgba", size=(32, 16), crop=(0, 0, 16, 16))
        with pytest.raises(g.GlavaError, match="overlay_scaled.*leaves"):
            r.overlay_frames([0], [img], None, "rgba", size=(32, 16), crop=(40, 0, 32, 16))
        with pytest.raises(g.GlavaError, match="overlay_scaled.*overlaps"):
            r.overlay_frames([0, 1], [img, img], None, "rgba", size=(32, 16), opacity=[0.0, 0.0])
        nv = torch.zeros((24, 32), dtype=torch.uint8, device="cuda")
        with pytest.raises(g.GlavaError, match="overlay_scaled.*even"):
            r.overlay_frames([0], [nv[:, :31]], None, "nv12", size=(31, 16))


def test_sharded_equals_one_handle(built):
    p = g.default_params("graph", n=1024, w=96, h=48)
    size, crop = (42, 20), (6, 4, 88, 42)
    with g.ShardedRenderer(p, 6, [0, 0, 0]) as sh, g.Renderer(p, batch=6) as one:
        rng = np.random.default_rng(1)
        for _ in range(3):
            lb = (rng.standard_normal((6, 1024)) * 0.3).astype(np.float32)
            rb = (rng.standard_normal((6, 1024)) * 0.3).astype(np.float32)
            sh.update(lb, rb); one.update(lb, rb, True)
        for op in ([0.5, 0.0, 1.0, 0.2], None):
            for fmt, planes in formats(*size):
                a = [Picture(fmt, *size, 4 + i) for i in range(4)]
                b = [Picture(fmt, *size, 4 + i) for i in range(4)]
                if planes:
                    sh.overlay_planes([5, 0, 3, 5], [x.planes_arg() for x in a], None, NAME[fmt], matrix="bt601", opacity=op,
                                      size=size, crop=crop)
                    one.overlay_planes([5, 0, 3, 5], [x.planes_arg() for x in b], None, NAME[fmt], matrix="bt601", opacity=op,
                                       size=size, crop=crop)
                else:
                    sh.overlay_frames([5, 0, 3, 5], [frames_arg(x) for x in a], None, FNAME[fmt], opacity=op, size=size, crop=crop)
                    one.overlay_frames([5, 0, 3, 5], [frames_arg(x) for x in b], None, FNAME[fmt], opacity=op, size=size, crop=crop)
                sh.sync()
                torch.cuda.synchronize()
                for x, y in zip(a, b):
                    same(x.host(), y.host(), ("sharded", fmt, op))
