"""-m gpu: the 4:2:2 export, YUV422P, YUV422P10 and UYVY (DESIGN 4.18).  Whole frames against the numpy restatement of
tests/export_422_np.py applied to glava_b200_readback of the same stream at the same point, for every module, encoding and
opacity, odd heights and widths of 4k + 2 included; the identities on the device (UYVY is YUV422P interleaved, and the
Y planes are I420's and YUV420P10's); scaled output as the format's arithmetic on the 8-bit scaled image and the whole
frame at its own size equal to export_frames; mixed ladders equal to their standalone calls; live, stale and absent marks,
the framebuffer ring, styles, 1024 streams; mosaics with sentinels; events, the sharded handle, the Python shapes and
dtypes, and the planes read as an ffmpeg-style consumer reads yuv422p10le."""
import ctypes

import numpy as np
import pytest

import glava_b200 as g
from tests.export_422_np import FORMATS, export422_np, planar_of
from tests.test_export_core import RGBA, over_np
from tests.test_export_scaled_core import scaled_np

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

BG = (30, 60, 200)
ENCS = [(dict(), 0), (dict(full_range=True), 1), (dict(matrix="bt601"), 2), (dict(matrix="bt601", full_range=True), 3)]


def host(t):
    return tuple(x.cpu().numpy() for x in t) if isinstance(t, tuple) else t.cpu().numpy()


def entry(got, i):
    return tuple(x[i] for x in got) if isinstance(got, tuple) else got[i]


def same(a, b):
    if isinstance(b, tuple):
        return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))
    return np.array_equal(a, b)


def feed(r, steps, seed=0, scale=0.3):
    rng = np.random.default_rng(seed)
    n = r.params.n
    for _ in range(steps):
        lb = (rng.standard_normal((r.batch, n)) * scale).astype(np.float32)
        rb = (rng.standard_normal((r.batch, n)) * scale).astype(np.float32)
        r.update(lb, rb, True)


def frame_np(frame, fmt, e, bg, native):
    return export422_np(over_np(frame[::-1], bg, native), fmt, e)


def check(r, streams, fmt, kw, e, bg=BG, what=""):
    got = host(r.export_frames(streams, fmt, background=bg, **kw))
    native = bool(r.params.premultiply_alpha)
    for i, s in enumerate(streams):
        assert same(entry(got, i), frame_np(r.readback(int(s)), fmt, e, bg, native)), (what, fmt, kw, i, int(s))


def check_identities(r, streams, kw, bg=BG):
    """on the device, same streams and call order: UYVY is YUV422P interleaved; YUV422P's Y is I420's Y and YUV422P10's
    Y is YUV420P10's Y (h even here); every YUV422P10 sample is LSB-aligned"""
    p = r.export_frames(streams, "yuv422p", background=bg, **kw)
    u = r.export_frames(streams, "uyvy", background=bg, **kw)
    assert torch.equal(u[..., 1::2], p[0]) and torch.equal(u[..., 0::4], p[1]) and torch.equal(u[..., 2::4], p[2]), kw
    if r.params.h % 2 == 0:
        assert torch.equal(p[0], r.export_frames(streams, "i420", background=bg, **kw)[0]), kw
        p10 = r.export_frames(streams, "yuv422p10", background=bg, **kw)
        assert torch.equal(p10[0].view(torch.int16), r.export_frames(streams, "yuv420p10", background=bg, **kw)[0].view(torch.int16))
        for t in p10:
            assert int(t.view(torch.int16).min()) >= 0 and int(t.view(torch.int16).max()) <= 1023


# ---- whole frames --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("native", [True, False], ids=["native", "blended"])
@pytest.mark.parametrize("module", g.MODULES)
def test_every_module_encoding_and_opacity(built, module, native):
    kw0 = {} if native else dict(premultiply_alpha=0, clear_color=[0.1, 0.2, 0.3, 1.0])
    for w, h in ((96, 64), (98, 63), (130, 5), (6, 3)):
        p = g.default_params(module, n=1024, w=w, h=h, **kw0)
        with g.Renderer(p, batch=3) as r:
            feed(r, 3, seed=w + h)
            for kw, e in ENCS:
                for fmt in FORMATS:
                    check(r, [0, 2, 1], fmt, kw, e, what=(module, w, h))
                check_identities(r, [2, 0], kw)


def test_bars_1080p_live_stale_and_absent_marks(built):
    p = g.default_params("bars", n=4096, w=1920, h=1080)
    p.lazy_smooth = 1
    with g.Renderer(p, batch=3) as r:
        for step in range(3):                                          # marks valid from the second pass on
            feed(r, 1, seed=step, scale=0.1 + 0.3 * step)
            for fmt in FORMATS:
                check(r, [2, 0], fmt, {}, 0, what=step)
        check(r, [1], "yuv422p10", dict(matrix="bt601", full_range=True), 3)
        check_identities(r, [0, 1, 2], {})
        q = r.params.copy(); q.bars_mirror_yx = 1                      # the generic kernel keeps no marks
        r.reconfigure(q)
        feed(r, 1, seed=9)
        for fmt in FORMATS:
            check(r, [1], fmt, {}, 0, what="no marks")


@pytest.mark.parametrize("slots", [1, 3])
def test_framebuffer_ring_styles_and_repeats(built, slots):
    p = g.default_params("graph", n=1024, w=128, h=63, fb_slots=slots)
    with g.Renderer(p, batch=5) as r:
        r.set_stream_styles([1, 4], [{"amplify": 500, "fg": "#ff8000"}, {"fg": (0.1, 0.9, 0.2, 1.0), "bg": (0.3, 0.3, 0.3, 0.5)}])
        feed(r, 3)
        for kw, e in ENCS:
            for fmt in FORMATS:
                check(r, [4, 0, 4, 1, 3], fmt, kw, e, bg=(255, 255, 255))


def test_a_thousand_streams_in_one_launch(built):
    p = g.default_params("bars", n=512, w=64, h=33)
    with g.Renderer(p, batch=1024) as r:
        feed(r, 2)
        for kw, e in ENCS[::3]:
            for fmt in FORMATS:
                l0 = r.launch_count
                got = host(r.export_frames(range(1024), fmt, **kw))
                assert r.launch_count == l0 + 1
                for s in list(range(0, 1024, 37)) + [1023]:
                    assert same(entry(got, s), frame_np(r.readback(s), fmt, e, (0, 0, 0), True)), (fmt, kw, s)


# ---- scaled, ladder, mosaic ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("native", [True, False], ids=["native", "blended"])
@pytest.mark.parametrize("module", ["bars", "radial", "wave"])
def test_scaled_is_the_format_on_the_scaled_image(built, module, native):
    kw0 = {} if native else dict(premultiply_alpha=0, clear_color=[0.1, 0.2, 0.3, 1.0])
    p = g.default_params(module, n=1024, w=300, h=170, **kw0)
    with g.Renderer(p, batch=3) as r:
        feed(r, 3, seed=5)
        for kw, e in ENCS:
            for size, crop in (((100, 56), None), ((64, 31), (10, 20, 200, 100)), ((38, 19), None), ((2, 1), None), ((34, 7), None)):
                for fmt in FORMATS:
                    got = host(r.export_scaled([2, 0], size, crop, fmt, background=BG, **kw))
                    for i, s in enumerate([2, 0]):
                        img = scaled_np(r.readback(s), RGBA, True, BG, native, size, crop)   # the 8-bit scaled image
                        assert same(entry(got, i), export422_np(img, fmt, e)), (fmt, kw, size, crop, s)
            for fmt in FORMATS:                                        # the whole frame at its own size is export_frames
                assert same(host(r.export_scaled([0, 1], (300, 170), None, fmt, **kw)),
                            host(r.export_frames([0, 1], fmt, **kw))), (fmt, kw)


def ladder_vs_standalone(r, streams, rungs):
    l0 = r.launch_count
    got = r.export_ladder(streams, rungs)
    assert r.launch_count == l0 + 1
    for j, rung in enumerate(rungs):
        kw = {k: v for k, v in rung.items() if k in ("over", "background", "matrix", "full_range")}
        want = (r.export_frames(streams, rung["fmt"], **kw) if rung.get("size") is None
                else r.export_scaled(streams, rung["size"], rung.get("crop"), rung["fmt"], **kw))
        assert same(host(got[j]), host(want)), (j, rung)


def test_mixed_ladders_equal_their_standalone_calls(built):
    p = g.default_params("bars", n=4096, w=1920, h=1080)
    p.lazy_smooth = 1
    rungs = [dict(size=None, fmt="yuv422p10"), dict(size=(1280, 720), fmt="nv12", matrix="bt601"),
             dict(size=(640, 360), fmt="yuv420p10", full_range=True), dict(size=(96, 54), fmt="rgba", over=True),
             dict(size=(480, 270), fmt="uyvy", matrix="bt601", full_range=True), dict(size=None, fmt="yuv422p", background=BG),
             dict(size=(640, 361), fmt="yuv422p10", full_range=True), dict(size=None, fmt="uyvy")]
    with g.Renderer(p, batch=3) as r:
        for step in range(2):
            feed(r, 1, seed=step, scale=0.2 + 0.3 * step)
            ladder_vs_standalone(r, [2, 0], rungs)
        ladder_vs_standalone(r, [1], rungs[:4])
    p = g.default_params("radial", n=1024, w=98, h=61)                # no marks, w % 4 == 2, odd h
    with g.Renderer(p, batch=2) as r:
        feed(r, 2)
        ladder_vs_standalone(r, [1, 0, 1], [dict(size=None, fmt="yuv422p", matrix="bt601"), dict(size=(48, 30), fmt="nv12"),
                                            dict(size=(34, 17), crop=(5, 5, 80, 40), fmt="yuv422p10", full_range=True),
                                            dict(size=None, fmt="uyvy"), dict(size=(40, 21), fmt="yuv444p10")])


@pytest.mark.parametrize("fmt,tile", [("yuv422p", (64, 27)), ("yuv422p10", (48, 28)), ("uyvy", (40, 27))])
@pytest.mark.parametrize("kw", [dict(), dict(matrix="bt601", full_range=True)], ids=["bt709", "jfif"])
def test_mosaics_with_sentinels(built, fmt, tile, kw):
    p = g.default_params("bars", n=1024, w=200, h=120)
    with g.Renderer(p, batch=7) as r:
        feed(r, 2, seed=3)
        streams, cols = [6, 1, 0, 3, 5], 3
        tw, th = tile
        W, H = cols * tw, 2 * th
        rows, row_bytes, align = g.api._export_layout(fmt, W, H)
        pitch = (row_bytes + 64 + align - 1) // align * align
        out = torch.full((rows, pitch), 0xA5, dtype=torch.uint8, device="cuda")
        r.export_mosaic(streams, cols, tile, fmt, background=BG, out=out, **kw)
        base = out.cpu().numpy()
        views = host(g.api._export_views(fmt, out, W, H))
        written = np.zeros(base.size, bool)
        P, sb = pitch, 2 if fmt == "yuv422p10" else 1
        for i, s in enumerate(streams):
            ty, tx = i // cols, i % cols
            want = entry(host(r.export_scaled([s], tile, None, fmt, background=BG, **kw)), 0)
            if fmt == "uyvy":
                assert np.array_equal(views[ty * th:(ty + 1) * th, 2 * tx * tw:2 * (tx + 1) * tw], want), i
                for rr in range(th):
                    o = (ty * th + rr) * P + tx * tw * 2
                    written[o:o + tw * 2] = True
                continue
            cw = tw // 2
            assert np.array_equal(views[0][ty * th:(ty + 1) * th, tx * tw:(tx + 1) * tw], want[0]), i
            assert np.array_equal(views[1][ty * th:(ty + 1) * th, tx * cw:(tx + 1) * cw], want[1]), i
            assert np.array_equal(views[2][ty * th:(ty + 1) * th, tx * cw:(tx + 1) * cw], want[2]), i
            for rr in range(th):
                o = (ty * th + rr) * P + tx * tw * sb
                written[o:o + tw * sb] = True
            for k in range(2):
                for rr in range(th):
                    o = P * H + k * (P // 2) * H + (ty * th + rr) * (P // 2) + tx * cw * sb
                    written[o:o + cw * sb] = True
        assert (base.reshape(-1)[~written] == 0xA5).all(), fmt
        # without out=, the empty tile is black in the encoding: Y 16 / 64 (0 in full range), chroma 128 / 512
        m = host(r.export_mosaic(streams, cols, tile, fmt, background=BG, **kw))
        ty, tx = 1, 2
        y0, c0 = (0 if kw else 64, 512) if fmt == "yuv422p10" else (0 if kw else 16, 128)
        if fmt == "uyvy":
            m = planar_of(m)
        cw = tw // 2
        assert (m[0][ty * th:(ty + 1) * th, tx * tw:(tx + 1) * tw] == y0).all()
        assert (m[1][ty * th:(ty + 1) * th, tx * cw:(tx + 1) * cw] == c0).all()
        assert (m[2][ty * th:(ty + 1) * th, tx * cw:(tx + 1) * cw] == c0).all()


# ---- consumer layout, events, the sharded handle, Python shapes -------------------------------------------------------------
def test_an_ffmpeg_style_consumer_reads_yuv422p10le_and_uyvy422(built):
    """the three uint16 planes of one yuv422p10 export, read from the raw bytes with linesizes (pitch, pitch / 2, pitch / 2)
    and plane offsets (0, pitch h, pitch h + pitch / 2 h) as AVFrame data[] / linesize[] describe yuv422p10le; and a UYVY
    export read with one linesize, the pitch"""
    p = g.default_params("radial", n=1024, w=160, h=91)
    with g.Renderer(p, batch=2) as r:
        feed(r, 2)
        pitch = 384                                                    # padded rows: a multiple of 32, above 2 w
        out = torch.full((1, 91 * 2, pitch), 0x5A, dtype=torch.uint8, device="cuda")
        r.export_frames([1], "yuv422p10", out=out)
        raw = out.cpu().numpy().reshape(-1)
        data = [0, pitch * 91, pitch * 91 + (pitch // 2) * 91]
        linesize = [pitch, pitch // 2, pitch // 2]
        dims = [(91, 160), (91, 80), (91, 80)]
        got = []
        for d, ls, (hh, ww) in zip(data, linesize, dims):
            rows = [raw[d + k * ls:d + k * ls + 2 * ww].view("<u2") for k in range(hh)]
            got.append(np.stack(rows))
        assert same(tuple(got), frame_np(r.readback(1), "yuv422p10", 0, (0, 0, 0), True))
        assert all(int(x.max()) < 1024 for x in got)                   # the top 6 bits are zero
        out = torch.full((1, 91, 336), 0x5A, dtype=torch.uint8, device="cuda")
        r.export_frames([0], "uyvy", out=out)
        raw = out.cpu().numpy().reshape(-1)
        u = np.stack([raw[k * 336:k * 336 + 320] for k in range(91)])
        assert np.array_equal(u, frame_np(r.readback(0), "uyvy", 0, (0, 0, 0), True))
        assert (raw.reshape(91, 336)[:, 320:] == 0x5A).all()


def test_events_sharded_and_python_shapes(built):
    p = g.default_params("graph", n=1024, w=128, h=64)
    rng = np.random.default_rng(4)
    lb = (rng.standard_normal((6, 1024)) * 0.3).astype(np.float32); rb = lb[::-1].copy()
    with g.ShardedRenderer(p, 6, [0, 0, 0]) as sh, g.Renderer(p, batch=6) as one:
        for _ in range(2):
            sh.update(lb, rb); one.update(lb, rb, True)
        order = [5, 0, 3, 3, 1]
        for fmt in FORMATS:
            for kw, e in (ENCS[0], ENCS[3]):
                a = sh.export_frames(order, fmt, background=BG, **kw)
                b = sh.export_scaled(order, (64, 31), None, fmt, **kw)
                c = sh.export_ladder(order, [dict(size=None, fmt=fmt, **kw), dict(size=(32, 16), fmt=fmt), dict(size=(32, 16), fmt="p010")])
                sh.sync()
                assert same(host(a), host(one.export_frames(order, fmt, background=BG, **kw))), (fmt, kw)
                assert same(host(b), host(one.export_scaled(order, (64, 31), None, fmt, **kw))), (fmt, kw)
                assert same(host(c[0]), host(one.export_frames(order, fmt, **kw))), (fmt, kw)
                assert same(host(c[1]), host(one.export_scaled(order, (32, 16), None, fmt))), (fmt, kw)
                assert same(host(c[2]), host(one.export_scaled(order, (32, 16), None, "p010"))), (fmt, kw)
        with pytest.raises(g.GlavaError, match="YUV422P pitch"):
            sh.export_frames([0], "yuv422p", out=torch.zeros((1, 128, 144), dtype=torch.uint8, device="cuda"))   # 144: not 32k
        # shapes, dtypes and pitches
        y, cb, cr = one.export_frames([0, 2], "yuv422p10")
        assert all(t.dtype == torch.uint16 for t in (y, cb, cr))
        assert y.shape == (2, 64, 128) and cb.shape == cr.shape == (2, 64, 64) and y.stride(1) == 128 and cb.stride(1) == 64
        assert cb.data_ptr() == y.data_ptr() + 256 * 64 and cr.data_ptr() == cb.data_ptr() + 128 * 64
        y8, cb8, cr8 = one.export_frames([1], "yuv422p")
        assert y8.dtype == torch.uint8 and y8.shape == (1, 64, 128) and cb8.shape == cr8.shape == (1, 64, 64)
        uy = one.export_frames([1, 2], "uyvy")
        assert uy.dtype == torch.uint8 and uy.shape == (2, 64, 256)
        out16 = torch.zeros((2, 128, 160), dtype=torch.uint16, device="cuda")    # pitch 320 bytes, planes back to back
        got = one.export_frames([1, 4], "yuv422p10", out=out16)
        assert got is out16
        views = host(g.api._export_views("yuv422p10", out16.view(torch.uint8), 128, 64))
        assert same(views, host(one.export_frames([1, 4], "yuv422p10")))
        side = torch.cuda.Stream()
        after, done = torch.cuda.Event(), torch.cuda.Event()
        base = torch.empty((1, 64, 256), dtype=torch.uint8, device="cuda")
        with torch.cuda.stream(side):
            torch.cuda._sleep(20_000_000)
            base.fill_(0x5A)
            after.record(side)
        frame = one.readback(3)
        one.export_frames([3], "uyvy", out=base, after=after, done=done)
        one.update(lb, rb, True)
        with torch.cuda.stream(side):
            side.wait_event(done)
            seen = base.clone()
        side.synchronize()
        assert same(host(seen[0]), frame_np(frame, "uyvy", 0, (0, 0, 0), True))
        for fmt in FORMATS:
            with pytest.raises(ValueError, match="overlay"):
                one.overlay_frames([0], torch.zeros((96, 128), dtype=torch.uint8, device="cuda"), fmt=fmt)
        n = ctypes.c_size_t()
        for fmt, want in (("yuv422p", 256 * 64 + 2 * 128 * 64), ("yuv422p10", 256 * 64 + 2 * 128 * 64), ("uyvy", 256 * 64)):
            d = g.api._export_desc(fmt, False, (0, 0, 0))
            d.pitch = 256
            assert one._L.glava_b200_export_bytes(one._h, ctypes.byref(d), ctypes.byref(n)) == 0 and n.value == want, fmt
