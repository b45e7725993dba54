"""-m gpu: I420, YUV 4:4:4 and P010 export (DESIGN 4.14).  Whole frames against the numpy restatement of
tests/test_export_formats_core.py applied to glava_b200_readback of the same stream at the same point; the identities with
NV12 (I420 = deinterleaved NV12, YUV444 Y = NV12 Y) on the device; scaled output as the format's arithmetic on the 8-bit
scaled image and the whole frame at its own size equal to export_frames; mixed-format ladders equal to their standalone
calls; live, stale and absent marks, the framebuffer ring, styles, 1024 streams; planar and P010 mosaics with sentinels;
events, the sharded handle and the Python shapes."""
import numpy as np
import pytest

import glava_b200 as g
from tests.test_export_formats_core import frame_np, yuv_np
from tests.test_export_scaled_core import scaled_np
from tests.test_export_core import RGBA

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

BG = (30, 60, 200)
NEW = ("i420", "yuv444", "p010")


def host(t):
    return tuple(x.cpu().numpy() for x in t) if isinstance(t, tuple) else t.cpu().numpy()


def entry(got, i):
    return tuple(x[i] for x in got) if isinstance(got, tuple) else got[i]


def same(a, b):
    if isinstance(b, tuple):
        return all(np.array_equal(x, y) for x, y in zip(a, b))
    return np.array_equal(a, b)


def feed(r, steps, seed=0, scale=0.3):
    rng = np.random.default_rng(seed)
    n = r.params.n
    for _ in range(steps):
        lb = (rng.standard_normal((r.batch, n)) * scale).astype(np.float32)
        rb = (rng.standard_normal((r.batch, n)) * scale).astype(np.float32)
        r.update(lb, rb, True)


def check(r, streams, fmt, bg=BG, what=""):
    got = host(r.export_frames(streams, fmt, background=bg))
    native = bool(r.params.premultiply_alpha)
    for i, s in enumerate(streams):
        assert same(entry(got, i), frame_np(r.readback(int(s)), fmt, bg, native)), (what, fmt, i, int(s))


def check_identities(r, streams, bg=BG):
    h = r.params.h
    nv12 = r.export_frames(streams, "nv12", background=bg)
    y, cb, cr = r.export_frames(streams, "i420", background=bg)
    assert torch.equal(y, nv12[:, :h]) and torch.equal(cb, nv12[:, h:, 0::2]) and torch.equal(cr, nv12[:, h:, 1::2])
    assert torch.equal(r.export_frames(streams, "yuv444", background=bg)[0], nv12[:, :h])


@pytest.mark.parametrize("native", [True, False], ids=["native", "blended"])
@pytest.mark.parametrize("module", g.MODULES)
def test_every_module_format_and_opacity(built, module, native):
    kw = {} if native else dict(premultiply_alpha=0, clear_color=[0.1, 0.2, 0.3, 1.0])
    for w, h, fmts in ((96, 64, NEW), (98, 62, NEW), (97, 63, ("yuv444",))):
        p = g.default_params(module, n=1024, w=w, h=h, **kw)
        with g.Renderer(p, batch=3) as r:
            feed(r, 3, seed=w)
            for fmt in fmts:
                check(r, [0, 2, 1], fmt, what=(module, w, h))
            if fmts == NEW:
                check_identities(r, [2, 0])


def test_bars_1080p_live_stale_and_absent_marks(built):
    p = g.default_params("bars", n=4096, w=1920, h=1080)
    p.lazy_smooth = 1
    with g.Renderer(p, batch=3) as r:
        for step in range(3):                                          # marks valid from the second pass on
            feed(r, 1, seed=step, scale=0.1 + 0.3 * step)
            for fmt in NEW:
                check(r, [2, 0], fmt, what=step)
        check_identities(r, [0, 1, 2])
        q = r.params.copy(); q.bars_mirror_yx = 1                      # the generic kernel keeps no marks
        r.reconfigure(q)
        feed(r, 1, seed=9)
        for fmt in NEW:
            check(r, [1], fmt, what="no marks")


@pytest.mark.parametrize("slots", [1, 3])
def test_framebuffer_ring_styles_and_repeats(built, slots):
    p = g.default_params("graph", n=1024, w=128, h=64, fb_slots=slots)
    with g.Renderer(p, batch=5) as r:
        r.set_stream_styles([1, 4], [{"amplify": 500, "fg": "#ff8000"}, {"fg": (0.1, 0.9, 0.2, 1.0), "bg": (0.3, 0.3, 0.3, 0.5)}])
        feed(r, 3)
        for fmt in NEW:
            check(r, [4, 0, 4, 1, 3], fmt, bg=(255, 255, 255))


def test_a_thousand_streams_in_one_launch(built):
    p = g.default_params("bars", n=512, w=64, h=32)
    with g.Renderer(p, batch=1024) as r:
        feed(r, 2)
        for fmt in NEW:
            l0 = r.launch_count
            got = host(r.export_frames(range(1024), fmt))
            assert r.launch_count == l0 + 1
            for s in list(range(0, 1024, 37)) + [1023]:
                assert same(entry(got, s), frame_np(r.readback(s), fmt, (0, 0, 0), True)), (fmt, s)


@pytest.mark.parametrize("native", [True, False], ids=["native", "blended"])
@pytest.mark.parametrize("module", ["bars", "radial", "wave"])
def test_scaled_is_the_format_on_the_scaled_image(built, module, native):
    kw = {} if native else dict(premultiply_alpha=0, clear_color=[0.1, 0.2, 0.3, 1.0])
    p = g.default_params(module, n=1024, w=300, h=170, **kw)
    with g.Renderer(p, batch=3) as r:
        feed(r, 3, seed=5)
        for size, crop in (((100, 56), None), ((64, 30), (10, 20, 200, 100)), ((300, 170), None), ((37, 19), None)):
            for fmt in NEW:
                if fmt != "yuv444" and (size[0] | size[1]) & 1:
                    continue
                got = host(r.export_scaled([2, 0], size, crop, fmt, background=BG))
                for i, s in enumerate([2, 0]):
                    img = scaled_np(r.readback(s), RGBA, True, BG, native, size, crop)   # the 8-bit scaled image
                    assert same(entry(got, i), yuv_np(img, fmt)), (fmt, size, crop, s)
        for fmt in NEW:                                                # the whole frame at its own size is export_frames
            assert same(host(r.export_scaled([0, 1], (300, 170), None, fmt)), host(r.export_frames([0, 1], fmt)))


def test_mixed_format_ladders_equal_their_standalone_calls(built):
    p = g.default_params("bars", n=4096, w=1920, h=1080)
    p.lazy_smooth = 1
    rungs = [dict(size=None, fmt="nv12"), dict(size=None, fmt="p010", background=BG), dict(size=(1280, 720), fmt="i420"),
             dict(size=(640, 360), fmt="p010"), dict(size=(480, 270), fmt="nv12"), dict(size=(321, 181), fmt="yuv444"),
             dict(size=None, fmt="yuv444"), dict(size=(96, 54), fmt="rgba", over=True)]
    with g.Renderer(p, batch=3) as r:
        for step in range(2):
            feed(r, 1, seed=step, scale=0.2 + 0.3 * step)
            l0 = r.launch_count
            got = r.export_ladder([2, 0], rungs)
            assert r.launch_count == l0 + 1
            for j, rung in enumerate(rungs):
                size = rung.get("size") or (1920, 1080)
                kw = dict(over=rung.get("over", False), background=rung.get("background", (0, 0, 0)))
                want = (r.export_frames([2, 0], rung["fmt"], **kw) if rung.get("size") is None
                        else r.export_scaled([2, 0], size, None, rung["fmt"], **kw))
                assert same(host(got[j]), host(want)), (step, j, rung)
    p = g.default_params("radial", n=1024, w=98, h=62)                # no marks, w % 4 == 2
    with g.Renderer(p, batch=2) as r:
        feed(r, 2)
        small = [dict(size=None, fmt="i420"), dict(size=(48, 30), fmt="p010"), dict(size=None, fmt="nv12"),
                 dict(size=(33, 17), crop=(5, 5, 80, 40), fmt="yuv444")]
        got = r.export_ladder([1, 0, 1], small)
        for j, rung in enumerate(small):
            want = (r.export_frames([1, 0, 1], rung["fmt"]) if rung.get("size") is None
                    else r.export_scaled([1, 0, 1], rung["size"], rung.get("crop"), rung["fmt"]))
            assert same(host(got[j]), host(want)), j


@pytest.mark.parametrize("fmt,tile", [("i420", (64, 36)), ("yuv444", (48, 27)), ("p010", (40, 24)), ("nv12", (48, 28))])
def test_mosaics_with_sentinels(built, fmt, tile):
    p = g.default_params("bars", n=1024, w=200, h=120)
    with g.Renderer(p, batch=7) as r:
        feed(r, 2, seed=3)
        streams, cols = [6, 1, 0, 3, 5], 3
        tw, th = tile
        W, H = cols * tw, 2 * th
        rows, row_bytes, align = g.api._export_layout(fmt, W, H)
        pitch = (row_bytes + 64 + align - 1) // align * align
        out = torch.full((rows, pitch), 0xA5, dtype=torch.uint8, device="cuda")
        mosaic = host(r.export_mosaic(streams, cols, tile, fmt, background=BG, out=out))
        assert mosaic is not None
        base = out.cpu().numpy()
        planes = host(g.api._export_views(fmt, out, W, H))
        # every tile equals its own scaled export; everything else keeps the sentinel
        written = np.zeros(base.shape, bool)
        flat = written.reshape(-1)
        P = pitch
        for i, s in enumerate(streams):
            ty, tx = i // cols, i % cols
            want = host(r.export_scaled([s], tile, None, fmt, background=BG))
            want = entry(want, 0)
            if fmt in ("nv12", "p010"):
                px = 2 if fmt == "p010" else 1
                view = base.view(np.uint16) if fmt == "p010" else base
                got_y = view[ty * th:(ty + 1) * th, tx * tw:(tx + 1) * tw]
                got_uv = view[H + ty * th // 2:H + (ty + 1) * th // 2, tx * tw:(tx + 1) * tw]
                assert np.array_equal(np.concatenate([got_y, got_uv]), want), (fmt, i)
                written[ty * th:(ty + 1) * th, tx * tw * px:(tx + 1) * tw * px] = True
                written[H + ty * th // 2:H + (ty + 1) * th // 2, tx * tw * px:(tx + 1) * tw * px] = True
            else:
                cw, ch, cp = (tw // 2, th // 2, P // 2) if fmt == "i420" else (tw, th, P)
                y, cb, cr = planes
                assert np.array_equal(y[ty * th:(ty + 1) * th, tx * tw:(tx + 1) * tw], want[0]), (fmt, i)
                assert np.array_equal(cb[ty * ch:(ty + 1) * ch, tx * cw:(tx + 1) * cw], want[1]), (fmt, i)
                assert np.array_equal(cr[ty * ch:(ty + 1) * ch, tx * cw:(tx + 1) * cw], want[2]), (fmt, i)
                written[ty * th:(ty + 1) * th, tx * tw:(tx + 1) * tw] = True
                plane = cp * (H // 2 if fmt == "i420" else H)
                for k in range(2):
                    o = P * H + k * plane + (ty * ch) * cp + tx * cw
                    for rr in range(ch):
                        flat[o + rr * cp:o + rr * cp + cw] = True
        assert (base[~written] == 0xA5).all(), fmt


def test_events_sharded_and_python_shapes(built):
    p = g.default_params("graph", n=1024, w=128, h=64)
    rng = np.random.default_rng(4)
    lb = (rng.standard_normal((6, 1024)) * 0.3).astype(np.float32); rb = lb[::-1].copy()
    with g.ShardedRenderer(p, 6, [0, 0, 0]) as sh, g.Renderer(p, batch=6) as one:
        for _ in range(2):
            sh.update(lb, rb); one.update(lb, rb, True)
        order = [5, 0, 3, 3, 1]
        for fmt in NEW:
            a = sh.export_frames(order, fmt, background=BG)
            b = sh.export_scaled(order, (64, 32), None, fmt)
            c = sh.export_ladder(order, [dict(size=None, fmt=fmt), dict(size=(32, 16), fmt=fmt)])
            sh.sync()
            assert same(host(a), host(one.export_frames(order, fmt, background=BG))), fmt
            assert same(host(b), host(one.export_scaled(order, (64, 32), None, fmt))), fmt
            assert same(host(c[0]), host(one.export_frames(order, fmt))), fmt
            assert same(host(c[1]), host(one.export_scaled(order, (32, 16), None, fmt))), fmt
        # shapes and pitches
        y, cb, cr = one.export_frames([0, 2], "i420")
        assert y.shape == (2, 64, 128) and cb.shape == cr.shape == (2, 32, 64) and y.stride(1) == 128 and cb.stride(1) == 64
        assert cb.data_ptr() == y.data_ptr() + 128 * 64 and cr.data_ptr() == cb.data_ptr() + 64 * 32
        y4 = one.export_frames([1], "yuv444")
        assert all(t.shape == (1, 64, 128) for t in y4) and y4[2].data_ptr() == y4[0].data_ptr() + 2 * 128 * 64
        q = one.export_frames([1], "p010")
        assert q.dtype == torch.uint16 and q.shape == (1, 96, 128) and q.stride(1) == 128
        z = host(q)
        assert ((z & 63) == 0).all() and z[0, :64].min() >= 64 << 6 and z[0, :64].max() <= 940 << 6
        out16 = torch.zeros((2, 96, 160), dtype=torch.uint16, device="cuda")
        got = one.export_frames([1, 4], "p010", out=out16)
        o16 = host(out16)
        assert got is out16 and (o16[:, :, 128:] == 0).all()
        assert np.array_equal(o16[:, :, :128], host(one.export_frames([1, 4], "p010")))
        side = torch.cuda.Stream()
        after, done = torch.cuda.Event(), torch.cuda.Event()
        base = torch.empty((1, 96, 128), dtype=torch.uint8, device="cuda")
        with torch.cuda.stream(side):
            torch.cuda._sleep(20_000_000)
            base.fill_(0x5A)
            after.record(side)
        frame = one.readback(3)
        one.export_frames([3], "i420", out=base, after=after, done=done)
        one.update(lb, rb, True)
        with torch.cuda.stream(side):
            side.wait_event(done)
            seen = base.clone()
        side.synchronize()
        views = g.api._export_views("i420", seen[0], 128, 64)
        assert same(host(views), frame_np(frame, "i420", (0, 0, 0), True))
        with pytest.raises(ValueError, match="overlay"):
            one.overlay_frames([0], torch.zeros((96, 128), dtype=torch.uint8, device="cuda"), fmt="i420")
        with pytest.raises(g.GlavaError, match="I420 pitch"):
            one.export_frames([0], "i420", out=torch.zeros((1, 96, 144), dtype=torch.uint8, device="cuda")[:, :, :136])
