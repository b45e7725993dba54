"""-m gpu: the overlay (glava_b200_overlay_frames, DESIGN 4.12).  What an overlay leaves in the caller's image must equal, bit
for bit, the numpy restatement of tests/test_overlay_core.py applied to glava_b200_readback of the same stream at the same
point in call order and to the image's bytes before the call: every module, format and opacity, the identities with
export_frames, live / stale / absent marks under both item shapes, the framebuffer ring, styles, 1024 streams, a mosaic of
rectangles in one image, untouched bytes around and between rectangles, ordering, events, refusals and the sharded
handle."""
import ctypes as C

import numpy as np
import pytest

import glava_b200 as g
from tests.test_export_core import BGRA, NV12, RGBA
from tests.test_overlay_core import overlay_np

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

FMT = {"rgba": RGBA, "bgra": BGRA, "nv12": NV12}


def feed(r, steps, seed=0, scale=0.3):
    rng = np.random.default_rng(seed)
    n = r.params.n
    for _ in range(steps):
        lb = (rng.standard_normal((r.batch, n)) * scale).astype(np.float32)
        rb = (rng.standard_normal((r.batch, n)) * scale).astype(np.float32)
        r.update(lb, rb, True)


def image(fmt, W, H, seed, count=None):
    """random W x H image(s), rows padded to a multiple of 16 bytes"""
    rng = np.random.default_rng(seed)
    row = W if fmt == "nv12" else W * 4
    rows = H * 3 // 2 if fmt == "nv12" else H
    host = rng.integers(0, 256, ((count,) if count else ()) + (rows, (row + 15) // 16 * 16), dtype=np.uint8)
    t = torch.from_numpy(host).cuda()[..., :row]
    return t if fmt == "nv12" else t.unflatten(-1, (W, 4))


def rect_of(img, fmt, x, y, w, h):
    """the rectangle's bytes of a host image, in overlay_np's layout"""
    if fmt != "nv12":
        return img[y:y + h, x:x + w]
    H = img.shape[0] * 2 // 3
    return np.concatenate([img[y:y + h, x:x + w], img[H + y // 2:H + (y + h) // 2, x:x + w]])


def put(img, fmt, x, y, rect):
    h = rect.shape[0] * 2 // 3 if fmt == "nv12" else rect.shape[0]
    w = rect.shape[1]
    if fmt != "nv12":
        img[y:y + h, x:x + w] = rect
        return
    H = img.shape[0] * 2 // 3
    img[y:y + h, x:x + w] = rect[:h]
    img[H + y // 2:H + (y + h) // 2, x:x + w] = rect[h:]


def expect(r, streams, imgs_before, fmt, at):
    """the images after the overlay, from readback and the images before"""
    w, h = r.params.w, r.params.h
    native = bool(r.params.premultiply_alpha)
    out = [im.copy() for im in imgs_before]
    for i, s in enumerate(streams):
        x, y = at[i]
        k = i if len(out) > 1 else 0
        put(out[k], fmt, x, y, overlay_np(r.readback(int(s)), rect_of(out[k], fmt, x, y, w, h), FMT[fmt], native))
    return out


def check(r, streams, fmt, at=None, pad=(0, 0), what=""):
    """one image per entry, `pad` pixels wider and taller than the frame, the frame at `at`"""
    w, h = r.params.w, r.params.h
    at = at or [(0, 0)] * len(streams)
    imgs = image(fmt, w + pad[0], h + pad[1], len(streams) * 7 + w, count=len(streams))
    before = [t.cpu().numpy() for t in imgs]
    r.overlay_frames(streams, imgs, at, fmt)
    got = imgs.cpu().numpy()
    want = expect(r, streams, before, fmt, at)
    for i in range(len(streams)):
        assert np.array_equal(got[i], want[i]), (what, fmt, i, int(streams[i]))


@pytest.mark.parametrize("native", [True, False], ids=["native", "blended"])
@pytest.mark.parametrize("module", g.MODULES)
def test_every_module_format_and_opacity(built, module, native):
    kw = {} if native else dict(premultiply_alpha=0, clear_color=[0.1, 0.2, 0.3, 1.0])
    for w, h in ((96, 64), (100, 62)):
        p = g.default_params(module, n=1024, w=w, h=h, **kw)
        with g.Renderer(p, batch=3) as r:
            feed(r, 3, seed=w)
            for fmt in ("rgba", "bgra", "nv12"):
                check(r, [0, 2, 1], fmt, what=(module, w, h))
                check(r, [2], fmt, at=[(16, 6)], pad=(32, 10), what=(module, w, h, "placed"))


@pytest.mark.parametrize("native", [True, False], ids=["native", "blended"])
def test_identities_with_export_frames(built, native):
    """RGBA / BGRA onto an opaque colour: export_frames with EXPORT_OVER over that colour (native), or export_frames'
    bytes whatever the image (other opacity); NV12 under other opacity: the NV12 export"""
    kw = {} if native else dict(premultiply_alpha=0)
    p = g.default_params("bars", n=1024, w=200, h=100, **kw)
    with g.Renderer(p, batch=2) as r:
        feed(r, 2)
        bg = (30, 60, 200)
        for fmt in ("rgba", "bgra"):
            img = torch.empty((2, 100, 200, 4), dtype=torch.uint8, device="cuda")
            img[..., :3] = torch.tensor(bg if fmt == "rgba" else bg[::-1], dtype=torch.uint8)
            img[..., 3] = 255
            r.overlay_frames([1, 0], img, fmt=fmt)
            assert torch.equal(img, r.export_frames([1, 0], fmt, over=True, background=bg)), fmt
        if not native:
            img = image("nv12", 200, 100, 3, count=2)
            r.overlay_frames([1, 0], img, fmt="nv12")
            assert torch.equal(img, r.export_frames([1, 0], "nv12")), "nv12"


@pytest.mark.parametrize("item", ["band"])                            # the only item shape under native opacity with marks
def test_bars_1080p_with_live_stale_and_no_marks(built, item):
    p = g.default_params("bars", n=4096, w=1920, h=1080)
    p.lazy_smooth = 1
    with g.Renderer(p, batch=3) as r:
        for step in range(3):                                          # live marks from the second pass on
            feed(r, 1, seed=step, scale=0.1 + 0.3 * step)
            check(r, [2, 0], "nv12", what=step)
            check(r, [1], "bgra", at=[(64, 2)], pad=(64, 2), what=step)
        q = r.params.copy(); q.bars_mirror_yx = 1                     # the generic kernel keeps no marks
        r.reconfigure(q)
        feed(r, 1, seed=20)
        check(r, [0, 1, 2], "nv12", what="no marks")
        q.bars_mirror_yx = 0                                           # marks stale for one pass, then valid again
        r.reconfigure(q)
        for step in range(2):
            feed(r, 1, seed=21 + step)
            check(r, [0, 1, 2], "nv12", what=("back", step))
            check(r, [2], "rgba", what=("back", step))


@pytest.mark.parametrize("rows", [7, 45])
def test_odd_band_heights(built, rows, monkeypatch):
    """bands whose NV12 row pairs straddle band edges (GLAVA_B200_ROWS sets the band height)"""
    monkeypatch.setenv("GLAVA_B200_ROWS", str(rows))
    for module in ("bars", "graph", "wave"):
        p = g.default_params(module, n=1024, w=320, h=180)
        with g.Renderer(p, batch=2) as r:
            for step in range(3):
                feed(r, 1, seed=step)
                check(r, [0, 1], "nv12", what=(module, step))
                check(r, [1], "rgba", what=(module, step))


@pytest.mark.parametrize("slots", [1, 3])
def test_framebuffer_ring(built, slots):
    p = g.default_params("graph", n=1024, w=128, h=64, fb_slots=slots)
    with g.Renderer(p, batch=5) as r:
        feed(r, 3)
        check(r, [0, 1, 2, 3, 4], "nv12")
        check(r, [4, 0, 4], "rgba")


def test_styles(built):
    p = g.default_params("bars", n=1024, w=160, h=90)
    with g.Renderer(p, batch=6) as r:
        r.set_stream_styles([1, 4], [{"amplify": 500, "fg": "#ff8000"}, {"fg": (0.1, 0.9, 0.2, 1.0), "bg": (0.3, 0.3, 0.3, 0.5)}])
        feed(r, 3)
        check(r, [5, 1, 1, 4, 0, 4], "rgba")
        check(r, [4, 2], "nv12")


def test_a_thousand_streams_in_one_launch(built):
    p = g.default_params("bars", n=512, w=1920, h=1080)
    p.lazy_smooth = 1
    with g.Renderer(p, batch=1024) as r:
        feed(r, 2)
        imgs = image("nv12", 1920, 1080, 5, count=1024)
        sample = list(range(0, 1024, 97)) + [1023]
        before = {s: imgs[s].cpu().numpy() for s in sample}
        l0 = r.launch_count
        r.overlay_frames(range(1024), imgs, fmt="nv12")
        assert r.launch_count == l0 + 1
        for s in sample:
            want = expect(r, [s], [before[s]], "nv12", [(0, 0)])[0]
            assert np.array_equal(imgs[s].cpu().numpy(), want), s


@pytest.mark.parametrize("fmt", ["nv12", "rgba"])
def test_a_mosaic_of_rectangles_in_one_image_leaves_the_rest(built, fmt):
    """7 frames of 64 x 36 in a 3 x 3 grid with gaps, one image with pitch padding: every rectangle blended, every other
    byte (gaps, padding, the two empty cells, the chroma between) as it was"""
    p = g.default_params("bars", n=1024, w=64, h=36)
    streams = [6, 0, 3, 3, 1, 5, 2]
    with g.Renderer(p, batch=7) as r:
        feed(r, 2)
        W, H = 3 * 80, 3 * 40
        img = image(fmt, W + 16, H, 11)
        at = [((i % 3) * 80, (i // 3) * 40) for i in range(len(streams))]
        before = img.cpu().numpy()
        r.overlay_frames(streams, [img] * len(streams), at, fmt)
        want = expect(r, streams, [before], fmt, at)[0]
        assert np.array_equal(img.cpu().numpy(), want)
        with pytest.raises(g.GlavaError, match="overlaps"):        # two frames 16 pixels apart
            r.overlay_frames([0, 1], [img, img], [(0, 0), (16, 0)], fmt)


def test_the_call_holds_the_frame_of_its_point_in_call_order(built):
    p = g.default_params("bars", n=1024, w=256, h=128)
    rng = np.random.default_rng(1)
    inputs = [(rng.standard_normal((2, 1024)) * s).astype(np.float32) for s in (0.5, 0.02, 0.4, 0.01)]
    frames = []
    with g.Renderer(p, batch=2) as a:
        for i in range(3):
            a.update(inputs[i], inputs[i][::-1].copy(), True)
            frames.append([a.readback(s) for s in range(2)])
    with g.Renderer(p, batch=2) as r:
        imgs = [image("nv12", 256, 128, 30 + i, count=2) for i in range(3)]
        before = [t.cpu().numpy() for t in imgs]
        for i in range(3):
            r.update(inputs[i], inputs[i][::-1].copy(), True)
            r.overlay_frames([0, 1], imgs[i], fmt="nv12")
        r.update(inputs[3], inputs[3], True)                        # right after the call: must not change it
        r.sync()
        for i in range(3):
            got = imgs[i].cpu().numpy()
            for s in range(2):
                assert np.array_equal(got[s], overlay_np(frames[i][s], before[i][s], NV12, True)), (i, s)


def test_after_and_done_events_order_a_side_stream(built):
    """the decoder → overlay → encoder hand-off: the side stream fills the image and records `after`; the overlay waits for
    it and records `done`, which the side stream waits for before it reads"""
    p = g.default_params("wave", n=1024, w=192, h=96)
    with g.Renderer(p, batch=2) as r:
        feed(r, 2)
        frame = r.readback(1)
        side = torch.cuda.Stream()
        img = torch.empty((96 * 3 // 2, 192), dtype=torch.uint8, device="cuda")
        after, done = torch.cuda.Event(), torch.cuda.Event()
        with torch.cuda.stream(side):
            torch.cuda._sleep(20_000_000)
            img.fill_(0x5A)
            after.record(side)
        r.overlay_frames([1], [img], fmt="nv12", after=after, done=done)
        feed(r, 1, seed=9)
        with torch.cuda.stream(side):
            side.wait_event(done)
            seen = img.clone()
        side.synchronize()
        want = overlay_np(frame, np.full((144, 192), 0x5A, np.uint8), NV12, True)
        assert np.array_equal(seen.cpu().numpy(), want)


def test_device_refusals_leave_nothing_enqueued(built):
    p = g.default_params("bars", n=1024, w=64, h=32)
    with g.Renderer(p, batch=2) as r:
        feed(r, 1)
        L = r._L
        d = g.Export(); d.format = g.EXPORT_NV12; d.pitch = 64
        s = np.zeros(1, np.int32)
        host = np.zeros(8192 + 64, np.uint8)
        dev = torch.empty(8192 + 64, dtype=torch.uint8, device="cuda")
        ok = dev.data_ptr()
        bad = [host.ctypes.data + (-host.ctypes.data) % 16, dev.data_ptr() + 8, r.framebuffer_device]
        if torch.cuda.device_count() > 1:
            bad.append(torch.empty(8192, dtype=torch.uint8, device="cuda:1").data_ptr())
        for ptr in bad:
            for dst, uv in (((ptr,), None), ((ok,), (ptr,))):
                l0 = r.launch_count
                rc = L.glava_b200_overlay_frames(r._h, s.ctypes.data, 1, (C.c_void_p * 1)(*dst),
                                                 None if uv is None else (C.c_void_p * 1)(*uv), C.byref(d), None, None)
                assert rc != 0 and b"glava_b200_overlay_frames" in L.glava_b200_last_error()
                assert r.launch_count == l0
        img = image("nv12", 64, 32, 1)
        with pytest.raises(g.GlavaError, match="takes none"):
            d.flags = g.EXPORT_OVER
            L_rc = L.glava_b200_overlay_frames(r._h, s.ctypes.data, 1, (C.c_void_p * 1)(ok), None, C.byref(d), None, None)
            g.api._check(L_rc)
        with pytest.raises(ValueError, match="leaves"):
            r.overlay_frames([0], [img], [(2, 0)], "nv12")
        with pytest.raises(ValueError, match="16 bytes"):
            r.overlay_frames([0], [image("nv12", 72, 32, 1)], [(4, 0)], "nv12")
        with pytest.raises(g.GlavaError, match="overlaps"):
            r.overlay_frames([0, 1], [img, img], None, "nv12")


def test_sharded_equals_one_handle(built):
    p = g.default_params("graph", n=1024, w=128, h=64)
    rng = np.random.default_rng(4)
    lb = (rng.standard_normal((6, 1024)) * 0.3).astype(np.float32); rb = lb[::-1].copy()
    with g.ShardedRenderer(p, 6, [0, 0, 0]) as sh, g.Renderer(p, batch=6) as one:
        for _ in range(2):
            sh.update(lb, rb); one.update(lb, rb, True)
        order = [5, 0, 3, 3, 1]
        for fmt in ("nv12", "rgba", "bgra"):
            a = image(fmt, 128, 64, 8, count=len(order))
            b = a.clone()
            sh.overlay_frames(order, a, fmt=fmt)
            sh.sync()
            one.overlay_frames(order, b, fmt=fmt)
            assert torch.equal(a, b), fmt
        img = image("nv12", 128, 64, 9)
        with pytest.raises(g.GlavaError, match="out of range"):
            sh.overlay_frames([6], [img])
        with pytest.raises(g.GlavaError, match="glava_b200_sharded_overlay_frames.*overlaps"):
            sh.overlay_frames([0, 5], [img, img])                     # streams of two shards, one rectangle
