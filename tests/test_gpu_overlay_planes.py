"""-m gpu: the overlay onto decoded pictures (glava_b200_overlay_planes, DESIGN 4.17).  What the call leaves in the caller's
planes must equal, bit for bit, the numpy restatement of tests/overlay_planes_np.py applied to glava_b200_readback of the
same stream at the same point in call order and to the planes before the call, with every byte outside the rectangles
untouched: every module, format, encoding and opacity; the identities with overlay_frames' NV12, I420 against NV12 and
YUV420P10 against P010; live, stale and absent marks; odd band heights; the framebuffer ring and styles; a mosaic in one
picture with its own chroma pitch and sentinel gaps; separate and batched plane tensors; an export-then-overlay round trip;
events, the Python refusals and the sharded handle."""
import numpy as np
import pytest

import glava_b200 as g
from tests.overlay_planes_np import C420, FORMATS, WIDE, planes_np

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

ENCS = [(dict(), 0), (dict(full_range=True), 1), (dict(matrix="bt601"), 2), (dict(matrix="bt601", full_range=True), 3)]


def feed(r, steps, seed=0, scale=0.3):
    rng = np.random.default_rng(seed)
    n = r.params.n
    for _ in range(steps):
        lb = (rng.standard_normal((r.batch, n)) * scale).astype(np.float32)
        rb = (rng.standard_normal((r.batch, n)) * scale).astype(np.float32)
        r.update(lb, rb, True)


def plane_shapes(fmt, W, H):
    """(rows, cols) in samples of each plane of a W x H picture"""
    ch = H // 2 if fmt in C420 else H
    cw = W // 2 if fmt in ("i420", "yuv420p10") else W
    return [(H, W), (ch, cw)] + ([] if fmt in ("nv12", "p010") else [(ch, cw)])


def picture(fmt, W, H, seed, count=None, pad=(16, 48)):
    """random planes (every bit random, padding bits of 10-bit samples included), each its own allocation with rows padded:
    luma by pad[0] bytes, chroma by pad[1] (so chroma_pitch != pitch / 2)"""
    rng = np.random.default_rng(seed)
    dt, sb = (np.uint16, 2) if fmt in WIDE else (np.uint8, 1)
    out = []
    for p, (rows, cols) in enumerate(plane_shapes(fmt, W, H)):
        pitch = (cols * sb + pad[min(p, 1)] + 15) // 16 * 16 // sb
        host = rng.integers(0, 1 << (8 * sb), ((count,) if count else ()) + (rows, pitch), dtype=dt)
        out.append(torch.from_numpy(host).cuda()[..., :cols])
    return tuple(out)


def crop(planes, fmt, x, y, w, h):
    """the rectangle's views of host planes"""
    cx, cw = (x // 2, w // 2) if fmt in ("i420", "yuv420p10") else (x, w)
    cy, chh = (y // 2, h // 2) if fmt in C420 else (y, h)
    return [planes[0][y:y + h, x:x + w]] + [p[cy:cy + chh, cx:cx + cw] for p in planes[1:]]


def host(pic):
    return [t.cpu().numpy() for t in pic]


def expect(r, streams, before, fmt, e, at, shared):
    """the pictures after the call: before[i] the host planes of entry i's picture (shared: one picture for all)"""
    w, h = r.params.w, r.params.h
    native = bool(r.params.premultiply_alpha)
    out = [[p.copy() for p in b] for b in before]
    for i, s in enumerate(streams):
        k = 0 if shared else i
        x, y = at[i]
        rect = crop(out[k], fmt, x, y, w, h)
        for dst, new in zip(rect, planes_np(r.readback(int(s)), [v.copy() for v in rect], fmt, e, native)):
            dst[...] = new
    return out


def same(got, want, what):
    for p, (a, b) in enumerate(zip(got, want)):
        if not np.array_equal(a, b):
            bad = np.argwhere(a != b)
            raise AssertionError(f"{what}: plane {p} differs at {len(bad)} samples, first {bad[0]}: {a[tuple(bad[0])]} != {b[tuple(bad[0])]}")


def check(r, streams, fmt, kw, e, at=None, size=None, batched=False, what=""):
    w, h = r.params.w, r.params.h
    at = at or [(0, 0)] * len(streams)
    W, H = size or (w, h)
    if batched:
        pic = picture(fmt, W, H, len(streams) * 7 + w, count=len(streams))
        before = [[p[i].cpu().numpy() for p in pic] for i in range(len(streams))]
        r.overlay_planes(streams, pic, at, fmt, **kw)
        got = [[p[i].cpu().numpy() for p in pic] for i in range(len(streams))]
    else:
        pics = [picture(fmt, W, H, i * 13 + w) for i in range(len(streams))]
        before = [host(p) for p in pics]
        r.overlay_planes(streams, pics, at, fmt, **kw)
        got = [host(p) for p in pics]
    want = expect(r, streams, before, fmt, e, at, False)
    for i in range(len(streams)):
        same(got[i], want[i], (what, fmt, e, i))


# ---- every module, format, encoding and opacity ----------------------------------------------------------------------------
@pytest.mark.parametrize("native", [True, False], ids=["native", "blended"])
@pytest.mark.parametrize("module", g.MODULES)
def test_every_module_format_encoding_and_opacity(built, module, native):
    kw0 = {} if native else dict(premultiply_alpha=0, clear_color=[0.1, 0.2, 0.3, 1.0])
    for w, h, fmts in ((96, 64, FORMATS), (98, 62, FORMATS), (97, 63, ("yuv444", "yuv444p10")), (99, 5, ("yuv444", "yuv444p10"))):
        p = g.default_params(module, n=1024, w=w, h=h, **kw0)
        with g.Renderer(p, batch=3) as r:
            feed(r, 3, seed=w)
            for kw, e in ENCS:
                for k, fmt in enumerate(fmts):
                    check(r, [0, 2, 1], fmt, kw, e, batched=k % 2 == 1, what=(module, w, h))


# ---- identities --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("native", [True, False], ids=["native", "blended"])
def test_identities_on_the_device(built, native):
    kw0 = {} if native else dict(premultiply_alpha=0)
    p = g.default_params("bars", n=1024, w=160, h=90, **kw0)
    with g.Renderer(p, batch=2) as r:
        feed(r, 3)
        h = 90
        rng = np.random.default_rng(5)
        for kw, e in ENCS:
            # NV12 through overlay_frames and overlay_planes: the same bytes
            y = rng.integers(0, 256, (h * 3 // 2, 160), dtype=np.uint8)
            a = torch.from_numpy(y).cuda()
            b = a.clone()
            r.overlay_frames([1], [a], None, "nv12", **kw)
            r.overlay_planes([1], [(b[:h], b[h:])], None, "nv12", **kw)
            assert torch.equal(a, b), e
            # I420 is NV12 deinterleaved
            nv = torch.from_numpy(y).cuda()
            src = (nv[:h].clone(), nv[h:, 0::2].contiguous(), nv[h:, 1::2].contiguous())
            r.overlay_planes([0], [(nv[:h], nv[h:])], None, "nv12", **kw)
            r.overlay_planes([0], [src], None, "i420", **kw)
            assert torch.equal(src[0], nv[:h]) and torch.equal(src[1], nv[h:, 0::2]) and torch.equal(src[2], nv[h:, 1::2]), e
            # YUV420P10 is P010 deinterleaved and >> 6, on pictures holding the same codes
            codes = rng.integers(0, 1024, (h * 3 // 2, 160), dtype=np.uint16)
            p010 = torch.from_numpy(codes << 6).cuda()
            planar = (torch.from_numpy(codes[:h].copy()).cuda(), torch.from_numpy(codes[h:, 0::2].copy()).cuda(),
                      torch.from_numpy(codes[h:, 1::2].copy()).cuda())
            r.overlay_planes([1], [(p010[:h], p010[h:])], None, "p010", **kw)
            r.overlay_planes([1], [planar], None, "yuv420p10", **kw)
            q = p010.cpu().numpy() >> 6
            assert np.array_equal(planar[0].cpu().numpy(), q[:h]), e
            assert np.array_equal(planar[1].cpu().numpy(), q[h:, 0::2]) and np.array_equal(planar[2].cpu().numpy(), q[h:, 1::2]), e


# ---- marks, band heights, ring, styles ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("full_store", [False, True], ids=["live", "stale"])
def test_bars_1080p_live_stale_and_absent_marks(built, full_store, monkeypatch):
    if full_store:
        monkeypatch.setenv("GLAVA_B200_FULL_STORE", "1")
    p = g.default_params("bars", n=4096, w=1920, h=1080)
    p.lazy_smooth = 1
    with g.Renderer(p, batch=3) as r:
        for step in range(3):                                          # marks valid from the second pass on
            feed(r, 1, seed=step, scale=0.1 + 0.3 * step)
            for fmt in FORMATS:
                check(r, [2, 0], fmt, {}, 0, what=step)
        check(r, [1], "yuv420p10", dict(matrix="bt601", full_range=True), 3)
        q = r.params.copy(); q.bars_mirror_yx = 1                      # the generic kernel keeps no marks
        r.reconfigure(q)
        feed(r, 1, seed=9)
        for fmt in FORMATS:
            check(r, [1], fmt, {}, 0, what="no marks")
        q.bars_mirror_yx = 0                                           # stale for one pass, then valid again
        r.reconfigure(q)
        for step in range(2):
            feed(r, 1, seed=21 + step)
            for fmt in ("i420", "p010", "yuv444p10"):
                check(r, [0, 1, 2], fmt, {}, 0, what=("back", step))


@pytest.mark.parametrize("rows", [7, 45])
def test_odd_band_heights(built, rows, monkeypatch):
    """bands whose 4:2:0 row pairs straddle band edges (GLAVA_B200_ROWS sets the band height)"""
    monkeypatch.setenv("GLAVA_B200_ROWS", str(rows))
    for module in ("bars", "graph", "wave"):
        p = g.default_params(module, n=1024, w=320, h=180)
        with g.Renderer(p, batch=2) as r:
            for step in range(3):
                feed(r, 1, seed=step)
                for fmt in FORMATS:
                    check(r, [0, 1], fmt, {}, 0, what=(module, step))


@pytest.mark.parametrize("slots", [1, 3])
def test_framebuffer_ring_and_styles(built, slots):
    p = g.default_params("graph", n=1024, w=128, h=64, fb_slots=slots)
    with g.Renderer(p, batch=5) as r:
        r.set_stream_styles([1, 4], [{"amplify": 500, "fg": "#ff8000"}, {"fg": (0.1, 0.9, 0.2, 1.0), "bg": (0.3, 0.3, 0.3, 0.5)}])
        feed(r, 3)
        for kw, e in ENCS:
            for fmt in FORMATS:
                check(r, [4, 0, 4, 1, 3], fmt, kw, e, batched=True)


# ---- geometry ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FORMATS)
def test_a_mosaic_in_one_picture_with_its_own_chroma_pitch(built, fmt):
    """2 x 3 tiles with gaps in one picture whose chroma pitch is not pitch / 2: every byte outside the tiles keeps its
    sentinel"""
    p = g.default_params("bars", n=1024, w=64, h=32)
    with g.Renderer(p, batch=6) as r:
        feed(r, 3)
        W, H = 3 * 64 + 2 * 32, 2 * 32 + 2
        pic = picture(fmt, W, H, 3, pad=(64, 80))
        at = [(c * 96, rr * 34) for rr in range(2) for c in range(3)]
        before = [host(pic)]
        r.overlay_planes(range(6), [pic] * 6, at, fmt)
        want = expect(r, list(range(6)), before, fmt, 0, at, True)
        same(host(pic), want[0], fmt)


def test_export_then_overlay_round_trip(built):
    """export_frames' plane views are pictures overlay_planes takes as they are"""
    p = g.default_params("wave", n=1024, w=128, h=64)
    with g.Renderer(p, batch=3) as r:
        feed(r, 3)
        for fmt in ("i420", "yuv444", "yuv420p10", "yuv444p10"):
            planes = r.export_frames([0, 1], fmt)
            before = [[t[i].cpu().numpy() for t in planes] for i in range(2)]
            r.overlay_planes([2, 1], planes, None, fmt)
            want = expect(r, [2, 1], before, fmt, 0, [(0, 0)] * 2, False)
            for i in range(2):
                same([t[i].cpu().numpy() for t in planes], want[i], fmt)


# ---- ordering, refusals, sharding ----------------------------------------------------------------------------------------------
def test_after_and_done_events_order_a_side_stream(built):
    p = g.default_params("bars", n=1024, w=128, h=64)
    with g.Renderer(p, batch=2) as r:
        feed(r, 2)
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            pic = (torch.zeros((64, 128), dtype=torch.uint8, device="cuda"), torch.zeros((32, 64), dtype=torch.uint8, device="cuda"),
                   torch.zeros((32, 64), dtype=torch.uint8, device="cuda"))
            pic[0].fill_(40)
            after, done = torch.cuda.Event(), torch.cuda.Event()
            after.record(side)
        before = [np.full((64, 128), 40, np.uint8), np.zeros((32, 64), np.uint8), np.zeros((32, 64), np.uint8)]
        r.overlay_planes([1], [pic], None, "i420", after=after, done=done)
        side.wait_event(done)
        side.synchronize()
        want = expect(r, [1], [before], "i420", 0, [(0, 0)], False)
        same(host(pic), want[0], "events")


def test_python_refusals(built):
    p = g.default_params("bars", n=1024, w=64, h=32)
    with g.Renderer(p, batch=2) as r:
        feed(r, 1)
        pic = picture("i420", 64, 32, 0)
        with pytest.raises(ValueError, match="overlay_frames"):
            r.overlay_planes([0], [pic], None, "rgba")
        with pytest.raises(ValueError, match="planes"):
            r.overlay_planes([0], [pic[:2]], None, "i420")
        with pytest.raises(ValueError, match="leaves"):
            r.overlay_planes([0], [pic], [(2, 0)], "i420")
        big = picture("i420", 128, 64, 1)
        with pytest.raises(ValueError, match="multiple of 16"):
            r.overlay_planes([0], [big], [(16, 0)], "i420")                # Cb would start at byte 8
        with pytest.raises(ValueError, match="even"):
            r.overlay_planes([0], [big], [(32, 1)], "i420")
        other = picture("i420", 64, 32, 2, pad=(48, 48))
        with pytest.raises(ValueError, match="pitch"):
            r.overlay_planes([0, 1], [pic, other], None, "i420")
        with pytest.raises(ValueError, match="uint8"):
            r.overlay_planes([0], [tuple(t.to(torch.int16) for t in pic)], None, "i420")
        with pytest.raises(g.GlavaError, match="overlaps"):
            r.overlay_planes([0, 1], [pic, pic], None, "i420")
        with pytest.raises(g.GlavaError, match="out of range"):
            r.overlay_planes([5], [pic], None, "i420")
        p10 = picture("p010", 64, 32, 3)
        r.overlay_planes([0], [tuple(t.view(torch.uint8) for t in p10)], None, "p010")   # uint8 views of doubled width


def test_sharded_equals_one_handle(built):
    p = g.default_params("graph", n=1024, w=96, h=48)
    with g.ShardedRenderer(p, 6, [0, 0, 0]) as sh, g.Renderer(p, batch=6) as one:
        rng = np.random.default_rng(1)
        for _ in range(3):
            lb = (rng.standard_normal((6, 1024)) * 0.3).astype(np.float32)
            rb = (rng.standard_normal((6, 1024)) * 0.3).astype(np.float32)
            sh.update(lb, rb); one.update(lb, rb, True)
        for fmt in FORMATS:
            a, b = picture(fmt, 96, 48, 4, count=4), picture(fmt, 96, 48, 4, count=4)
            sh.overlay_planes([5, 0, 3, 5], a, None, fmt, matrix="bt601")
            sh.sync()
            one.overlay_planes([5, 0, 3, 5], b, None, fmt, matrix="bt601")
            torch.cuda.synchronize()
            for x, y in zip(a, b):
                assert np.array_equal(x.cpu().numpy(), y.cpu().numpy()), fmt
        with pytest.raises(g.GlavaError, match="overlaps"):
            pic = picture("i420", 96, 48, 5)
            sh.overlay_planes([0, 5], [pic, pic], None, "i420")
