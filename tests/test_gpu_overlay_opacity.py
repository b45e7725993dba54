"""-m gpu: the overlay at a per-entry opacity (glava_b200_overlay_frames_opacity / glava_b200_overlay_planes_opacity, DESIGN
4.20).  What a call leaves in the caller's pictures must equal, bit for bit, the plain overlay's numpy restatement applied to
the pre-scaled frame (tests/test_overlay_opacity_core.py restated), from glava_b200_readback of the same stream at the same
point in call order and the pictures before the call, with every byte outside the rectangles untouched (row padding
included): every module, every overlay_frames and overlay_planes format and encoding, native and any other opacity, K in
{0, 1, 37, 128, 254, 255} and mixed lists; K = 255 equals the plain call byte for byte and K = 0 leaves the picture
alone; bars at 1080p under marks, the framebuffer ring and styles, a 1024-entry mosaic, after / done ordering and the
sharded handle against one handle."""
import numpy as np
import pytest

import glava_b200 as g
from tests.test_overlay_opacity_core import (BGRA, C420, FORMATS, I420, NAME, NV12, RGBA, UYVY, YUV422P, YUV422P10,
                                             plane_shapes, restated)

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

ENCS = [(dict(), 0), (dict(full_range=True), 1), (dict(matrix="bt601"), 2), (dict(matrix="bt601", full_range=True), 3)]
K_LIST = [0, 1, 37, 128, 254, 255]
FNAME = {RGBA: "rgba", BGRA: "bgra", NV12: "nv12"}


def feed(r, steps, seed=0, scale=0.3):
    rng = np.random.default_rng(seed)
    n = r.params.n
    for _ in range(steps):
        lb = (rng.standard_normal((r.batch, n)) * scale).astype(np.float32)
        rb = (rng.standard_normal((r.batch, n)) * scale).astype(np.float32)
        r.update(lb, rb, True)


def fits(fmt, w, h):
    return not ((fmt in C420 and (w | h) & 1) or (fmt in (YUV422P, YUV422P10, UYVY) and w & 1))


class Picture:
    """one entry's destination: each plane its own random uint8 allocation with padded rows; .views are the rectangle's
    byte planes [rows, row bytes], frames_arg() / planes_arg() what overlay_frames / overlay_planes take"""

    def __init__(self, fmt, w, h, seed, pad=48):
        rng = np.random.default_rng(seed)
        self.fmt, self.w, self.h = fmt, w, h
        if fmt == NV12:                                       # overlay_frames: one [h * 3 / 2, w] image; overlay_planes: (Y, CbCr)
            shapes = [(h * 3 // 2, w)]
        else:
            shapes = plane_shapes(fmt, w, h)
        self.full = [torch.from_numpy(rng.integers(0, 256, (rows, (cols + pad + 15) // 16 * 16), dtype=np.uint8)).cuda()
                     for rows, cols in shapes]
        self.views = [t[:, :cols] for t, (rows, cols) in zip(self.full, shapes)]

    def frames_arg(self):
        t = self.views[0]
        return t.view(self.h, self.w, 4) if self.fmt in (RGBA, BGRA) else t

    def planes_arg(self):
        if self.fmt == NV12:
            t = self.views[0]
            return (t[:self.h], t[self.h:])
        return tuple(self.views)

    def host(self):
        return [t.cpu().numpy() for t in self.full]

    def rect_planes(self, full):
        """the rectangle's byte planes (as restated() takes them) of host copies of the allocations"""
        if self.fmt == NV12:
            a = full[0][:, :self.w]
            return [a[:self.h], a[self.h:]]
        return [a[:, :v.shape[1]] for a, v in zip(full, self.views)]


def run(r, streams, fmt, pics, k, kw, planes=False):
    op = None if k is None else [v / 255.0 for v in k]
    if fmt in (RGBA, BGRA) or (fmt == NV12 and not planes):
        r.overlay_frames(streams, [p.frames_arg() for p in pics], None, FNAME[fmt], opacity=op, **kw)
    else:
        r.overlay_planes(streams, [p.planes_arg() for p in pics], None, NAME[fmt], opacity=op, **kw)
    torch.cuda.synchronize()


def expect(r, streams, pics, before, k, e):
    native = bool(r.params.premultiply_alpha)
    out = [[a.copy() for a in b] for b in before]
    for i, s in enumerate(streams):
        rect = pics[i].rect_planes(out[i])
        frame = r.readback(int(s))
        for dst, new in zip(rect, restated(frame, [v.copy() for v in rect], pics[i].fmt, e, k[i], native)):
            dst[...] = new
    return out


def same(got, want, what):
    for p, (a, b) in enumerate(zip(got, want)):
        if not np.array_equal(a, b):
            bad = np.argwhere(a != b)
            raise AssertionError(f"{what}: plane {p} differs at {len(bad)} bytes, first {bad[0]}: {a[tuple(bad[0])]} != {b[tuple(bad[0])]}")


def check(r, streams, fmt, k, kw, e, planes=False, seed=0, what=""):
    pics = [Picture(fmt, r.params.w, r.params.h, seed + 17 * i) for i in range(len(streams))]
    before = [p.host() for p in pics]
    run(r, streams, fmt, pics, k, kw, planes)
    want = expect(r, streams, pics, before, k, e)
    for i, p in enumerate(pics):
        same(p.host(), want[i], (what, fmt, e, k[i], i))


def frame_formats(w, h):
    return [(f, False) for f in (RGBA, BGRA, NV12) if fits(f, w, h)] + [(f, True) for f in FORMATS if f not in (RGBA, BGRA)
                                                                         and fits(f, w, h)]


# ---- every module, format, encoding and opacity ----------------------------------------------------------------------------
@pytest.mark.parametrize("native", [True, False], ids=["native", "blended"])
@pytest.mark.parametrize("module", g.MODULES)
def test_every_module_format_encoding_and_opacity(built, module, native):
    kw0 = {} if native else dict(premultiply_alpha=0, clear_color=[0.1, 0.2, 0.3, 1.0])
    streams = [0, 1, 2, 0, 1, 2]
    for w, h in ((98, 62), (97, 63)):
        p = g.default_params(module, n=1024, w=w, h=h, **kw0)
        with g.Renderer(p, batch=3) as r:
            feed(r, 3, seed=w)
            for fmt, planes in frame_formats(w, h):
                for kw, e in (ENCS if fmt not in (RGBA, BGRA) else ENCS[:1]):
                    check(r, streams, fmt, K_LIST, kw, e, planes, seed=w + e, what=(module, w, h))      # mixed list
                    k = [K_LIST[(e + fmt) % 6]] * 3                                                    # one K for all
                    check(r, streams[:3], fmt, k, kw, e, planes, seed=w + 5, what=(module, w, h))


@pytest.mark.parametrize("native", [True, False], ids=["native", "blended"])
def test_full_opacity_is_the_plain_call_and_zero_leaves_the_picture(built, native):
    kw0 = {} if native else dict(premultiply_alpha=0)
    p = g.default_params("bars", n=1024, w=160, h=90, **kw0)
    with g.Renderer(p, batch=3) as r:
        feed(r, 3)
        for fmt, planes in frame_formats(160, 90):
            for kw, e in (ENCS if fmt not in (RGBA, BGRA) else ENCS[:1]):
                a = [Picture(fmt, 160, 90, 9 + i) for i in range(3)]
                b = [Picture(fmt, 160, 90, 9 + i) for i in range(3)]
                before = [x.host() for x in a]
                run(r, [2, 0, 1], fmt, a, None, kw, planes)
                run(r, [2, 0, 1], fmt, b, [255] * 3, kw, planes)
                for x, y in zip(a, b):
                    same(x.host(), y.host(), (fmt, e, "K = 255"))
                run(r, [2, 0, 1], fmt, b, [0] * 3, kw, planes)
                for x, y in zip(a, b):
                    same(y.host(), x.host(), (fmt, e, "K = 0"))
                assert any(not np.array_equal(x, y) for x, y in zip(a[0].host(), before[0]))


# ---- marks, ring, styles ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("full_store", ["0", "1"], ids=["live", "stale"])
def test_bars_1080p_with_marks(built, full_store, monkeypatch):
    """the headline geometry: band items under marks the last pass kept; with GLAVA_B200_FULL_STORE the pass stores every
    row and the marks still describe the frame"""
    monkeypatch.setenv("GLAVA_B200_FULL_STORE", full_store)
    p = g.default_params("bars", n=1024, w=1920, h=1080)
    with g.Renderer(p, batch=2) as r:
        feed(r, 2)
        for fmt, planes in ((RGBA, False), (NV12, False), (I420, True), (YUV422P10, True)):
            check(r, [1, 0], fmt, [128, 37], {}, 0, planes, what="1080p")


@pytest.mark.parametrize("slots", [1, 3])
def test_framebuffer_ring_and_styles(built, slots):
    p = g.default_params("graph", n=1024, w=128, h=64, fb_slots=slots)
    with g.Renderer(p, batch=5) as r:
        r.set_stream_styles([1, 4], [{"amplify": 500, "fg": "#ff8000"}, {"fg": (0.1, 0.9, 0.2, 1.0), "bg": (0.3, 0.3, 0.3, 0.5)}])
        feed(r, 3)
        for fmt, planes in frame_formats(128, 64):
            check(r, [4, 0, 4, 1, 3], fmt, [1, 254, 0, 128, 200], {}, 0, planes, what=("ring", slots))


def test_a_mosaic_of_1024_entries(built):
    """1024 32 x 16 tiles in one RGBA picture and one NV12 picture, each tile at its own opacity"""
    tw, th = 32, 16
    p = g.default_params("bars", n=1024, w=tw, h=th)
    rng = np.random.default_rng(5)
    with g.Renderer(p, batch=64) as r:
        feed(r, 3)
        streams = [int(s) for s in rng.integers(0, 64, 1024)]
        k = [int(v) for v in rng.integers(0, 256, 1024)]
        at = [((i % 32) * tw, (i // 32) * th) for i in range(1024)]
        for fmt in (RGBA, NV12):
            W, H = 32 * tw, 32 * th
            host0 = rng.integers(0, 256, (H, W, 4) if fmt == RGBA else (H * 3 // 2, W), dtype=np.uint8)
            img = torch.from_numpy(host0).cuda()
            r.overlay_frames(streams, [img] * 1024, at, FNAME[fmt], opacity=[v / 255.0 for v in k])
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
                for dst, new in zip(rect, restated(r.readback(s), src, fmt, 0, k[i], True)):
                    dst[...] = new.reshape(dst.shape)
            assert np.array_equal(img.cpu().numpy(), want), fmt


# ---- ordering, sharding ----------------------------------------------------------------------------------------------------------
def test_after_and_done_events_order_a_side_stream(built):
    p = g.default_params("bars", n=1024, w=128, h=64)
    with g.Renderer(p, batch=2) as r:
        feed(r, 2)
        for opacity in ([0.5], [0.0]):
            side = torch.cuda.Stream()
            with torch.cuda.stream(side):
                pic = (torch.zeros((64, 128), dtype=torch.uint8, device="cuda"),
                       torch.zeros((32, 64), dtype=torch.uint8, device="cuda"), torch.zeros((32, 64), dtype=torch.uint8, device="cuda"))
                pic[0].fill_(40)
                after, done = torch.cuda.Event(), torch.cuda.Event()
                after.record(side)
            r.overlay_planes([1], [pic], None, "i420", after=after, done=done, opacity=opacity)
            side.wait_event(done)
            side.synchronize()
            before = [np.full((64, 128), 40, np.uint8), np.zeros((32, 64), np.uint8), np.zeros((32, 64), np.uint8)]
            want = restated(r.readback(1), before, I420, 0, int(opacity[0] * 255 + 0.5), True)
            for t, x in zip(pic, want):
                assert np.array_equal(t.cpu().numpy(), x), opacity


def test_python_refusals(built):
    p = g.default_params("bars", n=1024, w=64, h=32)
    with g.Renderer(p, batch=2) as r:
        feed(r, 1)
        img = torch.zeros((32, 64, 4), dtype=torch.uint8, device="cuda")
        for bad in (float("nan"), 1.5, -0.01, [0.5, 0.5]):
            with pytest.raises(ValueError, match="opacity"):
                r.overlay_frames([0], [img], None, "rgba", opacity=bad)
        with pytest.raises(g.GlavaError, match="overlay_frames_opacity.*overlaps"):
            r.overlay_frames([0, 1], [img, img], None, "rgba", opacity=[0.0, 0.0])


def test_sharded_equals_one_handle(built):
    p = g.default_params("graph", n=1024, w=96, h=48)
    with g.ShardedRenderer(p, 6, [0, 0, 0]) as sh, g.Renderer(p, batch=6) as one:
        rng = np.random.default_rng(1)
        for _ in range(3):
            lb = (rng.standard_normal((6, 1024)) * 0.3).astype(np.float32)
            rb = (rng.standard_normal((6, 1024)) * 0.3).astype(np.float32)
            sh.update(lb, rb); one.update(lb, rb, True)
        op = [0.5, 0.0, 1.0, 0.2]
        for fmt, planes in frame_formats(96, 48):
            a = [Picture(fmt, 96, 48, 4 + i) for i in range(4)]
            b = [Picture(fmt, 96, 48, 4 + i) for i in range(4)]
            if planes:
                sh.overlay_planes([5, 0, 3, 5], [x.planes_arg() for x in a], None, NAME[fmt], matrix="bt601", opacity=op)
                one.overlay_planes([5, 0, 3, 5], [x.planes_arg() for x in b], None, NAME[fmt], matrix="bt601", opacity=op)
            else:
                sh.overlay_frames([5, 0, 3, 5], [x.frames_arg() for x in a], None, FNAME[fmt], opacity=op)
                one.overlay_frames([5, 0, 3, 5], [x.frames_arg() for x in b], None, FNAME[fmt], opacity=op)
            sh.sync()
            torch.cuda.synchronize()
            for x, y in zip(a, b):
                same(x.host(), y.host(), ("sharded", fmt))
