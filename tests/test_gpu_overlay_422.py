"""-m gpu: the overlay onto 4:2:2 pictures, YUV422P, YUV422P10 and UYVY (glava_b200_overlay_planes, DESIGN 4.18).  What the
call leaves in the caller's planes must equal, bit for bit, the numpy restatement of tests/export_422_np.py applied to
glava_b200_readback of the same stream and to the planes before the call: every module, format, encoding and opacity,
with every byte outside the rectangles untouched and all 16 bits of 10-bit samples under zero pixels kept; the opaque
identity with export_frames; live and absent marks; a mosaic in one picture with its own chroma pitch; an
export-then-overlay round trip; the Python forms of a UYVY picture; the refusals and the sharded handle."""
import numpy as np
import pytest

import glava_b200 as g
from tests.export_422_np import FORMATS, overlay422_np

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
    return [(H, 2 * W)] if fmt == "uyvy" else [(H, W), (H, W // 2), (H, W // 2)]


def picture(fmt, W, H, seed, count=None, pad=(16, 48)):
    """random planes (every bit random, padding bits of 10-bit samples included), each its own allocation with rows padded:
    luma by pad[0] bytes, chroma by pad[1] (so chroma_pitch != pitch / 2)"""
    rng = np.random.default_rng(seed)
    dt, sb = (np.uint16, 2) if fmt == "yuv422p10" else (np.uint8, 1)
    out = []
    for p, (rows, cols) in enumerate(plane_shapes(fmt, W, H)):
        pitch = (cols * sb + pad[min(p, 1)] + 15) // 16 * 16 // sb
        host = rng.integers(0, 1 << (8 * sb), ((count,) if count else ()) + (rows, pitch), dtype=dt)
        out.append(torch.from_numpy(host).cuda()[..., :cols])
    return tuple(out)


def crop(planes, fmt, x, y, w, h):
    """the rectangle's views of host planes"""
    if fmt == "uyvy":
        return [planes[0][y:y + h, 2 * x:2 * (x + w)]]
    return [planes[0][y:y + h, x:x + w]] + [p[y:y + h, x // 2:(x + w) // 2] for p in planes[1:]]


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
        for dst, new in zip(rect, overlay422_np(r.readback(int(s)), [v.copy() for v in rect], fmt, e, native)):
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


@pytest.mark.parametrize("native", [True, False], ids=["native", "blended"])
@pytest.mark.parametrize("module", g.MODULES)
def test_every_module_format_encoding_and_opacity(built, module, native):
    kw0 = {} if native else dict(premultiply_alpha=0, clear_color=[0.1, 0.2, 0.3, 1.0])
    for w, h in ((96, 64), (98, 63), (130, 5)):
        p = g.default_params(module, n=1024, w=w, h=h, **kw0)
        with g.Renderer(p, batch=3) as r:
            feed(r, 3, seed=w)
            for kw, e in ENCS:
                for k, fmt in enumerate(FORMATS):
                    check(r, [0, 2, 1], fmt, kw, e, batched=k % 2 == 1, what=(module, w, h))


@pytest.mark.parametrize("native", [True, False], ids=["native", "blended"])
def test_opaque_pixels_and_other_opacities_give_the_export(built, native):
    """under any other opacity the rectangle gets export_frames' bytes; under native opacity so do the opaque pixels (Y)
    and the pixel pairs whose two pixels are opaque (chroma)"""
    kw0 = {} if native else dict(premultiply_alpha=0)
    p = g.default_params("bars", n=1024, w=128, h=63, **kw0)
    with g.Renderer(p, batch=2) as r:
        feed(r, 3)
        opaque = r.readback(1)[::-1, :, 3] == 255 if native else np.ones((63, 128), bool)
        pairs = opaque[:, 0::2] & opaque[:, 1::2]
        assert pairs.any()
        for kw, e in ENCS:
            for fmt in FORMATS:
                pic = picture(fmt, 128, 63, 7)
                r.overlay_planes([1], [pic], None, fmt, **kw)
                got = [t.cpu().numpy() for t in pic]
                want = r.export_frames([1], fmt, **kw)
                want = [t[0].cpu().numpy() for t in ((want,) if fmt == "uyvy" else want)]
                if fmt == "uyvy":
                    m = np.zeros((63, 256), bool)
                    m[:, 1::2] = opaque
                    m[:, 0::4] = m[:, 2::4] = pairs
                    masks = [m]
                else:
                    masks = [opaque, pairs, pairs]
                for a, b, m in zip(got, want, masks):
                    assert np.array_equal(a[m], b[m]), (fmt, e)


def test_bars_1080p_live_and_absent_marks(built):
    p = g.default_params("bars", n=4096, w=1920, h=1080)
    p.lazy_smooth = 1
    with g.Renderer(p, batch=3) as r:
        for step in range(3):
            feed(r, 1, seed=step, scale=0.1 + 0.3 * step)
            for fmt in FORMATS:
                check(r, [2, 0], fmt, {}, 0, what=step)
        q = r.params.copy(); q.bars_mirror_yx = 1                      # the generic kernel keeps no marks
        r.reconfigure(q)
        feed(r, 1, seed=9)
        for fmt in FORMATS:
            check(r, [1], fmt, dict(matrix="bt601"), 2, what="no marks")


@pytest.mark.parametrize("fmt", FORMATS)
def test_a_mosaic_in_one_picture_with_its_own_chroma_pitch(built, fmt):
    """2 x 3 tiles with gaps in one picture whose chroma pitch is not pitch / 2: every byte outside the tiles keeps its
    sentinel"""
    p = g.default_params("bars", n=1024, w=64, h=31)
    with g.Renderer(p, batch=6) as r:
        feed(r, 3)
        W, H = 3 * 64 + 2 * 32, 2 * 31 + 3
        pic = picture(fmt, W, H, 3, pad=(64, 80))
        at = [(c * 96, rr * 33) for rr in range(2) for c in range(3)]
        before = [host(pic)]
        r.overlay_planes(range(6), [pic] * 6, at, fmt)
        want = expect(r, list(range(6)), before, fmt, 0, at, True)
        same(host(pic), want[0], fmt)


def test_export_then_overlay_round_trip_and_uyvy_forms(built):
    """export_frames' results are pictures overlay_planes takes as they are: plane views, and a UYVY tensor alone, in a
    1-tuple, one per picture or batched"""
    p = g.default_params("wave", n=1024, w=128, h=64)
    with g.Renderer(p, batch=3) as r:
        feed(r, 3)
        for fmt in FORMATS:
            got = r.export_frames([0, 1], fmt)
            planes = (got,) if fmt == "uyvy" else got
            before = [[t[i].cpu().numpy() for t in planes] for i in range(2)]
            r.overlay_planes([2, 1], got, None, fmt)
            want = expect(r, [2, 1], before, fmt, 0, [(0, 0)] * 2, False)
            for i in range(2):
                same([t[i].cpu().numpy() for t in planes], want[i], fmt)
        u = r.export_frames([0, 1], "uyvy")
        for form in (lambda t: [t[0], t[1]], lambda t: [(t[0],), (t[1],)], lambda t: (t,)):
            a = u.clone()
            before = [[a[i].cpu().numpy()] for i in range(2)]
            r.overlay_planes([2, 1], form(a), None, "uyvy")
            want = expect(r, [2, 1], before, "uyvy", 0, [(0, 0)] * 2, False)
            for i in range(2):
                same([a[i].cpu().numpy()], want[i], "uyvy form")


def test_refusals_and_sharded(built):
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
        big = picture("yuv422p", 192, 48, 2)
        with pytest.raises(ValueError, match="even x"):
            one.overlay_planes([0], [big], [(33, 0)], "yuv422p")
        with pytest.raises(ValueError, match="multiple of 16"):
            one.overlay_planes([0], [big], [(16, 0)], "yuv422p")          # Cb would start at byte 8
        with pytest.raises(ValueError, match="planes"):
            one.overlay_planes([0], [picture("yuv422p10", 96, 48, 3)[:2]], None, "yuv422p10")
        pic = picture("uyvy", 96, 48, 5)
        with pytest.raises(g.GlavaError, match="overlaps"):
            sh.overlay_planes([0, 5], [pic, pic], None, "uyvy")
        with pytest.raises(ValueError, match="overlay"):
            one.overlay_frames([0], torch.zeros((72, 96), dtype=torch.uint8, device="cuda"), fmt="uyvy")
