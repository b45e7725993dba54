"""-m gpu: BT.2020 HDR exports and overlay (DESIGN 4.22).  Device bytes against the host build of export_core.h
(tests/export_hdr_shim.py) applied to glava_b200_readback of the same stream at the same point: whole frames of every HDR
format and transfer at 1920x1080 (bars with live marks, radial without) and odd sizes, scaled frames, a mosaic with
sentinels, a ladder mixing HDR and SDR rungs equal to its standalone calls, the framebuffer ring and styles, 1024 streams and
the sharded handle; overlay_planes, its opacity and overlay_scaled onto random 10-bit pictures whose unused bits are set."""
import numpy as np
import pytest

import glava_b200 as g
from tests import export_hdr_shim as S
from tests.export_hdr_np import HLG, PQ
from tests.test_export_core import RGBA, over_np
from tests.test_export_scaled_core import scaled_np

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

BG = (30, 60, 200)
FORMATS = {"p010": S.P010, "yuv420p10": S.YUV420P10, "yuv444p10": S.YUV444P10, "yuv422p10": S.YUV422P10}
TRANSFERS = {"pq": PQ, "hlg": HLG}


def feed(r, steps, seed=0, scale=0.3):
    rng = np.random.default_rng(seed)
    n = r.params.n
    for _ in range(steps):
        r.update((rng.standard_normal((r.batch, n)) * scale).astype(np.float32),
                 (rng.standard_normal((r.batch, n)) * scale).astype(np.float32), True)


def planes_of(got, fmt, i, h):
    """entry i of an export result as uint16 numpy planes laid out as export_hdr_shim.planes lays them"""
    if fmt == "p010":
        a = got[i].cpu().numpy()
        return a[:h], a[h:]
    return tuple(p[i].cpu().numpy() for p in got)


def want_whole(r, s, fmt, e, bg=BG):
    native = bool(r.params.premultiply_alpha)
    return S.planes(e, FORMATS[fmt], S.pack(over_np(r.readback(int(s))[::-1], bg, native)))


def same(got, want, what):
    for p, (a, b) in enumerate(zip(got, want)):
        if not np.array_equal(a, b):
            bad = np.argwhere(a != b)
            raise AssertionError(f"{what}: plane {p} differs at {len(bad)} samples, first {bad[0]}: {a[tuple(bad[0])]} != {b[tuple(bad[0])]}")


def check_whole(r, streams, fmt, tr, what):
    got = r.export_frames(streams, fmt, background=BG, matrix="bt2020", transfer=tr)
    for i, s in enumerate(streams):
        same(planes_of(got, fmt, i, r.params.h), want_whole(r, s, fmt, TRANSFERS[tr]), (what, fmt, tr, i))


@pytest.mark.parametrize("module", ["bars", "radial"])
def test_whole_frames_at_1080p(module):
    p = g.default_params(module, n=4096, w=1920, h=1080)
    with g.Renderer(p, batch=3) as r:
        feed(r, 3)
        for fmt in FORMATS:
            for tr in TRANSFERS:
                check_whole(r, [0, 2, 1], fmt, tr, module)


def test_stale_and_absent_marks_and_odd_sizes():
    for w, h, fmts in ((302, 171, ("yuv444p10", "yuv422p10")), (300, 170, tuple(FORMATS)), (6, 4, tuple(FORMATS))):
        for kw0 in ({}, dict(premultiply_alpha=0, clear_color=[0.1, 0.2, 0.3, 1.0])):
            p = g.default_params("bars", n=1024, w=w, h=h, **kw0)
            with g.Renderer(p, batch=2) as r:
                feed(r, 2)
                for fmt in fmts:
                    for tr in TRANSFERS:
                        check_whole(r, [0, 1], fmt, tr, (w, h, kw0))
                feed(r, 1, seed=5, scale=0.0)                 # quiet audio: the marks go stale as the bars fall
                for tr in TRANSFERS:
                    check_whole(r, [1], fmts[0], tr, "stale")


def test_framebuffer_ring_styles_and_1024_streams():
    p = g.default_params("graph", n=1024, w=128, h=64, fb_slots=3)
    with g.Renderer(p, batch=5) as r:
        r.set_stream_styles([1, 4], [{"amplify": 500, "fg": "#ff8000"}, {"fg": (0.1, 0.9, 0.2, 1.0), "bg": (0.3, 0.3, 0.3, 0.5)}])
        feed(r, 4)
        for fmt in FORMATS:
            check_whole(r, [4, 1, 1, 0], fmt, "pq", "ring")
    p = g.default_params("bars", n=512, w=64, h=32)
    with g.Renderer(p, batch=1024) as r:
        feed(r, 2)
        streams = np.arange(1024)[::-1]
        for fmt, tr in (("p010", "hlg"), ("yuv422p10", "pq")):
            got = r.export_frames(streams, fmt, background=BG, matrix="bt2020", transfer=tr)
            for i in (0, 1, 511, 1023):
                same(planes_of(got, fmt, i, 32), want_whole(r, streams[i], fmt, TRANSFERS[tr]), ("1024", fmt, i))


def test_scaled_mosaic_and_ladder():
    p = g.default_params("bars", n=4096, w=1920, h=1080)
    with g.Renderer(p, batch=2) as r:
        feed(r, 3)
        native = bool(r.params.premultiply_alpha)
        for fmt in FORMATS:
            for tr in TRANSFERS:
                got = r.export_scaled([1, 0], (480, 270) if fmt in ("yuv444p10", "yuv422p10") else (480, 270 - 0), fmt=fmt,
                                      background=BG, matrix="bt2020", transfer=tr)
                for i, s in enumerate([1, 0]):
                    img = S.pack(scaled_np(r.readback(s), RGBA, True, BG, native, (480, 270)))
                    same(planes_of(got, fmt, i, 270), S.planes(TRANSFERS[tr], FORMATS[fmt], img), ("scaled", fmt, tr, i))
        # a mosaic of 3 tiles in 2 columns: the fourth tile keeps HDR black (Y 64, C 512)
        m = r.export_mosaic([0, 1, 0], 2, (480, 270), fmt="yuv420p10", matrix="bt2020", transfer="pq")
        y, cb, cr = (x.cpu().numpy() for x in m)
        assert (y[270:, 480:] == 64).all() and (cb[135:, 240:] == 512).all() and (cr[135:, 240:] == 512).all()
        full = r.export_scaled([0], (480, 270), fmt="yuv420p10", matrix="bt2020", transfer="pq")
        assert all(torch.equal(m[k][:full[k].shape[1], :full[k].shape[2]], full[k][0]) for k in range(3))
        # a ladder mixing HDR and SDR rungs: each rung its standalone call
        rungs = [dict(fmt="p010", matrix="bt2020", transfer="pq"), dict(size=(960, 540), fmt="nv12"),
                 dict(size=(480, 270), fmt="yuv422p10", matrix="bt2020", transfer="hlg"),
                 dict(size=(640, 360), fmt="yuv420p10", full_range=True), dict(size=(320, 180), fmt="yuv444p10", matrix="bt2020",
                                                                               transfer="hlg", background=BG)]
        lad = r.export_ladder([0, 1], rungs)
        for j, rung in enumerate(rungs):
            kw = dict(rung)
            size = kw.pop("size", (1920, 1080))
            solo = r.export_scaled([0, 1], size, **kw)
            if isinstance(solo, tuple):
                assert all(torch.equal(a, b) for a, b in zip(lad[j], solo)), j
            else:
                assert torch.equal(lad[j], solo), j


def test_sharded_handle_on_one_device():
    p = g.default_params("bars", n=1024, w=256, h=128)
    with g.ShardedRenderer(p, 4, [0, 0]) as sh, g.Renderer(p, batch=4) as one:
        rng = np.random.default_rng(1)
        for _ in range(2):
            lb = (rng.standard_normal((4, 1024)) * 0.3).astype(np.float32)
            rb = (rng.standard_normal((4, 1024)) * 0.3).astype(np.float32)
            sh.update(lb, rb, np.ones(4, bool))
            one.update(lb, rb, True)
        for fmt in FORMATS:
            a = sh.export_frames([3, 0], fmt, matrix="bt2020", transfer="hlg")
            sh.sync()
            b = one.export_frames([3, 0], fmt, matrix="bt2020", transfer="hlg")
            torch.cuda.synchronize()
            assert all(torch.equal(x, y) for x, y in zip(a, b)) if isinstance(b, tuple) else torch.equal(a, b)


# ---- overlay onto HDR pictures ----------------------------------------------------------------------------------------------
def picture(fmt, W, H, seed):
    """random uint16 planes (every bit random, the unused six included), each its own allocation with padded rows"""
    rng = np.random.default_rng(seed)
    shapes = [(H, W), S.chroma_shape(FORMATS[fmt], W, H)]
    shapes += [] if fmt == "p010" else shapes[1:]
    out = []
    for p, (rows, cols) in enumerate(shapes):
        pitch = (cols * 2 + (16 if p == 0 else 48) + 15) // 16 * 16 // 2
        out.append(torch.from_numpy(rng.integers(0, 1 << 16, (rows, pitch), dtype=np.uint16)).cuda()[:, :cols])
    return tuple(out)


def host(pic):
    return [t.cpu().numpy() for t in pic]


@pytest.mark.parametrize("module", ["bars", "radial"])
def test_overlay_planes_opacity_and_scaled(module):
    p = g.default_params(module, n=2048, w=640, h=360)
    with g.Renderer(p, batch=2) as r:
        feed(r, 3)
        assert r.params.premultiply_alpha
        for fmt, F in FORMATS.items():
            for tr, e in TRANSFERS.items():
                kw = dict(matrix="bt2020", transfer=tr)
                pic = picture(fmt, 640, 360, 3 + F)
                before = host(pic)
                r.overlay_planes([1], [pic], None, fmt, **kw)
                got = host(pic)
                want = S.overlay(e, F, S.pack(r.readback(1)[::-1]), before)
                same(got, want, (module, fmt, tr))
                # K = 255 is the plain call, K = 0 leaves the picture
                again = picture(fmt, 640, 360, 3 + F)
                r.overlay_planes([1], [again], None, fmt, opacity=1.0, **kw)
                same(host(again), want, (module, fmt, tr, "K=255"))
                untouched = picture(fmt, 640, 360, 9 + F)
                keep = host(untouched)
                r.overlay_planes([1, 0], [untouched, picture(fmt, 640, 360, 1)], None, fmt, opacity=[0.0, 0.5], **kw)
                same(host(untouched), keep, (module, fmt, tr, "K=0"))
                # the scaled overlay: the premultiplied area average of the stored pixels, blended as above
                small = picture(fmt, 320, 180, 5 + F)
                before = host(small)
                r.overlay_planes([0], [small], None, fmt, size=(320, 180), **kw)
                img = S.pack(scaled_np(r.readback(0), RGBA, False, (0, 0, 0), True, (320, 180)))
                same(host(small), S.overlay(e, F, img, before), (module, fmt, tr, "scaled"))
