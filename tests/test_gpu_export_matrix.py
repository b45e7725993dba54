"""-m gpu: the Y'CbCr encodings of the exports and the NV12 overlay (DESIGN 4.15).  Every check is against a numpy
restatement applied to glava_b200_readback of the same stream at the same point, with the coefficient sets of
tests/test_export_matrix_core.py (the float64-pinned construction): whole frames of every module, format, encoding and
opacity; the identities with NV12; the framebuffer ring, styles and 1024 streams in one launch; scaled output, mosaics and
ladders that mix encodings per rung against their standalone calls; the overlay onto sentinel pictures; and the sharded
handle against one handle.  The 1080p cases are tests/test_z_gpu_export_matrix_large.py."""
import numpy as np
import pytest

import glava_b200 as g
from tests.test_export_core import RGBA, over_np
from tests.test_export_formats_core import yuv_np
from tests.test_export_matrix_core import coef_py
from tests.test_export_scaled_core import scaled_np

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

BG = (30, 60, 200)
FORMATS = ("nv12", "i420", "yuv444", "p010")
# the three new encodings as keyword arguments, and the encoding index export_core.h gives them
NEW = [(dict(matrix="bt709", full_range=True), 1), (dict(matrix="bt601"), 2), (dict(matrix="bt601", full_range=True), 3)]
NEW_IDS = ["bt709-full", "bt601-limited", "bt601-full"]


# ---- numpy restatement ------------------------------------------------------------------------------------------------------
def ycbcr_np(c, fmt, e):
    """a composited top-down image c [h][w][>= 3] in encoding e -> NV12 bytes [h * 3 / 2][w], (Y, Cb, Cr) planes for I420 /
    YUV444, P010 [h * 3 / 2][w] uint16"""
    c = np.asarray(c, np.int64)
    h, w = c.shape[:2]
    ky, kcb, kcr, yoff, coff, top, full = coef_py(e, 10 if fmt == "p010" else 8)
    code = (lambda acc, sh: np.minimum(acc >> sh, top)) if full else (lambda acc, sh: acc >> sh)
    dot = lambda k, v: k[0] * v[..., 0] + k[1] * v[..., 1] + k[2] * v[..., 2]
    y = code(dot(ky, c) + (yoff << 16) + (1 << 15), 16)
    if fmt == "p010":
        s = c[..., :3].reshape(h // 2, 2, w // 2, 2, 3).sum(axis=(1, 3))      # exact block sums
        cb, cr = code(dot(kcb, s) + (coff << 18) + (1 << 17), 18), code(dot(kcr, s) + (coff << 18) + (1 << 17), 18)
        return (np.concatenate([y, np.stack([cb, cr], axis=-1).reshape(h // 2, w)]) << 6).astype(np.uint16)
    if fmt in ("nv12", "i420"):
        c = (c[..., :3].reshape(h // 2, 2, w // 2, 2, 3).sum(axis=(1, 3)) + 2) >> 2
    cb, cr = code(dot(kcb, c) + (coff << 16) + (1 << 15), 16), code(dot(kcr, c) + (coff << 16) + (1 << 15), 16)
    if fmt == "nv12":
        return np.concatenate([y, np.stack([cb, cr], axis=-1).reshape(h // 2, w)]).astype(np.uint8)
    return y.astype(np.uint8), cb.astype(np.uint8), cr.astype(np.uint8)


def frame_np(frame, fmt, e, bg, native):
    return ycbcr_np(over_np(frame[::-1], bg, native), fmt, e)


def overlay_np(frame, pic, e):
    """NV12 picture pic [h * 3 / 2][w] (the frame's rectangle) after the native overlay of read-back frame [h][w][4]"""
    px = frame[::-1].astype(np.int64)
    h, w = px.shape[:2]
    ky, kcb, kcr, yoff, coff, _, _ = coef_py(e, 8)
    frac = lambda off, a, vd: (((off * a + (255 - a) * vd) << 16) + 127) // 255
    dot = lambda k, v: k[0] * v[..., 0] + k[1] * v[..., 1] + k[2] * v[..., 2]
    out = pic.copy()
    out[:h] = np.clip((dot(ky, px) + frac(yoff, px[..., 3], pic[:h].astype(np.int64)) + (1 << 15)) >> 16, 0, 255)
    m = (px.reshape(h // 2, 2, w // 2, 2, 4).sum(axis=(1, 3)) + 2) >> 2
    uv = pic[h:].astype(np.int64).reshape(h // 2, w // 2, 2)
    cb = np.clip((dot(kcb, m) + frac(coff, m[..., 3], uv[..., 0]) + (1 << 15)) >> 16, 0, 255)
    cr = np.clip((dot(kcr, m) + frac(coff, m[..., 3], uv[..., 1]) + (1 << 15)) >> 16, 0, 255)
    out[h:] = np.stack([cb, cr], axis=-1).reshape(h // 2, w)
    return out


# ---- helpers ---------------------------------------------------------------------------------------------------------------------
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


def check(r, streams, fmt, kw, e, bg=BG, what=""):
    got = host(r.export_frames(streams, fmt, background=bg, **kw))
    native = bool(r.params.premultiply_alpha)
    for i, s in enumerate(streams):
        assert same(entry(got, i), frame_np(r.readback(int(s)), fmt, e, bg, native)), (what, fmt, kw, i, int(s))


def check_identities(r, streams, kw, bg=BG):
    h = r.params.h
    nv12 = r.export_frames(streams, "nv12", background=bg, **kw)
    y, cb, cr = r.export_frames(streams, "i420", background=bg, **kw)
    assert torch.equal(y, nv12[:, :h]) and torch.equal(cb, nv12[:, h:, 0::2]) and torch.equal(cr, nv12[:, h:, 1::2]), kw
    assert torch.equal(r.export_frames(streams, "yuv444", background=bg, **kw)[0], nv12[:, :h]), kw


# ---- whole frames --------------------------------------------------------------------------------------------------------------
def test_the_restatement_is_todays_arithmetic_for_bt709_limited():
    rng = np.random.default_rng(0)
    c = rng.integers(0, 256, (6, 10, 4))
    for fmt in ("i420", "yuv444", "p010"):
        assert same(ycbcr_np(c, fmt, 0), yuv_np(c, fmt)), fmt


@pytest.mark.parametrize("native", [True, False], ids=["native", "blended"])
@pytest.mark.parametrize("module", g.MODULES)
def test_every_module_format_encoding_and_opacity(built, module, native):
    kw0 = {} if native else dict(premultiply_alpha=0, clear_color=[0.1, 0.2, 0.3, 1.0])
    for w, h, fmts in ((96, 64, FORMATS), (98, 62, FORMATS), (97, 63, ("yuv444",))):
        p = g.default_params(module, n=1024, w=w, h=h, **kw0)
        with g.Renderer(p, batch=3) as r:
            feed(r, 3, seed=w)
            for kw, e in NEW:
                for fmt in fmts:
                    check(r, [0, 2, 1], fmt, kw, e, what=(module, w, h))
                if fmts == FORMATS:
                    check_identities(r, [2, 0], kw)
            for fmt in fmts:                                           # the defaults set no colour bit
                assert same(host(r.export_frames([1, 0], fmt, matrix="bt709", full_range=False)),
                            host(r.export_frames([1, 0], fmt))), fmt


@pytest.mark.parametrize("slots", [1, 3])
def test_framebuffer_ring_styles_and_repeats(built, slots):
    p = g.default_params("graph", n=1024, w=128, h=64, fb_slots=slots)
    with g.Renderer(p, batch=5) as r:
        r.set_stream_styles([1, 4], [{"amplify": 500, "fg": "#ff8000"}, {"fg": (0.1, 0.9, 0.2, 1.0), "bg": (0.3, 0.3, 0.3, 0.5)}])
        feed(r, 3)
        for kw, e in NEW:
            for fmt in FORMATS:
                check(r, [4, 0, 4, 1, 3], fmt, kw, e, bg=(255, 255, 255))


def test_a_thousand_streams_in_one_launch(built):
    p = g.default_params("bars", n=512, w=64, h=32)
    with g.Renderer(p, batch=1024) as r:
        feed(r, 2)
        for kw, e in NEW:
            for fmt in FORMATS:
                l0 = r.launch_count
                got = host(r.export_frames(range(1024), fmt, **kw))
                assert r.launch_count == l0 + 1
                for s in list(range(0, 1024, 37)) + [1023]:
                    assert same(entry(got, s), frame_np(r.readback(s), fmt, e, (0, 0, 0), True)), (fmt, kw, s)


# ---- scaled, mosaic, ladder --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("native", [True, False], ids=["native", "blended"])
@pytest.mark.parametrize("module", ["bars", "radial", "wave"])
def test_scaled_is_the_encoding_on_the_scaled_image(built, module, native):
    kw0 = {} if native else dict(premultiply_alpha=0, clear_color=[0.1, 0.2, 0.3, 1.0])
    p = g.default_params(module, n=1024, w=300, h=170, **kw0)
    with g.Renderer(p, batch=3) as r:
        feed(r, 3, seed=5)
        for kw, e in NEW:
            for size, crop in (((100, 56), None), ((64, 30), (10, 20, 200, 100)), ((37, 19), None)):
                for fmt in FORMATS:
                    if fmt != "yuv444" and (size[0] | size[1]) & 1:
                        continue
                    got = host(r.export_scaled([2, 0], size, crop, fmt, background=BG, **kw))
                    for i, s in enumerate([2, 0]):
                        img = scaled_np(r.readback(s), RGBA, True, BG, native, size, crop)   # the 8-bit scaled image
                        assert same(entry(got, i), ycbcr_np(img, fmt, e)), (fmt, kw, size, crop, s)
            for fmt in FORMATS:                                        # the whole frame at its own size is export_frames
                assert same(host(r.export_scaled([0, 1], (300, 170), None, fmt, **kw)),
                            host(r.export_frames([0, 1], fmt, **kw))), (fmt, kw)


@pytest.mark.parametrize("fmt,tile", [("nv12", (48, 28)), ("i420", (64, 36)), ("yuv444", (48, 27)), ("p010", (40, 24))])
def test_mosaics_per_encoding(built, fmt, tile):
    p = g.default_params("bars", n=1024, w=200, h=120)
    with g.Renderer(p, batch=7) as r:
        feed(r, 2, seed=3)
        streams, cols = [6, 1, 0, 3, 5], 3
        tw, th = tile
        W, H = cols * tw, 2 * th
        for kw, e in NEW:
            m = host(r.export_mosaic(streams, cols, tile, fmt, background=BG, **kw))
            planes = m if isinstance(m, tuple) else (m[:H], m[H:])
            for i, s in enumerate(streams):
                ty, tx = i // cols, i % cols
                want = entry(host(r.export_scaled([s], tile, None, fmt, background=BG, **kw)), 0)
                if fmt in ("nv12", "p010"):
                    got = np.concatenate([planes[0][ty * th:(ty + 1) * th, tx * tw:(tx + 1) * tw],
                                          planes[1][ty * th // 2:(ty + 1) * th // 2, tx * tw:(tx + 1) * tw]])
                    assert np.array_equal(got, want), (kw, i)
                else:
                    cw, ch = (tw // 2, th // 2) if fmt == "i420" else (tw, th)
                    for k, (pl, sw, sh) in enumerate(((planes[0], tw, th), (planes[1], cw, ch), (planes[2], cw, ch))):
                        assert np.array_equal(pl[ty * sh:(ty + 1) * sh, tx * sw:(tx + 1) * sw], want[k]), (kw, i, k)
            # the empty tile is black in the encoding: Y 0 in full range, 16 (64 << 6) in limited range; chroma 128 (512 << 6)
            black = 0 if kw.get("full_range") else (64 << 6 if fmt == "p010" else 16)
            mid = 512 << 6 if fmt == "p010" else 128
            ty, tx = 1, 2
            assert (planes[0][ty * th:(ty + 1) * th, tx * tw:(tx + 1) * tw] == black).all(), kw
            cw, ch = (tw // 2, th // 2) if fmt in ("i420",) else (tw, th // 2) if fmt in ("nv12", "p010") else (tw, th)
            assert (planes[1][ty * ch:(ty + 1) * ch, tx * cw:(tx + 1) * cw] == mid).all(), kw


def ladder_vs_standalone(r, streams, rungs):
    l0 = r.launch_count
    got = r.export_ladder(streams, rungs)
    assert r.launch_count == l0 + 1
    for j, rung in enumerate(rungs):
        kw = {k: v for k, v in rung.items() if k in ("over", "background", "matrix", "full_range")}
        want = (r.export_frames(streams, rung["fmt"], **kw) if rung.get("size") is None
                else r.export_scaled(streams, rung["size"], rung.get("crop"), rung["fmt"], **kw))
        assert same(host(got[j]), host(want)), (j, rung)


def test_ladders_mixing_encodings_equal_their_standalone_calls(built):
    p = g.default_params("radial", n=1024, w=98, h=62)                # no marks, w % 4 == 2
    with g.Renderer(p, batch=2) as r:
        feed(r, 2)
        rungs = [dict(size=None, fmt="i420", matrix="bt601", full_range=True), dict(size=(48, 30), fmt="p010", full_range=True),
                 dict(size=None, fmt="nv12", matrix="bt601"), dict(size=(33, 17), crop=(5, 5, 80, 40), fmt="yuv444", full_range=True),
                 dict(size=None, fmt="nv12"), dict(size=(48, 30), fmt="nv12", matrix="bt601", full_range=True),
                 dict(size=(40, 20), fmt="rgba", over=True)]
        ladder_vs_standalone(r, [1, 0, 1], rungs)
        ladder_vs_standalone(r, [0], [dict(size=None, fmt="nv12", full_range=True), dict(size=(48, 30), fmt="nv12")])


# ---- overlay ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw,e", NEW, ids=NEW_IDS)
@pytest.mark.parametrize("module", ["bars", "radial", "graph"])
def test_nv12_overlay_per_encoding(built, module, kw, e):
    p = g.default_params(module, n=1024, w=128, h=64)
    rng = np.random.default_rng(e)
    with g.Renderer(p, batch=3) as r:
        for step in range(2):                                          # marks from the second pass
            feed(r, 1, seed=step)
            W, H, at = 256, 96, [(0, 0), (128, 32)]
            pic = torch.tensor(rng.integers(0, 256, (H * 3 // 2, W), dtype=np.uint8), device="cuda")
            before = pic.cpu().numpy()
            r.overlay_frames([0, 2], [pic, pic], at, **kw)
            after = pic.cpu().numpy()
            want = before.copy()
            for s, (x, y) in zip([0, 2], at):
                rect = np.concatenate([want[y:y + 64, x:x + 128], want[H + y // 2:H + y // 2 + 32, x:x + 128]])
                out = overlay_np(r.readback(s), rect, e)
                want[y:y + 64, x:x + 128], want[H + y // 2:H + y // 2 + 32, x:x + 128] = out[:64], out[64:]
            assert np.array_equal(after, want), (module, kw, step)
            # bytes under all-zero quads are untouched
            fr = r.readback(0)[::-1]
            zq = (fr.reshape(32, 2, 32, 4, 4) == 0).all(axis=(1, 3, 4))   # [row pair][quad]
            quads = lambda a: a[0:64, 0:128].reshape(32, 2, 32, 4).transpose(0, 2, 1, 3)
            assert zq.any() and (quads(after)[zq] == quads(before)[zq]).all()
        # an opaque frame (non-native opacity) gives the export's bytes
        q = r.params.copy(); q.premultiply_alpha = 0
        r.reconfigure(q)
        feed(r, 1, seed=7)
        pic = torch.full((96, 128), 0xA5, dtype=torch.uint8, device="cuda")
        r.overlay_frames([1], [pic], **kw)
        assert np.array_equal(pic.cpu().numpy(), host(r.export_frames([1], "nv12", **kw))[0]), kw


def test_overlay_native_opaque_pixels_give_the_export(built):
    """under native opacity, wherever a 2x2 block's stored pixels are all opaque its Y and CbCr bytes are the export's"""
    p = g.default_params("bars", n=1024, w=64, h=32, clear_color=[0.2, 0.4, 0.6, 1.0])
    with g.Renderer(p, batch=2) as r:
        feed(r, 2)
        fr = r.readback(0)[::-1]
        opaque = (fr[..., 3] == 255).reshape(16, 2, 32, 2).all(axis=(1, 3))   # [block row][block]
        assert opaque.any()
        for kw, e in NEW:
            pic = torch.full((48, 64), 0x5A, dtype=torch.uint8, device="cuda")
            r.overlay_frames([0], [pic], **kw)
            got, want = pic.cpu().numpy(), host(r.export_frames([0], "nv12", **kw))[0]
            blocks = lambda a: a[:32].reshape(16, 2, 32, 2).transpose(0, 2, 1, 3)
            assert (blocks(got)[opaque] == blocks(want)[opaque]).all(), kw
            uv = lambda a: a[32:].reshape(16, 32, 2)
            assert (uv(got)[opaque] == uv(want)[opaque]).all(), kw


# ---- the sharded handle -------------------------------------------------------------------------------------------------------
def test_sharded_equals_one_handle(built):
    p = g.default_params("graph", n=1024, w=128, h=64)
    rng = np.random.default_rng(4)
    lb = (rng.standard_normal((6, 1024)) * 0.3).astype(np.float32); rb = lb[::-1].copy()
    with g.ShardedRenderer(p, 6, [0, 0, 0]) as sh, g.Renderer(p, batch=6) as one:
        for _ in range(2):
            sh.update(lb, rb); one.update(lb, rb, True)
        order = [5, 0, 3, 3, 1]
        for kw, e in NEW:
            for fmt in FORMATS:
                a = sh.export_frames(order, fmt, background=BG, **kw)
                b = sh.export_scaled(order, (64, 32), None, fmt, **kw)
                c = sh.export_ladder(order, [dict(size=None, fmt=fmt, **kw), dict(size=(32, 16), fmt=fmt)])
                sh.sync()
                assert same(host(a), host(one.export_frames(order, fmt, background=BG, **kw))), (fmt, kw)
                assert same(host(b), host(one.export_scaled(order, (64, 32), None, fmt, **kw))), (fmt, kw)
                assert same(host(c[0]), host(one.export_frames(order, fmt, **kw))), (fmt, kw)
                assert same(host(c[1]), host(one.export_scaled(order, (32, 16), None, fmt))), (fmt, kw)
            pics = [torch.tensor(rng.integers(0, 256, (96, 128), dtype=np.uint8), device="cuda") for _ in range(2)]
            twins = [t.clone() for t in pics]
            sh.overlay_frames([5, 0], pics, **kw)
            sh.sync()
            one.overlay_frames([5, 0], twins, **kw)
            assert all(torch.equal(x, y) for x, y in zip(pics, twins)), kw
        with pytest.raises(g.GlavaError, match="no matrix or range"):
            sh.export_frames([0], "rgba", matrix="bt601")
        with pytest.raises(ValueError, match="matrix"):
            one.export_frames([0], "nv12", matrix="bt2020")
