"""-m gpu: the transparent exports, straight RGBA / BGRA, YUVA420P and YUVA444P10 (DESIGN 4.19).  Whole frames against the
numpy restatement of tests/export_alpha_np.py applied to glava_b200_readback of the same stream at the same point, for
every module (bars with live marks and with GLAVA_B200_FULL_STORE=1, the generic bars kernel), both opacities and every
encoding; the device's un-premultiply over all 65536 (c, a) pairs against the host build; scaled output, mixed ladders,
the framebuffer ring, styles, repeats and the sharded handle; bytes outside each rectangle and in the pitch padding left
as they were; the identities with the opaque exports and the Python shapes."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import glava_b200 as g
from tests.export_alpha_np import FORMATS, frame_alpha_np, scaled_alpha_np

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

BG = (30, 60, 200)
ENCS = [(dict(), 0), (dict(full_range=True), 1), (dict(matrix="bt601"), 2), (dict(matrix="bt601", full_range=True), 3)]
# (fmt, export keywords, encoding, name of the restatement)
CASES = ([(f, kw, e, f) for f in FORMATS for kw, e in ENCS] +
         [("rgba", dict(straight=True), 0, "rgba"), ("bgra", dict(straight=True), 0, "bgra")])
OPAQUE = dict(premultiply_alpha=0, clear_color=[0.1, 0.2, 0.3, 1.0])


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


def check(r, streams, what="", cases=CASES):
    native = bool(r.params.premultiply_alpha)
    for fmt, kw, e, name in cases:
        got = host(r.export_frames(streams, fmt, background=BG, **kw))
        for i, s in enumerate(streams):
            assert same(entry(got, i), frame_alpha_np(r.readback(int(s)), name, e, native)), (what, fmt, kw, i, int(s))


def unassociated(r, streams):
    """the pixels of the listed streams' frames whose colour exceeds their alpha (c > a: straight alpha clamps them)"""
    n = 0
    for s in streams:
        f = r.readback(int(s)).astype(np.int64)
        n += int((f[..., :3] > f[..., 3:4]).any(axis=-1).sum())
    return n


# ---- whole frames --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("native", [True, False], ids=["native", "opaque"])
@pytest.mark.parametrize("module", g.MODULES)
def test_every_module_encoding_and_opacity(built, module, native):
    for w, h in ((96, 64), (130, 6), (98, 34)):
        p = g.default_params(module, n=1024, w=w, h=h, **({} if native else OPAQUE))
        with g.Renderer(p, batch=3) as r:
            feed(r, 3, seed=w + h)
            check(r, [0, 2, 1], (module, w, h))
            if native:
                print(f"{module} {w}x{h}: {unassociated(r, range(3))} pixels with c > a")
    p = g.default_params(module, n=1024, w=67, h=33, **({} if native else OPAQUE))   # odd sizes: YUVA444P10 and straight
    with g.Renderer(p, batch=2) as r:
        feed(r, 2)
        check(r, [1, 0], (module, "odd"), [c for c in CASES if c[0] != "yuva420p"])


def test_bars_1080p_marks_full_store_and_the_generic_kernel(built):
    p = g.default_params("bars", n=4096, w=1920, h=1080)
    p.lazy_smooth = 1
    with g.Renderer(p, batch=3) as r:
        for step in range(3):                                          # marks valid from the second pass on
            feed(r, 1, seed=step, scale=0.1 + 0.3 * step)
            check(r, [2, 0], step, CASES[::3] + CASES[-2:])
        q = r.params.copy(); q.bars_mirror_yx = 1                      # the generic kernel keeps no marks
        r.reconfigure(q)
        feed(r, 1, seed=9)
        check(r, [1], "no marks", CASES[::2] + CASES[-1:])


def test_full_store_gives_the_same_bytes(built, tmp_path):
    """GLAVA_B200_FULL_STORE=1 makes the bars and wave rasters store every zero row; the exports read the same frames"""
    code = r"""
import sys, numpy as np
sys.path.insert(0, sys.argv[1])
import glava_b200 as g
from tests.export_alpha_np import frame_alpha_np
for module in ("bars", "wave", "graph"):
    p = g.default_params(module, n=1024, w=256, h=128)
    with g.Renderer(p, batch=2) as r:
        rng = np.random.default_rng(1)
        for _ in range(3):
            r.update((rng.standard_normal((2, 1024)) * 0.3).astype(np.float32), (rng.standard_normal((2, 1024)) * 0.3).astype(np.float32), True)
        for fmt, kw, name in (("yuva420p", {}, "yuva420p"), ("yuva444p10", dict(matrix="bt601"), "yuva444p10"), ("rgba", dict(straight=True), "rgba")):
            got = r.export_frames([1, 0], fmt, **kw)
            got = tuple(x.cpu().numpy() for x in got) if isinstance(got, tuple) else got.cpu().numpy()
            for i, s in enumerate([1, 0]):
                want = frame_alpha_np(r.readback(s), name, 2 if kw else 0)
                have = tuple(x[i] for x in got) if isinstance(got, tuple) else got[i]
                ok = all(np.array_equal(a, b) for a, b in zip(have, want)) if isinstance(want, tuple) else np.array_equal(have, want)
                assert ok, (module, fmt, s)
print("ok")
"""
    env = dict(os.environ, GLAVA_B200_FULL_STORE="1")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-c", code, root], env=env, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "ok" in out.stdout, out.stdout[-2000:] + out.stderr[-4000:]


@pytest.mark.parametrize("slots", [1, 3])
def test_framebuffer_ring_styles_and_repeats(built, slots):
    p = g.default_params("graph", n=1024, w=128, h=64, fb_slots=slots)
    with g.Renderer(p, batch=5) as r:
        r.set_stream_styles([1, 4], [{"amplify": 500, "fg": (1.0, 0.5, 0.0, 0.6)}, {"fg": (0.1, 0.9, 0.2, 0.4), "bg": (0.3, 0.3, 0.3, 0.5)}])
        feed(r, 3)
        check(r, [4, 0, 4, 1, 3], slots)
        print(f"graph, translucent colours: {unassociated(r, range(5))} pixels with c > a")


# ---- the device's arithmetic over every (c, a) -------------------------------------------------------------------------------------
def test_every_pair_on_the_device(built):
    """all 65536 (c, a) pairs written into a radial renderer's 256 x 256 framebuffer (radial keeps no marks, so the export
    reads every row, and the next raster pass rewrites every pixel): straight RGBA, YUVA444P10 and YUVA420P against the
    host restatement, which tests/test_export_alpha_core.py proves equal to the host build of export_core.h"""
    p = g.default_params("radial", n=1024, w=256, h=256)
    with g.Renderer(p, batch=1) as r:
        feed(r, 1)
        r.sync()
        a, c = np.divmod(np.arange(65536, dtype=np.int64), 256)
        px = np.stack([c, (c + 85) % 256, (c + 170) % 256, a], axis=-1).astype(np.uint8).reshape(256, 256, 4)
        t = torch.from_numpy(px.reshape(-1)).cuda()
        rt = C.CDLL("libcudart.so.12")
        torch.cuda.synchronize()
        assert rt.cudaMemcpy(C.c_void_p(r.framebuffer_device), C.c_void_p(t.data_ptr()), C.c_size_t(t.numel()), 3) == 0
        assert np.array_equal(r.readback(0), px)
        for fmt, kw, e, name in CASES:
            got = host(r.export_frames([0], fmt, **kw))
            assert same(entry(got, 0), frame_alpha_np(px, name, e)), (fmt, kw)
            got = host(r.export_scaled([0], (128, 64), None, fmt, **kw))
            assert same(entry(got, 0), scaled_alpha_np(px, name, (128, 64), None, e)), (fmt, kw)
        s = host(r.export_frames([0], "rgba", straight=True))[0][::-1].reshape(-1, 4).astype(np.int64)
        ok = c <= a
        assert np.array_equal(((2 * s[ok, 0] * a[ok] + 255) // 510), c[ok]), "mul_norm8(S, a) == c on the device's output"


# ---- scaled, ladders, rectangles ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("native", [True, False], ids=["native", "opaque"])
@pytest.mark.parametrize("module", ["bars", "radial", "wave", "graph"])
def test_scaled_is_the_format_on_the_scaled_image(built, module, native):
    p = g.default_params(module, n=1024, w=300, h=170, **({} if native else OPAQUE))
    with g.Renderer(p, batch=3) as r:
        feed(r, 3, seed=5)
        for fmt, kw, e, name in CASES:
            for size, crop in (((100, 56), None), ((64, 32), (10, 20, 200, 100)), ((38, 20), None), ((2, 2), None)):
                got = host(r.export_scaled([2, 0], size, crop, fmt, background=BG, **kw))
                for i, s in enumerate([2, 0]):
                    assert same(entry(got, i), scaled_alpha_np(r.readback(s), name, size, crop, e, native, BG)), (fmt, kw, size, crop)
            assert same(host(r.export_scaled([0, 1], (300, 170), None, fmt, **kw)), host(r.export_frames([0, 1], fmt, **kw)))


def ladder_vs_standalone(r, streams, rungs):
    l0 = r.launch_count
    got = r.export_ladder(streams, rungs)
    assert r.launch_count == l0 + 1
    for j, rung in enumerate(rungs):
        kw = {k: v for k, v in rung.items() if k in ("over", "background", "matrix", "full_range", "straight")}
        want = (r.export_frames(streams, rung["fmt"], **kw) if rung.get("size") is None
                else r.export_scaled(streams, rung["size"], rung.get("crop"), rung["fmt"], **kw))
        assert same(host(got[j]), host(want)), (j, rung)


def test_mixed_ladders_equal_their_standalone_calls(built):
    p = g.default_params("bars", n=4096, w=1920, h=1080)
    p.lazy_smooth = 1
    rungs = [dict(size=None, fmt="yuva420p"), dict(size=(1280, 720), fmt="nv12", matrix="bt601"),
             dict(size=(640, 360), fmt="yuva444p10", full_range=True), dict(size=(96, 54), fmt="rgba", straight=True),
             dict(size=None, fmt="bgra", straight=True), dict(size=(480, 270), fmt="yuva420p", matrix="bt601", full_range=True),
             dict(size=(640, 361), fmt="yuv422p10"), dict(size=(320, 180), fmt="rgba", over=True)]
    with g.Renderer(p, batch=3) as r:
        for step in range(2):
            feed(r, 1, seed=step, scale=0.2 + 0.3 * step)
            ladder_vs_standalone(r, [2, 0], rungs)
        ladder_vs_standalone(r, [1], rungs[:4])
    p = g.default_params("radial", n=1024, w=98, h=62, **OPAQUE)    # no marks, w % 4 == 2, opaque
    with g.Renderer(p, batch=2) as r:
        feed(r, 2)
        ladder_vs_standalone(r, [1, 0, 1], [dict(size=None, fmt="yuva444p10", matrix="bt601"), dict(size=(48, 30), fmt="nv12"),
                                            dict(size=(34, 18), crop=(5, 5, 80, 40), fmt="yuva420p"),
                                            dict(size=None, fmt="rgba", straight=True)])


@pytest.mark.parametrize("fmt,kw", [("yuva420p", {}), ("yuva444p10", dict(matrix="bt601")), ("rgba", dict(straight=True))])
def test_bytes_outside_the_rectangles_are_unchanged(built, fmt, kw):
    """exports into padded rows with uv_offset > one plane, and scaled exports, leave every byte outside their planes"""
    p = g.default_params("bars", n=1024, w=192, h=96)
    with g.Renderer(p, batch=3) as r:
        feed(r, 2, seed=8)
        for size in (None, (96, 48)):
            w, h = size or (192, 96)
            rows, row_bytes, align = g.api._export_layout(fmt, w, h)
            pitch = (row_bytes + 48 + align - 1) // align * align
            d = g.api._export_desc(fmt, False, (0, 0, 0), kw.get("matrix", "bt709"), False, kw.get("straight", False))
            d.pitch = pitch
            planar = fmt != "rgba"
            chroma = (pitch // 2) * (h // 2) if fmt == "yuva420p" else pitch * h
            d.uv_offset = chroma + 64 if planar else 0
            n = C.c_size_t()
            sc = g.api._export_scale((w, h), None)
            assert r._L.glava_b200_export_scaled_bytes(r._h, C.byref(d), C.byref(sc), C.byref(n)) == 0
            total = n.value + 256
            base = torch.full((2, total), 0x5A, dtype=torch.uint8, device="cuda")
            dst = (C.c_void_p * 2)(base.data_ptr() + 128, base.data_ptr() + total + 128)
            s = np.array([2, 1], np.int32)
            r.sync()
            torch.cuda.synchronize()
            assert r._L.glava_b200_export_scaled(r._h, s.ctypes.data, 2, dst, None, C.byref(d), C.byref(sc), None, None) == 0
            r.sync()
            raw = base.cpu().numpy()
            for i, st in enumerate([2, 1]):
                b = raw[i, 128:]
                written = np.zeros(b.size, bool)
                sb = 2 if fmt == "yuva444p10" else 1
                if not planar:
                    planes = [(0, h, pitch, 4 * w)]
                else:
                    cw, ch, cp = (w // 2, h // 2, pitch // 2) if fmt == "yuva420p" else (w, h, pitch)
                    planes = [(0, h, pitch, w * sb), (pitch * h, ch, cp, cw * sb), (pitch * h + d.uv_offset, ch, cp, cw * sb),
                              (pitch * h + 2 * d.uv_offset, h, pitch, w * sb)]
                got = []
                for off, nr, pp, nb in planes:
                    idx = off + np.arange(nr)[:, None] * pp + np.arange(nb)[None, :]
                    written[idx] = True
                    v = np.ascontiguousarray(b[idx])
                    got.append(v.view(np.uint16) if sb == 2 else v)
                assert (raw[i, :128] == 0x5A).all() and (b[~written] == 0x5A).all(), (fmt, size, i)
                want = scaled_alpha_np(r.readback(st), fmt, (w, h), None, 2 if "matrix" in kw else 0)
                assert same(tuple(got) if planar else got[0].reshape(h, w, 4), want), (fmt, size, i)


# ---- the sharded handle and Python -----------------------------------------------------------------------------------------------
def test_sharded_and_python_shapes(built):
    p = g.default_params("graph", n=1024, w=128, h=64)
    rng = np.random.default_rng(4)
    lb = (rng.standard_normal((6, 1024)) * 0.3).astype(np.float32); rb = lb[::-1].copy()
    with g.ShardedRenderer(p, 6, [0, 0]) as sh, g.Renderer(p, batch=6) as one:
        for _ in range(2):
            sh.update(lb, rb); one.update(lb, rb, True)
        order = [5, 0, 3, 3, 1]
        for fmt, kw, e, name in (CASES[0], CASES[7], CASES[-1]):
            a = sh.export_frames(order, fmt, **kw)
            b = sh.export_scaled(order, (64, 32), None, fmt, **kw)
            c = sh.export_ladder(order, [dict(size=None, fmt=fmt, **kw), dict(size=(32, 16), fmt="nv12")])
            sh.sync()
            assert same(host(a), host(one.export_frames(order, fmt, **kw))), fmt
            assert same(host(b), host(one.export_scaled(order, (64, 32), None, fmt, **kw))), fmt
            assert same(host(c[0]), host(one.export_frames(order, fmt, **kw))), fmt
            assert same(host(c[1]), host(one.export_scaled(order, (32, 16), None, "nv12"))), fmt
        y, cb, cr, al = one.export_frames([0, 2], "yuva420p")
        assert y.shape == al.shape == (2, 64, 128) and cb.shape == cr.shape == (2, 32, 64) and y.dtype == torch.uint8
        assert al.data_ptr() == y.data_ptr() + 128 * 64 + 2 * 64 * 32 and y.stride(0) == 128 * 160
        y, cb, cr, al = one.export_frames([1], "yuva444p10")
        assert all(t.dtype == torch.uint16 and t.shape == (1, 64, 128) for t in (y, cb, cr, al))
        assert al.data_ptr() == y.data_ptr() + 3 * 256 * 64 and int(al.view(torch.int16).max()) <= 1023
        with pytest.raises(ValueError, match="exclude each other"):
            one.export_frames([0], "rgba", over=True, straight=True)
        with pytest.raises(g.GlavaError, match="EXPORT_STRAIGHT is for RGBA and BGRA"):
            one.export_frames([0], "nv12", straight=True)
        with pytest.raises(g.GlavaError, match="never composited"):
            one.export_frames([0], "yuva420p", over=True)
        with pytest.raises(ValueError, match="yuva420p"):
            one.export_mosaic([0, 1], 2, (32, 16), "yuva420p")
        with pytest.raises(ValueError, match="overlay"):
            one.overlay_frames([0], torch.zeros((96, 128), dtype=torch.uint8, device="cuda"), fmt="yuva420p")
