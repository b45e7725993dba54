"""-m gpu: scaled and cropped export (glava_b200_export_scaled, DESIGN 4.11).  What an export writes must equal, bit for
bit, the numpy restatement of tests/test_export_scaled_core.py applied to glava_b200_readback of the same stream at the
same point in call order: every module, format, opacity and composite, crops, live / stale / absent marks, the framebuffer
ring, styles, repeats, 1024 thumbnails, untouched bytes around every destination, mosaics, ordering, events, refusals and
the sharded handle."""
import ctypes as C

import numpy as np
import pytest

import glava_b200 as g
from tests.test_export_core import NV12, RGBA, BGRA
from tests.test_export_scaled_core import scaled_np

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

BG = (30, 60, 200)
FMT = {"rgba": RGBA, "bgra": BGRA, "nv12": NV12}


def want(r, s, fmt, over, bg, size, crop=None):
    return scaled_np(r.readback(int(s)), FMT[fmt], over, bg, bool(r.params.premultiply_alpha), size, crop)


def check(r, streams, fmt, size, crop=None, over=False, bg=BG, what=""):
    got = r.export_scaled(streams, size, crop, fmt, over=over, background=bg)
    host = got.cpu().numpy() if not isinstance(got, list) else [t.cpu().numpy() for t in got]
    for i, s in enumerate(streams):
        exp = want(r, s, fmt, over, bg, size, crop)
        assert np.array_equal(np.asarray(host[i]).reshape(exp.shape), exp), (what, fmt, over, size, crop, i, int(s))


def feed(r, steps, seed=0, scale=0.3):
    rng = np.random.default_rng(seed)
    n = r.params.n
    for _ in range(steps):
        lb = (rng.standard_normal((r.batch, n)) * scale).astype(np.float32)
        rb = (rng.standard_normal((r.batch, n)) * scale).astype(np.float32)
        r.update(lb, rb, True)


@pytest.mark.parametrize("native", [True, False], ids=["native", "blended"])
@pytest.mark.parametrize("module", g.MODULES)
def test_every_module_format_and_opacity(built, module, native):
    kw = {} if native else dict(premultiply_alpha=0, clear_color=[0.1, 0.2, 0.3, 1.0])
    for w, h, cases in ((96, 64, [((96, 64), None), ((32, 16), None), ((14, 10), (5, 7, 80, 50))]),
                        (97, 63, [((13, 7), None), ((97, 63), None), ((30, 20), (33, 1, 61, 60))])):
        p = g.default_params(module, n=1024, w=w, h=h, **kw)
        with g.Renderer(p, batch=3) as r:
            feed(r, 3, seed=w)
            for size, crop in cases:
                for fmt in ("rgba", "bgra", "nv12"):
                    if fmt == "nv12" and (size[0] | size[1]) & 1:
                        continue
                    for over in (False, True):
                        check(r, [0, 2, 1], fmt, size, crop, over, what=(module, w, h))


def test_full_size_equals_export_frames(built):
    p = g.default_params("bars", n=1024, w=200, h=100)
    with g.Renderer(p, batch=2) as r:
        feed(r, 2)
        for fmt, over in (("nv12", True), ("rgba", False), ("bgra", True)):
            a = r.export_scaled([1, 0], (200, 100), None, fmt, over=over, background=BG)
            b = r.export_frames([1, 0], fmt, over=over, background=BG)
            assert torch.equal(a, b), fmt


def test_bars_1080p_with_live_stale_and_no_marks(built):
    p = g.default_params("bars", n=4096, w=1920, h=1080)
    p.lazy_smooth = 1
    with g.Renderer(p, batch=3) as r:
        for step in range(3):                                          # live marks from the second pass on
            feed(r, 1, seed=step, scale=0.1 + 0.3 * step)
            check(r, [2, 0], "nv12", (480, 270), what=step)
            check(r, [1], "rgba", (192, 108), over=True, what=step)
            check(r, [0], "bgra", (7, 3), crop=(1000, 540, 920, 540), what=step)    # the lower half, ragged
        q = r.params.copy(); q.bars_mirror_yx = 1                     # the generic kernel keeps no marks
        r.reconfigure(q)
        feed(r, 1, seed=20)
        check(r, [0, 1, 2], "nv12", (480, 270), what="no marks")
        q.bars_mirror_yx = 0                                           # marks stale for one pass, then valid again
        r.reconfigure(q)
        for step in range(2):
            feed(r, 1, seed=21 + step)
            check(r, [0, 1, 2], "nv12", (128, 72), what=("back", step))
            check(r, [2], "rgba", (97, 13), crop=(64, 900, 1800, 180), over=True, what=("back", step))


@pytest.mark.parametrize("module", ["radial", "circle", "graph", "wave"])
def test_other_modules_at_1080p(built, module):
    p = g.default_params(module, n=1024, w=1920, h=1080)
    with g.Renderer(p, batch=2) as r:
        feed(r, 2, seed=5)
        check(r, [0, 1], "nv12", (480, 270))
        check(r, [1], "rgba", (192, 108), crop=(480, 270, 960, 540), over=True)


@pytest.mark.parametrize("slots", [1, 3])
def test_framebuffer_ring(built, slots):
    p = g.default_params("graph", n=1024, w=128, h=64, fb_slots=slots)
    with g.Renderer(p, batch=5) as r:
        feed(r, 3)
        check(r, [0, 1, 2, 3, 4], "nv12", (64, 32))
        check(r, [4, 0, 4], "rgba", (40, 20), crop=(10, 10, 100, 40), over=True)


def test_styles_and_repeats(built):
    p = g.default_params("bars", n=1024, w=160, h=90)
    with g.Renderer(p, batch=6) as r:
        r.set_stream_styles([1, 4], [{"amplify": 500, "fg": "#ff8000"}, {"fg": (0.1, 0.9, 0.2, 1.0), "bg": (0.3, 0.3, 0.3, 0.5)}])
        feed(r, 3)
        check(r, [5, 1, 1, 4, 0, 4], "rgba", (40, 30), over=True, bg=(255, 255, 255))
        check(r, [4, 2], "nv12", (80, 44), bg=(12, 34, 56))


def test_a_thousand_thumbnails_in_one_launch(built):
    p = g.default_params("bars", n=512, w=1920, h=1080)
    p.lazy_smooth = 1
    with g.Renderer(p, batch=1024) as r:
        feed(r, 2)
        l0 = r.launch_count
        got = r.export_scaled(range(1024), (192, 108), fmt="nv12").cpu().numpy()
        assert r.launch_count == l0 + 1
        for s in list(range(0, 1024, 97)) + [1023]:
            assert np.array_equal(got[s], want(r, s, "nv12", True, (0, 0, 0), (192, 108))), s


def test_nothing_outside_the_rectangles_is_written(built):
    p = g.default_params("wave", n=1024, w=300, h=200)
    with g.Renderer(p, batch=3) as r:
        feed(r, 2)
        for fmt, size in (("rgba", (37, 21)), ("nv12", (50, 30)), ("bgra", (300, 200))):
            px = 1 if fmt == "nv12" else 4
            rows = size[1] * 3 // 2 if fmt == "nv12" else size[1]
            out = torch.full((3, rows + 3, 1280), 0x5A, dtype=torch.uint8, device="cuda")
            view = out[:, :rows]
            r.export_scaled([2, 0, 1], size, None, fmt, out=view)
            host = out.cpu().numpy()
            assert (host[:, rows:] == 0x5A).all() and (host[:, :, size[0] * px:] == 0x5A).all(), fmt
            for i, s in enumerate([2, 0, 1]):
                exp = want(r, s, fmt, False, (0, 0, 0), size)
                assert np.array_equal(host[i, :rows, :size[0] * px].reshape(exp.shape), exp), (fmt, i)


@pytest.mark.parametrize("fmt,tile", [("nv12", (32, 18)), ("rgba", (24, 18)), ("bgra", (20, 10))])
def test_mosaic_equals_separate_exports(built, fmt, tile):
    p = g.default_params("bars", n=1024, w=320, h=180)
    streams = [6, 0, 3, 3, 1, 5, 2]
    cols = 3
    with g.Renderer(p, batch=7) as r:
        feed(r, 2)
        m = r.export_mosaic(streams, cols, tile, fmt, background=BG)
        sep = r.export_scaled(streams, tile, None, fmt, background=BG).cpu().numpy()
        host = m.cpu().numpy()
        tw, th = tile
        H = 3 * th
        assert host.shape[:2] == ((H * 3 // 2, cols * tw) if fmt == "nv12" else (H, cols * tw))
        for i in range(len(streams)):
            ty, tx = divmod(i, cols)
            if fmt == "nv12":
                y = host[ty * th:(ty + 1) * th, tx * tw:(tx + 1) * tw]
                uv = host[H + ty * th // 2:H + (ty + 1) * th // 2, tx * tw:(tx + 1) * tw]
                assert np.array_equal(np.concatenate([y, uv]), sep[i]), i
            else:
                assert np.array_equal(host[ty * th:(ty + 1) * th, tx * tw:(tx + 1) * tw], sep[i]), i
        # the tiles past the last stream are black
        last = host[2 * th:3 * th, 1 * tw:]
        assert (last == (16 if fmt == "nv12" else 0)).all()
        # into a caller's surface with pitch padding: nothing but the tiles is written
        px = 1 if fmt == "nv12" else 4
        surf = torch.full((host.shape[0], cols * tw * px + 64), 0x33, dtype=torch.uint8, device="cuda")
        r.export_mosaic(streams, cols, tile, fmt, background=BG, out=surf)
        s2 = surf.cpu().numpy()
        assert (s2[:, cols * tw * px:] == 0x33).all()
        flat = host.reshape(host.shape[0], -1)
        written = np.zeros(flat.shape, bool)
        for i in range(len(streams)):
            ty, tx = divmod(i, cols)
            written[ty * th:(ty + 1) * th, tx * tw * px:(tx + 1) * tw * px] = True
            if fmt == "nv12":
                written[H + ty * th // 2:H + (ty + 1) * th // 2, tx * tw:(tx + 1) * tw] = True
        body = s2[:, :cols * tw * px]
        assert np.array_equal(body[written], flat[written]) and (body[~written] == 0x33).all()


def test_export_holds_the_frame_of_its_point_in_call_order(built):
    p = g.default_params("bars", n=1024, w=256, h=128)
    rng = np.random.default_rng(1)
    inputs = [(rng.standard_normal((2, 1024)) * s).astype(np.float32) for s in (0.5, 0.02, 0.4, 0.01)]
    frames = []
    with g.Renderer(p, batch=2) as a:
        for i in range(3):
            a.update(inputs[i], inputs[i][::-1].copy(), True)
            frames.append([a.readback(s) for s in range(2)])
    with g.Renderer(p, batch=2) as r:
        outs = []
        for i in range(3):
            r.update(inputs[i], inputs[i][::-1].copy(), True)
            outs.append(r.export_scaled([0, 1], (64, 40), (0, 8, 256, 120), "rgba", over=True))
        r.update(inputs[3], inputs[3], True)
        r.sync()
        for i in range(3):
            got = outs[i].cpu().numpy()
            for s in range(2):
                exp = scaled_np(frames[i][s], RGBA, True, (0, 0, 0), True, (64, 40), (0, 8, 256, 120))
                assert np.array_equal(got[s], exp), (i, s)


def test_after_and_done_events_order_a_side_stream(built):
    p = g.default_params("wave", n=1024, w=192, h=96)
    with g.Renderer(p, batch=2) as r:
        feed(r, 2)
        frame = r.readback(1)
        side = torch.cuda.Stream()
        out = torch.empty((1, 48, 96 * 4), dtype=torch.uint8, device="cuda")
        after, done = torch.cuda.Event(), torch.cuda.Event()
        with torch.cuda.stream(side):
            torch.cuda._sleep(20_000_000)
            out.fill_(0x5A)
            after.record(side)
        r.export_scaled([1], (96, 48), None, "bgra", over=True, out=out, after=after, done=done)
        feed(r, 1, seed=9)
        with torch.cuda.stream(side):
            side.wait_event(done)
            seen = out.clone()
        side.synchronize()
        exp = scaled_np(frame, BGRA, True, (0, 0, 0), True, (96, 48))
        assert np.array_equal(seen.cpu().numpy().reshape(exp.shape), exp)


def test_device_refusals_leave_nothing_enqueued(built):
    p = g.default_params("bars", n=1024, w=64, h=32)
    with g.Renderer(p, batch=2) as r:
        feed(r, 1)
        L = r._L
        d = g.Export(); d.format = g.EXPORT_NV12; d.pitch = 32
        sc = g.ExportScale(); sc.out_w, sc.out_h = 32, 16
        s = np.zeros(1, np.int32)
        host = np.zeros(4096 + 64, np.uint8)
        dev = torch.empty(4096 + 64, dtype=torch.uint8, device="cuda")
        ok = dev.data_ptr()
        bad = [host.ctypes.data + (-host.ctypes.data) % 16, dev.data_ptr() + 8]
        if torch.cuda.device_count() > 1:
            bad.append(torch.empty(4096, dtype=torch.uint8, device="cuda:1").data_ptr())
        for ptr in bad:
            for dst, uv in (((ptr,), None), ((ok,), (ptr,))):
                l0 = r.launch_count
                rc = L.glava_b200_export_scaled(r._h, s.ctypes.data, 1, (C.c_void_p * 1)(*dst),
                                                None if uv is None else (C.c_void_p * 1)(*uv), C.byref(d), C.byref(sc), None, None)
                assert rc != 0 and b"glava_b200_export_scaled" in L.glava_b200_last_error()
                assert r.launch_count == l0
        rc = L.glava_b200_export_scaled(r._h, s.ctypes.data, 1, (C.c_void_p * 1)(ok), (C.c_void_p * 1)(ok + 1024), C.byref(d),
                                        C.byref(sc), None, None)
        assert rc == 0
        with pytest.raises(g.GlavaError, match="upscaling"):
            r.export_scaled([0], (65, 32))
        with pytest.raises(g.GlavaError, match="leaves"):
            r.export_scaled([0], (8, 8), (60, 0, 8, 8))


def test_sharded_equals_one_handle(built):
    p = g.default_params("graph", n=1024, w=128, h=64)
    rng = np.random.default_rng(4)
    lb = (rng.standard_normal((6, 1024)) * 0.3).astype(np.float32); rb = lb[::-1].copy()
    with g.ShardedRenderer(p, 6, [0, 0, 0]) as sh, g.Renderer(p, batch=6) as one:
        for _ in range(2):
            sh.update(lb, rb); one.update(lb, rb, True)
        order = [5, 0, 3, 3, 1]
        for fmt, over, size, crop in (("nv12", True, (64, 32), None), ("rgba", False, (30, 17), (3, 5, 120, 50)),
                                      ("bgra", True, (128, 64), None)):
            a = sh.export_scaled(order, size, crop, fmt, over=over, background=BG)
            sh.sync()
            b = one.export_scaled(order, size, crop, fmt, over=over, background=BG)
            assert torch.equal(a, b), fmt
        with pytest.raises(g.GlavaError, match="out of range"):
            sh.export_scaled([6], (8, 8))
        with pytest.raises(g.GlavaError, match="glava_b200_sharded_export_scaled"):
            sh.export_scaled([0, 5], (8, 9), fmt="nv12")
