"""-m gpu: encoder ladder (glava_b200_export_ladder, DESIGN 4.13).  Every rung of a ladder must equal, bit for bit, the
standalone call it stands for — glava_b200_export_frames for a whole-frame rung, glava_b200_export_scaled otherwise —
issued at the same point in call order: every module and opacity with a mixed ladder (NV12 beside composited RGBA and a
BGRA thumbnail), live / stale / absent marks, the framebuffer ring, styles, repeats, widths that are not a multiple of 4,
1024 streams x 4 rungs in one launch, untouched bytes around every destination, ordering, events, refusals and the
sharded handle."""
import ctypes as C

import numpy as np
import pytest

import glava_b200 as g

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

BG = (30, 60, 200)
LADDER_1080 = [dict(size=(1920, 1080)), dict(size=(1280, 720)), dict(size=(640, 360)), dict(size=(480, 270))]


def even(v):
    return max(2, int(v) // 2 * 2)


def mixed(w, h):
    """a whole-frame NV12 rung, a 2/3 NV12 rung, a cropped RGBA rung composited over BG and a BGRA thumbnail"""
    return [dict(size=None, fmt="nv12", background=BG), dict(size=(even(w * 2 / 3), even(h * 2 / 3)), fmt="nv12"),
            dict(size=(w // 4, h // 4), crop=(w // 8, h // 8, w // 2, h // 2), fmt="rgba", over=True, background=BG),
            dict(size=(max(w // 8, 1), max(h // 8, 1)), fmt="bgra")]


def standalone(r, streams, rung):
    """the call rung stands for: export_frames for the whole frame at its own size, else export_scaled"""
    p = r.params
    size, crop = rung.get("size") or (p.w, p.h), rung.get("crop")
    kw = dict(over=rung.get("over", False), background=rung.get("background", (0, 0, 0)))
    fmt = rung.get("fmt", "nv12")
    if tuple(size) == (p.w, p.h) and crop in (None, (0, 0, p.w, p.h)):
        return r.export_frames(streams, fmt, **kw)
    return r.export_scaled(streams, size, crop, fmt, **kw)


def check(r, streams, rungs, what=""):
    l0 = r.launch_count
    got = r.export_ladder(streams, rungs)
    assert r.launch_count == l0 + 1, what
    assert len(got) == len(rungs)
    for j, rung in enumerate(rungs):
        want = standalone(r, streams, rung)
        assert got[j].shape == want.shape and torch.equal(got[j], want), (what, j, rung)


def feed(r, steps, seed=0, scale=0.3):
    rng = np.random.default_rng(seed)
    n = r.params.n
    for _ in range(steps):
        lb = (rng.standard_normal((r.batch, n)) * scale).astype(np.float32)
        rb = (rng.standard_normal((r.batch, n)) * scale).astype(np.float32)
        r.update(lb, rb, True)


@pytest.mark.parametrize("native", [True, False], ids=["native", "blended"])
@pytest.mark.parametrize("module", g.MODULES)
def test_every_module_and_opacity_with_a_mixed_ladder(built, module, native):
    kw = {} if native else dict(premultiply_alpha=0, clear_color=[0.1, 0.2, 0.3, 1.0])
    for w, h in ((96, 64), (98, 62)):                                  # 98: rows of a width that is not a multiple of 4
        p = g.default_params(module, n=1024, w=w, h=h, **kw)
        with g.Renderer(p, batch=3) as r:
            feed(r, 3, seed=w)
            check(r, [0, 2, 1], mixed(w, h), (module, w, h))


def test_bars_1080p_with_live_stale_and_no_marks(built):
    p = g.default_params("bars", n=4096, w=1920, h=1080)
    p.lazy_smooth = 1
    rungs = LADDER_1080 + [dict(size=(97, 13), crop=(64, 900, 1800, 180), fmt="rgba", over=True)]
    with g.Renderer(p, batch=3) as r:
        for step in range(3):                                          # live marks from the second pass on
            feed(r, 1, seed=step, scale=0.1 + 0.3 * step)
            check(r, [2, 0], rungs, step)
        q = r.params.copy(); q.bars_mirror_yx = 1                     # the generic kernel keeps no marks
        r.reconfigure(q)
        feed(r, 1, seed=20)
        check(r, [0, 1, 2], rungs, "no marks")
        q.bars_mirror_yx = 0                                           # marks stale for one pass, then valid again
        r.reconfigure(q)
        for step in range(2):
            feed(r, 1, seed=21 + step)
            check(r, [0, 1, 2], rungs, ("back", step))


@pytest.mark.parametrize("slots", [1, 3])
def test_framebuffer_ring(built, slots):
    p = g.default_params("graph", n=1024, w=130, h=64, fb_slots=slots)
    with g.Renderer(p, batch=5) as r:
        feed(r, 3)
        check(r, [0, 1, 2, 3, 4], mixed(130, 64))
        check(r, [4, 0, 4], [dict(size=(40, 20), crop=(10, 10, 100, 40), fmt="rgba", over=True), dict(size=None, fmt="bgra")])


def test_styles_and_repeats(built):
    p = g.default_params("bars", n=1024, w=162, h=90)
    with g.Renderer(p, batch=6) as r:
        r.set_stream_styles([1, 4], [{"amplify": 500, "fg": "#ff8000"}, {"fg": (0.1, 0.9, 0.2, 1.0), "bg": (0.3, 0.3, 0.3, 0.5)}])
        feed(r, 3)
        check(r, [5, 1, 1, 4, 0, 4], mixed(162, 90) + [dict(size=(40, 30), fmt="rgba", over=True, background=(255, 255, 255))])


def test_a_thousand_streams_by_four_rungs_in_one_launch(built):
    p = g.default_params("bars", n=512, w=1920, h=1080)
    p.lazy_smooth = 1
    with g.Renderer(p, batch=1024) as r:
        feed(r, 2)
        l0 = r.launch_count
        got = r.export_ladder(range(1024), LADDER_1080)
        assert r.launch_count == l0 + 1
        for j, rung in enumerate(LADDER_1080):
            want = standalone(r, range(1024), rung)
            assert torch.equal(got[j], want), j
            del want


def test_nothing_outside_the_rectangles_is_written(built):
    p = g.default_params("wave", n=1024, w=300, h=200)
    rungs = [dict(size=None, fmt="nv12"), dict(size=(37, 21), fmt="rgba"), dict(size=(50, 30), fmt="nv12"),
             dict(size=(300, 200), fmt="bgra", over=True)]
    with g.Renderer(p, batch=3) as r:
        feed(r, 2)
        outs, views = [], []
        for rung in rungs:
            w, h = rung["size"] or (300, 200)
            rows = h * 3 // 2 if rung["fmt"] == "nv12" else h
            out = torch.full((3, rows + 3, 1280), 0x5A, dtype=torch.uint8, device="cuda")
            outs.append(out)
            views.append(out[:, :rows])
        r.export_ladder([2, 0, 1], rungs, out=views)
        for rung, out in zip(rungs, outs):
            w, h = rung["size"] or (300, 200)
            px = 1 if rung["fmt"] == "nv12" else 4
            rows = h * 3 // 2 if rung["fmt"] == "nv12" else h
            host = out.cpu().numpy()
            assert (host[:, rows:] == 0x5A).all() and (host[:, :, w * px:] == 0x5A).all(), rung
            want = standalone(r, [2, 0, 1], rung).cpu().numpy()
            assert np.array_equal(host[:, :rows, :w * px].reshape(want.shape), want), rung


def test_export_holds_the_frame_of_its_point_in_call_order(built):
    p = g.default_params("bars", n=1024, w=256, h=128)
    rng = np.random.default_rng(1)
    inputs = [(rng.standard_normal((2, 1024)) * s).astype(np.float32) for s in (0.5, 0.02, 0.4, 0.01)]
    rungs = [dict(size=None), dict(size=(64, 40), crop=(0, 8, 256, 120), fmt="rgba", over=True), dict(size=(128, 64))]
    with g.Renderer(p, batch=2) as a, g.Renderer(p, batch=2) as r:
        wants, outs = [], []
        for i in range(3):
            a.update(inputs[i], inputs[i][::-1].copy(), True)
            wants.append([standalone(a, [0, 1], rung).clone() for rung in rungs])
            r.update(inputs[i], inputs[i][::-1].copy(), True)
            outs.append(r.export_ladder([0, 1], rungs))
        r.update(inputs[3], inputs[3], True)
        r.sync()
        for i in range(3):
            for j in range(len(rungs)):
                assert torch.equal(outs[i][j], wants[i][j]), (i, j)


def test_after_and_done_events_order_a_side_stream(built):
    p = g.default_params("wave", n=1024, w=192, h=96)
    rungs = [dict(size=(96, 48), fmt="bgra", over=True), dict(size=(64, 32))]
    with g.Renderer(p, batch=2) as r:
        feed(r, 2)
        want = [standalone(r, [1], rung).clone() for rung in rungs]
        side = torch.cuda.Stream()
        outs = [torch.empty((1, 48, 96 * 4), dtype=torch.uint8, device="cuda"),
                torch.empty((1, 48, 64), dtype=torch.uint8, device="cuda")]
        after, done = torch.cuda.Event(), torch.cuda.Event()
        with torch.cuda.stream(side):
            torch.cuda._sleep(20_000_000)
            for o in outs:
                o.fill_(0x5A)
            after.record(side)
        r.export_ladder([1], rungs, out=outs, after=after, done=done)
        feed(r, 1, seed=9)
        with torch.cuda.stream(side):
            side.wait_event(done)
            seen = [o.clone() for o in outs]
        side.synchronize()
        for j in range(2):
            assert torch.equal(seen[j].reshape(want[j].shape), want[j]), j


def test_device_refusals_leave_nothing_enqueued(built):
    p = g.default_params("bars", n=1024, w=64, h=32)
    with g.Renderer(p, batch=2) as r:
        feed(r, 1)
        L = r._L
        rungs = (g.ExportRung * 2)()
        rungs[0].desc.format = g.EXPORT_NV12; rungs[0].desc.pitch = 64
        rungs[0].scale.out_w, rungs[0].scale.out_h = 64, 32
        rungs[1].desc.format = g.EXPORT_RGBA; rungs[1].desc.pitch = 64
        rungs[1].scale.out_w, rungs[1].scale.out_h = 16, 8
        s = np.zeros(1, np.int32)
        host = np.zeros(8192 + 64, np.uint8)
        dev = torch.empty(8192 + 64, dtype=torch.uint8, device="cuda")
        ok, ok2 = dev.data_ptr(), dev.data_ptr() + 4096
        bad = [host.ctypes.data + (-host.ctypes.data) % 16, dev.data_ptr() + 8]
        if torch.cuda.device_count() > 1:
            bad.append(torch.empty(4096, dtype=torch.uint8, device="cuda:1").data_ptr())
        for ptr in bad:
            for dst, uv, j in (((ptr, ok2), None, 0), ((ok, ptr), None, 1), ((ok, ok2), (ptr, None), 0)):
                l0 = r.launch_count
                rc = L.glava_b200_export_ladder(r._h, s.ctypes.data, 1, rungs, 2, (C.c_void_p * 2)(*dst),
                                                None if uv is None else (C.c_void_p * 2)(*uv), None, None)
                assert rc != 0 and f"glava_b200_export_ladder: rung {j}".encode() in L.glava_b200_last_error()
                assert r.launch_count == l0
        l0 = r.launch_count
        assert L.glava_b200_export_ladder(r._h, s.ctypes.data, 1, rungs, 2, (C.c_void_p * 2)(ok, ok2), None, None, None) == 0
        assert r.launch_count == l0 + 1
        with pytest.raises(g.GlavaError, match="rung 1: .*upscaling"):
            r.export_ladder([0], [dict(size=(32, 16)), dict(size=(65, 32))])
        with pytest.raises(g.GlavaError, match="nrungs 9"):
            r.export_ladder([0], [dict(size=(8, 8))] * 9)


def test_sharded_equals_one_handle(built):
    p = g.default_params("graph", n=1024, w=128, h=64)
    rng = np.random.default_rng(4)
    lb = (rng.standard_normal((6, 1024)) * 0.3).astype(np.float32); rb = lb[::-1].copy()
    with g.ShardedRenderer(p, 6, [0, 0, 0]) as sh, g.Renderer(p, batch=6) as one:
        for _ in range(2):
            sh.update(lb, rb); one.update(lb, rb, True)
        order = [5, 0, 3, 3, 1]
        rungs = mixed(128, 64)
        a = sh.export_ladder(order, rungs)
        sh.sync()
        b = one.export_ladder(order, rungs)
        for j in range(len(rungs)):
            assert torch.equal(a[j], b[j]), j
        with pytest.raises(g.GlavaError, match="out of range"):
            sh.export_ladder([6], rungs)
        with pytest.raises(g.GlavaError, match="glava_b200_sharded_export_ladder: rung 1"):
            sh.export_ladder([0, 5], [dict(size=(8, 8)), dict(size=(8, 9), fmt="nv12")])
