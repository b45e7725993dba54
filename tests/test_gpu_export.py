"""-m gpu: frame export (glava_b200_export_frames, DESIGN 4.10).  What an export writes must equal, bit for bit, the
numpy restatement of tests/test_export_core.py applied to glava_b200_readback of the same stream at the same point in
call order: every module and format, composited or not, native and blended opacity, with the dirty-row marks live,
stale or absent, through the framebuffer ring, styles, repeats, 1024 streams, events, refusals and the sharded handle."""
import ctypes as C

import numpy as np
import pytest

import glava_b200 as g
from tests.test_export_core import nv12_np, over_np

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

BG = (30, 60, 200)


def want(frame, fmt, over, bg, native):
    """the expected export of one read-back frame ([h][w][4], row 0 = bottom)"""
    if fmt == "nv12":
        return nv12_np(frame, bg, native)
    out = (over_np(frame, bg, native).astype(np.uint8) if over else frame)[::-1]
    return out[..., [2, 1, 0, 3]] if fmt == "bgra" else out


def check(r, streams, fmt, over=False, bg=BG, what=""):
    got = r.export_frames(streams, fmt, over=over, background=bg)
    host = got.cpu().numpy() if not isinstance(got, list) else [t.cpu().numpy() for t in got]
    native = bool(r.params.premultiply_alpha)
    for i, s in enumerate(streams):
        exp = want(r.readback(int(s)), fmt, over, bg, native)
        assert np.array_equal(np.asarray(host[i]).reshape(exp.shape), exp), (what, fmt, over, i, int(s))


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
    for w, h, fmts in ((96, 64, ("rgba", "bgra", "nv12")), (97, 63, ("rgba", "bgra"))):
        p = g.default_params(module, n=1024, w=w, h=h, **kw)
        with g.Renderer(p, batch=3) as r:
            feed(r, 3, seed=w)
            for fmt in fmts:
                for over in (False, True):
                    check(r, [0, 1, 2], fmt, over, what=(module, w, h))


def test_bars_1080p_with_live_marks(built):
    p = g.default_params("bars", n=4096, w=1920, h=1080)
    p.lazy_smooth = 1
    with g.Renderer(p, batch=4) as r:
        for step in range(4):
            feed(r, 1, seed=step, scale=0.1 + 0.3 * step)
            for fmt, over in (("nv12", True), ("rgba", True), ("bgra", False)):
                check(r, [3, 0, 2], fmt, over, what=step)


@pytest.mark.parametrize("module", ["bars", "graph", "wave"])
def test_marks_valid_stale_and_reset(built, module):
    p = g.default_params(module, n=1024, w=332, h=180)
    with g.Renderer(p, batch=3) as r:
        for step in range(4):                                          # marks valid from the second pass on
            feed(r, 1, seed=10 + step, scale=0.05 if step % 2 else 0.5)
            check(r, [0, 1, 2], "nv12", what=step)
            check(r, [2], "rgba", True, what=step)
        if module == "bars":                                           # the generic kernel keeps no marks, and back
            q = r.params.copy(); q.bars_mirror_yx = 1
            r.reconfigure(q)
            feed(r, 1, seed=20)
            check(r, [0, 1, 2], "rgba", True, what="mirror")
            q.bars_mirror_yx = 0
            r.reconfigure(q)
            for step in range(2):
                feed(r, 1, seed=21 + step)
                check(r, [0, 1, 2], "nv12", what=("back", step))
        r.sizereq(256, 120)
        check(r, [0, 1], "rgba", True, what="before the resize applies")
        feed(r, 2, seed=30)
        check(r, [0, 1, 2], "nv12", what="resized")
        r.reset_streams([1, 0, 1])
        check(r, [0, 1, 2], "bgra", True, what="after reset")
        feed(r, 1, seed=31)
        check(r, [0, 1, 2], "nv12", what="reset, updated")


@pytest.mark.parametrize("slots", [1, 3])
def test_framebuffer_ring(built, slots):
    p = g.default_params("graph", n=1024, w=128, h=64, fb_slots=slots)
    with g.Renderer(p, batch=5) as r:
        feed(r, 3)
        check(r, [0, 1, 2, 3, 4], "nv12")
        check(r, [4, 0, 4], "rgba", True)


def test_styles_subsets_and_repeats(built):
    p = g.default_params("bars", n=1024, w=160, h=90)
    with g.Renderer(p, batch=6) as r:
        r.set_stream_styles([1, 4], [{"amplify": 500, "fg": "#ff8000"}, {"fg": (0.1, 0.9, 0.2, 1.0), "bg": (0.3, 0.3, 0.3, 0.5)}])
        feed(r, 3)
        check(r, [5, 1, 1, 4, 0, 4], "rgba", True, bg=(255, 255, 255))
        check(r, [4, 2], "nv12", bg=(12, 34, 56))


def test_a_thousand_streams_in_one_launch(built):
    p = g.default_params("bars", n=512, w=64, h=32)
    with g.Renderer(p, batch=1024) as r:
        feed(r, 2)
        l0 = r.launch_count
        got = r.export_frames(range(1024), "nv12").cpu().numpy()
        assert r.launch_count == l0 + 1
        for s in list(range(0, 1024, 7)) + [1023]:
            assert np.array_equal(got[s], want(r.readback(s), "nv12", True, (0, 0, 0), True)), s


def test_export_holds_the_frame_of_its_point_in_call_order(built):
    p = g.default_params("bars", n=1024, w=256, h=128)
    rng = np.random.default_rng(1)
    inputs = [(rng.standard_normal((2, 1024)) * s).astype(np.float32) for s in (0.5, 0.02, 0.4, 0.01)]
    frames = []
    with g.Renderer(p, batch=2) as a:                                   # the frames, one sync per update
        for i in range(3):
            a.update(inputs[i], inputs[i][::-1].copy(), True)
            frames.append([a.readback(s) for s in range(2)])
    with g.Renderer(p, batch=2) as r:                                   # the same calls without a sync in between
        outs = []
        for i in range(3):
            r.update(inputs[i], inputs[i][::-1].copy(), True)
            outs.append(r.export_frames([0, 1], "rgba", over=True))
        r.update(inputs[3], inputs[3], True)
        r.sync()
        for i in range(3):
            got = outs[i].cpu().numpy()
            for s in range(2):
                assert np.array_equal(got[s], want(frames[i][s], "rgba", True, (0, 0, 0), True)), (i, s)


def test_after_and_done_events_order_a_side_stream(built):
    p = g.default_params("wave", n=1024, w=192, h=96)
    with g.Renderer(p, batch=2) as r:
        feed(r, 2)
        frame = r.readback(1)
        side = torch.cuda.Stream()
        out = torch.empty((1, 96, 192 * 4), dtype=torch.uint8, device="cuda")
        after, done = torch.cuda.Event(), torch.cuda.Event()
        with torch.cuda.stream(side):
            torch.cuda._sleep(20_000_000)                               # the producer is still busy with the buffer
            out.fill_(0x5A)
            after.record(side)
        r.export_frames([1], "bgra", over=True, out=out, after=after, done=done)
        feed(r, 1, seed=9)                                              # the next frame does not wait for the consumer
        with torch.cuda.stream(side):
            side.wait_event(done)
            seen = out.clone()
        side.synchronize()
        assert np.array_equal(seen.cpu().numpy().reshape(96, 192, 4), want(frame, "bgra", True, (0, 0, 0), True))


def test_device_refusals_leave_nothing_enqueued(built):
    p = g.default_params("bars", n=1024, w=64, h=32)
    with g.Renderer(p, batch=2) as r:
        feed(r, 1)
        L = r._L
        d = g.Export(); d.format = g.EXPORT_RGBA; d.pitch = 256
        s = np.zeros(1, np.int32)
        host = np.zeros(64 * 32 * 4 + 64, np.uint8)
        dev = torch.empty(64 * 32 * 4 + 64, dtype=torch.uint8, device="cuda")
        bad = [host.ctypes.data + (-host.ctypes.data) % 16, dev.data_ptr() + 8]
        if torch.cuda.device_count() > 1:
            other = torch.empty(64 * 32 * 4, dtype=torch.uint8, device="cuda:1")
            bad.append(other.data_ptr())
        for ptr in bad:
            l0 = r.launch_count
            rc = L.glava_b200_export_frames(r._h, s.ctypes.data, 1, (C.c_void_p * 1)(ptr), C.byref(d), None, None)
            assert rc != 0 and b"glava_b200_export_frames" in L.glava_b200_last_error()
            assert r.launch_count == l0
        rc = L.glava_b200_export_frames(r._h, s.ctypes.data, 1, (C.c_void_p * 1)(dev.data_ptr()), C.byref(d), None, None)
        assert rc == 0
        with pytest.raises(g.GlavaError, match="out of range"):
            r.export_frames([2], "rgba")


def test_sharded_equals_one_handle(built):
    p = g.default_params("graph", n=1024, w=128, h=64)
    rng = np.random.default_rng(4)
    lb = (rng.standard_normal((6, 1024)) * 0.3).astype(np.float32); rb = lb[::-1].copy()
    with g.ShardedRenderer(p, 6, [0, 0, 0]) as sh, g.Renderer(p, batch=6) as one:
        for _ in range(2):
            sh.update(lb, rb); one.update(lb, rb, True)
        order = [5, 0, 3, 3, 1]
        for fmt, over in (("nv12", True), ("rgba", False), ("bgra", True)):
            a = sh.export_frames(order, fmt, over=over, background=BG)
            sh.sync()
            b = one.export_frames(order, fmt, over=over, background=BG)
            assert torch.equal(a, b), fmt
        with pytest.raises(g.GlavaError, match="out of range"):
            sh.export_frames([6], "rgba")


def test_python_shapes_and_pitches(built):
    p = g.default_params("bars", n=1024, w=100, h=50)
    with g.Renderer(p, batch=3) as r:
        feed(r, 2)
        a = r.export_frames([0, 2], "rgba")
        assert a.shape == (2, 50, 100, 4) and a.dtype == torch.uint8 and a.stride(1) == 400 and a.stride(2) == 4
        b = r.export_frames([1], "nv12")
        assert b.shape == (1, 75, 100) and b.stride(1) == 112                  # rows padded to 16 bytes
        base = torch.zeros((2, 50, 512), dtype=torch.uint8, device="cuda")
        c = r.export_frames([2, 0], "bgra", over=True, out=base)
        assert c is base and (base[:, :, 400:] == 0).all()
        lst = [torch.zeros((75, 128), dtype=torch.uint8, device="cuda") for _ in range(2)]
        d = r.export_frames([1, 1], "nv12", out=lst)
        assert d is lst and torch.equal(lst[0][:, :100], b[0]) and torch.equal(lst[1][:, :100], b[0])
        assert torch.equal(base[0, :, :400].reshape(50, 100, 4), torch.from_numpy(want(r.readback(2), "bgra", True, (0, 0, 0), True)).cuda())
        with pytest.raises(ValueError):
            r.export_frames([0], "rgba", out=torch.zeros((1, 49, 400), dtype=torch.uint8, device="cuda"))
        with pytest.raises(g.GlavaError, match="pitch"):
            r.export_frames([0], "nv12", out=torch.zeros((1, 75, 104), dtype=torch.uint8, device="cuda"))
