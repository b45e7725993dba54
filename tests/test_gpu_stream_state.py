"""-m gpu: reset, save and load of individual streams (glava_b200_reset_streams / _save_streams / _load_streams).

A reset stream must render exactly what a newly created batch-1 renderer renders when fed the same calls; a saved stream
loaded into any slot of any renderer with the same parameters must continue exactly as the source would have.  Every
comparison is bit for bit over spectra, textures and frames, over the configurations of test_gpu_masked.py plus
setbufscale 2."""
import ctypes as C

import numpy as np
import pytest

import glava_b200 as g

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

CASES = [
    ("bars", dict(), "pipeline B, full K5"),
    ("bars", dict(lazy_smooth=1), "pipeline B, lazy K5"),
    ("bars", dict(accel_fft=0), "pipeline A"),
    ("bars", dict(accel_fft=0, avg_frames=3, lazy_smooth=1), "pipeline A, F=3, lazy"),
    ("graph", dict(avg_frames=7), "generic F"),
    ("circle", dict(), "circle"),
    ("wave", dict(), "wave chain"),
    ("bars", dict(transform_smooth=1), "appended transform_smooth"),
    ("radial", dict(smooth_pass=0), "no K5"),
    ("bars", dict(bufscale=2), "setbufscale 2"),
]
IDS = [c[2] for c in CASES]
N = 1024


def _params(module, over):
    return g.default_params(module, n=N, w=128, h=64, **over)


class Feed:
    """per-step inputs of `logical` streams; a renderer maps each of its slots to a logical stream (-1: inputs of its own)"""

    def __init__(self, seed, logical):
        self.rng = np.random.default_rng(seed)
        self.logical = logical

    def step(self, p_uneven=0.55):
        m = self.rng.random(self.logical) < p_uneven if p_uneven < 1 else np.ones(self.logical, bool)
        return m, (self.rng.random((self.logical, N), np.float32) - 0.5) * 0.3, (self.rng.random((self.logical, N), np.float32) - 0.5) * 0.3


def _apply(r, slots, m, l, rr, rng, plain=False):
    """update renderer r: slot s takes logical stream slots[s] (or fresh noise and a random flag for -1)"""
    b = r.batch
    lb = (rng.random((b, N), np.float32) - 0.5) * 0.3; rb = (rng.random((b, N), np.float32) - 0.5) * 0.3
    mask = rng.random(b) < 0.5
    for s, q in enumerate(slots):
        if q >= 0:
            lb[s], rb[s], mask[s] = l[q], rr[q], m[q]
    if plain:
        r.update(lb, rb, True)
    else:
        r.update_masked(lb, rb, mask)


def _same(ra, sa, rb, sb, what, frames=True):
    (al, ar), (bl, br) = ra.spectrum(), rb.spectrum()
    assert np.array_equal(al[sa].view(np.uint32), bl[sb].view(np.uint32)) and np.array_equal(ar[sa].view(np.uint32), br[sb].view(np.uint32)), what
    (al, ar), (bl, br) = ra.textures(), rb.textures()
    assert np.array_equal(al[sa], bl[sb]) and np.array_equal(ar[sa], br[sb]), what
    if frames:
        assert np.array_equal(ra.readback(sa), rb.readback(sb)), what


@pytest.mark.parametrize("module,over,what", CASES, ids=IDS)
def test_reset_equals_a_fresh_renderer(built, module, over, what):
    p = _params(module, over)
    batch, steps, t_reset, reset = 5, 12, 6, (1, 3)
    feed = Feed(hash(what) & 0xffff, batch)
    singles = [g.Renderer(p, batch=1) for _ in range(batch)]
    try:
        with g.Renderer(p, batch=batch) as r:
            for t in range(steps):
                m, l, rr = feed.step()
                m[0] = t < 2 or m[0]
                if t == t_reset:
                    mask = np.zeros(batch, bool); mask[list(reset)] = True
                    r.reset_streams(mask)
                    for s in reset:
                        singles[s].close(); singles[s] = g.Renderer(p, batch=1)
                    m[list(reset)] = False                  # the first call after the reset re-rasters (modified = 0)
                r.update_masked(l, rr, m)
                for s in range(batch):
                    singles[s].update(l[s:s + 1], rr[s:s + 1], bool(m[s]))
                if t >= t_reset - 1:
                    for s in range(batch):
                        _same(r, s, singles[s], 0, (what, t, s))
                if t == t_reset:
                    for s in reset:
                        assert not r.textures()[0][s].any()
            assert r.textures()[0].any()
    finally:
        for q in singles:
            q.close()


def _history(r, feed, slots, steps, rng, plain=False):
    for _ in range(steps):
        m, l, rr = feed.step()
        _apply(r, slots, m, l, rr, rng, plain)


@pytest.mark.parametrize("lock_step", [False, True], ids=["desync", "lock-step"])
@pytest.mark.parametrize("module,over,what", CASES, ids=IDS)
def test_save_load_continues_the_stream(built, module, over, what, lock_step):
    p = _params(module, over)
    rng = np.random.default_rng(len(what) * 7 + lock_step)
    own = Feed(hash(what) & 0xfff, 5)
    with g.Renderer(p, batch=5) as x, g.Renderer(p, batch=7) as y:
        _history(x, own, list(range(5)), 8, rng)                              # X: desynchronised cursors
        _history(y, Feed(99, 7), list(range(7)), 4 if lock_step else 9, rng, plain=lock_step)
        blobs = x.save_streams(range(5))
        assert blobs.shape == (5, g.stream_state_bytes(p))
        perm = [6, 0, 4, 2, 5]                                                 # X stream i -> Y slot perm[i]
        y.load_streams(perm, blobs)
        for i in range(5):
            _same(x, i, y, perm[i], (what, "after load", i), frames=False)
        slots_y = [-1] * 7
        for i, s in enumerate(perm):
            slots_y[s] = i
        feed = Feed(5, 5)
        for t in range(7):
            m, l, rr = feed.step(1.0 if lock_step else 0.55)
            _apply(x, list(range(5)), m, l, rr, rng, plain=lock_step)
            _apply(y, slots_y, m, l, rr, rng, plain=lock_step)
            if t in (0, 1, 4, 6):
                for i in range(5):
                    _same(x, i, y, perm[i], (what, t, i))


@pytest.mark.parametrize("module,over,what", CASES, ids=IDS)
def test_swap_and_roll_back(built, module, over, what):
    """two streams swapped within one renderer; and a whole renderer rolled back to a save k steps earlier"""
    p = _params(module, over)
    rng = np.random.default_rng(3)
    with g.Renderer(p, batch=5) as a, g.Renderer(p, batch=5) as ref:
        feed = Feed(21, 5)
        for _ in range(6):                                                     # identical histories
            m, l, rr = feed.step()
            a.update_masked(l, rr, m); ref.update_masked(l, rr, m)
        blobs = a.save_streams([1, 3])
        a.load_streams([3, 1], blobs)                                          # swap
        swap = [0, 3, 2, 1, 4]                                                 # a's slot s holds ref's stream swap[s]
        at_t = a.save_streams(range(5))
        for _ in range(3):                                                     # k = 3 steps that are rolled back
            m, l, rr = feed.step()
            _apply(a, swap, m, l, rr, rng)
        a.load_streams(range(5), at_t)
        for t in range(6):
            m, l, rr = feed.step()
            _apply(a, swap, m, l, rr, rng)
            ref.update_masked(l, rr, m)
            if t in (0, 2, 5):
                for s in range(5):
                    _same(a, s, ref, swap[s], (what, t, s))


def test_device_fifo_rings_move_with_the_stream(built):
    p = _params("bars", dict())
    hop = 256
    rng = np.random.default_rng(17)
    with g.Renderer(p, batch=3) as a, g.Renderer(p, batch=4) as b:
        for t in range(6):
            a.ingest_fifo(rng.integers(-20000, 20000, size=(3, hop * 2), dtype=np.int16)); a.update_rings(True)
            if t < 4:
                b.ingest_fifo(rng.integers(-20000, 20000, size=(4, hop * 2), dtype=np.int16)); b.update_rings(True)
        b.load_streams([3, 1], a.save_streams([0, 2]))
        for t in range(6):                                                     # 6 * 256 frames: the old ring content leaves
            ca = rng.integers(-20000, 20000, size=(3, hop * 2), dtype=np.int16)
            cb = rng.integers(-20000, 20000, size=(4, hop * 2), dtype=np.int16)
            cb[3], cb[1] = ca[0], ca[2]
            a.ingest_fifo(ca); b.ingest_fifo(cb)
            if t % 2 == 0:
                a.update_rings(True); b.update_rings(True)
            _same(a, 0, b, 3, ("fifo", t, 0)); _same(a, 2, b, 1, ("fifo", t, 2))


def test_sharded_reset_and_move_between_shards(built):
    p = _params("bars", dict())
    batch = 11
    rng = np.random.default_rng(8)
    with g.ShardedRenderer(p, batch, [0, 0, 0]) as sh, g.Renderer(p, batch=batch) as one:
        shards = sh.shards
        assert [f for _d, f, _c in shards] == [0, 4, 8]
        lb = np.zeros((batch, N), np.float32); rb = np.zeros_like(lb)

        def step(mask=None):
            lb[:] = (rng.random((batch, N), np.float32) - 0.5) * 0.3; rb[:] = (rng.random((batch, N), np.float32) - 0.5) * 0.3
            sh.update(lb, rb, mask)
            if mask is None:
                one.update(lb, rb, True)
            else:
                one.update_masked(lb, rb, mask)

        for t in range(5):
            step(None if t % 2 == 0 else rng.random(batch) < 0.6)
        mask = np.zeros(batch, bool); mask[[2, 9]] = True
        sh.reset_streams(mask); one.reset_streams(mask)
        blob = sh.save_streams([1])                                           # shard 0 -> shard 2
        assert np.array_equal(blob[:, 4096:], one.save_streams([1])[:, 4096:])
        sh.load_streams([10], blob); one.load_streams([10], one.save_streams([1]))
        for t in range(4):
            step(rng.random(batch) < 0.6 if t % 2 else None)
        sh.sync(); one.sync()
        a, b = sh.textures(), one.textures()
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[0].any()
        for s in range(batch):
            assert np.array_equal(sh.readback(s), one.readback(s)), s
        with pytest.raises(g.GlavaError, match="listed twice"):
            sh.load_streams([4, 4], np.concatenate([blob, blob]))


def test_calls_are_ordered_without_sync(built):
    """updates, resets and loads back to back with asynchronous read-backs equal the same calls with a sync after each"""
    p = _params("bars", dict(lazy_smooth=1))
    batch, steps = 4, 10
    feed = Feed(31, batch)
    seq = [feed.step() for _ in range(steps)]
    with g.Renderer(p, batch=batch) as src:
        for m, l, rr in seq[:3]:
            src.update_masked(l, rr, m)
        blobs = src.save_streams([0, 1])

    def run(sync):
        outs = []
        with g.Renderer(p, batch=batch) as r:
            for t, (m, l, rr) in enumerate(seq):
                if t == 3:
                    r.reset_streams([0, 1, 0, 1])
                if t == 6:
                    r.load_streams([2, 0], blobs)
                if t in (3, 6) and sync:
                    r.sync()
                r.update_masked(l, rr, m)
                for s in range(batch):
                    if sync:
                        r.sync(); outs.append(r.readback(s))
                    else:
                        buf = g.pinned_empty((p.h, p.w, 4), np.uint8); r.readback_async(s, buf); outs.append(buf)
                if t in (3, 6) and not sync:
                    buf = g.pinned_empty((p.h, p.w, 4), np.uint8); r.readback_async(1, buf); outs.append(buf)
                elif t in (3, 6):
                    r.sync(); outs.append(r.readback(1))
            r.sync()
            return [o.copy() for o in outs], r.textures()

    a, ta = run(False)
    b, tb = run(True)
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert np.array_equal(x, y), i
    assert np.array_equal(ta[0], tb[0]) and np.array_equal(ta[1], tb[1])


def _snapshot(r):
    (tl, tr) = r.textures()
    return tl, tr, [r.readback(s) for s in range(r.batch)]


def _unchanged(r, snap):
    tl, tr, frames = snap
    a, b = r.textures()
    assert np.array_equal(a, tl) and np.array_equal(b, tr)
    for s in range(r.batch):
        assert np.array_equal(r.readback(s), frames[s])


def test_rejections_leave_the_destination_untouched(built):
    z = np.zeros((2, 512), np.float32)
    pi = g.default_params("wave", n=512, w=64, h=32, interpolate=1, fr=400.0)
    with g.Renderer(pi, batch=2) as r:
        r.update(z + 0.1, z + 0.1, True)
        snap = _snapshot(r)
        one, buf = (C.c_int * 1)(0), C.create_string_buffer(1 << 16)
        for call in (lambda: r.reset_streams([1, 0]),
                     lambda: g.api._check(r._L.glava_b200_save_streams(r._h, one, 1, buf)),
                     lambda: g.api._check(r._L.glava_b200_load_streams(r._h, one, 1, buf))):
            with pytest.raises(g.GlavaError, match="interpolation"):
                call()
        _unchanged(r, snap)

    p = _params("bars", dict())
    rng = np.random.default_rng(4)
    lb = (rng.random((3, N), np.float32) - 0.5) * 0.3
    with g.Renderer(p, batch=3) as a, g.Renderer(_params("bars", dict(bars_amplify=p.bars_amplify * 2)), batch=3) as other, \
            g.Renderer(p, batch=3) as d:
        for r in (a, other, d):
            r.update(lb, lb[::-1].copy(), True)
        d.update(lb[::-1].copy(), lb, True)
        good = a.save_streams([0, 1])
        snap = _snapshot(d)
        with pytest.raises(g.GlavaError, match="other parameters"):
            d.load_streams([0, 1], other.save_streams([0, 1]))
        for off, what in ((0, "magic"), (4, "version"), (8, "size"), (16, "size")):
            bad = good.copy(); bad[1, off] ^= 0x5a
            with pytest.raises(g.GlavaError, match=what):
                d.load_streams([0, 1], bad)
        for streams, what in (([0, 3], "out of range"), ([-1, 0], "out of range"), ([2, 2], "twice")):
            with pytest.raises(g.GlavaError, match=what):
                d.load_streams(streams, good)
            with pytest.raises(g.GlavaError, match=what):
                d.save_streams(streams)
        _unchanged(d, snap)
        d.load_streams([2, 0], good)                                          # and a good blob still loads
        _same(a, 0, d, 2, "good", frames=False)
