"""-m gpu: the device FIFO ingest (glava_b200_ingest_fifo / _ingest_float, fifo_ingest_kernel) bit for bit against a numpy
restatement of fifo.c:89-110 and pulse_input.c:146-174, read straight out of the rings.

The rings are read from save_streams blobs: the FIFO ring is the last segment of each channel (stream_state_core.h).  The
restatement: the ring slides by `frames` and the new frames land at its end; int16 converts as float32(a) / float32(65535);
the int16 mono mix (channels = 1 or setmirror) is the C integer mean (a + b) / 2, truncating toward zero, then converted;
the float mono mix is (a + b) / 2 in float32.  Stereo rings compare bit for bit, NaN payloads included; the mono float mix
compares NaN for NaN (the payload of a sum is the hardware's)."""
import numpy as np
import pytest

import glava_b200 as g

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

HEADER = g.STATE_HEADER_BYTES
EINVAL = -1                      # GLAVA_B200_EINVAL


# ---- the restatement ----------------------------------------------------------------------------------------------------
def ingest_ref(rl, rr, chunk, mono, is_float):
    """one stream's rings after one ingest of `chunk` (interleaved L, R)"""
    frames = chunk.shape[0] // 2
    n = rl.shape[0]
    rl = np.concatenate([rl[frames:], np.zeros(frames, np.float32)]) if frames < n else np.zeros(n, np.float32)
    rr = np.concatenate([rr[frames:], np.zeros(frames, np.float32)]) if frames < n else np.zeros(n, np.float32)
    if is_float:
        a = chunk[0::2].astype(np.float32); b = chunk[1::2].astype(np.float32)
        with np.errstate(all="ignore"):
            l, r = ((a + b) / np.float32(2),) * 2 if mono else (a, b)
    else:
        a = chunk[0::2].astype(np.int32); b = chunk[1::2].astype(np.int32)
        if mono:
            s = a + b
            q = np.where(s < 0, -((-s) // 2), s // 2)          # C's int division truncates toward zero (not floor: //)
            l = r = q.astype(np.float32) / np.float32(65535)
        else:
            l = a.astype(np.float32) / np.float32(65535); r = b.astype(np.float32) / np.float32(65535)
    rl[n - frames:] = l; rr[n - frames:] = r
    return rl, rr


def rings_of(r, streams=None):
    """(l, r) FIFO rings [streams][n_in] read from save_streams blobs"""
    p = r.params
    streams = list(range(r.batch)) if streams is None else list(streams)
    n_in = p.n; n = p.n // p.bufscale
    k = p.copy()
    if k.transform_smooth == 1 and k.module != g.MODULES.index("wave"):
        k.accel_fft = 0
    esz = 2 if k.accel_fft else 4
    chan = (1 + p.avg_frames) * n * esz + n * 4 + n * 2 + n * 2 + n_in * 4
    blobs = r.save_streams(streams)
    assert blobs.shape[1] == HEADER + 2 * chan
    out = []
    for ch in (0, 1):
        off = HEADER + ch * chan + chan - n_in * 4
        out.append(np.ascontiguousarray(blobs[:, off: off + n_in * 4]).view(np.float32))
    return out


def same_ring(got, want, mono_float):
    if not mono_float:
        return np.array_equal(got.view(np.uint32), want.view(np.uint32))
    nan = np.isnan(want)
    return np.array_equal(np.isnan(got), nan) and np.array_equal(got.view(np.uint32)[~nan], want.view(np.uint32)[~nan])


# ---- inputs -------------------------------------------------------------------------------------------------------------
INT_EDGES = [(-32768, -32768), (32767, 32767), (-32768, 32767), (32767, -32768), (-3, 0), (-1, 0), (1, 0), (-32767, -2),
             (-5, 2), (0, -1), (3, 0), (0, 0)]
F32 = np.float32
FLOAT_EDGES = [(F32(0.0), F32(-0.0)), (F32(-0.0), F32(-0.0)), (F32(1e-45), F32(1e-45)), (F32(-1e-40), F32(3e-39)),
               (F32(np.inf), F32(1.0)), (F32(-np.inf), F32(np.inf)), (F32(3e38), F32(3e38)), (F32(-3.4e38), F32(-3.4e38)),
               (F32(3.4028235e38), F32(-3.4028235e38)), (F32(1.0), F32(-1.0))]
NAN_BITS = [0x7fc00001, 0xffc12345, 0x7fa00002, 0x7fffffff]          # quiet and signalling payloads, both signs


def chunk_of(rng, batch, frames, is_float):
    """[batch][frames * 2] interleaved samples: random over the whole range, the edge pairs at rotating positions"""
    if is_float:
        c = ((rng.random((batch, frames * 2), np.float32) - 0.5) * 2).astype(np.float32)
        edges = list(FLOAT_EDGES) + [(np.uint32(b).view(np.float32), F32(0.5)) for b in NAN_BITS]
    else:
        c = rng.integers(-32768, 32768, size=(batch, frames * 2), dtype=np.int32).astype(np.int16)
        edges = INT_EDGES
    for s in range(batch):
        for j, (a, b) in enumerate(edges):
            q = (s * 7 + j * 3) % frames
            if j < frames:
                c[s, 2 * q] = a; c[s, 2 * q + 1] = b
    return c


# ---- one ring per configuration, over the frame counts -----------------------------------------------------------------
SIZES = [dict(n=256), dict(n=1024), dict(n=4096), dict(n=16384), dict(n=2048, bufscale=2), dict(n=4096, bufscale=4)]
CHANNELS = {"stereo": dict(), "channels1": dict(channels=1), "mirror": dict(channels=2, mirror_input=1)}
BATCHES = [1, 5, 33]


def _params(size, chans, accel):
    return g.default_params("bars", w=64, h=16, accel_fft=accel, **size, **CHANNELS[chans])


CONFIGS = [(i, fmt, ch) for i in range(len(SIZES)) for fmt in ("int16", "float") for ch in CHANNELS]


@pytest.mark.parametrize("si,fmt,chans", CONFIGS, ids=[f"{SIZES[i]}-{f}-{c}" for i, f, c in CONFIGS])
def test_ingest_rings_bit_for_bit(si, fmt, chans, built):
    size = SIZES[si]
    k = CONFIGS.index((si, fmt, chans))
    batch = BATCHES[k % 3]
    p = _params(size, chans, accel=k % 2)
    n_in = p.n
    is_float = fmt == "float"
    mono = chans != "stereo"
    rng = np.random.default_rng([si, k])
    rl = np.zeros((batch, n_in), np.float32); rr = np.zeros((batch, n_in), np.float32)
    with g.Renderer(p, batch=batch) as r:
        for frames in [f for f in (1, 2, 3, 255, 256, 257) if f < n_in - 1] + [n_in - 1, n_in, 3]:
            c = chunk_of(rng, batch, frames, is_float)
            (r.ingest_float if is_float else r.ingest_fifo)(c)
            for s in range(batch):
                rl[s], rr[s] = ingest_ref(rl[s], rr[s], c[s], mono, is_float)
            gl, gr = rings_of(r)
            for s in range(batch):
                assert same_ring(gl[s], rl[s], mono and is_float), (frames, s, "l")
                assert same_ring(gr[s], rr[s], mono and is_float), (frames, s, "r")


# ---- sequences: ingests, updates and stream state, against update() on the restated rings -------------------------------
@pytest.mark.parametrize("chans", ["stereo", "mirror"])
@pytest.mark.parametrize("size", [dict(n=1024), dict(n=4096, bufscale=2)], ids=["1024", "4096-bs2"])
def test_ingest_sequences_match_update_on_the_restated_rings(size, chans, built):
    p = _params(size, chans, accel=1)
    p.lazy_smooth = 1
    batch, n_in = 5, p.n
    mono = chans != "stereo"
    rng = np.random.default_rng(11)
    rl = np.zeros((batch, n_in), np.float32); rr = np.zeros((batch, n_in), np.float32)
    with g.Renderer(p, batch=batch) as a, g.Renderer(p, batch=batch) as b:
        def ingest(frames, is_float=False):
            c = chunk_of(rng, batch, frames, is_float)
            if is_float:
                c = (c * F32(0.25)).astype(np.float32)
                c[~np.isfinite(c)] = 0                          # finite audio for the spectra
            (a.ingest_float if is_float else a.ingest_fifo)(c)
            for s in range(batch):
                rl[s], rr[s] = ingest_ref(rl[s], rr[s], c[s], mono, is_float)

        def compare(tag):
            for ch, (x, y) in enumerate(zip(a.spectrum(), b.spectrum())):
                assert np.array_equal(x, y, equal_nan=True), (tag, "spectrum", ch)
            for ch, (x, y) in enumerate(zip(a.textures(), b.textures())):
                assert np.array_equal(x, y), (tag, "texture", ch)
            for s in range(batch):
                assert np.array_equal(a.readback(s), b.readback(s)), (tag, "frame", s)
            gl, gr = rings_of(a)
            for s in range(batch):
                assert same_ring(gl[s], rl[s], False) and same_ring(gr[s], rr[s], False), (tag, "ring", s)

        # the chunk buffer grows, shrinks and grows again; several ingests between updates
        for frames in (64, n_in, 7, 300, n_in // 2):
            ingest(frames)
        a.update_rings(True); b.update(rl, rr, True); compare("grow-shrink")
        ingest(n_in - 1); ingest(1, is_float=True); ingest(257)
        a.update_rings(False); b.update(rl, rr, False); compare("unmodified")
        a.update_rings(True); b.update(rl, rr, True); compare("modified")
        m = np.array([1, 0, 1, 1, 0], bool)
        ingest(96)
        a.update_rings_masked(m); b.update_masked(rl, rr, m); compare("masked")
        # stream 3 reset (its ring empties), then stream 1 loaded from stream 4 (ring included)
        reset = np.zeros(batch, bool); reset[3] = True
        a.reset_streams(reset); b.reset_streams(reset)
        rl[3] = 0; rr[3] = 0
        ingest(200)
        a.update_rings(True); b.update(rl, rr, True); compare("reset")
        a.load_streams([1], a.save_streams([4])); b.load_streams([1], b.save_streams([4]))
        rl[1], rr[1] = rl[4].copy(), rr[4].copy()
        ingest(33); ingest(n_in)
        a.update_rings(True); b.update(rl, rr, True); compare("load")


# ---- refusals -----------------------------------------------------------------------------------------------------------
def test_refused_ingests_leave_every_ring_alone(built):
    p = _params(dict(n=1024), "stereo", accel=1)
    batch = 3
    rng = np.random.default_rng(5)
    with g.Renderer(p, batch=batch) as r:
        r.ingest_fifo(chunk_of(rng, batch, 300, False)); r.ingest_float(chunk_of(rng, batch, 100, True))
        before = [x.copy() for x in rings_of(r)]
        count = r.launch_count
        for fn, dtype in ((r._L.glava_b200_ingest_fifo, np.int16), (r._L.glava_b200_ingest_float, np.float32)):
            big = np.zeros((batch, 2 * (p.n + 1)), dtype)
            for ptr, frames in ((big.ctypes.data, 0), (big.ctypes.data, -1), (big.ctypes.data, p.n + 1), (None, 16)):
                assert fn(r._h, ptr, frames) == EINVAL, (frames, ptr)
        assert r.launch_count == count
        for x, y in zip(rings_of(r), before):
            assert np.array_equal(x.view(np.uint32), y.view(np.uint32))


# ---- sharded ------------------------------------------------------------------------------------------------------------
def test_sharded_ingest_equals_one_handle(built):
    p = _params(dict(n=1024), "channels1", accel=1)
    batch = 7
    rng = np.random.default_rng(9)
    with g.ShardedRenderer(p, batch, [0, 0, 0]) as sh, g.Renderer(p, batch=batch) as one:
        for frames in (256, 1, 1024, 77):
            c = chunk_of(rng, batch, frames, False)
            sh.ingest_fifo(c)
            one.ingest_fifo(c); one.update_rings(True)
            for ch, (x, y) in enumerate(zip(sh.textures(), one.textures())):
                assert np.array_equal(x, y), (frames, ch)
            for s in (0, 3, 6):
                assert np.array_equal(sh.readback(s), one.readback(s)), (frames, s)
            blobs_sh, blobs_one = sh.save_streams(range(batch)), one.save_streams(range(batch))
            assert np.array_equal(blobs_sh[:, HEADER:], blobs_one[:, HEADER:]), frames
