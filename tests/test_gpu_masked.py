"""-m gpu: per-stream `modified` (glava_b200_update_masked).

glava.c:528-537 copies the rings and passes modified = true only when ITS audio thread ticked; rd_update then either
runs the chain or re-rasters the previous texture (render.c:2122, 2268-2272).  In a batch every stream has its own
flag: the masked update must give, for every stream, exactly what a single-stream renderer gives when it is called
with that stream's flag — spectra, textures and frames bit for bit — for both pipelines, lazy and full K5, the wave
chain and the appended "smooth" transform."""
import numpy as np
import pytest

import glava_b200 as g

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

CASES = [
    ("bars", dict(), "pipeline B, full K5"),
    ("bars", dict(lazy_smooth=1), "pipeline B, lazy K5 (need-list, shared-memory taps)"),
    ("bars", dict(accel_fft=0), "pipeline A"),
    ("bars", dict(accel_fft=0, avg_frames=3, lazy_smooth=1), "pipeline A, F=3, lazy"),
    ("graph", dict(avg_frames=7), "generic F"),
    ("circle", dict(), "circle (texmm)"),
    ("wave", dict(), "wave chain"),
    ("bars", dict(transform_smooth=1), "appended transform_smooth (post chain)"),
    ("radial", dict(smooth_pass=0), "no K5"),
]


@pytest.mark.parametrize("module,over,what", CASES, ids=[c[2] for c in CASES])
def test_masked_update_equals_single_stream_renderers(built, module, over, what):
    n, batch, steps = 1024, 5, 14
    p = g.default_params(module, n=n, w=128, h=64, **over)
    rng = np.random.default_rng(hash(what) & 0xffff)
    lb = np.zeros((batch, n), np.float32); rb = np.zeros_like(lb)
    masks = rng.random((steps, batch)) < 0.55
    masks[3] = False                                  # nobody: plain modified = 0
    masks[6] = True                                   # everybody (after the streams have drifted apart)
    masks[0, 0] = False; masks[0, 1] = True           # uneven from the very first update
    singles = [g.Renderer(p, batch=1) for _ in range(batch)]
    try:
        with g.Renderer(p, batch=batch) as r:
            for t in range(steps):
                for s in range(batch):
                    if masks[t, s]:                   # rows of unmodified streams keep their old content (glava.c:531-536)
                        lb[s] = (rng.random(n, np.float32) - 0.5) * 0.3; rb[s] = (rng.random(n, np.float32) - 0.5) * 0.3
                r.update_masked(lb, rb, masks[t])
                for s in range(batch):
                    singles[s].update(lb[s:s + 1], rb[s:s + 1], bool(masks[t, s]))
                if t in (0, 3, 6, 9, steps - 1):
                    sl, sr = r.spectrum(); tl, tr = r.textures()
                    for s in range(batch):
                        a = singles[s].spectrum(); b = singles[s].textures()
                        assert np.array_equal(sl[s], a[0][0], equal_nan=True) and np.array_equal(sr[s], a[1][0], equal_nan=True), (what, t, s)   # (transform_smooth writes NaN into b[0], render.c:694-718)
                        assert np.array_equal(tl[s], b[0][0]) and np.array_equal(tr[s], b[1][0]), (what, t, s)
                        assert np.array_equal(r.readback(s), singles[s].readback(0)), (what, t, s)
            assert r.spectrum()[0].any()
    finally:
        for q in singles:
            q.close()


def test_plain_updates_after_an_uneven_one_keep_per_stream_cursors(built):
    """after streams drifted apart, glava_b200_update(modified = 1) still advances every stream on ITS ring cursor"""
    n, batch = 512, 3
    p = g.default_params("bars", n=n, w=64, h=32)
    rng = np.random.default_rng(5)
    seq = [np.array([1, 0, 1]), np.array([0, 1, 1]), None, None, np.array([1, 1, 0]), None, None, None]
    lb = np.zeros((batch, n), np.float32); rb = np.zeros_like(lb)
    singles = [g.Renderer(p, batch=1) for _ in range(batch)]
    try:
        with g.Renderer(p, batch=batch) as r:
            for m in seq:
                mm = np.ones(batch, bool) if m is None else m.astype(bool)
                for s in range(batch):
                    if mm[s]:
                        lb[s] = (rng.random(n, np.float32) - 0.5) * 0.3; rb[s] = (rng.random(n, np.float32) - 0.5) * 0.3
                if m is None:
                    r.update(lb, rb, True)
                else:
                    r.update_masked(lb, rb, mm)
                for s in range(batch):
                    singles[s].update(lb[s:s + 1], rb[s:s + 1], bool(mm[s]))
            tl, tr = r.textures()
            for s in range(batch):
                b = singles[s].textures()
                assert np.array_equal(tl[s], b[0][0]) and np.array_equal(tr[s], b[1][0])
                assert np.array_equal(r.readback(s), singles[s].readback(0))
    finally:
        for q in singles:
            q.close()


def test_uneven_mask_with_interpolation_is_rejected(built):
    p = g.default_params("wave", n=512, w=64, h=32, interpolate=1, fr=400.0)
    z = np.zeros((2, 512), np.float32)
    with g.Renderer(p, batch=2) as r:
        r.update_masked(z, z, [1, 1])
        r.update_masked(z, z, [0, 0])
        with pytest.raises(g.GlavaError, match="interpolation"):
            r.update_masked(z, z, [1, 0])


def test_null_right_channel_is_rejected_for_two_channel_modules(built):
    p = g.default_params("bars", n=512, w=64, h=32)
    z = np.zeros((1, 512), np.float32)
    with g.Renderer(p, batch=1) as r:
        with pytest.raises(g.GlavaError, match="rb is null"):
            r.update(z, None, True)
        r.update(z, None, False)                      # modified = 0 does not read the buffers
    with g.Renderer(g.default_params("wave", n=512, w=64, h=32), batch=1) as r:
        r.update(z, None, True)                       # wave samples audio_l only (wave/1.frag:7)


PERSISTENT_CASES = [("bars", dict(), "bars"), ("wave", dict(), "wave"), ("bars", dict(accel_fft=0), "pipeline A"),
                    ("graph", dict(avg_frames=7), "generic F")]


@pytest.mark.parametrize("n", [256, 1024, 2048])
@pytest.mark.parametrize("module,over,what", PERSISTENT_CASES, ids=[c[2] for c in PERSISTENT_CASES])
def test_persistent_spectrum_grid_with_uneven_masks(built, monkeypatch, n, module, over, what):
    """At the default settings with the K5 taps in shared memory (lazy_smooth=1, FFT < 4096) the spectrum kernel runs as a
    persistent grid of 2 CTAs per SM whenever there are more units than that (launch_spectrum_t): a CTA walks units
    blockIdx.x, + grid, ...  Masks chosen per CTA: one skips its first unit and runs a later one, one the reverse, one
    skips all of its units, while the mbarrier parity flips, the next unit's PCM is prefetched and the tap table stays
    resident.  The whole batch must equal one CTA per unit (GLAVA_B200_SPEC_CTAS_PER_SM=0) bit for bit, and probe streams
    past the first grid stride must equal single-stream renderers fed the same flags."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    batch, steps = 2 * sms + 37, 7                            # odd, not a multiple of 32, more units than CTAs
    grid = 2 * sms                                            # (even: a CTA stays on one channel)
    stride = grid // 2 if module != "wave" else grid          # unit u = plane u (stream u >> 1); wave: unit u = stream u
    p = g.default_params(module, n=n, w=64, h=16, lazy_smooth=1, **over)
    rng = np.random.default_rng(n + len(what))
    masks = rng.random((steps, batch)) < 0.6
    masks[0] = True
    a, b, c, d = 3, 11, 5, 40                                 # FFT modules: streams < 37 have a third unit, 40 has two
    for t in (1, 2, 4, 5):
        masks[t, a] = False; masks[t, a + stride::stride] = True      # the CTAs of stream a: skip the first unit, run the later ones
        masks[t, b] = True; masks[t, b + stride::stride] = False      # the reverse
        masks[t, c::stride] = False; masks[t, d::stride] = False       # every unit skipped
    masks[3] = ~masks[2]
    seq = []
    lb = np.zeros((batch, n), np.float32); rb = np.zeros_like(lb)
    for t in range(steps):
        for s in np.flatnonzero(masks[t]):
            lb[s] = (rng.random(n, np.float32) - 0.5) * 0.3; rb[s] = (rng.random(n, np.float32) - 0.5) * 0.3
        seq.append((lb.copy(), rb.copy()))
    probes = sorted({a + stride, b + stride, c + stride, min(d + stride, batch - 1), stride + 17, batch - 2})

    def run(per_sm):
        monkeypatch.delenv("GLAVA_B200_SPEC_CTAS_PER_SM", raising=False)
        if per_sm is not None:
            monkeypatch.setenv("GLAVA_B200_SPEC_CTAS_PER_SM", per_sm)
        with g.Renderer(p, batch=batch) as r:
            for (l, rr), m in zip(seq, masks):
                r.update_masked(l, rr, m)
            return r.spectrum(), r.textures(), {s: r.readback(s) for s in probes + [0, a, b, c]}

    persistent, per_unit = run(None), run("0")
    for x, y in zip(persistent[0] + persistent[1], per_unit[0] + per_unit[1]):
        assert np.array_equal(x, y), what
    for s, frame in persistent[2].items():
        assert np.array_equal(frame, per_unit[2][s]), (what, s)
    assert persistent[1][0].any()
    for s in probes:
        with g.Renderer(p, batch=1) as one:
            for (l, rr), m in zip(seq, masks):
                one.update(l[s:s + 1], rr[s:s + 1], bool(m[s]))
            (sl, sr), (tl, tr) = one.spectrum(), one.textures()
            assert np.array_equal(sl[0], persistent[0][0][s]) and np.array_equal(sr[0], persistent[0][1][s]), (what, s)
            assert np.array_equal(tl[0], persistent[1][0][s]) and np.array_equal(tr[0], persistent[1][1][s]), (what, s)
            assert np.array_equal(one.readback(0), persistent[2][s]), (what, s)
