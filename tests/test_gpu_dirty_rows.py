"""-m gpu: the dirty-row marks of the bars / graph / wave rasters leave every frame bit-exact.

Those kernels skip the zero rows that the previous frame in the same framebuffer slot already left at zero (raster_core.h
dirty_pack).  What is in memory therefore depends on the previous frame and on how it was drawn, so these tests drive
sequences of frames through one renderer: textures at full height, single spikes, silence and ramps, with the band height,
the framebuffer ring, the geometry, the kernel (a reconfigure to bars MIRROR_YX runs the generic kernel) and per-stream
`modified` masks changing between steps.  After every step, every stream's frame must equal the host build of the same
textures, bit for bit."""
import numpy as np
import pytest

import glava_b200 as g
from tests import emul

pytestmark = pytest.mark.gpu

N = 1024
W, H = 332, 181


def _patterns(n, k):
    """full height, spikes, silence and a ramp; pattern k, left / right differ"""
    k %= 4
    if k == 0:
        t = np.full(n, 65535, np.uint16)
    elif k == 1:
        t = np.zeros(n, np.uint16); t[:: max(1, n // 7)] = 65535; t[n // 2] = 40000
    elif k == 2:
        t = np.zeros(n, np.uint16)
    else:
        t = np.linspace(0, 65535, n).astype(np.uint16)
    return t, t[::-1].copy()


def _textures(batch, n, step):
    rows = [_patterns(n, step + s) for s in range(batch)]
    return np.stack([r[0] for r in rows]), np.stack([r[1] for r in rows])


def _want(p, tl, tr):
    fast = not (p.module == g.default_params("bars").module and p.bars_mirror_yx)
    return emul.raster(p, tl, tr, fast=fast)


def _check(r, tl, tr, what):
    """every slot holds the frame of the highest stream mapped to it"""
    p = r.refresh_params()
    slots = p.fb_slots if 0 < p.fb_slots < r.batch else r.batch
    for k in range(slots):
        s = max(t for t in range(r.batch) if t % slots == k)
        got = r.readback(s)
        want = _want(p, tl[s], tr[s])
        assert np.array_equal(got, want), (what, s, int((got != want).any(axis=2).sum()))


CASES = {
    "bars": dict(module="bars"),
    "bars_flip": dict(module="bars", bars_flip=1),
    "graph": dict(module="graph"),
    "graph_invert": dict(module="graph", graph_invert=1),
    "wave": dict(module="wave"),
}


def _params(case, w=W, h=H, **kw):
    d = dict(CASES[case]); m = d.pop("module")
    p = g.default_params(m, n=N, w=w, h=h)
    for k, v in {**d, **kw}.items():
        setattr(p, k, v)
    return p


@pytest.mark.parametrize("case", sorted(CASES))
def test_sequence_across_band_heights(case, monkeypatch, built):
    """the band height changes between steps: marks written at one height must not be trusted at another"""
    batch = 4
    with g.Renderer(_params(case), batch=batch) as r:
        for step, rows in enumerate([None, None, "16", "16", "7", "7", None, "181", "181", "45", None, None]):
            if rows is None:
                monkeypatch.delenv("GLAVA_B200_ROWS", raising=False)
            else:
                monkeypatch.setenv("GLAVA_B200_ROWS", rows)
            tl, tr = _textures(batch, r.nsz, step)
            r.raster_textures(tl, tr)
            _check(r, tl, tr, (case, step, rows))


@pytest.mark.parametrize("slots", [1, 3])
@pytest.mark.parametrize("case", ["bars", "graph", "wave"])
def test_sequence_with_framebuffer_ring(case, slots, built):
    """fb_slots < batch: a slot's previous frame is another stream's"""
    batch = 7
    with g.Renderer(_params(case, fb_slots=slots), batch=batch) as r:
        for step in range(9):
            tl, tr = _textures(batch, r.nsz, step * 3 + 1)
            r.raster_textures(tl, tr)
            _check(r, tl, tr, (case, slots, step))


@pytest.mark.parametrize("case", ["bars", "bars_flip", "graph", "wave"])
def test_sequence_across_resizes(case, built):
    """sizereq replaces the framebuffer and the marks between steps"""
    batch = 3
    with g.Renderer(_params(case), batch=batch) as r:
        for step, geo in enumerate([None, (200, 96), None, (W, H), None, (512, 64), None]):
            if geo is not None:
                r.sizereq(*geo)
            tl, tr = _textures(batch, r.nsz, step)
            r.raster_textures(tl, tr)
            _check(r, tl, tr, (case, step, geo))


@pytest.mark.parametrize("case", ["bars", "bars_flip"])
def test_sequence_across_mirror_reconfigure(case, built):
    """bars MIRROR_YX runs the generic kernel, which keeps no marks: the first bars launch after it stores every row"""
    batch = 3
    with g.Renderer(_params(case), batch=batch) as r:
        for step, mirror in enumerate([0, 0, 1, 1, 0, 0, 1, 0, 0]):
            if mirror != r.params.bars_mirror_yx:
                q = r.params.copy(); q.bars_mirror_yx = mirror
                r.reconfigure(q)
            tl, tr = _textures(batch, r.nsz, step)
            r.raster_textures(tl, tr)
            _check(r, tl, tr, (case, step, mirror))


@pytest.mark.parametrize("case", ["bars", "graph", "wave"])
def test_sequence_with_masks_and_unmodified_updates(case, built):
    """per-stream masked updates and modified = false re-raster some or all textures unchanged; loud, quiet and silent
    audio makes the frames rise and fall"""
    batch = 5
    rng = np.random.default_rng(11)
    p = _params(case)
    with g.Renderer(p, batch=batch) as r:
        n = r.params.n
        t = np.arange(n, dtype=np.float32)
        for step in range(10):
            amp = [0.5, 0.02, 0.0, 0.3][step % 4]
            lb = (amp * np.sin(t[None, :] * (0.05 + 0.01 * np.arange(batch)[:, None]))).astype(np.float32)
            rb = (lb[:, ::-1] * 0.7 + amp * 0.1 * rng.standard_normal((batch, n))).astype(np.float32)
            if step % 3 == 2:
                r.update(lb, rb, modified=False)
            else:
                r.update_masked(lb, rb, rng.random(batch) < 0.6)
            r.sync()
            tl, tr = r.textures()
            _check(r, tl, tr, (case, step))
