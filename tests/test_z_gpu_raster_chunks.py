"""-m gpu: the raster launch past its 32768-stream chunk, and the framebuffer ring, for every module.

launch_raster covers at most 32768 streams (grid z) or `fb_slots` streams per launch, whichever is fewer, and starts each
launch at stream0 > 0.  The column table (graph / wave), the per-stream texture min / max (circle) and the framebuffer slot
are all indexed by the global stream; the geometry cache (radial / circle) is shared.  Probe streams on both sides of the
chunk boundary must equal the oracle on the same textures, and each pass must issue the launches raster_plan.h plans for it
(one set per chunk).  Tiny frames and parameters that light pixels inside them keep
the host side small: on an H100 the device holds about 1.5 GB during the 32771-stream cases, CUDA context included."""
import numpy as np
import pytest

import glava_b200 as g
from oracle.oracle import params_from
from tests import emul

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

SMALL_PARAMS = {
    "bars": dict(bars_amplify=60.0),
    "graph": dict(graph_vscale=40.0),
    "wave": dict(wave_amplify=60.0),
    "radial": dict(radial_radius=8.0, radial_amplify=12.0),
    "circle": dict(circle_radius=8.0, circle_amplify=12.0),
    "test": dict(),
}


def _raster(r, p, batch, slots, tl, tr):
    """r.raster_textures(tl, tr), checking the pass's launch count against the plan"""
    before = r.launch_count
    r.raster_textures(tl, tr)
    assert r.launch_count - before == emul.raster_plan(p, batch, slots, {})["launches"], (g.MODULES[p.module], batch, slots)


def _textures(n, batch, seed, wave=False):
    """[batch][n] uint16 left / right: a few base rows times a per-stream gain (distinct streams at any batch, cheaply)"""
    rng = np.random.default_rng(seed)
    base_l = rng.random((7, n), np.float32); base_r = rng.random((5, n), np.float32)
    s = np.arange(batch, dtype=np.uint64)
    gain = (0.15 + 0.85 * ((s * np.uint64(2654435761)) % np.uint64(1009)).astype(np.float32) / np.float32(1009))[:, None]
    tl = base_l[np.arange(batch) % 7] * gain; tr = base_r[(2 * np.arange(batch)) % 5] * gain
    if wave:                                                 # lines around 0.5
        tl = 0.375 + tl / 4; tr = 0.375 + tr / 4
    return (tl * 65535).astype(np.uint16), (tr * 65535).astype(np.uint16)


@pytest.mark.parametrize("module", ["graph", "wave", "radial", "circle"])
def test_raster_past_the_stream_chunk(orc_pm, module, built):
    n, batch = 256, 32771
    p = g.default_params(module, n=n, w=32, h=24, **SMALL_PARAMS[module]); op = params_from(p)
    tl, tr = _textures(n, batch, 7, wave=module == "wave")
    with g.Renderer(p, batch=batch) as r:
        _raster(r, p, batch, batch, tl, tr)
        for s in (0, 1, 32767, 32768, 32769, batch - 1):
            got = r.readback(s)
            assert got.any(), (module, s)
            assert np.array_equal(got, orc_pm.raster(op, tl[s], tr[s])), (module, s)


@pytest.mark.parametrize("slots", [1, 3])
@pytest.mark.parametrize("module", g.MODULES)
def test_framebuffer_ring(orc_pm, module, slots, built):
    """fb_slots < batch: slot j holds the frame of the highest stream s with s % slots == j, after raster_textures and after
    an unmodified update, which re-rasters the textures the renderer holds"""
    n, batch = 1024, 8
    p = g.default_params(module, n=n, w=96, h=48, fb_slots=slots, **SMALL_PARAMS[module]); op = params_from(p)
    tops = [max(s for s in range(batch) if s % slots == j) for j in range(slots)]
    tl, tr = _textures(n, batch, 3 + slots, wave=module == "wave")
    rng = np.random.default_rng(slots)
    lb = ((rng.random((batch, n), np.float32) - 0.5) * 0.4); rb = ((rng.random((batch, n), np.float32) - 0.5) * 0.4)
    with g.Renderer(p, batch=batch) as r:
        _raster(r, p, batch, slots, tl, tr)
        for j, s in enumerate(tops):
            got = r.readback(j)
            assert got.any(), (module, s)
            assert np.array_equal(got, orc_pm.raster(op, tl[s], tr[s])), (module, slots, s)
        r.update(lb, rb, True)
        r.update(lb, rb, False)
        ul, ur = r.textures()
        for j, s in enumerate(tops):
            assert np.array_equal(r.readback(j), orc_pm.raster(op, ul[s], ur[s])), (module, slots, s, "unmodified update")
