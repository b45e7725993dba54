"""-m gpu: setopacity other than "native" (premultiply_alpha = 0).  The reference then draws every module stage with
GL_BLEND, glBlendFunc(GL_SRC_ALPHA, GL_ONE_MINUS_SRC_ALPHA), over the target glClear'd to the `setbg` colour and skips the
premultiply stages (render.c:1467-1470, 1700, 2028).  Kernels (the generic per-pixel path: plan_raster's rule) against
frames computed from the reference's shader text with that blend state (tests/golden/glsl_golden.npz, *_blend cases),
against the oracle, and against the host build of the same arithmetic."""
import json
import os

import numpy as np
import pytest

import glava_b200 as g
from oracle.oracle import params_from
from tests.conftest import GOLDEN

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]
N = 512


def _blend_cases():
    z = np.load(os.path.join(GOLDEN, "glsl_golden.npz"))
    return [str(c) for c in z["case_names"] if str(c).endswith(("_blend", "_blend_opaque", "_nopremult"))]


@pytest.mark.parametrize("case", _blend_cases())
def test_kernels_blend_every_stage_over_the_clear_colour(orc_pm, case, built):
    from tests import emul
    z = np.load(os.path.join(GOLDEN, "glsl_golden.npz"))
    module = str(z[f"{case}_module"]); w, h = (int(v) for v in z[f"{case}_size"])
    p = g.default_params(module, n=N, w=w, h=h, **json.loads(str(z[f"{case}_params"])))
    assert p.premultiply_alpha == 0
    tl, tr, want = z[f"{case}_tl"], z[f"{case}_tr"], z[f"{case}_frame"]
    with g.Renderer(p, batch=2) as r:
        r.raster_textures(np.stack([tl, tr]), np.stack([tr, tl]))
        got, swapped = r.readback(0), r.readback(1)
    assert np.array_equal(got, emul.raster(p, tl, tr)) and np.array_equal(swapped, emul.raster(p, tr, tl))
    assert np.array_equal(got, orc_pm.raster(params_from(p), tl, tr))
    assert int(np.abs(got.astype(int) - want.astype(int)).max()) <= 1
    assert (got != want).any(axis=2).sum() <= 0.002 * w * h


def test_full_size_non_native_frame(orc_pm, built):
    """1920x1080 bars over an opaque background: rows spot-checked against the oracle"""
    p = g.default_params("bars", n=4096, w=1920, h=1080, premultiply_alpha=0, clear_color=[0.05, 0.05, 0.1, 1.0])
    op = params_from(p)
    rng = np.random.default_rng(12)
    tl = orc_pm.smooth_pass(op, (rng.random(4096) ** 2 * 65535).astype(np.uint16))
    tr = orc_pm.smooth_pass(op, (rng.random(4096) ** 3 * 65535).astype(np.uint16))
    with g.Renderer(p, batch=1) as r:
        r.raster_textures(tl[None], tr[None])
        got = r.readback(0)
    for y0, y1 in ((0, 4), (100, 104), (298, 304), (1076, 1080)):
        assert np.array_equal(got[y0:y1], orc_pm.raster(op, tl, tr, rows=(y0, y1))[y0:y1])
    assert (got[1079, 0] == [13, 13, 26, 255]).all()


def test_radial_bar_outline_through_the_per_pixel_kernel(orc_pm, built):
    """BAR_OUTLINE_WIDTH > 0 (deprecated, radial.glsl:33-36): three values per pixel, so plan_raster leaves the geometry
    cache for the per-pixel radial kernel"""
    from tests import emul
    z = np.load(os.path.join(GOLDEN, "glsl_golden.npz"))
    case = "radial_outline"
    w, h = (int(v) for v in z[f"{case}_size"])
    p = g.default_params("radial", n=N, w=w, h=h, **json.loads(str(z[f"{case}_params"])))
    tl, tr, want = z[f"{case}_tl"], z[f"{case}_tr"], z[f"{case}_frame"]
    with g.Renderer(p, batch=2) as r:
        r.raster_textures(np.stack([tl, tr]), np.stack([tr, tl]))
        got = r.readback(0)
    assert np.array_equal(got, emul.raster(p, tl, tr))
    assert np.array_equal(got, orc_pm.raster(params_from(p), tl, tr))
    assert int(np.abs(got.astype(int) - want.astype(int)).max()) <= 1 and (got != want).any(axis=2).sum() <= 0.002 * w * h
    big = g.default_params("radial", n=4096, w=1280, h=720, radial_bar_outline_width=2.0, radial_bar_outline=[1.0, 1.0, 0.0, 1.0])
    rng = np.random.default_rng(3)
    op = params_from(big)
    tl = orc_pm.smooth_pass(op, (rng.random(4096) ** 2 * 65535).astype(np.uint16)); tr = tl[::-1].copy()
    with g.Renderer(big, batch=1) as r:
        r.raster_textures(tl[None], tr[None])
        got = r.readback(0)
    assert np.array_equal(got, orc_pm.raster(op, tl, tr))


def test_graph_join_channels(orc_pm, built):
    """JOIN_CHANNELS 1 (graph/1.frag:93-96,126): generic kernel; the lazy K5 need-list must hold the texels `middle` samples"""
    from tests import emul
    z = np.load(os.path.join(GOLDEN, "glsl_golden.npz"))
    case = "graph_join"
    w, h = (int(v) for v in z[f"{case}_size"])
    p = g.default_params("graph", n=N, w=w, h=h, **json.loads(str(z[f"{case}_params"])))
    tl, tr, want = z[f"{case}_tl"], z[f"{case}_tr"], z[f"{case}_frame"]
    with g.Renderer(p, batch=1) as r:
        r.raster_textures(tl[None], tr[None])
        got = r.readback(0)
    assert np.array_equal(got, emul.raster(p, tl, tr))
    assert int(np.abs(got.astype(int) - want.astype(int)).max()) <= 1 and (got != want).any(axis=2).sum() <= 0.002 * w * h
    # whole pipeline, lazy K5 (only the sampled texels are smoothed) against full K5: identical frames
    frames = []
    for lazy in (0, 1):
        q = g.default_params("graph", n=1024, w=320, h=200, graph_join_channels=1, lazy_smooth=lazy)
        rings = g.StreamRings(2, 1024)
        with g.Renderer(q, batch=2) as r:
            for _ in range(6):
                rings.advance(); r.update(rings.lb, rings.rb, True)
            frames.append([r.readback(0), r.readback(1)])
    assert np.array_equal(frames[0][0], frames[1][0]) and np.array_equal(frames[0][1], frames[1][1]) and frames[0][0].any()


@pytest.mark.parametrize("case", ["graph_aa", "graph_aa_invert"])
def test_graph_anti_alias_stage(orc_pm, case, built):
    """ANTI_ALIAS 1 (graph/3.frag): per-pixel column walks in the generic kernel; exact (no transcendental on this path)"""
    z = np.load(os.path.join(GOLDEN, "glsl_golden.npz"))
    w, h = (int(v) for v in z[f"{case}_size"])
    p = g.default_params("graph", n=N, w=w, h=h, **json.loads(str(z[f"{case}_params"])))
    tl, tr, want = z[f"{case}_tl"], z[f"{case}_tr"], z[f"{case}_frame"]
    with g.Renderer(p, batch=2) as r:
        r.raster_textures(np.stack([tl, tr]), np.stack([tr, tl]))
        got, swapped = r.readback(0), r.readback(1)
    assert np.array_equal(got, want) and np.array_equal(swapped, orc_pm.raster(params_from(p), tr, tl))
    big = g.default_params("graph", n=2048, w=1280, h=720, graph_anti_alias=1)
    op = params_from(big)
    rng = np.random.default_rng(2)
    tl = orc_pm.smooth_pass(op, (rng.random(2048) ** 2 * 65535).astype(np.uint16)); tr = orc_pm.smooth_pass(op, (rng.random(2048) ** 3 * 65535).astype(np.uint16))
    with g.Renderer(big, batch=1) as r:
        r.raster_textures(tl[None], tr[None])
        got = r.readback(0)
    assert np.array_equal(got, orc_pm.raster(op, tl, tr))


@pytest.mark.parametrize("module", ["bars", "radial", "circle", "graph"])
def test_stage1_shader_belief_about_its_textures(orc_pm, module, built):
    """params.shader_pre_smoothed: the raster launch sees the module shader's (possibly stale) `_PRE_SMOOTHED_AUDIO`, not the
    K5 decision.  On the same textures, "believes smoothed although K5 is off" renders like smooth_pass = 1, and "believes raw
    although K5 ran" like smooth_pass = 0."""
    n, w, h = 512, 320, 200
    rng = np.random.default_rng(6)
    tl = (rng.random(n) ** 2 * 65535).astype(np.uint16); tr = (rng.random(n) ** 3 * 65535).astype(np.uint16)
    frames = {}
    for key, over in (("on", dict(smooth_pass=1)), ("off", dict(smooth_pass=0)),
                      ("stale_on", dict(smooth_pass=0, shader_pre_smoothed=1)), ("stale_off", dict(smooth_pass=1, shader_pre_smoothed=2))):
        p = g.default_params(module, n=n, w=w, h=h, **over)
        with g.Renderer(p, batch=1) as r:
            r.raster_textures(tl[None], tr[None])
            frames[key] = r.readback(0)
        assert np.array_equal(frames[key], orc_pm.raster(params_from(p), tl, tr)), (module, key)
    assert np.array_equal(frames["stale_on"], frames["on"]) and np.array_equal(frames["stale_off"], frames["off"])
    assert not np.array_equal(frames["on"], frames["off"])
