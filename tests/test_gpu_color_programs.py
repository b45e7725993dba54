"""-m gpu: the colour-expression programs of tests/color_programs.py in every kernel that runs them, bit for bit against the
host build of the same arithmetic (emul).  Each case renders edge textures (silence, saturation, spikes at texel 0 and
n - 1, and the height ramps or polar bands of tests/test_gpu_raster_variants.py, so that every row and radius is lit) in
a batch mixing the styles of color_programs.styles_for: slot 0, AMPLIFY only, bg only, fg + bg.  CPU tier:
tests/test_color_programs.py."""
import numpy as np
import pytest

import glava_b200 as g
from tests import color_programs as cp
from tests import emul
from tests import test_gpu_raster_variants as rv

pytestmark = pytest.mark.gpu
CASES = cp.cases()


def _textures(p):
    m, w, h = g.MODULES[p.module], p.w, p.h
    rows = rv._edges(cp.N)
    if m in ("bars", "graph"):
        amp = getattr(p, cp.AMP[m])
        per = int((w / 2) // (p.bars_width + p.bars_gap)) if m == "bars" else w // 2
        rows = rows + rv._height_ramps(cp.N, h, amp, max(per, 16))[0][:8]
    else:
        rows = rows + rv._polar_bands(cp.N, w + h)
    return rv._stack(rows)


class _Want:
    """emul frames per (styled parameters, texture pair): the hoisted form where the host build has one, radial from its
    geometry computed once per parameter set"""

    def __init__(self):
        self.geo = {}

    def __call__(self, q, tl, tr):
        m = g.MODULES[q.module]
        if m == "radial":
            key = bytes(q)
            if key not in self.geo:
                self.geo[key] = emul.RadialGeo(q)
            return self.geo[key].frame(tl, tr)
        fast = (m == "bars" and not q.bars_mirror_yx) or (m == "graph" and not q.graph_anti_alias)
        return emul.raster(q, tl, tr, fast=fast)


def _env(monkeypatch, env):
    for k in rv.KNOBS + ("FULL_STORE",):
        monkeypatch.delenv("GLAVA_B200_" + k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv("GLAVA_B200_" + k, str(v))


@pytest.mark.parametrize("case", [c[0] for c in CASES])
def test_programs_on_the_device(case, monkeypatch, built):
    _, site, name, p = next(c for c in CASES if c[0] == case)
    _env(monkeypatch, site[6])
    tl0, tr0 = _textures(p)
    sty = cp.styles_for(p)
    k = tl0.shape[0]
    tl, tr = np.concatenate([tl0] * len(sty)), np.concatenate([tr0] * len(sty))
    styles = [st for st in sty for _ in range(k)]
    want = _Want()
    with g.Renderer(p, batch=tl.shape[0]) as r:
        r.set_stream_styles(range(tl.shape[0]), styles)
        r.raster_textures(tl, tr)
        for s in range(tl.shape[0]):
            got = r.readback(s)
            exp = want(g.style_params(p, styles[s]), tl[s], tr[s])
            bad = (got != exp).any(axis=2)
            if bad.any():
                ys, xs = np.nonzero(bad)
                pytest.fail(f"{case} ({site[6]}) stream {s} style {styles[s]}: {int(bad.sum())} pixels differ, "
                            f"first (x, y) = ({xs[0]}, {ys[0]}): got {got[ys[0], xs[0]]} want {exp[ys[0], xs[0]]}")
    assert any(want(p, tl0[1], tr0[1]).any(axis=2).any(axis=1)), case


def test_tall_bars_pass_two_to_the_31_quadrants(built):
    """sin(d * 1e6) on a 16384-row frame: d * 1e6 passes 2^31 pi/2 (about 3.4e9) from row 3400 on"""
    _, site, name, p = next(c for c in CASES if c[0] == "bars-256x16384-trig_large")
    full = np.full((1, cp.N), 65535, np.uint16)
    with g.Renderer(p, batch=1) as r:
        r.raster_textures(full, full)
        got = r.readback(0)
    want = emul.raster(p, full[0], full[0], fast=True)
    assert np.float32(16383.5) * np.float32(1e6) > 2 ** 31 * np.pi / 2
    bad = (got != want).any(axis=2)
    assert not bad.any(), ("rows", sorted(set(np.nonzero(bad)[0].tolist()))[:20], int(bad.sum()))


def test_radial_over_the_cache_budget_keeps_the_program(monkeypatch, tmp_path_factory, built):
    """so many bg-only styles that their radial caches together pass 512 MiB: the styled per-pixel kernel runs the
    program for every (fg, bg) pair"""
    from tests.test_stream_styles import styled_plan
    _env(monkeypatch, {})
    p = cp.params("radial", 1920, 1080, cp.program_text("atan_quadrants", "radial"), radial_radius=128.0)
    one = styled_plan(tmp_path_factory, [p], 1, 1, 1, {})
    pairs = (512 << 20) // one["geo_bytes"] + 1
    styles = [{"bg": (k / pairs, 0.5, 1 - k / pairs, 1.0)} for k in range(pairs)]
    assert styled_plan(tmp_path_factory, [p] + [g.style_params(p, s) for s in styles], pairs, pairs, pairs, {})["kernel"] == "radial"
    tl0, tr0 = _textures(p)
    tl = np.stack([tl0[s % tl0.shape[0]] for s in range(pairs)]); tr = np.stack([tr0[s % tr0.shape[0]] for s in range(pairs)])
    with g.Renderer(p, batch=pairs) as r:
        r.set_stream_styles(range(pairs), styles)
        r.raster_textures(tl, tr)
        for s in (1, pairs // 2, pairs - 1):
            want = emul.RadialGeo(g.style_params(p, styles[s])).frame(tl[s], tr[s])
            assert np.array_equal(r.readback(s), want), s


def test_reconfigure_swaps_programs_with_live_marks(monkeypatch, built):
    """a closed-form colour, then a program swapped in, changed, and taken out between frames, on the same textures at
    every step: only the colour changes what the stored rows hold, and every frame equals the host build"""
    _env(monkeypatch, {})
    w, h = 332, 181
    plain = g.default_params("bars", n=cp.N, w=w, h=h, bars_amplify=1.25 * h, bars_outline_width=1.0)
    a = cp.params("bars", w, h, cp.program_text("log_domain", "bars"), cp.program_text("alpha_toggle", "bars"),
                  bars_amplify=1.25 * h, bars_outline_width=1.0)
    b = cp.params("bars", w, h, cp.program_text("trig_large", "bars"), None, bars_amplify=1.25 * h, bars_outline_width=1.0)
    tl0, tr0 = _textures(plain)
    with g.Renderer(plain, batch=2) as r:
        for step, q in enumerate([plain, a, a, b, plain, b]):
            if step == 0 or q is not [plain, a, a, b, plain, b][step - 1]:
                r.reconfigure(q)
            tl, tr = tl0[4:6], tr0[4:6]
            r.raster_textures(tl, tr)
            for s in range(2):
                assert np.array_equal(r.readback(s), emul.raster(q, tl[s], tr[s], fast=True)), (step, s)


@pytest.mark.parametrize("name", cp.llvmpipe_names())
def test_llvmpipe_frames_replayed_through_the_kernels(name, built):
    """the reference's own frames on Mesa llvmpipe, from its own textures: the kernels equal the host build bit for bit,
    and so meet the same criterion against llvmpipe"""
    p, tex, want = cp.llvmpipe_case(name)
    with g.Renderer(p, batch=2) as r:
        r.raster_textures(np.stack([tex[0], tex[1]]), np.stack([tex[1], tex[0]]))
        got, swapped = r.readback(0), r.readback(1)
    assert np.array_equal(got, cp.host_frame(p, tex[0], tex[1])), name
    assert np.array_equal(swapped, cp.host_frame(p, tex[1], tex[0])), name
    cp.check_against_llvmpipe(name, got, want)
