"""-m gpu: the styled raster kernels (DESIGN 4.9) in every launch form, bit for bit against the oracle at each stream's
styled parameters, and their dirty-row marks across the styled / plain switch.

A stream of style `s` must render what the oracle renders at style_params(p, s).  The styled twins read their stream's
style slot (parameters, row table, geometry cache) instead of the kernel parameter; two of them (wave, circle) are kept by
hand beside the plain kernels' text.  Every case and launch variant of tests/test_gpu_raster_variants.py runs here again,
with GLAVA_B200_FULL_STORE added, on a batch in which every texture of the case is rendered in each AMPLIFY group of
styles: the renderer's own AMPLIFY (unstyled, constant and gradient fg, bg), x0.5, x1.7 (which grows the polar box beyond
the base parameters' box) and, for radial and circle, the negated AMPLIFY.  Within a group the styles cycle over the
streams, so each style lands on several streams and radial builds a cache for several (fg, bg) pairs.  Height ramps are
built for the AMPLIFY of their group.  The coverage assertions, computed from the oracle frames, keep the cases reaching
the per-stream bounds: ramp heights, lines that leave the frame, the polar reach and ring culls per styled AMPLIFY,
pixels outside the base box, and a circle CTA region outside one stream's reach where another stream draws.

The dirty-row sequences drive one renderer through styles set, changed (AMPLIFY x1.7 to x0.3 on unchanged textures, so
that only the style shrinks the frame) and cleared, at several band heights and framebuffer rings.  The marks' key is the
plain plan's, so marks written by a styled twin are trusted by the plain kernel and the reverse."""
import ctypes as C

import numpy as np
import pytest

import glava_b200 as g
from oracle.oracle import params_from
from tests import emul
from tests import test_gpu_dirty_rows as dr
from tests import test_gpu_raster_variants as rv
from tests.test_stream_styles import _plan_lib

pytestmark = pytest.mark.gpu

N = rv.N
KNOBS = rv.KNOBS + ("FULL_STORE",)
AMP = dict(bars="bars_amplify", radial="radial_amplify", circle="circle_amplify", graph="graph_vscale", wave="wave_amplify")
GRAD = ((0.9, 0.1, 0.2, 1.0), (0.1, 0.2, 0.9, 0.6), 17.0)
FG1, FG2, BG = "#ff8000", (0.2, 0.9, 0.4, 0.8), (0.4, 0.5, 0.1, 1.0)


def _module(p):
    return g.MODULES[p.module]


def _amp(p):
    return getattr(p, AMP[_module(p)])


def _groups(p):
    """[(AMPLIFY, styles)]: every texture of the case is rendered once per group, the group's styles cycling over it"""
    m, a = _module(p), _amp(p)
    grad = g.Color(0, (C.c_float * 4)(*GRAD[0]), (C.c_float * 4)(*GRAD[1]), GRAD[2])
    own = [None, {"fg": FG1}]
    if m in ("bars", "radial", "graph"):
        own.append({"fg": grad})
    if m != "circle":
        own += [{"bg": BG}, {"fg": FG2, "bg": BG}]
    groups = [(a, own), (0.5 * a, [{"amplify": 0.5 * a}, {"amplify": 0.5 * a, "fg": FG2}]),
              (1.7 * a, [{"amplify": 1.7 * a}, {"amplify": 1.7 * a, "fg": FG1}])]
    if m in ("radial", "circle"):
        groups.append((-a, [{"amplify": -a}, {"amplify": -a, "fg": FG2}]))
    return groups


def _ramp_top(h, amp):
    """the highest column height a ramp built for `amp` reaches in every one of its bands"""
    return h if amp >= 1.05 * h else int(0.95 * amp)


def _textures(p, amp):
    """the case's textures (tests/test_gpu_raster_variants.py) with the height ramps built for `amp`, and the ramp bands"""
    m, w, h = _module(p), p.w, p.h
    rows, bands = rv._edges(N), None
    if m in ("bars", "graph"):
        per = int((w / 2) // (p.bars_width + p.bars_gap)) if m == "bars" else w // 2
        ramps, bands = rv._height_ramps(N, _ramp_top(h, amp), amp, per)
        rows = rows + ramps
    elif m == "wave":
        rows = rows + rv._wave_rows(N, w + h)
    else:
        rows = rows + rv._polar_bands(N, w + h)
    return rows, bands


def _styled_batch(p):
    """(tl, tr, styles, groups): groups = [(AMPLIFY, first stream, streams, ramp bands)]"""
    rows, styles, groups = [], [], []
    for amp, st in _groups(p):
        tex, bands = _textures(p, amp)
        groups.append((amp, len(rows), len(tex), bands))
        rows += tex
        styles += [st[k % len(st)] for k in range(len(tex))]
    tl, tr = rv._stack(rows)
    return tl, tr, styles, groups


def _base_box(tmp_path_factory, p):
    box = (C.c_int * 4)()
    lib = _plan_lib(tmp_path_factory)
    lib.emul_styled_geo_box.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    lib.emul_styled_geo_box(C.byref(p), 1, box)
    return tuple(box)


def _check_heights(frames, bands, top, h):
    """as test_gpu_raster_variants._check_heights, with the bands covering 0..top (top < h: a ramp AMPLIFY below h)"""
    assert not frames[0].any() and rv._column_heights(frames[1]).max() >= top
    covered = set()
    for k, (lo, hi) in enumerate(bands):
        got = set(rv._column_heights(frames[4 + k]).tolist())
        missing = sorted(set(range(lo, hi + 1)) - got)
        assert not missing, ("ramp stream", 4 + k, "misses column heights", missing[:10])
        covered |= set(range(lo, hi + 1))
    assert covered == set(range(top + 1))


def _circle_cta_split(p, want, styles, groups):
    """1080p circle: some 128 x 128 CTA region (CIRCLE_TILES default) lies outside one styled stream's static reach while
    a x1.7 stream lights a pixel in it, so the whole-CTA zero region is decided per stream"""
    cx, cy = p.w // 2, p.h // 2
    lit_big = [(want[s] != 0).any(axis=2) for s in range(groups[2][1], groups[2][1] + groups[2][2])]
    reaches = []
    for amp, first, count, _ in groups:
        q = g.style_params(p, styles[first + 1])
        reaches.append(np.float32(q.circle_radius) + abs(np.float32(q.circle_amplify)) + abs(np.float32(q.circle_line)) + 3)
    for tx0 in range(0, p.w, 128):
        bx0, bx1 = tx0 - 1 - cx, tx0 + 128 - cx
        nx = bx0 if bx0 > 0 else (-bx1 if bx1 < 0 else 0)
        for y0 in range(0, p.h, 128):
            y1 = min(p.h, y0 + 128)
            cb0, cb1 = y0 - 1 - cy, y1 - cy
            ny = cb0 if cb0 > 0 else (-cb1 if cb1 < 0 else 0)
            if nx * nx + ny * ny > min(reaches) ** 2 and any(f[y0:y1, tx0:tx0 + 128].any() for f in lit_big):
                return
    pytest.fail("no circle CTA region outside one stream's reach that a x1.7 stream lights")


def _coverage(p, want, styles, groups, tmp_path_factory):
    m, h = _module(p), p.h
    for amp, first, count, bands in groups:
        fr = want[first:first + count]
        if m in ("bars", "graph"):
            if not p.graph_invert or m == "bars":
                _check_heights(fr, bands, _ramp_top(h, amp), h)
        elif m == "wave":
            if abs(amp) <= abs(_amp(p)):
                rv._check_wave(fr, h)
            lit = (fr[7] != 0).any(axis=(1, 2))
            assert lit[0] and lit[h - 1], (amp, "the ramp's line does not leave the frame at both ends")
        else:
            if m == "radial":
                cx, cy, radius, ring = p.w // 2 - p.radial_off_x, p.h // 2 - p.radial_off_y, p.radial_radius, False
            else:
                cx, cy, radius, ring = p.w // 2, p.h // 2, p.circle_radius, amp > 0 and not p.circle_fill
            if amp > 0 or _amp(p) < 0:
                rv._check_polar(fr, cx, cy, radius, amp, ring)
            else:                                          # the negated AMPLIFY: only the curve near the base circle draws
                d = [rv._lit_radii(f, cx, cy) for f in fr]
                assert any(x.size for x in d) and all(abs(x.min() - radius) < 0.2 * abs(amp) + 4 for x in d if x.size)
    if m in ("radial", "circle") and _amp(p) > 0:
        x0, y0, bw, bh = _base_box(tmp_path_factory, p)
        outside = np.ones((p.h, p.w), bool)
        outside[y0:y0 + bh, x0:x0 + bw] = False
        _, first, count, _ = groups[2]
        assert any(((want[s] != 0).any(axis=2) & outside).any() for s in range(first, first + count)), \
            ("no x1.7 stream lights a pixel outside the base box", (x0, y0, bw, bh))
    if m == "circle" and (p.w, p.h) == rv.HD:
        _circle_cta_split(p, want, styles, groups)


def _render(p, tl, tr, styles, env, monkeypatch):
    for k in KNOBS:
        monkeypatch.delenv("GLAVA_B200_" + k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv("GLAVA_B200_" + k, str(v))
    batch = tl.shape[0]
    with g.Renderer(p, batch=batch) as r:
        r.set_stream_styles(range(batch), styles)
        before = r.launch_count
        r.raster_textures(tl, tr)
        assert r.launch_count - before == emul.raster_plan(p, batch, batch, env)["launches"], env
        return [r.readback(s) for s in range(batch)]


def _variants(variants):
    return list(variants) + [dict(FULL_STORE=1)]


def _run_case(orc, p, tl, tr, styles, variants, monkeypatch):
    ops = {}
    want = []
    for s in range(tl.shape[0]):
        key = None if styles[s] is None else bytes(g.stream_style(styles[s]))
        if key not in ops:
            ops[key] = params_from(g.style_params(p, styles[s]))
        want.append(orc.raster(ops[key], tl[s], tr[s]))
    for env in variants:
        got = _render(p, tl, tr, styles, env, monkeypatch)
        for s in range(tl.shape[0]):
            bad = (got[s] != want[s]).any(axis=2)
            if bad.any():
                ys, xs = np.nonzero(bad)
                pytest.fail(f"{env} stream {s} style {styles[s]}: {int(bad.sum())} pixels differ, first (x, y) = ({xs[0]}, {ys[0]})")
    return want


def _cases():
    c = [(name, make, _variants(v)) for name, make, v in rv.CASES]
    for w, h in rv.SMALL:
        geo = [{}, dict(ROWS=1), dict(ROWS=h), dict(NO_GEO=1)]
        c.append((f"radial-nbars1030-off-{w}x{h}",
                  lambda w=w, h=h: rv._polar_case("radial", w, h, radial_nbars=1030, radial_off_x=w / 2 - 12.0, radial_off_y=-30.0),
                  _variants(geo)))
    return c


CASES = _cases()


@pytest.mark.parametrize("case", [c[0] for c in CASES])
def test_styled_raster_variants_equal_the_oracle(orc_pm, case, monkeypatch, tmp_path_factory, built):
    _, make, variants = next(c for c in CASES if c[0] == case)
    p, _, _ = make()
    tl, tr, styles, groups = _styled_batch(p)
    assert len({(a.tobytes(), b.tobytes(), None if s is None else bytes(g.stream_style(s)))
                for a, b, s in zip(tl, tr, styles)}) == tl.shape[0]
    want = _run_case(orc_pm, p, tl, tr, styles, variants, monkeypatch)
    _coverage(p, want, styles, groups, tmp_path_factory)


# ---- dirty-row marks across styles -----------------------------------------------------------------------------------
SEQ_BATCH = 7


def _seq_styles(p, kind):
    """per-stream styles: "grow" (AMPLIFY x1.7, some with a colour), "shrink" (the same streams at x0.3), "none" """
    a = _amp(p)
    if kind == "none":
        return [None] * SEQ_BATCH
    f = 1.7 if kind == "grow" else 0.3
    return [{"amplify": f * a}, None, {"amplify": f * a, "fg": FG1}, {"amplify": f * a}, {"fg": FG2},
            {"amplify": f * a, "bg": BG}, {"amplify": f * a}]


def _seq_check(r, p, styles, tl, tr, what):
    """every slot holds the frame of the highest stream mapped to it, at that stream's styled parameters"""
    slots = p.fb_slots if 0 < p.fb_slots < SEQ_BATCH else SEQ_BATCH
    for k in range(slots):
        s = max(t for t in range(SEQ_BATCH) if t % slots == k)
        got = r.readback(s)
        want = emul.raster(g.style_params(p, styles[s]), tl[s], tr[s], fast=True)
        assert np.array_equal(got, want), (what, s, styles[s], int((got != want).any(axis=2).sum()))


@pytest.mark.parametrize("fb_slots", [0, 1, 3])
@pytest.mark.parametrize("case", sorted(dr.CASES))
def test_styled_sequence_across_band_heights(case, fb_slots, monkeypatch, built):
    """styles set, changed and cleared between steps, on unchanged textures where the style alone moves the rows, with the
    band height changing in between"""
    for k in KNOBS:
        monkeypatch.delenv("GLAVA_B200_" + k, raising=False)
    p = dr._params(case, fb_slots=fb_slots)
    h = str(p.h)
    steps = [(None, "none", 0), (None, "grow", 0), (None, "shrink", 0), ("16", "shrink", 1), ("16", "grow", 1),
             ("16", "none", 1), ("7", "grow", 2), ("7", "shrink", 2), ("1", "shrink", 3), ("1", "none", 3), (h, "grow", 0),
             (h, "shrink", 0), (h, "none", 0), (None, "grow", 1)]
    with g.Renderer(p, batch=SEQ_BATCH) as r:
        cur = None
        for step, (rows, kind, tex) in enumerate(steps):
            if rows is None:
                monkeypatch.delenv("GLAVA_B200_ROWS", raising=False)
            else:
                monkeypatch.setenv("GLAVA_B200_ROWS", rows)
            styles = _seq_styles(p, kind)
            if kind != cur:
                r.set_stream_styles(range(SEQ_BATCH), styles)
                cur = kind
            tl, tr = dr._textures(SEQ_BATCH, r.nsz, tex)
            r.raster_textures(tl, tr)
            _seq_check(r, p, styles, tl, tr, (case, fb_slots, step, rows, kind))
