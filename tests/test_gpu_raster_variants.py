"""-m gpu: every launch form of the raster pass, bit for bit against the oracle.

raster_plan.h plan_raster picks one of eleven kernels and template instantiations and takes its tile shape from the
environment (GLAVA_B200_ROWS, _BX, _GW_MINB, _CIRCLE_TILES, _NO_COLTAB, _NO_TEXMM at every launch; _NO_GEO, _CTILE when the
tables are built; DESIGN 6.2); launch_raster executes the plan.  tests/test_raster_plan.py checks which plan each variant
gets on the host; here every variant's pass must issue the plan's launches.  The row band moves the warp-uniform splits of the specialised kernels (bars z0/z1/f0/f1, graph b1/b2/b3, wave
ra/rb, radial_geo band_live), and those splits exist only in the kernels.  Each case computes the oracle's frames once and
runs every variant on them through raster_textures.  The textures reach the edges: silence, saturation, single spikes at
texel 0 and n - 1, height ramps whose columns take every row value from 0 to h (bars, graph), lines that leave the frame
(wave), narrow value bands that make each per-stream cull bound live somewhere (radial, circle).  Each coverage claim is
asserted from the oracle frames."""
import math

import numpy as np
import pytest

import glava_b200 as g
from oracle.oracle import params_from
from tests import emul

pytestmark = pytest.mark.gpu

N = 1024
KNOBS = ("ROWS", "BX", "GW_MINB", "NO_COLTAB", "CIRCLE_TILES", "CTILE", "NO_TEXMM", "NO_GEO")
SMALL = [(332, 181), (333, 181)]          # 83 quads: no candidate block width tiles them; w % 4 != 0; odd height
HD = (1920, 1080)


# ---- textures --------------------------------------------------------------------------------------------------------
def _edges(n):
    """silence, saturation, and single spikes at texel 0 and n - 1 (left / right swapped in the second spike stream)"""
    z = np.zeros(n, np.uint16); f = np.full(n, 65535, np.uint16)
    a = z.copy(); a[0] = 65535
    b = z.copy(); b[-1] = 65535
    return [(z, z), (f, f), (a, b), (b, a)]


def _stack(rows):
    return np.stack([r[0] for r in rows]), np.stack([r[1] for r in rows])


def _height_ramps(n, h, amp, per_channel):
    """streams whose left texture ramps up and right texture down through heights a little beyond [lo, hi] (height = texel /
    65535 * amp); the bands [lo, hi] partition 0..h and are narrow enough that `per_channel` evenly spread samples of a ramp
    are less than one row apart"""
    bands = max(2, math.ceil((h + 1) / (0.6 * per_channel - 6)))
    cuts = np.linspace(0, h + 1, bands + 1).round().astype(int)
    rows, want = [], []
    for k in range(bands):
        lo, hi = int(cuts[k]), int(cuts[k + 1]) - 1
        m = 3 + 0.08 * (hi - lo)                      # graph tapers the outer and centre columns: the ramp ends land there
        u = np.clip(np.rint(np.linspace(lo - m, hi + m, n) / amp * 65535), 0, 65535).astype(np.uint16)
        rows.append((u, u[::-1].copy()))
        want.append((lo, hi))
    return rows, want


def _column_heights(frame):
    return (frame != 0).any(axis=2).sum(axis=0)


def _check_heights(frames, bands, h):
    """stream 4 + k lights every column height of band k (bands cover 0..h); silence lights nothing, saturation reaches h"""
    assert not frames[0].any() and _column_heights(frames[1]).max() == h
    covered = set()
    for k, (lo, hi) in enumerate(bands):
        got = set(_column_heights(frames[4 + k]).tolist())
        missing = sorted(set(range(lo, hi + 1)) - got)
        assert not missing, ("ramp stream", 4 + k, "misses column heights", missing[:10])
        covered |= set(range(lo, hi + 1))
    assert covered == set(range(h + 1))


def _polar_bands(n, seed):
    """narrow value bands (as test_polar_per_stream_reach_cull), each stream's right channel the band of another stream"""
    rng = np.random.default_rng(seed)
    bands = [(0, 1), (0, 700), (3000, 3400), (20000, 21000), (64000, 65535), (100, 40000)]
    tl = [rng.integers(lo, hi + 1, n).astype(np.uint16) for lo, hi in bands]
    tr = [rng.integers(lo, hi + 1, n).astype(np.uint16) for lo, hi in bands]
    return [(tl[k], tr[k]) for k in range(len(bands))]


def _lit_radii(frame, cx, cy):
    ys, xs = np.nonzero((frame != 0).any(axis=2))
    return np.hypot(xs + 0.5 - cx, ys + 0.5 - cy)


def _check_polar(frames, cx, cy, radius, amp, ring):
    """some stream's curve stays within a fifth of AMPLIFY of C_RADIUS (the per-stream reach / tile cull cut the rest),
    another reaches past four fifths of it; with `ring` (circle without fill) most of some stream's curve lies outside the
    base circle, which the inner-ring cull skips.  A negative AMPLIFY draws only where the curve is near the base circle:
    some stream lights the whole ring, another almost nothing."""
    near, far, outside, sizes = [], [], [], []
    for f in frames[4:]:                                   # the band streams
        d = _lit_radii(f, cx, cy)
        assert d.size, "band stream lights nothing"
        ext = d.max() if amp > 0 else d.min()
        near.append(abs(ext - radius) < 0.2 * abs(amp) + 4)
        far.append(abs(ext - radius) > 0.8 * abs(amp))
        outside.append(np.percentile(d, 5) > radius + 0.6 * amp)
        sizes.append(d.size)
    assert any(near), near
    if amp > 0:
        assert any(far), far
    else:
        assert min(sizes) * 10 < _lit_radii(frames[0], cx, cy).size <= max(sizes), sizes
    if ring:
        assert any(outside), "no stream whose curve lies mostly outside the base circle"


def _wave_rows(n, seed):
    """lines around 0.5 (PCM-like, as the other wave tests), then a full ramp whose line leaves the frame at both ends"""
    rng = np.random.default_rng(seed)
    rows = []
    for k in range(3):
        u = (rng.random(n) * 16383 + 24576 + (k - 1) * 2000).astype(np.uint16)
        rows.append((u, u[::-1].copy()))
    ramp = np.linspace(0, 65535, n).round().astype(np.uint16)
    rows.append((ramp, ramp[::-1].copy()))
    return rows


def _check_wave(frames, h):
    inside, ramp = frames[4:7], frames[7]
    for f in inside:
        lit = (f != 0).any(axis=(1, 2))
        assert lit.any() and not lit[0] and not lit[h - 1], "line around 0.5 touches the top or bottom row"
    lit = (ramp != 0).any(axis=(1, 2))
    assert lit[0] and lit[h - 1], "the ramp's line does not leave the frame at both ends"


# ---- cases -----------------------------------------------------------------------------------------------------------
def _bars_case(w, h, **over):
    p = g.default_params("bars", n=N, w=w, h=h, bars_amplify=1.25 * h, **over)
    ramps, bands = _height_ramps(N, h, p.bars_amplify, int((w / 2) // (p.bars_width + p.bars_gap)))
    return p, _stack(_edges(N) + ramps), lambda fr: _check_heights(fr, bands, h)


def _graph_case(w, h, **over):
    p = g.default_params("graph", n=N, w=w, h=h, graph_vscale=1.25 * h, **over)
    ramps, bands = _height_ramps(N, h, p.graph_vscale, w // 2)
    return p, _stack(_edges(N) + ramps), (None if p.graph_invert else (lambda fr: _check_heights(fr, bands, h)))


def _wave_case(w, h, **over):
    p = g.default_params("wave", n=N, w=w, h=h, wave_amplify=2.5 * h, **over)
    return p, _stack(_edges(N) + _wave_rows(N, w + h)), lambda fr: _check_wave(fr, h)


def _polar_case(module, w, h, **over):
    small = h < 1080
    base = (dict(radial_radius=30.0, radial_amplify=50.0) if module == "radial" else dict(circle_radius=30.0, circle_amplify=50.0)) \
        if small else {}
    base.update(over)
    p = g.default_params(module, n=N, w=w, h=h, **base)
    if module == "radial":
        cx, cy, radius, amp, ring = w // 2 - p.radial_off_x, h // 2 - p.radial_off_y, p.radial_radius, p.radial_amplify, False
    else:
        cx, cy, radius, amp = w // 2, h // 2, p.circle_radius, p.circle_amplify
        ring = amp > 0 and not p.circle_fill
    return p, _stack(_edges(N) + _polar_bands(N, w + h)), lambda fr: _check_polar(fr, cx, cy, radius, amp, ring)


def _rows_variants(h, rows):
    return [dict(ROWS=r) for r in rows]


def _gw_variants(h, rows=(1, 3, 16, 30, None), bx=64):
    """{column table, NO_COLTAB, 48-register budget} x row bands, with a block width that leaves a partial last CTA"""
    out = [{}, dict(NO_COLTAB=1), dict(GW_MINB=5)]
    for tab in ({}, dict(NO_COLTAB=1), dict(GW_MINB=5)):
        for r in rows:
            out.append(dict(tab, ROWS=h if r is None else r, BX=bx))
    return out


def _cases():
    c = []
    for w, h in SMALL:
        for flip in (0, 1):
            v = _rows_variants(h, (1, 2, 7, 135, h - 1, h, h + 37))
            if not flip:
                v += [dict(BX=b) for b in (32, 64, 96, 128, 160, 192, 256)]
            c.append((f"bars-flip{flip}-{w}x{h}", lambda w=w, h=h, flip=flip: _bars_case(w, h, bars_flip=flip), v))
        for module, mk in (("graph", _graph_case), ("wave", _wave_case)):
            c.append((f"{module}-{w}x{h}", lambda w=w, h=h, mk=mk: mk(w, h), _gw_variants(h)))
        c.append((f"graph-invert-{w}x{h}", lambda w=w, h=h: _graph_case(w, h, graph_invert=1), _gw_variants(h, rows=(1, 30, None))))
        geo = [dict(NO_GEO=1, ROWS=r) for r in (1, 45, h)] + [dict(ROWS=r) for r in (1, 45, h)]
        for name, over in (("", {}), ("-nbars200", dict(radial_nbars=200)), ("-nbars300", dict(radial_nbars=300)),
                           ("-nbars1030", dict(radial_nbars=1030)), ("-off-left", dict(radial_off_x=w / 2 - 12.0)),
                           ("-off-right", dict(radial_off_x=-(w / 2 - 9.0), radial_off_y=20.0))):
            v = [{}] + geo + ([dict(BX=b) for b in (32, 256)] + [dict(NO_GEO=1, BX=256)] if not over else [])
            c.append((f"radial{name}-{w}x{h}", lambda w=w, h=h, over=over: _polar_case("radial", w, h, **over), v))
        cv = [{}] + [dict(CIRCLE_TILES=t) for t in (1, 3, 16, (h + 7) // 8 + 5)] + \
             [dict(CTILE=1), dict(CTILE=1, CIRCLE_TILES=1), dict(NO_TEXMM=1), dict(NO_GEO=1), dict(NO_GEO=1, CIRCLE_TILES=3)]
        for name, over in (("", {}), ("-nosmooth", dict(smooth_pass=0)), ("-fill", dict(circle_fill=1)),
                           ("-negamp", dict(circle_amplify=-25.0))):
            c.append((f"circle{name}-{w}x{h}", lambda w=w, h=h, over=over: _polar_case("circle", w, h, **over), cv))
    w, h = HD
    c.append(("bars-flip0-1920x1080", lambda: _bars_case(w, h), [{}] + _rows_variants(h, (135, h - 1, h, h + 1)) + [dict(BX=160)]))
    c.append(("bars-flip1-1920x1080", lambda: _bars_case(w, h, bars_flip=1), _rows_variants(h, (135, h - 1, h))))
    for module, mk in (("graph", _graph_case), ("wave", _wave_case)):
        c.append((f"{module}-1920x1080", lambda mk=mk: mk(w, h), _gw_variants(h, rows=(16, 30, None), bx=96)[3:]))
    c.append(("radial-1920x1080", lambda: _polar_case("radial", w, h), [{}, dict(ROWS=h), dict(NO_GEO=1)]))
    c.append(("circle-1920x1080", lambda: _polar_case("circle", w, h), [{}, dict(CTILE=1), dict(CIRCLE_TILES=1), dict(NO_TEXMM=1)]))
    return c


CASES = _cases()


def _render(p, tl, tr, env, monkeypatch):
    for k in KNOBS:
        monkeypatch.delenv("GLAVA_B200_" + k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv("GLAVA_B200_" + k, str(v))
    with g.Renderer(p, batch=tl.shape[0]) as r:
        before = r.launch_count
        r.raster_textures(tl, tr)
        assert r.launch_count - before == emul.raster_plan(p, tl.shape[0], tl.shape[0], env)["launches"], env
        return [r.readback(s) for s in range(tl.shape[0])]


def _compare(orc, p, tl, tr, variants, monkeypatch):
    op = params_from(p)
    want = [orc.raster(op, tl[s], tr[s]) for s in range(tl.shape[0])]
    for env in variants:
        got = _render(p, tl, tr, env, monkeypatch)
        for s in range(tl.shape[0]):
            bad = (got[s] != want[s]).any(axis=2)
            if bad.any():
                ys, xs = np.nonzero(bad)
                pytest.fail(f"{env} stream {s}: {int(bad.sum())} pixels differ, first (x, y) = ({xs[0]}, {ys[0]})")
    return want


@pytest.mark.parametrize("case", [c[0] for c in CASES])
def test_raster_variants_equal_the_oracle(orc_pm, case, monkeypatch, built):
    _, make, variants = next(c for c in CASES if c[0] == case)
    p, (tl, tr), coverage = make()
    assert tl.shape[0] >= 3 and len({(a.tobytes(), b.tobytes()) for a, b in zip(tl, tr)}) == tl.shape[0]
    want = _compare(orc_pm, p, tl, tr, variants, monkeypatch)
    if coverage:
        coverage(want)


@pytest.mark.parametrize("w,h", SMALL)
@pytest.mark.parametrize("case", ["blend", "mirror_yx"])
def test_generic_kernel_block_widths(orc_pm, case, w, h, monkeypatch, built):
    """raster_generic_kernel is __launch_bounds__(128): a GLAVA_B200_BX above that must not fail the launch (nor may it for
    the two radial kernels, above), and every width must give the oracle's pixels"""
    if case == "blend":
        p = g.default_params("graph", n=N, w=w, h=h, premultiply_alpha=0, clear_color=[0.05, 0.05, 0.1, 1.0], graph_vscale=1.25 * h)
    else:
        p = g.default_params("bars", n=N, w=w, h=h, bars_mirror_yx=1, bars_amplify=1.25 * w)
    tl, tr = _stack(_edges(N) + _height_ramps(N, h, 1.25 * h, w // 2)[0][:2])
    _compare(orc_pm, p, tl, tr, [dict(BX=b) for b in (32, 128, 256)], monkeypatch)
