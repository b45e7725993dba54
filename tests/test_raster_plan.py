"""The raster pass the library plans (glava_b200/csrc/raster_plan.h, compiled into the host build), against a restatement of
DESIGN 4.2's kernel table and tile defaults: for every case and launch environment of tests/test_gpu_raster_variants.py and
for the option fallbacks, the kernel, tile shape, the kernels in front of it, the batch chunk, the dirty-row mark key and the
launches of one pass.  The GPU tier checks the same launch counts on the device."""
import pytest

import glava_b200 as g
from tests import emul
from tests import test_gpu_raster_variants as rv

BLOCK_WIDTHS = (96, 160, 128, 192, 256, 64)      # candidates in order of preference: the first that tiles w / 4 exactly


def _knob(env, name, default, ok=lambda v: v > 0):
    v = int(env.get(name, 0) or 0)
    return v if name in env and ok(v) else default


def restated(p, batch, slots, env):
    """DESIGN 4.2: which kernel a frame gets, its tile shape and what runs in front of it"""
    m = g.MODULES[p.module]
    native = p.premultiply_alpha != 0
    # the geometry cache is built for the real smooth pass; the raster view drops the circle cache under shader_pre_smoothed
    geo = (m == "radial" or (m == "circle" and bool(p.smooth_pass))) and "NO_GEO" not in env \
        and not (m == "circle" and p.shader_pre_smoothed)
    texmm = m == "circle" and geo and "NO_TEXMM" not in env
    bars = native and m == "bars" and not p.bars_mirror_yx and p.w % 4 == 0
    graph = native and m == "graph" and not p.graph_join_channels and not p.graph_anti_alias
    wave = native and m == "wave"
    rgeo = native and m == "radial" and geo and p.radial_nbars <= 1024 and not p.radial_bar_outline_width > 0
    wide = bars or graph or wave
    coltab = (graph or wave) and "NO_COLTAB" not in env
    minb = (5 if str(env.get("GW_MINB")) == "5" else 4) if coltab else (1 if graph or wave else 0)
    if bars: kernel = "bars"
    elif graph or wave: kernel = ("graph" if graph else "wave") + (f"_tab{minb}" if coltab else "")
    elif rgeo: kernel = "radial_geo"
    elif native and m in ("radial", "circle"): kernel = m
    else: kernel = "generic"
    rows = 540 if bars else ((16 if wave else 30) if coltab else 720) if graph or wave else 45 if rgeo else 8
    rows = min(_knob(env, "ROWS", rows), p.h)
    quads = (p.w + 3) // 4
    bx = _knob(env, "BX", next((c for c in BLOCK_WIDTHS if quads % c == 0), 128) if wide else 128,
               lambda v: 32 <= v <= 256 and v % 32 == 0)
    if not wide:
        bx = min(bx, 128)
    circle = kernel == "circle"
    chunk = min(slots, 32768)
    return dict(kernel=kernel, bx=256 if circle else bx, rows=rows, minb=minb,
                circle_tiles=_knob(env, "CIRCLE_TILES", 16) if circle else 0, coltab=int(coltab), texmm=int(texmm),
                ctile=int(texmm and "CTILE" in env), rowtab=int(m in ("bars", "graph")), geo=int(geo), chunk=chunk,
                mark_key=((1 if bars else 2 if graph else 3) | rows << 2) if wide else 0,
                launches=int(texmm) + -(-batch // chunk) * (2 if coltab else 1))


def _check(p, batch, slots, env):
    got = emul.raster_plan(p, batch, slots, env)
    got.pop("marks_valid")
    assert got == restated(p, batch, slots, env), env


@pytest.mark.parametrize("case", [c[0] for c in rv.CASES])
def test_plan_of_every_raster_variant(case, built):
    _, make, variants = next(c for c in rv.CASES if c[0] == case)
    p, (tl, _), _ = make()
    for env in [{}] + variants:
        _check(p, tl.shape[0], tl.shape[0], env)


def _params(module, **over):
    return g.default_params(module, n=1024, w=over.pop("w", 1920), h=over.pop("h", 1080), **over)


FALLBACKS = [
    ("bars-mirror_yx", "bars", dict(bars_mirror_yx=1), "generic"),
    ("bars-w%4", "bars", dict(w=333), "generic"),
    ("bars-blend", "bars", dict(premultiply_alpha=0), "generic"),
    ("graph-join", "graph", dict(graph_join_channels=1), "generic"),
    ("graph-aa", "graph", dict(graph_anti_alias=1), "generic"),
    ("radial-outline", "radial", dict(radial_bar_outline_width=1.0), "radial"),
    ("radial-nbars1030", "radial", dict(radial_nbars=1030), "radial"),
    ("circle-nosmooth", "circle", dict(smooth_pass=0), "circle"),
    ("circle-stale_on", "circle", dict(smooth_pass=0, shader_pre_smoothed=1), "circle"),
    ("circle-stale_off", "circle", dict(smooth_pass=1, shader_pre_smoothed=2), "circle"),
    ("test", "test", {}, "generic"),
]


@pytest.mark.parametrize("name,module,over,kernel", FALLBACKS, ids=[f[0] for f in FALLBACKS])
def test_option_fallbacks(name, module, over, kernel, built):
    p = _params(module, **over)
    assert emul.raster_plan(p, 4, 4, {})["kernel"] == kernel
    for env in ({}, dict(BX=256), dict(ROWS=7), dict(NO_GEO=1), dict(NO_TEXMM=1), dict(CTILE=1)):
        _check(p, 4, 4, env)
    if module == "circle":                       # neither the stale belief nor a raw texture may use the cache
        assert not emul.raster_plan(p, 4, 4, {})["texmm"]


@pytest.mark.parametrize("module", g.MODULES)
@pytest.mark.parametrize("batch,slots", [(32771, 32771), (32768, 32768), (8, 3), (8, 1), (70000, 70000)])
def test_batch_chunks(module, batch, slots, built):
    """one launch covers at most 32768 streams, and at most `slots` with a framebuffer ring"""
    p = _params(module, w=96, h=48)
    for env in ({}, dict(NO_COLTAB=1)):
        _check(p, batch, slots, env)
    plan = emul.raster_plan(p, batch, slots, {})
    assert plan["chunk"] == min(slots, 32768) and plan["launches"] >= -(-batch // plan["chunk"])


def _key(p, env=None):
    return emul.raster_plan(p, 8, 8, env or {})["mark_key"]


def _valid(p, last_key, env=None):
    return bool(emul.raster_plan(p, 8, 8, env or {}, last_key=last_key)["marks_valid"])


def test_mark_key_rules(built):
    bars, graph, wave = _params("bars"), _params("graph"), _params("wave")
    mirror = _params("bars", bars_mirror_yx=1)
    for p in (bars, graph, wave):
        k = _key(p)
        assert k != 0 and _valid(p, k)                                      # the same kernel at the same rows
        assert not _valid(p, _key(p, dict(ROWS=135)))                       # another band height
        assert not _valid(p, k, dict(FULL_STORE=1))                         # forced full store
        assert _valid(p, k, dict(FULL_STORE=0))
        assert not _valid(p, 0)                                             # nothing recorded yet
    rows = dict(ROWS=30)
    keys = {_key(p, rows) for p in (bars, graph, wave)}
    assert len(keys) == 3                                                   # another kernel at the same rows
    assert not _valid(graph, _key(bars, rows), rows)
    # a kernel that keeps no marks records 0, so the next marks kernel stores every zero row
    assert _key(mirror) == 0 and not _valid(bars, _key(mirror))
    assert not _valid(mirror, _key(bars))
