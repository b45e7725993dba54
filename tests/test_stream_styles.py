"""Stream styles on the host (DESIGN 4.9): the ABI mirror, glava_b200_style_params' field mapping and refusals, its
equality with the `--pipe fg / bg` binds of the shipped configs, and the raster plan of a styled renderer (raster_plan.h
compiled for the host)."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import glava_b200 as g
from tests import emul
from tests import test_gpu_raster_variants as rv

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COLOURED = ("bars", "radial", "circle", "graph", "wave")
AMPLIFY = dict(bars="bars_amplify", radial="radial_amplify", circle="circle_amplify", graph="graph_vscale", wave="wave_amplify")


def _bytes(p):
    return C.string_at(C.addressof(p), C.sizeof(p))


def _style_params(base, style):
    return g.style_params(base, style)


def _einval(base, style):
    with pytest.raises(g.GlavaError):
        g.style_params(base, style)


def test_stream_style_struct_matches_header(built):
    hdr = open(os.path.join(ROOT, "include", "glava_b200.h")).read()
    m = re.search(r"typedef struct \{([^}]*)\} glava_b200_stream_style;", hdr)
    assert m and hdr.index("} glava_b200_params;") < m.start()
    fields = [re.sub(r"\[.*\]", "", d.strip()).split()[-1] for d in m.group(1).split(";") if d.strip()]
    assert fields == [f[0] for f in g.StreamStyle._fields_]
    assert C.sizeof(g.StreamStyle) == 4 + 4 + C.sizeof(g.Color) + 16
    for name, v in (("AMPLIFY", 1), ("FG", 2), ("BG", 4)):
        assert re.search(rf"#define GLAVA_B200_STYLE_{name}\s+{v}u", hdr)
        assert getattr(g, "STYLE_" + name) == v


def test_style_symbols_are_exported(built):
    L = C.CDLL(g.lib_path())
    for n in ("glava_b200_style_params", "glava_b200_set_stream_styles", "glava_b200_get_stream_styles",
              "glava_b200_sharded_set_stream_styles", "glava_b200_sharded_get_stream_styles"):
        assert hasattr(L, n), n


@pytest.mark.parametrize("module", COLOURED)
def test_field_mapping(module, built):
    base = g.load_config(force_module=module)
    assert _bytes(_style_params(base, None)) == _bytes(base)
    # amplify
    q = _style_params(base, {"amplify": -37.5})
    want = base.copy(); setattr(want, AMPLIFY[module], -37.5)
    assert _bytes(q) == _bytes(want)
    # constant fg
    fg = (0.25, 0.5, 0.75, 1.0)
    q = _style_params(base, {"fg": fg})
    want = base.copy()
    if module in ("bars", "radial", "graph"):
        col = getattr(want, module + "_color")
        col.mode = 1; col.lo = (C.c_float * 4)(*fg); col.hi = (C.c_float * 4)(*fg)
        getattr(want, module + "_color_prog").n_ops = 0
    else:
        setattr(want, "circle_outline" if module == "circle" else "wave_base_color", (C.c_float * 4)(*fg))
    assert _bytes(q) == _bytes(want)
    # gradient fg: taken whole where the module has a gradient, refused where fg is a plain colour
    grad = g.Color(0, (C.c_float * 4)(1, 0, 0, 1), (C.c_float * 4)(0, 0, 1, 0.5), 33.0)
    if module in ("bars", "radial", "graph"):
        q = _style_params(base, {"fg": grad})
        col = getattr(q, module + "_color")
        assert col.mode == 0 and tuple(col.hi) == (0, 0, 1, 0.5) and col.gradient == 33.0
    else:
        _einval(base, {"fg": grad})
    # bg
    bg = (0.125, 0.25, 0.375, 0.5)
    if module == "circle":
        _einval(base, {"bg": bg})
    else:
        q = _style_params(base, {"bg": bg})
        want = base.copy()
        if module == "bars":
            want.bars_outline_mode = 1; want.bars_outline = (C.c_float * 4)(*bg)
        elif module == "radial":
            want.radial_outline = (C.c_float * 4)(*bg); want.radial_bar_outline = (C.c_float * 4)(*bg)
        else:
            setattr(want, module + "_outline", (C.c_float * 4)(*bg))
        assert _bytes(q) == _bytes(want)
    # refusals common to every module
    bad = g.Color(2, (C.c_float * 4)(), (C.c_float * 4)(), 1.0)
    _einval(base, {"fg": bad})
    _einval(base, {"amplify": float("nan")})
    _einval(base, {"amplify": float("inf")})
    s = g.StreamStyle(); s.set = 8
    _einval(base, s)


def test_hex_colours_parse_as_pipe_binds(built):
    for text in ("#ff8000", "#ff8000c0", "#1A2B3C", "#00000000"):
        want = tuple(g.load_config(force_module="circle", binds={"fg": text}).circle_outline)
        assert g.stream_style({"fg": text}).fg.lo[:] == list(want), text
    for bad in ("ff8000x", "#zz0000", "", "#12345g"):
        with pytest.raises(g.GlavaError):
            g.stream_style({"fg": bad})


def test_test_module_has_no_style(built):
    base = g.default_params("test")
    assert _bytes(_style_params(base, None)) == _bytes(base)
    for st in ({"amplify": 2}, {"fg": (1, 1, 1, 1)}, {"bg": (0, 0, 0, 1)}):
        _einval(base, st)


def test_bars_fg_against_an_outline_expression(built):
    base = g.load_config(force_module="bars")
    base.bars_outline_mode = 2
    base.bars_outline_prog.n_ops = 1                        # SPLAT into register 0
    base.bars_outline_prog.result = 0
    _einval(base, {"fg": (1, 0, 0, 1)})                      # compiled against the renderer's own COLOR
    q = _style_params(base, {"fg": (1, 0, 0, 1), "bg": (0, 1, 0, 1)})
    assert q.bars_outline_mode == 1 and tuple(q.bars_outline) == (0, 1, 0, 1)
    q = _style_params(base, {"amplify": 9})                  # the outline stays
    assert q.bars_outline_mode == 2


def test_validation_of_styled_parameters(built):
    base = g.load_config(force_module="bars")
    bad = g.Color(-1, (C.c_float * 4)(), (C.c_float * 4)(), 1.0)
    _einval(base, {"fg": bad})


@pytest.mark.parametrize("module", COLOURED)
def test_style_equals_pipe_binds(module, built):
    """a style is the reference's `--pipe fg / bg` binding of the shipped configs, applied to one stream"""
    fg, bg = "#ff8000c0", "#1a2b3cff"
    base = g.load_config(force_module=module)
    binds = {"fg": fg} if module == "circle" else {"fg": fg, "bg": bg}
    want = g.load_config(force_module=module, binds=binds)
    got = g.style_params(base, binds)
    assert _bytes(got) == _bytes(want), module
    if module != "circle":                                   # one bind alone
        assert _bytes(g.style_params(base, {"bg": bg})) == _bytes(g.load_config(force_module=module, binds={"bg": bg}))
    assert _bytes(g.style_params(base, {"fg": fg})) == _bytes(g.load_config(force_module=module, binds={"fg": fg}))


# ---- the plan of a styled renderer (raster_plan.h on the host) ------------------------------------------------------------
_PLAN = ("kernel", "bx", "rows", "minb", "circle_tiles", "coltab", "texmm", "ctile", "rowtab", "geo", "chunk", "mark_key",
         "launches", "styled", "box_w", "box_h", "geo_bytes", "geo_caches")
_lib = None


def _plan_lib(tmp_path_factory):
    global _lib
    if _lib is None:
        so = str(tmp_path_factory.mktemp("style_plan") / "libstyle_plan.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-o", so,
                        os.path.join(ROOT, "tests", "emul", "style_plan.cpp")], check=True)
        _lib = C.CDLL(so)
        _lib.emul_styled_raster_plan.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                                 C.c_int, C.c_void_p]
    return _lib


def styled_plan(tmp_path_factory, slot_params, geo_caches, batch, fb_slots, env):
    arr = (g.Params * len(slot_params))(*slot_params)
    out = np.zeros(len(_PLAN), np.int64)
    _plan_lib(tmp_path_factory).emul_styled_raster_plan(arr, len(slot_params), geo_caches, batch, fb_slots,
                                                        *emul._env_arrays(env), out.ctypes.data)
    plan = dict(zip(_PLAN, out.tolist()))
    plan["kernel"] = emul.RASTER_KERNELS[plan["kernel"]]
    return plan


_COMMON = ("kernel", "bx", "rows", "minb", "circle_tiles", "coltab", "texmm", "ctile", "rowtab", "geo", "chunk", "mark_key",
           "launches")


def _styles_for(p):
    m = g.MODULES[p.module]
    if m == "test":
        return []
    out = [{"amplify": getattr(p, AMPLIFY[m]) * 1.5}, {"fg": (0.2, 0.9, 0.1, 1.0)}]
    if m != "circle":
        out.append({"bg": (0.3, 0.3, 0.3, 1.0), "amplify": getattr(p, AMPLIFY[m]) * 0.5})
    return out


@pytest.mark.parametrize("case", [c[0] for c in rv.CASES])
def test_styled_plan_of_every_raster_variant(case, tmp_path_factory, built):
    """no styles: the plan of today; styles: the same launches in the styled instantiation"""
    _, make, variants = next(c for c in rv.CASES if c[0] == case)
    p, (tl, _), _ = make()
    batch = tl.shape[0]
    for env in [{}] + variants:
        plain = emul.raster_plan(p, batch, batch, env)
        mine = styled_plan(tmp_path_factory, [p], 1, batch, batch, env)
        assert {k: mine[k] for k in _COMMON} == {k: plain[k] for k in _COMMON} and mine["styled"] == 0, env
        styles = _styles_for(p)
        if not styles:
            continue
        sp = [p] + [g.style_params(p, s) for s in styles]
        caches = len(sp) - 1 if g.MODULES[p.module] == "radial" else 1     # the amplify-only slot shares slot 0's cache
        st = styled_plan(tmp_path_factory, sp, caches, batch, batch, env)
        assert st["styled"] == 1 and st["launches"] == plain["launches"] and st["mark_key"] == plain["mark_key"], env
        for k in ("kernel", "rows", "bx", "coltab", "texmm"):
            if not (k == "kernel" and g.MODULES[p.module] == "radial"):
                assert st[k] == plain[k], (env, k)


def test_radial_cache_budget(tmp_path_factory, built):
    """radial keeps a cache per (fg, bg) pair in a box for the largest |AMPLIFY|; past 512 MiB together: the per-pixel kernel"""
    p = g.default_params("radial", n=1024, w=1920, h=1080)
    one = styled_plan(tmp_path_factory, [p], 1, 8, 8, {})
    assert one["kernel"] == "radial_geo" and one["geo_bytes"] > 0
    per = one["geo_bytes"]
    limit = (512 << 20) // per
    assert per * limit <= 512 << 20 < per * (limit + 1)
    for caches, kernel in ((limit, "radial_geo"), (limit + 1, "radial")):
        sp = [p, g.style_params(p, {"fg": (1, 0, 0, 1)})]
        plan = styled_plan(tmp_path_factory, sp, caches, 8, 8, {})
        assert plan["kernel"] == kernel and plan["styled"] == 1, caches
    # the box follows the largest |AMPLIFY| of the slots, in either sign
    big = styled_plan(tmp_path_factory, [p, g.style_params(p, {"amplify": -3 * p.radial_amplify})], 1, 8, 8, {})
    assert big["box_w"] > one["box_w"] and big["box_h"] > one["box_h"]
    small = styled_plan(tmp_path_factory, [p, g.style_params(p, {"amplify": 0.5 * p.radial_amplify})], 1, 8, 8, {})
    assert (small["box_w"], small["box_h"]) == (one["box_w"], one["box_h"])


def test_circle_box_follows_the_largest_amplify(tmp_path_factory, built):
    p = g.default_params("circle", n=1024, w=1920, h=1080)
    one = styled_plan(tmp_path_factory, [p], 1, 8, 8, {})
    big = styled_plan(tmp_path_factory, [p, g.style_params(p, {"amplify": 4 * p.circle_amplify})], 5, 8, 8, {})
    assert big["geo_caches"] == 1 and big["box_w"] > one["box_w"] and big["kernel"] == "circle"
