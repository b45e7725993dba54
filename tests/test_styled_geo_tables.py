"""The polar geometry caches that a styled renderer really builds, without a GPU: capi.cu built against the fake runtime of
tests/fakecuda, whose launch_polar_geo records the parameters and the box of every call.

A renderer with stream styles (DESIGN 4.9) builds its radial / circle geometry cache in one box for the largest |AMPLIFY|
of its style slots, so that a slot whose AMPLIFY grows the disc still finds its pixels in the cache.  Radial keeps one
cache per distinct (fg, bg) pair of the slots, built from the first slot with that pair; circle keeps one, built from the
renderer's own parameters.  Each set_stream_styles rebuilds the tables; the calls it makes must match that, with styles
set, changed to a smaller and to a negative AMPLIFY, and cleared.  Every cache must start 16-byte aligned: the radial
caches lie back to back, and at 332x181 the box has a pixel count that is not a multiple of 16."""
import ctypes as C

import pytest

import glava_b200 as g
from tests import fakecuda
from tests.test_stream_styles import _plan_lib

BATCH = 6
AMP = dict(radial="radial_amplify", circle="circle_amplify")
KNOBS = ("ROWS", "BX", "GW_MINB", "NO_COLTAB", "CIRCLE_TILES", "CTILE", "NO_TEXMM", "NO_GEO", "FULL_STORE")
SIZES = {"332x181": dict(w=332, h=181, radius=30.0, amplify=50.0), "1920x1080": dict(w=1920, h=1080)}


@pytest.fixture(scope="module")
def fake(built):
    if fakecuda.cuda_include() is None:
        pytest.skip("no CUDA toolkit headers")
    L = fakecuda.lib()
    vp, i32 = C.c_void_p, C.c_int
    P = C.POINTER(g.Params)
    for name, (res, args) in {"glava_b200_new": (vp, [P, i32, i32]), "glava_b200_destroy": (None, [vp]),
                              "glava_b200_set_stream_styles": (i32, [vp, vp, i32, vp]),
                              "glava_b200_set_abort_hook": (None, [vp]), "fake_geo_calls": (C.c_long, []),
                              "fake_geo_call": (i32, [C.c_long, P, vp])}.items():
        f = getattr(L, name)
        f.restype, f.argtypes = res, args
    quiet = C.CFUNCTYPE(None, C.c_char_p)(lambda msg: None)
    L.glava_b200_set_abort_hook(C.cast(quiet, vp))
    L._quiet = quiet
    return L


def _bytes(p):
    return C.string_at(C.addressof(p), C.sizeof(p))


def _calls(L):
    out = []
    for i in range(L.fake_geo_calls()):
        p, box = g.Params(), (C.c_int * 4)()
        assert L.fake_geo_call(i, C.byref(p), box) == 0, ("cache", i, "is not 16-byte aligned")
        out.append((p, tuple(box)))
    return out


def _styled_box(tmp_path_factory, slot_params):
    arr = (g.Params * len(slot_params))(*slot_params)
    box = (C.c_int * 4)()
    lib = _plan_lib(tmp_path_factory)
    lib.emul_styled_geo_box.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    lib.emul_styled_geo_box(arr, len(slot_params), box)
    return tuple(box)


def _key(style):
    return None if style is None else bytes(g.stream_style(style))


def _expected(p, styles):
    """slot 0 (the renderer's own parameters), then every distinct style in stream order; radial: the first slot of each
    distinct (fg, bg) pair builds that pair's cache, circle: slot 0 builds the one cache"""
    slots, seen = [p], {None}
    pair_rep, pairs = [p], {(None, None)}
    for st in styles:
        if _key(st) in seen:
            continue
        seen.add(_key(st))
        q = g.style_params(p, st)
        slots.append(q)
        pair = tuple(None if st.get(k) is None else bytes(getattr(g.stream_style({k: st[k]}), k)) for k in ("fg", "bg"))
        if pair not in pairs:
            pairs.add(pair)
            pair_rep.append(q)
    return slots, (pair_rep if g.MODULES[p.module] == "radial" else [p])


@pytest.mark.parametrize("size", sorted(SIZES))
@pytest.mark.parametrize("module", ["radial", "circle"])
def test_styled_geo_caches_follow_the_slots(fake, module, size, monkeypatch, tmp_path_factory):
    for k in KNOBS:
        monkeypatch.delenv("GLAVA_B200_" + k, raising=False)
    L = fake
    sz = dict(SIZES[size])
    over = {}
    if "radius" in sz:
        over = {module + "_radius": sz.pop("radius"), AMP[module]: sz.pop("amplify")}
    p = g.default_params(module, n=1024, **sz, **over)
    a = getattr(p, AMP[module])
    fg_a, fg_b = (0.9, 0.2, 0.1, 1.0), (0.1, 0.3, 0.9, 0.8)
    bg = None if module == "circle" else (0.2, 0.2, 0.25, 1.0)
    with_bg = (lambda d: dict(d, bg=bg)) if bg else (lambda d: dict(d, fg=fg_b))
    steps = [
        ("set, AMPLIFY x1.7", [None, {"amplify": 1.7 * a}, {"fg": fg_a}, with_bg({"fg": fg_a}),
                               {"amplify": 1.7 * a, "fg": fg_a}, {"amplify": -0.5 * a}]),
        ("changed to x0.3", [None, {"amplify": 0.3 * a}, {"fg": fg_a}, with_bg({"fg": fg_a}),
                             {"amplify": 0.3 * a, "fg": fg_a}, {"amplify": -0.5 * a}]),
        ("negative x-2", [{"fg": fg_b}, {"amplify": 0.3 * a}, None, None, {"amplify": -2.0 * a, "fg": fg_a}, None]),
        ("cleared", [None] * BATCH),
    ]
    base_box = _styled_box(tmp_path_factory, [p])
    assert base_box[2] > 0 and base_box[3] > 0
    L.fake_clear()
    h = L.glava_b200_new(C.byref(p), BATCH, 0)
    assert h
    try:
        for what, styles in [("created", [None] * BATCH)] + steps:
            if what != "created":
                L.fake_clear()
                arr = (g.StreamStyle * BATCH)(*[g.stream_style(s) for s in styles])
                idx = (C.c_int * BATCH)(*range(BATCH))
                assert L.glava_b200_set_stream_styles(h, idx, BATCH, arr) == 0, what
            slots, reps = _expected(p, styles)
            box = _styled_box(tmp_path_factory, slots)
            calls = _calls(L)
            assert len(calls) == len(reps), (what, len(calls), len(reps))
            for (got, got_box), want in zip(calls, reps):
                assert got_box == box, (what, got_box, box)
                assert _bytes(got) == _bytes(want), what
            # the box really moves with the slots' AMPLIFY: grown for the larger |AMPLIFY|, the base box otherwise
            grows = max(abs(getattr(q, AMP[module])) for q in slots) > abs(a)
            assert (box != base_box) == grows, (what, box, base_box)
            if module == "radial":
                assert len(calls) == (1 if what in ("created", "cleared") else 3), what
            else:
                assert len(calls) == 1, what
    finally:
        L.glava_b200_destroy(h)
