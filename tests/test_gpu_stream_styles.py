"""-m gpu: stream styles (DESIGN 4.9).  A stream whose style is `s` renders, byte for byte, what a batch-1 renderer created
with style_params(base, s) renders when fed the same calls, in every raster launch form; textures do not depend on styles;
styles survive reconfigure / resize / stream state I/O, and a refused call changes nothing."""
import ctypes as C

import numpy as np
import pytest

import glava_b200 as g

pytestmark = pytest.mark.gpu

N, W, H, BATCH = 1024, 96, 64, 7
AMP = dict(bars="bars_amplify", radial="radial_amplify", circle="circle_amplify", graph="graph_vscale", wave="wave_amplify")
KNOBS = ("ROWS", "BX", "GW_MINB", "NO_COLTAB", "CIRCLE_TILES", "CTILE", "NO_TEXMM", "NO_GEO", "FULL_STORE")


def _base(module, **over):
    p = g.default_params(module, n=N, w=over.pop("w", W), h=over.pop("h", H))
    for k, v in over.items():
        setattr(p, k, v)
    if module == "radial":
        p.radial_radius = 12.0                       # the disc and its bars fit the small frame
    if module == "circle":
        p.circle_radius = 12.0
    return p


def _styles(p):
    """none, amplify only, constant fg, gradient fg, bg only, all three, a duplicate of another stream's style"""
    m = g.MODULES[p.module]
    a = getattr(p, AMP[m])
    grad = g.Color(0, (C.c_float * 4)(0.9, 0.1, 0.2, 1.0), (C.c_float * 4)(0.1, 0.2, 0.9, 0.6), 17.0)
    fg2 = grad if m in ("bars", "radial", "graph") else (0.1, 0.8, 0.3, 0.9)
    bg = None if m == "circle" else (0.4, 0.5, 0.1, 1.0)
    return [None, {"amplify": a * 1.7}, {"fg": "#ff8000"}, {"fg": fg2}, {"bg": bg} if bg else {"amplify": -a * 0.6},
            {"amplify": a * 0.5, "fg": (0.7, 0.7, 0.2, 1.0), "bg": bg}, {"amplify": a * 1.7}]


def _env(monkeypatch, env):
    for k in KNOBS:
        monkeypatch.delenv("GLAVA_B200_" + k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv("GLAVA_B200_" + k, str(v))


def _pcm(rng, batch):
    return [(rng.standard_normal((batch, N)) * 0.3).astype(np.float32) for _ in range(2)]


def _frames(r, streams):
    r.sync()
    return [r.readback(s).copy() for s in streams]


def _singles(p, styles):
    return [g.Renderer(g.style_params(p, s), batch=1) for s in styles]


def _run_against_singles(p, styles, steps=4, seed=1, masked=False, fb_slots=0):
    q = p.copy(); q.fb_slots = fb_slots
    rng = np.random.default_rng(seed)
    own = range(BATCH) if not fb_slots else range(BATCH - fb_slots, BATCH)   # streams that own their framebuffer slot last
    with g.Renderer(q, batch=BATCH) as r, g.Renderer(q, batch=BATCH) as plain:
        r.set_stream_styles(range(BATCH), styles)
        singles = _singles(p, styles)
        try:
            for step in range(steps):
                lb, rb = _pcm(rng, BATCH)
                if masked and step:
                    m = rng.integers(0, 2, BATCH).astype(np.uint8)
                    r.update_masked(lb, rb, m); plain.update_masked(lb, rb, m)
                    for s, one in enumerate(singles):
                        one.update(lb[s:s + 1], rb[s:s + 1], modified=bool(m[s]))
                else:
                    r.update(lb, rb); plain.update(lb, rb)
                    for s, one in enumerate(singles):
                        one.update(lb[s:s + 1], rb[s:s + 1])
                got = _frames(r, own)
                for s, f in zip(own, got):
                    want = singles[s].readback(0)
                    assert np.array_equal(f, want), ("stream", s, "step", step, "style", styles[s])
                tl, tr = r.textures(); ul, ur = plain.textures()
                assert np.array_equal(tl, ul) and np.array_equal(tr, ur)
            return got
        finally:
            for one in singles:
                one.close()


VARIANTS = [{}, dict(ROWS=1), dict(ROWS=H), dict(NO_COLTAB=1), dict(GW_MINB=5), dict(NO_GEO=1), dict(CTILE=1),
            dict(NO_TEXMM=1), dict(FULL_STORE=1)]


@pytest.mark.parametrize("env", VARIANTS, ids=lambda e: "-".join(f"{k}{v}" for k, v in e.items()) or "default")
@pytest.mark.parametrize("module", ["bars", "radial", "circle", "graph", "wave"])
def test_styled_streams_equal_batch1_renderers(module, env, monkeypatch, built):
    _env(monkeypatch, env)
    p = _base(module)
    frames = _run_against_singles(p, _styles(p))
    assert any(f.any() for f in frames)


OPTIONS = [("bars", dict(premultiply_alpha=0)), ("bars", dict(bars_mirror_yx=1)), ("graph", dict(graph_join_channels=1)),
           ("graph", dict(graph_anti_alias=1)), ("radial", dict(radial_bar_outline_width=2.0)),
           ("radial", dict(premultiply_alpha=0)), ("circle", dict(premultiply_alpha=0)), ("wave", dict(premultiply_alpha=0))]


@pytest.mark.parametrize("module,over", OPTIONS, ids=[f"{m}-{list(o)[0]}" for m, o in OPTIONS])
def test_styled_streams_in_the_option_fallbacks(module, over, monkeypatch, built):
    _env(monkeypatch, {})
    p = _base(module, **over)
    _run_against_singles(p, _styles(p))


@pytest.mark.parametrize("fb_slots", [1, 3])
@pytest.mark.parametrize("module", ["bars", "radial", "circle", "graph", "wave"])
def test_styled_streams_with_a_framebuffer_ring(module, fb_slots, monkeypatch, built):
    _env(monkeypatch, {})
    p = _base(module)
    _run_against_singles(p, _styles(p), fb_slots=fb_slots)


def test_radial_over_the_cache_budget(monkeypatch, tmp_path_factory, built):
    """so many (fg, bg) pairs that their caches together pass 512 MiB: the styled per-pixel kernel runs, and every stream
    still equals a batch-1 renderer, which draws from its own cache"""
    from tests.test_stream_styles import styled_plan
    _env(monkeypatch, {})
    p = _base("radial", w=1920, h=1080)
    p.radial_radius = 128.0
    one = styled_plan(tmp_path_factory, [p], 1, 1, 1, {})
    assert one["kernel"] == "radial_geo"
    pairs = (512 << 20) // one["geo_bytes"] + 1
    styles = [{"fg": (k / pairs, 0.5, 1 - k / pairs, 1.0)} for k in range(pairs)]
    sp = [p] + [g.style_params(p, s) for s in styles]
    assert styled_plan(tmp_path_factory, sp, pairs, len(styles), len(styles), {})["kernel"] == "radial"
    batch = len(styles)
    rng = np.random.default_rng(19)
    check = [0, batch // 2, batch - 1]
    with g.Renderer(p, batch=batch) as r:
        r.set_stream_styles(range(batch), styles)
        singles = [g.Renderer(g.style_params(p, styles[s]), batch=1) for s in check]
        try:
            for _ in range(2):
                lb = (rng.standard_normal((batch, N)) * 0.3).astype(np.float32)
                rb = (rng.standard_normal((batch, N)) * 0.3).astype(np.float32)
                r.update(lb, rb)
                for s, one_r in zip(check, singles):
                    one_r.update(lb[s:s + 1], rb[s:s + 1])
                for s, one_r in zip(check, singles):
                    f = r.readback(s)
                    assert f.any() and np.array_equal(f, one_r.readback(0)), s
        finally:
            for x in singles:
                x.close()


@pytest.mark.parametrize("module", ["bars", "radial", "circle", "graph", "wave"])
def test_styled_streams_with_masked_updates(module, monkeypatch, built):
    _env(monkeypatch, {})
    p = _base(module)
    _run_against_singles(p, _styles(p), steps=5, masked=True)


@pytest.mark.parametrize("module", ["bars", "graph", "wave", "radial", "circle"])
def test_styles_set_changed_and_cleared_mid_run(module, monkeypatch, built):
    """checked at every step, across the styled / plain switch and its dirty-row marks; cleared = never styled"""
    _env(monkeypatch, {})
    p = _base(module)
    st = _styles(p)
    plans = [dict(), {1: st[1], 4: st[4]}, {1: st[5], 2: st[2], 6: st[3]}, {0: st[1]}, {1: None, 2: None, 4: None, 6: None, 0: None}]
    rng = np.random.default_rng(7)
    with g.Renderer(p, batch=BATCH) as r, g.Renderer(p, batch=BATCH) as never:
        cur = [None] * BATCH
        singles = _singles(p, [None] * BATCH)
        try:
            for step, change in enumerate(plans * 2):
                if change:
                    r.set_stream_styles(list(change), list(change.values()))
                    for s, v in change.items():
                        cur[s] = v
                        singles[s].close()
                        singles[s] = g.Renderer(g.style_params(p, v), batch=1)   # fed the batch's textures below
                got = [x.set for x in r.get_stream_styles(range(BATCH))]
                assert got == [0 if c is None else g.stream_style(c).set for c in cur]
                lb, rb = _pcm(rng, BATCH)
                before = r.launch_count; nb = never.launch_count
                r.update(lb, rb); never.update(lb, rb)
                if all(c is None for c in cur):
                    assert r.launch_count - before == never.launch_count - nb
                tl, tr = r.textures()
                assert np.array_equal((tl, tr), never.textures())
                for s in range(BATCH):
                    singles[s].raster_textures(tl[s:s + 1], tr[s:s + 1])
                for s, f in enumerate(_frames(r, range(BATCH))):
                    assert np.array_equal(f, singles[s].readback(0)), (step, s)
                if all(c is None for c in cur):
                    for s, f in enumerate(_frames(never, range(BATCH))):
                        assert np.array_equal(f, r.readback(s)), (step, s)
        finally:
            for one in singles:
                one.close()


def test_unmodified_update_rerasters_in_the_new_style(monkeypatch, built):
    _env(monkeypatch, {})
    p = _base("bars")
    st = _styles(p)
    rng = np.random.default_rng(3)
    with g.Renderer(p, batch=BATCH) as r:
        lb, rb = _pcm(rng, BATCH)
        r.update(lb, rb)
        before = _frames(r, range(BATCH))
        r.set_stream_styles(range(BATCH), st)
        r.update(lb, rb, modified=False)
        tl, tr = r.textures()
        after = _frames(r, range(BATCH))
        for s in range(BATCH):
            with g.Renderer(g.style_params(p, st[s]), batch=1) as one:
                one.raster_textures(tl[s:s + 1], tr[s:s + 1])
                assert np.array_equal(after[s], one.readback(0)), s
        assert np.array_equal(after[0], before[0]) and not np.array_equal(after[5], before[5])


@pytest.mark.parametrize("module", ["bars", "radial", "graph"])
def test_styles_survive_reconfigure_and_resize(module, monkeypatch, built):
    _env(monkeypatch, {})
    p = _base(module)
    st = _styles(p)
    rng = np.random.default_rng(5)
    with g.Renderer(p, batch=BATCH) as r:
        r.set_stream_styles(range(BATCH), st)
        q = p.copy(); setattr(q, AMP[module], getattr(p, AMP[module]) * 1.3)
        r.reconfigure(q)
        r.sizereq(W + 16, H + 8)
        for _ in range(2):
            lb, rb = _pcm(rng, BATCH)
            r.update(lb, rb)
        assert (r.params.w, r.params.h) == (W + 16, H + 8)
        assert [x.set for x in r.get_stream_styles(range(BATCH))] == [g.stream_style(x).set for x in st]
        tl, tr = r.textures()
        frames = _frames(r, range(BATCH))
        for s in range(BATCH):
            with g.Renderer(g.style_params(r.params, st[s]), batch=1) as one:
                one.raster_textures(tl[s:s + 1], tr[s:s + 1])
                assert np.array_equal(frames[s], one.readback(0)), s


def test_reconfigure_that_breaks_a_style_is_refused(monkeypatch, built):
    _env(monkeypatch, {})
    p = _base("bars")
    with g.Renderer(p, batch=BATCH) as r:
        r.set_stream_styles([2], [{"fg": (1, 0, 0, 1)}])
        q = p.copy(); q.bars_outline_mode = 2; q.bars_outline_prog.n_ops = 1
        with pytest.raises(g.GlavaError):
            r.reconfigure(q)
        assert r.params.bars_outline_mode == p.bars_outline_mode


def test_stream_state_beside_styled_streams(monkeypatch, built):
    """reset / save / load touch state only; a blob loads into a slot whatever the styles of either renderer"""
    _env(monkeypatch, {})
    p = _base("bars")
    st = _styles(p)
    rng = np.random.default_rng(11)
    with g.Renderer(p, batch=BATCH) as r, g.Renderer(p, batch=BATCH) as plain:
        r.set_stream_styles(range(BATCH), st)
        for _ in range(3):
            lb, rb = _pcm(rng, BATCH)
            r.update(lb, rb); plain.update(lb, rb)
        blobs = plain.save_streams([1, 4])
        r.load_streams([3, 5], blobs)
        tl, tr = r.textures(); pl_, pr_ = plain.textures()
        assert np.array_equal(tl[3], pl_[1]) and np.array_equal(tl[5], pl_[4])
        mask = np.zeros(BATCH, np.uint8); mask[6] = 1
        r.reset_streams(mask); plain.reset_streams(mask)
        assert [x.set for x in r.get_stream_styles(range(BATCH))] == [g.stream_style(x).set for x in st]
        lb, rb = _pcm(rng, BATCH)
        r.update(lb, rb); plain.update(lb, rb)
        tl, tr = r.textures(); pl_, pr_ = plain.textures()
        for s in (0, 1, 2, 4, 6):
            assert np.array_equal(tl[s], pl_[s]) and np.array_equal(tr[s], pr_[s])
        frames = _frames(r, range(BATCH))
        for s in range(BATCH):
            with g.Renderer(g.style_params(p, st[s]), batch=1) as one:
                one.raster_textures(tl[s:s + 1], tr[s:s + 1])
                assert np.array_equal(frames[s], one.readback(0)), s


def test_refused_calls_change_nothing(monkeypatch, built):
    _env(monkeypatch, {})
    p = _base("circle")
    st = _styles(p)
    rng = np.random.default_rng(13)
    with g.Renderer(p, batch=BATCH) as r:
        r.set_stream_styles([1, 2], [st[1], st[2]])
        lb, rb = _pcm(rng, BATCH)
        r.update(lb, rb)
        before = _frames(r, range(BATCH))
        launches = r.launch_count
        bad_fg = g.Color(2, (C.c_float * 4)(), (C.c_float * 4)(), 1.0)
        refused = [([7], [st[1]]), ([-1], [st[1]]), ([3, 3], [st[1], st[2]]), ([3], [{"bg": (0, 0, 0, 1)}]),
                   ([3], [{"amplify": float("nan")}]), ([3], [{"fg": bad_fg}]), ([0, 3], [st[1], {"bg": (0, 0, 0, 1)}])]
        for streams, styles in refused:
            with pytest.raises(g.GlavaError):
                r.set_stream_styles(streams, styles)
            with pytest.raises(g.GlavaError):
                r.get_stream_styles([7]) if streams == [7] else r.get_stream_styles([3, 3])
        assert r.launch_count == launches
        assert [x.set for x in r.get_stream_styles(range(BATCH))] == [0, g.stream_style(st[1]).set, g.stream_style(st[2]).set, 0, 0, 0, 0]
        r.update(lb, rb, modified=False)
        assert all(np.array_equal(a, b) for a, b in zip(before, _frames(r, range(BATCH))))


def test_sharded_handle_equals_a_single_device_handle(monkeypatch, built):
    _env(monkeypatch, {})
    p = _base("graph")
    st = _styles(p)
    rng = np.random.default_rng(17)
    with g.ShardedRenderer(p, BATCH, devices=[0, 0, 0]) as sh, g.Renderer(p, batch=BATCH) as one:
        order = [5, 0, 3, 6, 1, 4, 2]
        sh.set_stream_styles(order, [st[s] for s in order])
        one.set_stream_styles(range(BATCH), st)
        got = sh.get_stream_styles(range(BATCH))
        assert [C.string_at(C.addressof(x), C.sizeof(x)) for x in got] == \
               [C.string_at(C.addressof(x), C.sizeof(x)) for x in one.get_stream_styles(range(BATCH))]
        with pytest.raises(g.GlavaError):
            sh.set_stream_styles([1, 1], [st[1], st[2]])
        for _ in range(3):
            lb, rb = _pcm(rng, BATCH)
            sh.update(lb, rb); one.update(lb, rb)
        sh.sync(); one.sync()
        for s in range(BATCH):
            assert np.array_equal(sh.readback(s), one.readback(s)), s
