"""-m gpu: keyframe interpolation (setinterpolate) over its parameter space (tests/keyframe_cases.py), bit for bit against the
host build.

Each case runs its cadence of modified and unmodified frames through three inputs: host update, update_device, and
ingest_float of the whole ring followed by update_rings.  On every frame:
  a. streams 0, batch // 2 and batch - 1 against the host restatement (keyframe_cases.host_keyframes): textures bit for bit
     (sampled texels for the wide windows), spectra of the latest modified update in every bin (NaN for NaN), frames equal
     to emul.raster of the kernels' own textures;
  b. every stream: the three inputs give identical spectra and textures;
  c. the frame's launch count against keyframe_cases.launch_structure;
  d. for the cheap cases, the last stream's textures within 2 LSB16 of the oracle (OracleStream with setinterpolate).
Past the 0.9 boundary the run must equal an interpolate = 0 renderer bit for bit, launch counts included.  Then mid-stream:
a resize, reconfigures of fr and of the smoothing, a refused reconfigure, a refused update and a refused masked update."""
import numpy as np
import pytest

import glava_b200 as g
from tests import emul
from tests import keyframe_cases as kc
from tests import spectrum_cases as sc

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

CASES = kc.build_cases()
FORMS = ("host", "device", "rings")


def _env(monkeypatch, env):
    for k in sc.ENV_KEYS:
        monkeypatch.delenv("GLAVA_B200_" + k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv("GLAVA_B200_" + k, v)


def _ingest(r, form, modified, lb, rb):
    """the rings input's ingest in front of its update: the whole ring replaced, float samples land as they are"""
    if form == "rings" and modified:
        chunks = np.empty((r.batch, 2 * lb.shape[1]), np.float32)
        chunks[:, 0::2] = lb; chunks[:, 1::2] = rb
        r.ingest_float(chunks)


def _feed(r, form, modified, lb, rb, keep):
    """one frame's update through one of the three inputs (lb / rb: setbufsize floats per stream; ignored when not
    modified; the rings input's ingest is _ingest)"""
    wave = r.params.module == g.MODULES.index("wave")
    if form == "host":
        r.update(lb, None if wave else rb, modified)
    elif form == "device":
        import torch
        dl = torch.from_numpy(np.ascontiguousarray(lb)).cuda(); dr = torch.from_numpy(np.ascontiguousarray(rb)).cuda()
        torch.cuda.synchronize()
        keep.append((dl, dr))                                # alive until the run ends: the kernels read them later
        r.update_device(dl.data_ptr(), None if wave else dr.data_ptr(), modified)
    else:
        r.update_rings(modified)


def _run(monkeypatch, case, form, params=None, env=None):
    """-> per frame (textures, spectra, frames of the checked streams, launches before the raster pass)"""
    _env(monkeypatch, case.env if env is None else env)
    out, keep = [], []
    with g.Renderer(params or case.params(), batch=case.batch) as r:
        for t, m in enumerate(case.cadence):
            lb, rb = kc.batch_pcm(case, t)
            _ingest(r, form, bool(m), lb, rb)
            before = r.launch_count
            _feed(r, form, bool(m), lb, rb, keep)
            launches = r.launch_count - before
            tex, spec = r.textures(), r.spectrum()
            out.append((tex, spec, [r.readback(s) for s in kc.checked_streams(case)], launches))
        before = r.launch_count
        r.raster_textures(*out[-1][0])
        raster = r.launch_count - before                     # the raster pass's own launches
    return [(tex, spec, frames, launches - raster) for tex, spec, frames, launches in out]


@pytest.mark.parametrize("case", CASES, ids=str)
def test_keyframes_in_every_input_form(orc_pm, monkeypatch, case, built):
    k = case.kernel_params(); user = case.params()
    labels, launches, refusal = kc.launch_structure(case)
    if refusal:
        _env(monkeypatch, case.env)
        with g.Renderer(user, batch=case.batch) as r:
            spec0, count0 = r.spectrum(), r.launch_count
            lb, rb = kc.batch_pcm(case, 0)
            for form, modified in (("host", True), ("host", False), ("rings", False)):
                with pytest.raises(g.GlavaError, match="tap span"):
                    _feed(r, form, modified, lb, rb, [])
            assert r.launch_count == count0
            for a, b in zip(r.spectrum(), spec0):
                assert np.array_equal(a, b, equal_nan=True)
        return
    if launches is None:                                     # past the boundary: the plain renderer, launches included
        plain = user.copy(); plain.interpolate = 0
        for form in FORMS:
            a = _run(monkeypatch, case, form)
            b = _run(monkeypatch, case, form, params=plain)
            for t, (x, y) in enumerate(zip(a, b)):
                assert x[3] == y[3], (form, t)
                for ch in (0, 1):
                    assert np.array_equal(x[0][ch], y[0][ch]) and np.array_equal(x[1][ch], y[1][ch], equal_nan=True), (form, t)
                for f1, f2 in zip(x[2], y[2]):
                    assert np.array_equal(f1, f2), (form, t)
        return

    chans = (0,) if case.module == "wave" else (0, 1)
    streams = kc.checked_streams(case)
    idx = kc.texels(case)
    host = {s: kc.host_keyframes(case, s) for s in streams}
    runs = {form: _run(monkeypatch, case, form) for form in FORMS}
    base = runs["host"]
    for t, (tex, spec, frames, n_launch) in enumerate(base):
        m = bool(case.cadence[t])
        assert n_launch == launches[m], (t, m, n_launch, launches)
        for j, s in enumerate(streams):
            hs, ht = host[s][t]
            for ch in chans:
                assert np.array_equal(spec[ch][s], hs[ch], equal_nan=True), ("spectrum", t, s, ch)
                assert np.array_equal(tex[ch][s, idx], ht[ch]), ("texture", t, s, ch)
            assert np.array_equal(frames[j], emul.raster(k, tex[0][s], tex[1][s])), ("frame", t, s)
        for form in FORMS[1:]:
            o = runs[form][t]
            assert o[3] == n_launch, (form, t)
            for ch in chans:
                assert np.array_equal(o[0][ch], tex[ch]), (form, "textures", t, ch)
                assert np.array_equal(o[1][ch], spec[ch], equal_nan=True), (form, "spectra", t, ch)
            for a, b in zip(o[2], frames):
                assert np.array_equal(a, b), (form, "frames", t)
    if not kc.heavy(case) and k.n <= 4096:
        from oracle.oracle import OracleStream, ext_from, params_from
        s = case.batch - 1
        st = OracleStream(orc_pm, params_from(user), ext_from(user))
        for t, m in enumerate(case.cadence):
            want = st.update(*kc.stream_pcm(case, t, s), bool(m))
            for ch in chans:
                assert np.abs(base[t][0][ch][s].astype(int) - want[2 + ch].astype(int)).max() <= 2, ("oracle", t, ch)


# ---- mid-stream ---------------------------------------------------------------------------------------------------------
MID = kc.build_cases()[2]                                    # graph, pipeline A, setbufsize 1024, F = 5
CADENCE = (1, 0, 1, 1, 0, 0, 1, 0, 0, 0, 0, 0, 1, 0, 0)


def _mid_params(**over):
    return g.default_params(MID.module, **dict(MID.over, **over))


def _host_streams(frames, streams):
    """host restatement of streams over `frames` = [(modified, user params of the frame)] -> per frame [(spec, tex)]"""
    out = {}
    for s in streams:
        p0 = frames[0][1]
        h = kc.HostKeyframes(_kernel(p0), p0.bufscale)
        res = []
        for t, (m, p) in enumerate(frames):
            k = _kernel(p)
            res.append(h.step(m, kc.stream_pcm(MID, t, s), k, np.arange(k.n)))
        out[s] = res
    return out


def _kernel(p):
    k = p.copy(); k.n = p.n // p.bufscale; k.bufscale = 1
    return k


def _step(r, t, m):
    lb, rb = kc.batch_pcm(MID, t)
    r.update(lb, rb, bool(m))


def _check(r, want, t, streams):
    tex, spec = r.textures(), r.spectrum()
    k = _kernel(r.params)
    for s in streams:
        hs, ht = want[s][t]
        for ch in (0, 1):
            assert np.array_equal(tex[ch][s], ht[ch]), ("texture", t, s, ch)
            assert np.array_equal(spec[ch][s], hs[ch], equal_nan=True), ("spectrum", t, s, ch)
        assert np.array_equal(r.readback(s), emul.raster(k, tex[0][s], tex[1][s])), ("frame", t, s)


def test_resize_mid_stream_keeps_keys_and_kcounter(monkeypatch, built):
    """sizereq between two unmodified frames: afterwards every frame equals a renderer created at the new size fed the same
    history, so the keyframes and kcounter survived the rebuild"""
    _env(monkeypatch, {})
    small, big = _mid_params(), _mid_params(w=257, h=93)
    with g.Renderer(small, batch=MID.batch) as a, g.Renderer(big, batch=MID.batch) as b:
        for t, m in enumerate(CADENCE):
            if t == 8:
                a.sizereq(257, 93)
            _step(a, t, m); _step(b, t, m)
            if t >= 8:
                assert (a.params.w, a.params.h) == (257, 93)
                ta, tb = a.textures(), b.textures()
                for ch in (0, 1):
                    assert np.array_equal(ta[ch], tb[ch]), (t, ch)
                for s in range(MID.batch):
                    assert np.array_equal(a.readback(s), b.readback(s)), (t, s)


@pytest.mark.parametrize("what", ["fr", "smoothing"])
def test_reconfigure_mid_stream(monkeypatch, what, built):
    """a reconfigure of fr applies its ratio from the next frame on (kcounter and the keys kept); one of the smoothing
    parameters rebuilds the K5 table for the next frame's upload"""
    _env(monkeypatch, {})
    p0 = _mid_params()
    if what == "fr":
        p1 = _mid_params(fr=float(np.float32(p0.ur) * np.float32(7.0)))
    else:
        p1 = _mid_params(smooth_factor=0.04, sample_range=0.8, sample_scale=4.0, sample_mode=2, round_formula=1)
    at = 8
    frames = [(m, p0 if t < at else p1) for t, m in enumerate(CADENCE)]
    streams = kc.checked_streams(MID)
    want = _host_streams(frames, streams)
    with g.Renderer(p0, batch=MID.batch) as r:
        for t, m in enumerate(CADENCE):
            if t == at:
                r.reconfigure(p1)
            _step(r, t, m)
            _check(r, want, t, streams)
    # the new ratio really changed the frames after it
    old = _host_streams([(m, p0) for m in CADENCE], [0])
    assert any(not np.array_equal(old[0][t][1][0], want[0][t][1][0]) for t in range(at, len(CADENCE)))


def test_refused_calls_leave_the_keyframes_alone(monkeypatch, built):
    """a reconfigure that would switch interpolation off, an update the K5 span refuses (after a reconfigure to a window
    past k5_planes_kernel's shared memory, undone again) and a masked update: each fails, and the next frame equals a run
    without the refused call"""
    _env(monkeypatch, dict(NO_K5_TABLE="1"))
    n = 16384
    p0 = g.default_params("bars", **dict(MID.over, n=n, w=96, h=24, sample_mode=1, smooth_factor=0.01))
    wide = g.default_params("bars", **dict(MID.over, n=n, w=96, h=24, sample_mode=1, smooth_factor=0.04, **sc.WIDE))
    off = p0.copy(); off.fr = p0.ur                             # ur / fr = 1 > 0.9: interpolation would switch off
    lb0 = np.zeros((3, n), np.float32)
    with g.Renderer(p0, batch=3) as a, g.Renderer(p0, batch=3) as b:
        def step(t, m):
            for r in (a, b):
                rng = np.random.default_rng([t, 5])
                lb = (rng.random((3, n), np.float32) - 0.5) * 0.4; rb = (rng.random((3, n), np.float32) - 0.5) * 0.4
                r.update(lb, rb, bool(m))
            ta, tb = a.textures(), b.textures()
            for ch in (0, 1):
                assert np.array_equal(ta[ch], tb[ch]), (t, ch)
            assert np.array_equal(a.spectrum()[0], b.spectrum()[0], equal_nan=True), t
            assert np.array_equal(a.readback(2), b.readback(2)), t
        for t, m in enumerate((1, 0, 1, 1, 0)):
            step(t, m)
        def refused(match, call, *args):
            count = a.launch_count
            with pytest.raises(g.GlavaError, match=match):
                call(*args)
            assert a.launch_count == count, match              # the refused call enqueued nothing

        refused("interpolation", a.reconfigure, off)
        step(5, 0)
        a.reconfigure(wide)
        refused("tap span", a.update, lb0, lb0, True)
        refused("tap span", a.update_rings, False)
        a.reconfigure(p0)
        step(6, 0)
        refused("masks", a.update_masked, lb0, lb0, np.array([1, 0, 1], bool))
        refused("masks", a.update_rings_masked, np.array([0, 1, 0], bool))
        step(7, 1)
        step(8, 0)
