"""The spectrum path over its parameter space (tests/spectrum_cases.py), in every launch structure.

Each case runs seven updates (noise, edge signals, an all-silent update, two uneven masks) and is checked three ways:
  a. streams 0, batch // 2 and batch - 1 against the host build (tests/emul), bit for bit: spectra in every bin each launch
     structure writes, the texels the texture defines (under lazy K5 the sampled ones; every other texel must be zero),
     and frames equal to emul.raster of the kernels' own textures;
  b. the same streams against the oracle: spectra within 1e-5 of peak (2.5e-5 above FFT 4096), textures within 2 LSB16;
  c. every launch environment the case draws (spectrum_cases.ENVS, rotated over the cases) against the default run, all
     streams, bit for bit, and each run's launch count against the structure launch_structure predicts.
test_every_instantiation_is_reached (no GPU) shows that the environments and cases reach every kernel instantiation and
branch the parameters select, from the table sizes the host build of tables.h computes."""
import numpy as np
import pytest

import glava_b200 as g
from tests import emul
from tests import spectrum_cases as sc

CASES = sc.build_cases()


def _renderer(monkeypatch, case, env):
    for k in sc.ENV_KEYS:
        monkeypatch.delenv("GLAVA_B200_" + k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv("GLAVA_B200_" + k, v)
    return g.Renderer(case.params(), batch=case.batch)


def _run(monkeypatch, case, env):
    wave = case.module == "wave"
    with _renderer(monkeypatch, case, env) as r:
        for t, m in enumerate(sc.masks(case)):
            pcm = [sc.stream_pcm(case, t, s) for s in range(case.batch)]
            lb = np.stack([x[0] for x in pcm]); rb = np.stack([x[1] for x in pcm])
            before = r.launch_count
            if m is None:
                r.update(lb, None if wave else rb, True)
            else:
                r.update_masked(lb, rb, m)
            if t == 2:
                launches = r.launch_count - before
        tl, tr = r.textures()
        spec = r.spectrum()
        frames = [r.readback(s) for s in sc.checked_streams(case)]
        before = r.launch_count
        r.raster_textures(tl, tr)
        launches -= r.launch_count - before                     # the raster pass's own launches
    return (tl, tr), spec, frames, launches


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=str)
def test_spectrum_parameters_in_every_launch_structure(orc_pm, monkeypatch, case, built):
    k = case.kernel_params()
    wave = case.module == "wave"
    chans = (0,) if wave else (0, 1)
    bins = sc.spec_bins(case)
    idx = sc.texel_sets(case)
    lazy = sc.launch_class(case) == "lazy"
    tol = 1e-5 if k.n <= 4096 else 2.5e-5
    streams = sc.checked_streams(case)
    host = {s: sc.host_stream(case, s) for s in streams}
    orac = {s: sc.oracle_stream(orc_pm, case, s) for s in streams}

    base = _run(monkeypatch, case, {})
    structure, want_launches, _ = sc.launch_structure(case, {})
    assert base[3] == want_launches, (structure, base[3], want_launches)
    tex, spec, frames = base[0], base[1], base[2]
    assert tex[0].any()
    for j, s in enumerate(streams):
        for ch in chans:
            got = spec[ch][s, :bins]
            assert np.array_equal(got, host[s][0][ch][:bins], equal_nan=True), ("spectrum", s, ch)
            assert np.array_equal(tex[ch][s, idx[ch]], host[s][1][ch]), ("texture", s, ch)
            if lazy:
                rest = np.ones(k.n, bool); rest[idx[ch]] = False
                assert not tex[ch][s, rest].any(), ("unsampled texels", s, ch)
            assert sc.spectrum_error(case, got, orac[s][0][ch][:bins]) <= tol, ("oracle spectrum", s, ch)
            assert np.abs(tex[ch][s, idx[ch]].astype(int) - orac[s][1][ch].astype(int)).max(initial=0) <= 2, ("oracle texture", s, ch)
        assert np.array_equal(frames[j], emul.raster(k, tex[0][s], tex[1][s])), ("frame", s)

    for env in case.envs:
        structure, want_launches, refused = sc.launch_structure(case, env)
        if refused:
            with _renderer(monkeypatch, case, env) as r:
                spec0, count0 = r.spectrum(), r.launch_count
                lb, rb = sc.stream_pcm(case, 0, 0)
                assert lb.any()
                with pytest.raises(g.GlavaError, match=refused):
                    r.update(np.tile(lb, (case.batch, 1)), None if wave else np.tile(rb, (case.batch, 1)), True)
                # the refused update enqueued nothing and changed no state
                assert r.launch_count == count0, (env, r.launch_count, count0)
                for a, b in zip(r.spectrum(), spec0):
                    assert np.array_equal(a, b, equal_nan=True), (env, "spectrum after the refused update")
            continue
        got = _run(monkeypatch, case, env)
        assert got[3] == want_launches, (env, structure, got[3], want_launches)
        for ch in chans:
            assert np.array_equal(got[0][ch], tex[ch]), (env, "textures", ch)
            assert np.array_equal(got[1][ch][:, :bins], spec[ch][:, :bins], equal_nan=True), (env, "spectra", ch)
        for a, b in zip(got[2], frames):
            assert np.array_equal(a, b), (env, "frames")


def test_every_instantiation_is_reached(built):
    """each kernel instantiation and parameter-selected branch (spectrum_cases.REQUIRED) is reached by some case and
    environment, as launch_structure derives it from the host build's table sizes; the GPU test checks each run's launch
    count against the same derivation"""
    reach = {}
    for c in CASES:
        for env in [{}] + c.envs:
            for label in sc.launch_structure(c, env)[0]:
                reach.setdefault(label, []).append((c.id, env))
    missing = [label for label in sc.REQUIRED if label not in reach]
    assert not missing, missing
    assert not set(sc.UNREACHABLE) & set(reach)
    # every environment runs against several parameter classes
    for cls, envs in sc.ENVS.items():
        for env in envs:
            users = [c for c in CASES if any(env.items() <= e.items() for e in c.envs)]
            assert len(users) >= (1 if cls != "any" else 3), (cls, env)
    # every size in both pipelines, pipeline B under lazy K5 split off on each side of 4096, every F on each side
    for n in sc.SIZES:
        for accel in (0, 1):
            assert any(c.kernel_params().n == n and c.kernel_params().accel_fft == accel for c in CASES), (n, accel)
    for side in (lambda n: n < 4096, lambda n: n >= 4096):
        assert any(side(c.kernel_params().n) and any(lab.startswith("split need-list") for lab in sc.launch_structure(c, e)[0])
                   and c.kernel_params().accel_fft for c in CASES for e in [{}] + c.envs)
        for accel in (0, 1):
            fs = {c.kernel_params().avg_frames for c in CASES if side(c.kernel_params().n) and c.kernel_params().accel_fft == accel
                  and c.module != "wave"}
            assert set(sc.F_VALUES) <= fs, (accel, fs)
    assert {(c.kernel_params().sample_mode, c.kernel_params().round_formula) for c in CASES} == set(sc.MODES)
