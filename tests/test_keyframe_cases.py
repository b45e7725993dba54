"""Keyframe interpolation's host restatement (tests/keyframe_cases.py) against the oracle, and the coverage of its cases.

test_restatement_rotation_matches_the_oracle pins the restatement's key rotation, kcounter, upload and K5 to render.c as
the oracle restates it (OracleStream with setinterpolate), independently of the kernels: fed the oracle's own per-update
chain results, it must give the oracle's textures bit for bit on every frame of every case's cadence.
test_every_form_is_reached_under_interpolation shows that the cases reach every whole-plane K5 form, every post-chain
combination and both sides of the 0.9 boundary, as the library's plan (emul.spectrum_plan) derives them."""
import numpy as np
import pytest

from tests import keyframe_cases as kc
from tests import spectrum_cases as sc

CASES = kc.build_cases()


@pytest.mark.parametrize("case", CASES, ids=str)
def test_restatement_rotation_matches_the_oracle(orc_pm, case, built):
    from oracle.oracle import OracleStream, ext_from, params_from
    k = case.kernel_params(); user = case.params()
    if not kc.interp_on(user):
        pytest.skip("interpolation is off past the boundary (the GPU tier compares it with an interpolate = 0 renderer)")
    cheap = not kc.heavy(case)
    q = user.copy()
    if not cheap:
        q.smooth_pass = 0                      # the wide windows: the upload alone (whole-plane K5 per frame costs seconds)
    s = case.batch - 1
    st = OracleStream(orc_pm, params_from(q), ext_from(user))
    spectra, want = [], []
    for t, m in enumerate(case.cadence):
        l, r = kc.stream_pcm(case, t, s)
        sl, sr, tl, tr = st.update(l, r, bool(m))
        spectra.append([sl, sr]); want.append([tl, tr])
    got = kc.keyframes_from_spectra(case, spectra, pre_only=not cheap)
    chans = (0,) if case.module == "wave" else (0, 1)
    moved = 0
    for t in range(len(case.cadence)):
        for ch in chans:
            assert np.array_equal(got[t][ch], want[t][ch]), (t, ch)
        if t and not case.cadence[t]:
            moved += int(not np.array_equal(want[t][0], want[t - 1][0]))
    assert moved >= 1                          # unmodified frames really move the texture
    assert k.n == st.n


def test_every_form_is_reached_under_interpolation(built):
    reach = {}
    for c in CASES:
        labels, launches, refusal = kc.launch_structure(c)
        for label in labels:
            reach.setdefault(label, []).append(c.id)
        if launches is not None:
            assert launches[True] > launches[False] >= 1, (c.id, launches)
    missing = [x for x in kc.REQUIRED if x not in reach]
    assert not missing, missing
    assert not set(kc.UNREACHABLE) & set(reach)
    # the plan confirms both: with a post chain neither lazy_smooth nor FUSED_K5 moves K5 off the whole-plane kernels
    k = CASES[0].kernel_params(); k.lazy_smooth = 1
    for env in ({}, dict(FUSED_K5="1")):
        plan = emul_plan(k, env)
        assert not plan["need_list"] and plan["k5"] in ("full_table", "full_planes"), (env, plan)
    interp = [c for c in CASES if kc.interp_on(c.params())]
    assert {c.params().n for c in interp} == set(kc.SIZES)
    for module in ("bars", "radial", "graph", "circle"):
        assert any(c.module == module and not c.params().accel_fft for c in interp), module
    assert {c.params().accel_fft for c in interp if c.module == "wave"} == {0, 1}
    assert any(c.params().accel_fft and c.kernel_params().accel_fft == 0 for c in interp)    # setaccelfft cleared
    for F in kc.F_VALUES:
        assert {c.params().avg_window for c in interp if c.params().avg_frames == F} == {0, 1}, F
    assert {(c.kernel_params().sample_mode, c.kernel_params().round_formula) for c in interp} == set(kc.MODES)
    # the cadences: fr / ur of 4, 2.5 and 3.3, two modified updates in a row, runs of unmodified frames past fr / ur
    ratios = {round(float(np.float32(c.params().fr) / np.float32(c.params().ur)), 3) for c in interp}
    assert {4.0, 2.5, 3.3} <= ratios, ratios
    for cad in kc.CADENCES:
        assert cad[0] == 1 and "11" in "".join(map(str, cad))
        longest = max(len(run) for run in "".join(map(str, cad)).split("1"))
        assert longest > max(kc.RATIOS), cad
    # the boundary cases sit exactly on 0.9f and one float step past it
    at = [c for c in CASES if c.id.endswith("at-0.9")][0].params()
    past = [c for c in CASES if c.id.endswith("past-0.9")][0].params()
    assert np.float32(at.ur) / np.float32(at.fr) == np.float32(0.9) and kc.interp_on(at)
    assert np.float32(past.ur) / np.float32(past.fr) == np.nextafter(np.float32(0.9), np.float32(1)) and not kc.interp_on(past)
    # the wide cases move K5 to 4 and 2 planes per CTA, and NO_K5_TABLE's span past shared memory is refused
    assert any(kc.launch_structure(c)[2] for c in CASES)


def emul_plan(k, env):
    from tests import emul
    return emul.spectrum_plan(k, True, 4, sc.SM_COUNT, env)
