"""The launch structure the library chooses for a spectrum update (glava_b200/csrc/spectrum_plan.h, compiled into the host
build), against spectrum_cases.launch_structure's independent restatement of it: for every case and launch environment of
tests/spectrum_cases.py, the kernels the plan names, the launches one update issues before the raster pass, and the refusal.
The GPU tier (tests/test_gpu_spectrum_params.py) checks the same launch counts on the device."""
import pytest

import glava_b200 as g
from tests import emul
from tests import spectrum_cases as sc

CASES = sc.build_cases()


def post_chain(k):
    """capi.cu derive: the appended smooth transform or active keyframe interpolation"""
    fr = k.fr if k.fr > 0 else k.ur
    interp = k.interpolate and not (k.accel_fft and k.module != g.MODULES.index("wave")) and k.ur / fr <= 0.9
    return k.transform_smooth == 1 or bool(interp)


def plan_structure(c, env, plan):
    """launch_structure's labels, launch count and refusal for the plan the library chose"""
    p = c.kernel_params(); user = c.params()
    wave = p.module == g.MODULES.index("wave")
    post = post_chain(p)
    F = p.avg_frames
    FT = F if F in (3, 4, 5, 6) else 0
    mode = int(p.sample_mode != 0)
    k5 = plan["k5"]
    got = set()
    launches = 1 + (user.bufscale > 1)
    if not wave and p.accel_fft:
        if plan["split_epilogue"]:
            got.add(f"epilogue_b_kernel<{FT}>" + (" F=1" if F == 1 else ""))
            launches += 1
        else:
            got.add(f"in-kernel epilogue FT={FT}")
    if k5 == "taps_smem":
        got.add("in-kernel lazy K5, shared-memory taps")
    elif k5 == "taps_l2":
        ku = plan["tap_ku"]
        got.add(f"in-kernel lazy K5, L2 taps KU={8 if ku >= 8 else 4 if ku >= 4 else 2}")
    elif k5 == "taps_direct":
        got.add("in-kernel lazy K5, no tap table")
    elif k5 in ("need_smem", "need_l2"):
        mod = g.MODULES[p.module] + ("+join" if p.graph_join_channels and p.module == g.MODULES.index("graph") else "")
        got.add(f"split need-list: {mod}")
        if k5 == "need_smem":
            got.add(f"k5_need_smem_kernel<{mode}>")
            launches += 1
        else:
            if env.get("K5N_SMEM") != "0":
                got.add("k5_need_smem -> av_transpose + k5_need fall-back")
            S = plan["k5n_s"]
            if S == 2 and env.get("K5N_S") not in ("1", "2", "4"):
                got.add("k5_need_kernel automatic S=2")
            got.add(f"k5_need_kernel<{mode}, S={S}>")
            if S == 4 and c.batch > 64 and c.batch % 128:
                got.add("k5_need_kernel S=4, partial stream group")
            launches += 2
    elif k5 == "fused":
        got.add("in-kernel full-plane K5")
    elif k5 == "full_table":
        got.add(f"k5_table_kernel<{'avg' if p.sample_mode == 0 else 'max'}, {plan['table_planes']}>")
    elif k5 == "full_planes":
        got.add("k5_planes_kernel refused: tap span too large" if plan["refusal"] else "k5_planes_kernel")
    if k5 in ("full_table", "full_planes"):
        launches += 1
    if post:
        launches += 2                         # transform_smooth and the upload
    return got, launches, plan["refusal"]


@pytest.mark.parametrize("case", CASES, ids=str)
def test_plan_matches_launch_structure(case, built):
    k = case.kernel_params()
    for env in [{}] + case.envs:
        plan = emul.spectrum_plan(k, post_chain(k), case.batch, sc.SM_COUNT, env)
        got, launches, refusal = plan_structure(case, env, plan)
        want, want_launches, want_refusal = sc.launch_structure(case, env)
        assert got == want, (env, plan)
        assert launches == want_launches, (env, plan)
        if want_refusal is None:
            assert refusal is None, (env, refusal)
        else:
            assert refusal and want_refusal in refusal, (env, refusal)
