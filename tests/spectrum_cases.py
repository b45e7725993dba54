"""Seeded cases over the spectrum path's parameter space, shared by the CPU tier (tests/test_emul_parity.py: host build
against the oracle) and the GPU tier (tests/test_gpu_spectrum_params.py: kernels against the host build, the oracle and
each other).

A case is (module, parameters, batch, launch environments).  Coverage is forced, not left to the seed: every size in both
pipelines, every F on each side of 4096 in each pipeline, all nine sample_mode x round_formula pairs, all five modules,
post-chain, setbufscale and setmirror, and the wide windows that move K5 onto its fall-backs.  `launch_structure` restates
the choices capi.cu build_tables / run_update and spectrum_kernels.cu make from the parameters, the environment and the
table sizes (tests/emul table_sizes), so that the coverage of each kernel instantiation is computed, not claimed."""
import itertools

import numpy as np

import glava_b200 as g

SIZES = [256, 512, 1024, 2048, 4096, 8192, 16384]
F_VALUES = [1, 2, 3, 4, 5, 6, 7, 16]
MODES = list(itertools.product(range(3), range(3)))          # sample_mode x round_formula
SM_COUNT = 132                                              # H100 SXM: k5_need_kernel's automatic S = 2 depends on it
GEOMETRY = {"bars": [(1920, 8), (333, 12)], "radial": [(96, 64)], "graph": [(96, 24)], "wave": [(96, 24)],
            "circle": [(48, 48)]}
WIDE = dict(sample_range=0.999999, sample_scale=13.8)       # scale_audio reaches 1 at texel n: a window as wide as 0.8 n

# Launch environments (GLAVA_B200_<key>, DESIGN 6.2).  Each applies to the launch structures named by its class.
ENVS = {
    "lazy": [dict(K5_SPLIT="0"), dict(K5_SPLIT="1"), dict(K5_SPLIT="1", SPLIT_EPI="0"), dict(K5_SPLIT="1", SPLIT_EPI="1"),
             dict(K5_SPLIT="1", K5N_SMEM="0"), dict(K5_SPLIT="1", K5N_SMEM="1"),
             dict(K5_SPLIT="1", K5N_SMEM="0", K5N_S="1"), dict(K5_SPLIT="1", K5N_SMEM="0", K5N_S="2"),
             dict(K5_SPLIT="1", K5N_SMEM="0", K5N_S="4"),
             dict(K5_SPLIT="1", K5N_ROWS="64", K5N_TPB="3", K5N_WARPS="2"), dict(K5_SPLIT="1", K5N_SMEM="0", K5N_WARPS="7"),
             dict(K5_SPLIT="0", NO_SMEM_TAPS="1"), dict(NO_TAPTAB="1"),
             dict(K5_SPLIT="0", NO_SMEM_TAPS="1", TAP_KU="2"), dict(K5_SPLIT="0", NO_SMEM_TAPS="1", TAP_KU="4"),
             dict(K5_SPLIT="0", NO_SMEM_TAPS="1", TAP_KU="8"), dict(NO_EPI_PRUNE="1")],
    "full": [dict(NO_K5_TABLE="1"), dict(FUSED_K5="1")],
    "any": [dict(SPEC_CTAS_PER_SM="1")],
}
# one non-default FFT instantiation per size (launch_spectrum_fft: the default is in place at the size's thread count,
# out of place with 256 threads at 8192)
SPEC_VARIANT = {256: ("1", "128"), 512: ("1", "256"), 1024: ("1", "128"), 2048: ("1", "256"), 4096: ("1", "128"),
                8192: ("0", "256"), 16384: ("1", "1024")}
ENV_KEYS = sorted({k for envs in ENVS.values() for e in envs for k in e} | {"SPEC_OOP", "SPEC_T"})


class Case:
    def __init__(self, seed, cid, module, over, batch, envs):
        self.seed, self.id, self.module, self.over, self.batch, self.envs = seed, cid, module, over, batch, envs

    def params(self):
        return g.default_params(self.module, **self.over)

    def kernel_params(self):
        """the parameters the kernels run with (capi.cu derive): n = setbufsize / setbufscale, post-chain without setaccelfft"""
        p = self.params()
        n = p.n // p.bufscale
        q = g.default_params(self.module, **dict(self.over, n=n, bufscale=1))
        if q.transform_smooth == 1 and self.module != "wave":
            q.accel_fft = 0
        return q

    def __repr__(self):
        return self.id


def _random_knobs(rng):
    return dict(fft_scale=float(rng.uniform(0.5, 20.0)),
                fft_cutoff=float(rng.choice([0.0, rng.uniform(0.05, 1.0), 1.2])),
                gravity_step=float(rng.choice([0.0, rng.uniform(0.5, 12.0)])),
                ur=float(rng.uniform(20.0, 250.0)),
                sample_range=float(rng.uniform(0.6, 0.95)), sample_scale=float(rng.uniform(3.0, 10.0)),
                smooth_factor=float(np.exp(rng.uniform(np.log(0.005), np.log(0.06)))))


def build_cases(seed=2026):
    rng = np.random.default_rng(seed)
    cases = []
    modes = itertools.cycle(MODES)
    fft_modules = itertools.cycle(["bars", "bars", "radial", "graph", "circle"])

    def add(tag, module, over, batch=37):
        w, h = GEOMETRY[module][len(cases) % len(GEOMETRY[module])]
        sm, rf = next(modes)
        base = dict(_random_knobs(rng), w=w, h=h, sample_mode=sm, round_formula=rf)
        base.update(over)
        cases.append(Case(seed + len(cases), f"{len(cases):02d}-{module}-{tag}", module, base, batch, []))

    # every F on each side of 4096, in each pipeline (pipeline B half lazy, half full K5; lazy B from 4096 up splits)
    for accel in (0, 1):
        for side in (SIZES[:4], SIZES[4:]):
            fs = list(F_VALUES)
            rng.shuffle(fs)
            for i, F in enumerate(fs):
                n = side[i % len(side)]
                lazy = int(i % 2 == 0) if accel else int(rng.integers(0, 2))
                module = next(fft_modules)
                add(f"{'AB'[accel]}{n}F{F}", module, dict(n=n, accel_fft=accel, avg_frames=F, avg_window=int(F == 2 or i % 3 != 0),
                                                        lazy_smooth=lazy))
    # modules through the need-list, the smooth pass off, setmirror, post-chain, setbufscale
    add("wave-lazy", "wave", dict(n=8192, lazy_smooth=1))
    add("wave-full", "wave", dict(n=1024, lazy_smooth=0))
    add("graph-join", "graph", dict(n=4096, lazy_smooth=1, accel_fft=1, graph_join_channels=1))
    add("graph-join-small", "graph", dict(n=1024, lazy_smooth=1, accel_fft=1, graph_join_channels=1, avg_frames=4))
    add("radial-lazy", "radial", dict(n=16384, lazy_smooth=1, accel_fft=1, avg_frames=6))
    add("mirror", "bars", dict(n=2048, lazy_smooth=1, accel_fft=1, channels=1, mirror_input=1))
    add("mirror-big", "bars", dict(n=8192, lazy_smooth=1, accel_fft=1, channels=1, mirror_input=1, avg_frames=3))
    add("nosmooth", "bars", dict(n=4096, smooth_pass=0, accel_fft=1, lazy_smooth=1))
    add("nosmooth-a", "graph", dict(n=512, smooth_pass=0, accel_fft=0))
    add("post", "bars", dict(n=1024, transform_smooth=1))
    add("post-big", "graph", dict(n=8192, transform_smooth=1, lazy_smooth=1, smooth_distance=0.02, smooth_ratio=2.0))
    add("bs2", "bars", dict(n=2048, bufscale=2, lazy_smooth=1, accel_fft=1))
    add("bs4", "bars", dict(n=16384, bufscale=4, lazy_smooth=1, accel_fft=1, avg_frames=4))
    add("bs4-full", "radial", dict(n=4096, bufscale=4, lazy_smooth=0, accel_fft=0))
    # wide windows at 16384: the need-list tile past 200 KiB (k5_need_kernel from a transposed copy), and the full-plane
    # table past 6400 and 12800 texels (k5_table_kernel with 4 and 2 planes; k5_planes_kernel refuses the wider one)
    add("wide-lazy", "bars", dict(n=16384, lazy_smooth=1, accel_fft=1, smooth_factor=0.02, sample_range=0.9, sample_scale=2.0))
    add("wide-s4", "bars", dict(n=16384, lazy_smooth=0, accel_fft=1, smooth_factor=0.02, sample_mode=0, **WIDE), batch=21)
    add("wide-s2", "circle", dict(n=16384, lazy_smooth=0, accel_fft=0, smooth_factor=0.04, sample_mode=2, **WIDE), batch=11)
    add("narrow", "bars", dict(n=16384, lazy_smooth=1, accel_fft=1, smooth_factor=0.005))
    # batch: k5_need_kernel's automatic S = 2 (wide tile: no shared-memory form), S = 4 over a partial stream group
    add("s2-auto", "bars", dict(n=4096, lazy_smooth=1, accel_fft=1, smooth_factor=0.15, sample_range=0.9, sample_scale=2.0,
                                avg_frames=5, w=1920, h=8), batch=700)
    add("s4-partial", "bars", dict(n=4096, lazy_smooth=1, accel_fft=1, avg_frames=5), batch=70)

    # the launch environments, rotated through the cases each class applies to
    rot = {k: itertools.cycle(v) for k, v in ENVS.items()}
    for i, c in enumerate(cases):
        cls = launch_class(c)
        if cls in ("lazy", "full"):
            c.envs += [next(rot[cls]), next(rot[cls])]
        other = next(rot["any"]) if i % 3 == 0 else {}
        if c.module != "wave":
            oop, t = SPEC_VARIANT[c.over["n"] // c.over.get("bufscale", 1)]
            other = dict(other, SPEC_OOP=oop, SPEC_T=t)
        c.envs.append(other)
        if c.id.endswith("s4-partial"):
            c.envs.append(dict(K5_SPLIT="1", K5N_SMEM="0", K5N_S="4"))
        if c.id.endswith(("wide-s2", "wide-s4")):
            c.envs.append(dict(NO_K5_TABLE="1"))
        c.envs = [e for k, e in enumerate(c.envs) if e and e not in c.envs[:k]]
    return cases


# ---- what a case is driven with, and the host build's and the oracle's expectations for one stream -------------------
STEPS = 7
AMPS = [0.3, 0.05, 0.3, 0.0, 0.2, 0.004, 0.3]                # update 3 is all-silent: gravity falls


def stream_pcm(c, t, s):
    """(lb, rb) of stream s at update t: noise at the update's amplitude (every 4th stream 50x quieter); at update 1 every
    third stream's left channel is an edge signal (tests/pcm.py)"""
    from tests.pcm import EDGE_SIGNALS, edge_signal
    n = c.params().n
    rng = np.random.default_rng([c.seed, t, s])
    amp = AMPS[t] * (0.02 if s % 4 == 3 else 1.0)
    l = ((rng.random(n, dtype=np.float32) - 0.5) * np.float32(2 * amp)).astype(np.float32)
    r = ((rng.random(n, dtype=np.float32) - 0.5) * np.float32(2 * amp)).astype(np.float32)
    if t == 1 and s % 3 == 0:
        l = edge_signal(EDGE_SIGNALS[(s // 3) % len(EDGE_SIGNALS)], n)
    return l, r


def masks(c):
    """per update: None (every stream) or an uneven mask; the checked streams 0, batch // 2 and batch - 1 take both values"""
    b = c.batch
    rng = np.random.default_rng([c.seed, 99])
    out = [None] * STEPS
    for t, on in ((4, (1, 0, 1)), (6, (0, 1, 0))):
        m = rng.random(b) < (0.6 if t == 4 else 0.35)
        m[0], m[b // 2], m[b - 1] = on
        out[t] = m
    return out


def checked_streams(c):
    return sorted({0, c.batch // 2, c.batch - 1})


def texel_sets(c):
    """per channel, the texels each update's texture defines: the need-list under lazy K5 (others stay zero), else all;
    for windows wide enough that a full host K5 costs seconds, every 7th texel and the last 128"""
    from tests import emul
    k = c.kernel_params()
    if launch_class(c) == "lazy":
        return [emul.lazy_k5(k, ch, 1, np.zeros(k.n, np.uint16))[0] for ch in (0, 1)]
    if heavy(c):
        idx = np.union1d(np.arange(0, k.n, 7), np.arange(k.n - 128, k.n))
    else:
        idx = np.arange(k.n)
    return [idx, idx]


def heavy(c):
    return c.kernel_params().n * sizes(c)["planes_span"] > 2e7


def spec_bins(c):
    """bins of `spec` every launch structure writes: lazy pipeline B writes only up to epi_n (each form rounds it up)"""
    k = c.kernel_params()
    if launch_class(c) == "lazy" and k.accel_fft and k.module != g.MODULES.index("wave"):
        return sizes(c)["epi_n"]
    return k.n


def spectrum_error(c, got, want):
    """max error of a spectrum against the oracle's over its peak, NaN where the oracle has NaN (post chain), after a per-bin
    floor of the reference's own float rounding: render.c:844 rounds |X| + 1 to float (2^-24 of it) and the output again,
    so a bin carries up to 2^-23 * ramp / 3 whatever the transform.  That floor only shows on near-silent streams: the last
    stream of s2-auto (every 4th stream is 50x quieter; it was last updated with amplitude 8e-5) measured 9.97e-8 off at a
    peak of 4.06e-3, 2.5e-5 of peak, in the kernels and the host build alike (bit-identical), on an H100 at batch 600."""
    from tests.pcm import fft_ramp
    k = c.kernel_params()
    got = np.asarray(got, np.float64); want = np.asarray(want, np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want)
    floor = 0.0 if k.module == g.MODULES.index("wave") else 2.0 ** -23 * fft_ramp(k.n, k.fft_scale, k.fft_cutoff)[:len(want)] / 3
    err = np.maximum(np.abs(got - want) - floor, 0)[ok]
    return err.max(initial=0.0) / max(np.abs(want[ok]).max(initial=0.0), 1e-30)


def host_stream(c, s):
    """the host build (tests/emul) over the case's updates for stream s, advanced only when its mask bit is set
    -> ([spec_l, spec_r], [texture_l, texture_r] at texel_sets)"""
    from tests import emul
    k = c.kernel_params(); user = c.params()
    q = k.copy(); q.smooth_pass = 0
    chans = [emul.Channel(q), emul.Channel(q)]
    spec, pre = [None, None], [None, None]
    wave = k.module == g.MODULES.index("wave")
    for t, m in enumerate(masks(c)):
        if m is not None and not m[s]:
            continue
        for ch, x in enumerate(stream_pcm(c, t, s)):
            if user.bufscale > 1:
                x = emul.bufscale(x, user.bufscale)
            sp, av = chans[ch].update(x, is_fft=not wave)
            if k.transform_smooth == 1:
                sp = emul.transform_smooth(sp, k.smooth_distance, k.smooth_ratio)
                av = emul.upload(sp, None, k.ur, k.ur, 0)
            spec[ch], pre[ch] = sp, av
    tex = [emul.smooth_at(k, pre[ch], idx) if k.smooth_pass else pre[ch][idx] for ch, idx in enumerate(texel_sets(c))]
    return spec, tex


def oracle_stream(orc, c, s):
    """the oracle (OracleStream: setbufscale and the post chain as render.c orders them) for stream s -> as host_stream.
    Its own K5 where that takes well under a second; for the wide windows the host build's K5 (bit-identical to the
    oracle's: tests/test_emul_parity.py) on the oracle's pre-smoothing texture."""
    from oracle.oracle import OracleStream, ext_from, params_from
    from tests import emul
    k = c.kernel_params(); user = c.params()
    q = user.copy(); q.smooth_pass = 0
    st = OracleStream(orc, params_from(q), ext_from(user))
    for t, m in enumerate(masks(c)):
        l, r = stream_pcm(c, t, s)
        sl, sr, tl, tr = st.update(l, r, m is None or bool(m[s]))
    tex = []
    for ch, (pre, idx) in enumerate(zip((tl, tr), texel_sets(c))):
        if not k.smooth_pass:
            tex.append(pre[idx])
        elif heavy(c):
            tex.append(emul.smooth_at(k, pre, idx))
        else:
            tex.append(orc.smooth_pass(params_from(k), pre)[idx])
    return [sl, sr], tex


def launch_class(c):
    """'lazy' (need-list K5), 'full' (whole-plane K5 after the spectrum kernel) or 'none' (no smooth pass).  From the
    case's overrides alone (the defaults: smooth pass on, lazy_smooth and transform_smooth off), so that the case list
    is built without the native library."""
    o = c.over
    if not o.get("smooth_pass", 1):
        return "none"
    if o.get("lazy_smooth", 0) and o.get("transform_smooth", 0) != 1 and c.module != "circle":
        return "lazy"
    return "full"


_SIZES = {}


def sizes(c, env=None):
    env = env or {}
    target = int(env.get("K5N_ROWS", -105)); tpb = int(env.get("K5N_TPB", 16))
    target = target if (target >= 32 or target < 0) else -105
    key = (c.id, target, tpb)
    if key not in _SIZES:
        from tests import emul
        _SIZES[key] = emul.table_sizes(c.kernel_params(), target, max(tpb, 1), full=launch_class(c) == "full")
    return _SIZES[key]


def launch_structure(c, env, sm_count=SM_COUNT):
    """-> (set of kernel instantiations / branches one update of case `c` runs under `env`, kernel launches of that update
    before the raster pass, or the error text the update is refused with)"""
    p = c.kernel_params(); user = c.params()
    s = sizes(c, env)
    wave = p.module == g.MODULES.index("wave")
    post = p.transform_smooth == 1
    F = p.avg_frames
    got = set()
    launches = 1 + (user.bufscale > 1)
    need = launch_class(c) == "lazy" and s["need"]
    epi_n = 0 if "NO_EPI_PRUNE" in env else s["epi_n"]
    split_lazy = taptab = csr = False
    max_rows = s["max_rows"]
    if need:
        taptab = s["tap_bytes"] <= 64 << 20 and "NO_TAPTAB" not in env
        if taptab:
            csr = s["spec_smem"] + s["blob"] <= 112 * 1024 and "NO_SMEM_TAPS" not in env
            split_lazy = env["K5_SPLIT"] != "0" if "K5_SPLIT" in env else (not csr or p.n >= 4096)
    fft_b = not wave and p.accel_fft
    epi8 = (epi_n + 7) // 8 * 8
    split_epi = split_lazy and fft_b and env.get("SPLIT_EPI", "1") != "0" and 0 < epi8 <= p.n
    if fft_b:
        if split_epi:
            got.add(f"epilogue_b_kernel<{F if F in (3, 4, 5, 6) else 0}>" + (" F=1" if F == 1 else ""))
            launches += 1
        else:
            got.add(f"in-kernel epilogue FT={F if F in (3, 4, 5, 6) else 0}")
    if need and not split_lazy:
        if taptab and csr:
            got.add("in-kernel lazy K5, shared-memory taps")
        elif taptab:
            ku = int(env.get("TAP_KU", 8))
            got.add(f"in-kernel lazy K5, L2 taps KU={8 if ku >= 8 else 4 if ku >= 4 else 2}")
        else:
            got.add("in-kernel lazy K5, no tap table")
    if split_lazy:
        mod = g.MODULES[p.module] + ("+join" if p.graph_join_channels and p.module == g.MODULES.index("graph") else "")
        got.add(f"split need-list: {mod}")
        mode = int(p.sample_mode != 0)
        if max_rows * 33 * 4 <= 200 * 1024 and env.get("K5N_SMEM") != "0" and s["nblk"] > 0:
            got.add(f"k5_need_smem_kernel<{mode}>")
            launches += 1
        else:
            if env.get("K5N_SMEM") != "0":
                got.add("k5_need_smem -> av_transpose + k5_need fall-back")
            S = 2 if (c.batch >= 256 and (1 if wave else 2) * s["need_count"] * ((c.batch + 63) // 64) >= sm_count * 24) else 1
            if env.get("K5N_S") in ("1", "2", "4"):
                S = int(env["K5N_S"])
            elif S == 2:
                got.add("k5_need_kernel automatic S=2")
            got.add(f"k5_need_kernel<{mode}, S={S}>")
            if S == 4 and c.batch > 64 and c.batch % 128:        # (the third 32-stream slice of a lane partly past the batch)
                got.add("k5_need_kernel S=4, partial stream group")
            launches += 2
    full = launch_class(c) == "full"
    if full and not post and "FUSED_K5" in env:
        got.add("in-kernel full-plane K5")
    elif full:
        launches += 1 + 2 * post              # (post-chain: transform_smooth and the upload before K5)
        table = ("NO_K5_TABLE" not in env and 2 * s["k5_span"] * 4 <= 200 * 1024 and s["k5_ent_bytes"] <= 256 << 20)
        if table:
            S = 8 if 8 * s["k5_span"] * 4 <= 200 * 1024 else 4 if 4 * s["k5_span"] * 4 <= 200 * 1024 else 2
            got.add(f"k5_table_kernel<{'avg' if p.sample_mode == 0 else 'max'}, {S}>")
        elif 8 * max(s["planes_span"], 1) * 2 > 200 * 1024:
            got.add("k5_planes_kernel refused: tap span too large")
            return got, launches, "tap span"
        else:
            got.add("k5_planes_kernel")
    elif post:
        launches += 2                         # transform_smooth and the upload
    return got, launches, None


# Every instantiation or branch the cases must reach, with the labels launch_structure gives it.  Unreachable ones are
# listed with the reason.
REQUIRED = (["epilogue_b_kernel<3>", "epilogue_b_kernel<4>", "epilogue_b_kernel<5>", "epilogue_b_kernel<6>",
             "epilogue_b_kernel<0>", "epilogue_b_kernel<0> F=1", "in-kernel epilogue FT=4", "in-kernel epilogue FT=0",
             "k5_need_smem_kernel<0>", "k5_need_smem_kernel<1>", "k5_need_kernel<0, S=1>", "k5_need_kernel<1, S=1>",
             "k5_need_kernel<0, S=2>", "k5_need_kernel<1, S=2>", "k5_need_kernel<0, S=4>", "k5_need_kernel automatic S=2",
             "k5_need_kernel S=4, partial stream group", "k5_need_smem -> av_transpose + k5_need fall-back",
             "k5_table_kernel<avg, 8>", "k5_table_kernel<max, 8>", "k5_table_kernel<avg, 4>", "k5_table_kernel<max, 2>",
             "in-kernel lazy K5, shared-memory taps", "in-kernel lazy K5, L2 taps KU=8", "in-kernel lazy K5, L2 taps KU=4",
             "in-kernel lazy K5, L2 taps KU=2", "in-kernel lazy K5, no tap table", "in-kernel full-plane K5",
             "k5_planes_kernel", "k5_planes_kernel refused: tap span too large"]
            + [f"split need-list: {m}" for m in ("bars", "radial", "graph", "graph+join", "wave")])
UNREACHABLE = {
    "split need-list: circle": "build_need_list returns false for circle (its angle samples any texel): circle always "
                               "smooths whole planes",
    "build_k5_table refusal (2 * max_span * 4 > 200 KiB)": "max_span <= n <= 16384 and 2 * 16384 * 4 = 128 KiB",
}
