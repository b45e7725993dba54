"""Seeded cases over keyframe interpolation (setinterpolate), shared by the CPU tier (tests/test_keyframe_cases.py: the host
restatement against the oracle) and the GPU tier (tests/test_gpu_keyframes.py: the kernels against the host build).

With interpolation active every frame has a new texture: the R16 upload of s + (e - s) * mod, where s and e are the chain
results of the two previous modified updates (the keyframes, zero until two exist), mod = min(ur / fr * kcounter, 1) and
kcounter counts the frames since the last modified update (render.c:1792-1809, 2347-2353, 2380-2383).  A modified frame
still shows the lerp of the old keyframes with the old kcounter; its own chain result becomes the end keyframe afterwards.
Whole-plane K5 follows the upload (a post chain never runs the need-list forms).

A case is (module, parameters, batch, launch environment, cadence).  Coverage is forced, not left to the seed: every
setbufsize, bars / radial / graph / circle under pipeline A and wave under both, F in {1, 3, 5, 16} with the average window on
and off, all nine sample_mode x round_formula pairs, the smooth pass off, every whole-plane K5 form (k5_table_kernel with 8, 4
and 2 planes per CTA, partial CTA groups, k5_planes_kernel and its refusal), the appended transform, setbufscale 2 and 4 and
both together, setaccelfft with the appended transform (derive() clears it, so interpolation stays on), and both sides of
the 0.9 boundary of ur / fr.  `launch_structure` derives each frame's kernels from the library's own plan
(emul.spectrum_plan), so that coverage is computed, not claimed."""
import itertools

import numpy as np

import glava_b200 as g
from tests import spectrum_cases as sc

SIZES = sc.SIZES
F_VALUES = [1, 3, 5, 16]
MODES = sc.MODES
RATIOS = [4.0, 2.5, 3.3]                         # fr / ur
# cadences (1 = modified update): each starts before two keyframes exist, has two modified updates in a row and a run of
# unmodified frames longer than fr / ur (mod clamps at 1)
CADENCES = [(1, 0, 1, 1, 0, 0, 0, 0, 0, 0, 1, 0),
            (1, 1, 0, 0, 0, 1, 0, 0, 0, 0, 0, 1, 0),
            (1, 0, 0, 0, 0, 0, 1, 1, 0, 1, 0, 0)]
AMPS = [0.3, 0.05, 0.3, 0.0, 0.2, 0.004, 0.3, 0.1, 0.25, 0.02, 0.3, 0.15, 0.08]   # update 3 is silent: gravity falls


def _past_boundary(ur):
    """(ur', fr) with ur' the first float at or above ur for which some fr gives ur' / fr (in float) one float step above
    0.9f: the interpolation just switched off"""
    target = np.nextafter(np.float32(0.9), np.float32(1))
    u = np.float32(ur)
    for _ in range(256):
        fr = np.float32(u / target)
        for _ in range(8):
            q = u / fr
            if q == target:
                return float(u), float(fr)
            fr = np.nextafter(fr, np.float32(0) if q < target else np.float32(1e9))
        u = np.nextafter(u, np.float32(1e9))
    raise AssertionError("no fr found")


class Case:
    def __init__(self, seed, cid, module, over, batch, env, cadence):
        self.seed, self.id, self.module, self.over, self.batch = seed, cid, module, over, batch
        self.env, self.cadence = env, cadence

    def params(self):
        return g.default_params(self.module, **self.over)

    def kernel_params(self):
        """as capi.cu derive: n = setbufsize / setbufscale, setaccelfft cleared by the appended transform"""
        p = self.params()
        q = g.default_params(self.module, **dict(self.over, n=p.n // p.bufscale, bufscale=1))
        if q.transform_smooth == 1 and self.module != "wave":
            q.accel_fft = 0
        return q

    def __repr__(self):
        return self.id


def interp_on(p):
    """capi.cu derive: setinterpolate, not pushed to the GPU passes, and ur / fr <= 0.9 in float"""
    k = p.copy()
    if k.transform_smooth == 1 and k.module != g.MODULES.index("wave"):
        k.accel_fft = 0
    fr = np.float32(k.fr if k.fr > 0 else k.ur)
    return bool(k.interpolate and not (k.accel_fft and k.module != g.MODULES.index("wave"))
                and np.float32(k.ur) / fr <= np.float32(0.9))


def build_cases(seed=2027):
    rng = np.random.default_rng(seed)
    cases = []
    modes = itertools.cycle(MODES)
    ratios = itertools.cycle(RATIOS)
    cadences = itertools.cycle(CADENCES)

    def add(tag, module, over, batch=7, env=None, ratio=None):
        w, h = sc.GEOMETRY[module][len(cases) % len(sc.GEOMETRY[module])]
        sm, rf = next(modes)
        knobs = sc._random_knobs(rng)
        ratio = next(ratios) if ratio is None else ratio
        base = dict(knobs, w=w, h=h, sample_mode=sm, round_formula=rf, interpolate=1, accel_fft=0, lazy_smooth=0)
        base["fr"] = float(np.float32(base["ur"]) * np.float32(ratio))
        base.update(over)
        cases.append(Case(seed + len(cases), f"{len(cases):02d}-{module}-{tag}", module, base, batch, env or {},
                          next(cadences)))

    # every setbufsize; the five modules (wave in both pipelines); F on and off the average window
    add("256F1", "bars", dict(n=256, avg_frames=1, avg_window=0))
    add("512F3", "radial", dict(n=512, avg_frames=3, avg_window=1))
    add("1024F5", "graph", dict(n=1024, avg_frames=5, avg_window=0))
    add("2048F16", "circle", dict(n=2048, avg_frames=16, avg_window=1), batch=5)
    add("4096F3-A", "wave", dict(n=4096, avg_frames=3, avg_window=0))
    add("8192F5-B", "wave", dict(n=8192, avg_frames=5, avg_window=1, accel_fft=1))
    add("16384F16", "bars", dict(n=16384, avg_frames=16, avg_window=0, smooth_factor=0.005), batch=9)
    add("1024F16-B", "wave", dict(n=1024, avg_frames=16, accel_fft=1), batch=3)
    add("4096F1", "graph", dict(n=4096, avg_frames=1, graph_join_channels=1), batch=11)
    add("8192F3", "radial", dict(n=8192, avg_frames=3), batch=5)
    # the smooth pass off: the upload writes the texture
    add("nosmooth", "bars", dict(n=1024, smooth_pass=0))
    add("nosmooth-circle", "circle", dict(n=512, smooth_pass=0, avg_frames=5))
    # whole-plane K5 forms: wide windows at 16384 (4 and 2 planes per CTA, groups partial), k5_planes_kernel and its refusal
    add("wide-t4", "bars", dict(n=16384, smooth_factor=0.02, sample_mode=0, **sc.WIDE), batch=5)
    add("wide-t2", "circle", dict(n=16384, smooth_factor=0.04, sample_mode=2, **sc.WIDE), batch=3)
    add("planes", "bars", dict(n=4096), batch=5, env=dict(NO_K5_TABLE="1"))
    add("planes-refused", "bars", dict(n=16384, smooth_factor=0.04, sample_mode=1, **sc.WIDE), batch=3,
        env=dict(NO_K5_TABLE="1"))
    # post chains: the appended transform, setbufscale 2 and 4, both; setaccelfft under the appended transform
    add("post", "bars", dict(n=1024, transform_smooth=1))
    add("post-accel", "bars", dict(n=2048, transform_smooth=1, accel_fft=1, smooth_distance=0.02, smooth_ratio=2.0))
    add("bs2", "radial", dict(n=2048, bufscale=2))
    add("bs4", "graph", dict(n=4096, bufscale=4, avg_frames=3))
    add("bs2-post", "bars", dict(n=8192, bufscale=2, transform_smooth=1))
    add("bs4-post-accel", "bars", dict(n=4096, bufscale=4, transform_smooth=1, accel_fft=1), batch=6)
    # the boundary of ur / fr <= 0.9f: exactly on it (interpolation on), one float step past it (off)
    add("at-0.9", "bars", dict(n=1024, ur=90.0, fr=100.0))
    ur, fr = _past_boundary(90.0)
    add("past-0.9", "bars", dict(n=1024, ur=ur, fr=fr))
    return cases


# ---- inputs -------------------------------------------------------------------------------------------------------------
def stream_pcm(c, t, s):
    """(lb, rb) of stream s at frame t (setbufsize floats): noise at the frame's amplitude (every 4th stream 50x quieter)"""
    n = c.params().n
    rng = np.random.default_rng([c.seed, t, s])
    amp = AMPS[t % len(AMPS)] * (0.02 if s % 4 == 3 else 1.0)
    l = ((rng.random(n, dtype=np.float32) - 0.5) * np.float32(2 * amp)).astype(np.float32)
    r = ((rng.random(n, dtype=np.float32) - 0.5) * np.float32(2 * amp)).astype(np.float32)
    return l, r


def batch_pcm(c, t):
    pcm = [stream_pcm(c, t, s) for s in range(c.batch)]
    return np.stack([x[0] for x in pcm]), np.stack([x[1] for x in pcm])


def checked_streams(c):
    return sorted({0, c.batch // 2, c.batch - 1})


def heavy(c):
    """windows wide enough that a whole host K5 per frame costs seconds"""
    return c.kernel_params().n >= 16384 and c.over.get("sample_scale", 0) == sc.WIDE["sample_scale"]


def texels(c):
    """the texels compared per frame: all of them, or for the heavy cases every 61st and the last 32"""
    n = c.kernel_params().n
    if heavy(c):
        return np.union1d(np.arange(0, n, 61), np.arange(n - 32, n))
    return np.arange(n)


# ---- the host restatement -----------------------------------------------------------------------------------------------
class HostKeyframes:
    """one stream through the host build's pieces: emul.Channel (the chain, smooth pass off), emul.bufscale,
    emul.transform_smooth, the rotation of the keyframes, emul.upload(start, end, ur, fr, kcounter), emul.smooth_at.
    step(modified, pcm, k) takes the kernel parameters k of that frame (a reconfigure may change fr or the smoothing)."""

    def __init__(self, k, bufscale):
        self.bufscale = bufscale
        q = k.copy(); q.smooth_pass = 0
        self.q = q
        self.chans = [emul().Channel(q), emul().Channel(q)]
        self.keys = [[np.zeros(k.n, np.float32), np.zeros(k.n, np.float32)] for _ in range(2)]
        self.spec = [np.zeros(k.n, np.float32), np.zeros(k.n, np.float32)]
        self.kcounter = 0

    def chain(self, pcm, k):
        """the post-transform chain results of one modified update"""
        wave = k.module == g.MODULES.index("wave")
        out = []
        for ch, x in enumerate(pcm):
            if wave and ch == 1:
                out.append(np.zeros(k.n, np.float32))              # wave runs plane 0 only: plane 1 of its keys stays 0
                continue
            if self.bufscale > 1:
                x = emul().bufscale(x, self.bufscale)
            sp, _ = self.chans[ch].update(x, is_fft=not wave)
            if k.transform_smooth == 1:
                sp = emul().transform_smooth(sp, k.smooth_distance, k.smooth_ratio)
            out.append(sp)
        return out

    def upload(self, k):
        fr = k.fr if k.fr > 0 else k.ur
        return [emul().upload(self.keys[ch][0], self.keys[ch][1], k.ur, fr, self.kcounter) for ch in (0, 1)]

    def rotate(self, spec):
        for ch in (0, 1):
            self.keys[ch] = [self.keys[ch][1], spec[ch]]

    def step(self, modified, pcm, k, idx):
        """-> (spectra of the latest modified update, textures at idx)"""
        if modified:
            self.spec = self.chain(pcm, k)
        pre = self.upload(k)                                       # a modified frame: the old keys and the old kcounter
        tex = [emul().smooth_at(k, pre[ch], idx) if k.smooth_pass else pre[ch][idx] for ch in (0, 1)]
        if modified:
            self.rotate(self.spec)
        self.kcounter = 0 if modified else self.kcounter + 1
        return [x.copy() for x in self.spec], tex


def emul():
    from tests import emul as e
    return e


def host_keyframes(c, s):
    """per frame of case c, stream s: (spectra of the latest modified update, textures at texels(c))"""
    k = c.kernel_params()
    h = HostKeyframes(k, c.params().bufscale)
    idx = texels(c)
    return [h.step(m, stream_pcm(c, t, s), k, idx) for t, m in enumerate(c.cadence)]


def keyframes_from_spectra(c, spectra, pre_only=False):
    """the restatement's rotation, upload and K5 fed per-frame chain results (from another implementation: the oracle):
    spectra[t] = [spec_l, spec_r] after frame t -> per-frame textures (all texels; the upload alone with pre_only)"""
    k = c.kernel_params()
    h = HostKeyframes(k, 1)
    out = []
    for t, m in enumerate(c.cadence):
        pre = h.upload(k)
        if pre_only or not k.smooth_pass:
            out.append(pre)
        else:
            out.append([emul().smooth(k, x) for x in pre])
        if m:
            h.rotate([np.asarray(x, np.float32) for x in spectra[t]])
        h.kcounter = 0 if m else h.kcounter + 1
    return out


# ---- the launch structure -----------------------------------------------------------------------------------------------
_PLANS = {}


def plan(c, env=None):
    env = c.env if env is None else env
    key = (c.id, tuple(sorted(env.items())))
    if key not in _PLANS:
        _PLANS[key] = emul().spectrum_plan(c.kernel_params(), True, c.batch, sc.SM_COUNT, env)
    return _PLANS[key]


def post_label(c):
    k = c.kernel_params(); user = c.params()
    parts = ["interp"]
    if k.transform_smooth == 1:
        parts.append("transform_smooth")
        if user.accel_fft and c.module != "wave":
            parts.append("setaccelfft cleared")
    if user.bufscale > 1:
        parts.append(f"bufscale {user.bufscale}")
    return "post chain: " + " + ".join(parts)


def launch_structure(c):
    """-> (labels of what a frame of case c runs, {modified: launches before the raster pass}, refusal or None); for a
    case past the 0.9 boundary interpolation is off: (labels, None, None), compared with an interpolate = 0 renderer"""
    k = c.kernel_params(); user = c.params()
    if not interp_on(c.params()):
        return {"interpolation off: ur / fr one float step past 0.9f"}, None, None
    labels = {post_label(c)}
    if np.float32(k.ur) / np.float32(k.fr) == np.float32(0.9):
        labels.add("interpolation on: ur / fr exactly 0.9f")
    pl = plan(c)
    assert not pl["need_list"] and pl["k5"] in ("none", "full_table", "full_planes"), pl
    k5 = 0
    if pl["k5"] == "full_table":
        planes = pl["table_planes"]
        labels.add(f"k5_table_kernel<{'avg' if k.sample_mode == 0 else 'max'}, {planes}>")
        if (2 * c.batch) % planes:
            labels.add("k5_table_kernel partial CTA group")
        k5 = 1
    elif pl["k5"] == "full_planes":
        labels.add("k5_planes_kernel refused: tap span too large" if pl["refusal"] else "k5_planes_kernel")
        k5 = 1
    else:
        labels.add("smooth pass off: the upload writes the texture")
    spectrum = 1 + pl["split_epilogue"]                      # spectrum_kernel (no need-list, no in-kernel K5: skip_tex)
    modified = (user.bufscale > 1) + spectrum + (k.transform_smooth == 1) + 1 + k5
    return labels, {True: modified, False: 1 + k5}, pl["refusal"]


REQUIRED = (["k5_table_kernel<avg, 8>", "k5_table_kernel<max, 8>", "k5_table_kernel<avg, 4>", "k5_table_kernel<max, 2>",
             "k5_table_kernel partial CTA group", "k5_planes_kernel", "k5_planes_kernel refused: tap span too large",
             "smooth pass off: the upload writes the texture",
             "interpolation on: ur / fr exactly 0.9f", "interpolation off: ur / fr one float step past 0.9f"]
            + ["post chain: " + x for x in ("interp", "interp + transform_smooth",
                                              "interp + transform_smooth + setaccelfft cleared", "interp + bufscale 2",
                                              "interp + bufscale 4", "interp + transform_smooth + bufscale 2",
                                              "interp + transform_smooth + setaccelfft cleared + bufscale 4")])
UNREACHABLE = {
    "need-list K5 (lazy_smooth) under interpolation": "plan_spectrum builds no need-list with a post chain: every texel "
                                                      "moves on an interpolated frame",
    "in-kernel full-plane K5 (FUSED_K5) under interpolation": "plan_spectrum keeps K5 out of spectrum_kernel with a "
                                                               "post chain: it follows the upload",
}
