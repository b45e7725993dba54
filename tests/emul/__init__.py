"""TEST INFRASTRUCTURE — host emulation of the CUDA kernels' arithmetic (see emul.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None


def lib():
    global _lib
    if _lib is None:
        so = os.path.join(HERE, "libglava_emul.so")
        src = os.path.join(HERE, "emul.cpp")
        csrc = os.path.join(HERE, "..", "..", "glava_b200", "csrc")
        newest = max(os.path.getmtime(os.path.join(csrc, f)) for f in os.listdir(csrc) if f.endswith(".h"))
        if not os.path.exists(so) or os.path.getmtime(so) < max(newest, os.path.getmtime(src)):
            subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas",
                            "-o", so, src], check=True)
        L = C.CDLL(so)
        vp, i32 = C.c_void_p, C.c_int
        L.emul_fft.argtypes = [i32, vp, vp, C.c_float, C.c_float]
        L.emul_chan_new.restype = vp
        L.emul_chan_new.argtypes = [vp]
        L.emul_chan_free.argtypes = [vp]
        L.emul_chan_update.argtypes = [vp, vp, vp, i32, vp, vp]
        L.emul_smooth.argtypes = [vp, vp, vp]
        L.emul_smooth_at.argtypes = [vp, vp, vp, i32, vp]
        L.emul_raster.argtypes = [vp, vp, vp, vp, i32, i32]
        L.emul_raster_fast.argtypes = [vp, vp, vp, vp]
        L.emul_eval_color.argtypes = [vp, C.c_float, vp]
        L.emul_radial_geo.argtypes = [vp, vp]
        L.emul_radial_from_geo.argtypes = [vp, vp, vp, vp, vp]
        L.emul_lazy_k5.argtypes = [vp, i32, i32, vp, vp, vp]
        L.emul_lazy_epi_n.argtypes = [vp]
        L.emul_k5_table.argtypes = [vp, vp, vp]
        L.emul_table_sizes.argtypes = [vp, i32, i32, i32, vp]
        L.emul_spectrum_plan.argtypes = [vp, i32, i32, i32, vp, vp, i32, vp, vp, i32]
        L.emul_raster_plan.argtypes = [vp, i32, i32, vp, vp, i32, i32, vp]
        L.emul_bufscale.argtypes = [vp, i32, i32, vp]
        L.emul_transform_smooth.argtypes = [vp, i32, C.c_float, C.c_float]
        L.emul_upload.argtypes = [vp, vp, i32, C.c_float, C.c_float, i32, vp]
        _lib = L
    return _lib


def fft(pcm, fft_scale=10.2, fft_cutoff=0.3):
    x = np.ascontiguousarray(pcm, dtype=np.float32)
    out = np.empty_like(x)
    assert lib().emul_fft(x.shape[0], x.ctypes.data, out.ctypes.data, fft_scale, fft_cutoff) == 0
    return out


class Channel:
    def __init__(self, params):
        self.p = params
        self.h = lib().emul_chan_new(C.addressof(params))

    def update(self, pcm, is_fft=True):
        x = np.ascontiguousarray(pcm, dtype=np.float32)
        spec = np.empty(self.p.n, np.float32); tex = np.empty(self.p.n, np.uint16)
        assert lib().emul_chan_update(self.h, C.addressof(self.p), x.ctypes.data, 1 if is_fft else 0,
                                      spec.ctypes.data, tex.ctypes.data) == 0
        return spec, tex

    def __del__(self):
        try: lib().emul_chan_free(self.h)
        except Exception: pass


def smooth(params, tex):
    t = np.ascontiguousarray(tex, dtype=np.uint16)
    out = np.empty_like(t)
    lib().emul_smooth(C.addressof(params), t.ctypes.data, out.ctypes.data)
    return out


def smooth_at(params, tex, idx):
    """smooth(params, tex)[idx] without computing the other texels"""
    t = np.ascontiguousarray(tex, dtype=np.uint16)
    ix = np.ascontiguousarray(idx, dtype=np.int32)
    out = np.empty(ix.shape[0], np.uint16)
    lib().emul_smooth_at(C.addressof(params), t.ctypes.data, ix.ctypes.data, ix.shape[0], out.ctypes.data)
    return out


def raster(params, tex_l, tex_r, fast=False):
    tl = np.ascontiguousarray(tex_l, dtype=np.uint16)
    tr = np.ascontiguousarray(tex_r if tex_r is not None else tex_l, dtype=np.uint16)
    out = np.zeros((params.h, params.w, 4), dtype=np.uint8)
    if fast:
        assert lib().emul_raster_fast(C.addressof(params), tl.ctypes.data, tr.ctypes.data, out.ctypes.data) == 0
    else:
        lib().emul_raster(C.addressof(params), tl.ctypes.data, tr.ctypes.data, out.ctypes.data, 0, params.h)
    return out


class RadialGeo:
    """raster(params, tl, tr) for radial, with the audio-independent half of every pixel (the colour program included)
    computed once: frames(tl, tr) is then cheap for each further texture pair"""

    def __init__(self, params):
        self.p = params
        self.geo = np.empty(params.w * params.h * lib().emul_radial_geo_bytes(), np.uint8)
        lib().emul_radial_geo(C.addressof(params), self.geo.ctypes.data)

    def frame(self, tex_l, tex_r):
        tl = np.ascontiguousarray(tex_l, dtype=np.uint16)
        tr = np.ascontiguousarray(tex_r, dtype=np.uint16)
        out = np.zeros((self.p.h, self.p.w, 4), dtype=np.uint8)
        lib().emul_radial_from_geo(C.addressof(self.p), self.geo.ctypes.data, tl.ctypes.data, tr.ctypes.data, out.ctypes.data)
        return out


def bufscale(pcm, k):
    x = np.ascontiguousarray(pcm, dtype=np.float32)
    out = np.empty(x.shape[0] // k, np.float32)
    lib().emul_bufscale(x.ctypes.data, x.shape[0], k, out.ctypes.data)
    return out


def transform_smooth(buf, smooth_distance=0.01, smooth_ratio=4.0):
    b = np.array(buf, dtype=np.float32, copy=True)
    lib().emul_transform_smooth(b.ctypes.data, b.shape[0], smooth_distance, smooth_ratio)
    return b


def upload(start, end, ur, fr, kcounter):
    s = np.ascontiguousarray(start, dtype=np.float32)
    e = None if end is None else np.ascontiguousarray(end, dtype=np.float32)
    out = np.empty(s.shape[0], np.uint16)
    lib().emul_upload(s.ctypes.data, None if e is None else e.ctypes.data, s.shape[0], ur, fr, kcounter, out.ctypes.data)
    return out


def lazy_k5(p, chan, path, av):
    """(texel indices, values) of the need-list texels of channel `chan`, through the tap-major table (path 0) or the
    texel-major blob (path 1)"""
    av = np.ascontiguousarray(av, dtype=np.uint16)
    out = np.zeros(p.n, np.uint16); need = np.zeros(p.n, np.int32)
    cnt = lib().emul_lazy_k5(C.byref(p), chan, path, av.ctypes.data, out.ctypes.data, need.ctypes.data)
    if cnt < -1:
        raise AssertionError(f"blocks-of-texels walk: error {cnt} (emul.cpp emul_lazy_k5)")
    if cnt < 0:
        return None, None
    idx = need[:cnt].copy()
    return idx, out[idx]


def lazy_epi_n(p):
    return lib().emul_lazy_epi_n(C.byref(p))


TABLE_SIZES = ("need", "need_count", "blob", "tap_bytes", "epi_n", "max_rows", "nblk", "k5_span", "k5_ent_bytes",
               "planes_span", "spec_smem")


def table_sizes(p, target_rows=-105, texels_per_block=16, full=True):
    """the table sizes plan_spectrum chooses the K5 launch structure from (emul.cpp emul_table_sizes);
    target_rows / texels_per_block as GLAVA_B200_K5N_ROWS / _TPB, defaults as build_tables; full=False skips the
    full-plane table (k5_span, k5_ent_bytes read 0)"""
    out = np.zeros(len(TABLE_SIZES), np.int64)
    lib().emul_table_sizes(C.byref(p), target_rows, texels_per_block, 1 if full else 0, out.ctypes.data)
    return dict(zip(TABLE_SIZES, out.tolist()))


PLAN_FIELDS = ("need_list", "tap_table", "full_table", "split_epilogue", "epi_n", "av_t_len", "k5", "tap_ku", "table_planes",
               "k5n_s", "k5n_warps", "fft_oop", "fft_t", "spec_grid", "spec_resident")
K5_FORMS = ("none", "taps_smem", "taps_l2", "taps_direct", "need_smem", "need_l2", "full_table", "full_planes", "fused")


def _env_arrays(env):
    """env ({"K5_SPLIT": "1", ...}, names without GLAVA_B200_) -> (names, values, count) for the C side"""
    names = [("GLAVA_B200_" + k).encode() for k in env]
    values = [str(v).encode() for v in env.values()]
    n = max(len(names), 1)
    return (C.c_char_p * n)(*names), (C.c_char_p * n)(*values), len(names)


def spectrum_plan(p, post_chain, batch, sm_count, env):
    """the launch structure the library chooses (spectrum_plan.h plan_spectrum) for the effective parameters p under the
    environment overrides env ({"K5_SPLIT": "1", ...}, names without GLAVA_B200_) -> dict of PLAN_FIELDS (k5 as a K5_FORMS
    name) and "refusal" (None: none)"""
    out = np.zeros(len(PLAN_FIELDS), np.int64)
    refusal = C.create_string_buffer(256)
    lib().emul_spectrum_plan(C.byref(p), int(post_chain), batch, sm_count, *_env_arrays(env), out.ctypes.data,
                             refusal, len(refusal))
    plan = dict(zip(PLAN_FIELDS, out.tolist()))
    plan["k5"] = K5_FORMS[plan["k5"]]
    plan["refusal"] = refusal.value.decode() or None
    return plan


RASTER_PLAN_FIELDS = ("kernel", "bx", "rows", "minb", "circle_tiles", "coltab", "texmm", "ctile", "rowtab", "geo", "chunk",
                      "mark_key", "launches", "marks_valid")
RASTER_KERNELS = ("generic", "bars", "graph", "graph_tab4", "graph_tab5", "wave", "wave_tab4", "wave_tab5", "radial",
                  "radial_geo", "circle")


def raster_plan(p, batch, slots, env, last_key=0):
    """the raster pass the library plans (raster_plan.h) for the effective parameters p, `batch` streams and `slots`
    framebuffer slots under the environment overrides env (names without GLAVA_B200_, set when the tables are built and at
    the launch) -> dict of RASTER_PLAN_FIELDS (kernel as a RASTER_KERNELS name); marks_valid: whether a launch whose
    renderer last recorded `last_key` may trust its dirty-row marks"""
    out = np.zeros(len(RASTER_PLAN_FIELDS), np.int64)
    lib().emul_raster_plan(C.byref(p), batch, slots, *_env_arrays(env), last_key, out.ctypes.data)
    plan = dict(zip(RASTER_PLAN_FIELDS, out.tolist()))
    plan["kernel"] = RASTER_KERNELS[plan["kernel"]]
    return plan


def k5_table(p, tex):
    tex = np.ascontiguousarray(tex, dtype=np.uint16)
    out = np.empty_like(tex)
    lib().emul_k5_table(C.byref(p), tex.ctypes.data, out.ctypes.data)
    return out


def eval_color(prog, x):
    """a compiled colour expression (glava_b200.api.ColorProg) at X -> float32[4]"""
    out = np.zeros(4, np.float32)
    lib().emul_eval_color(C.byref(prog), float(x), out.ctypes.data)
    return out
