"""The overlay onto decoded pictures (glava_b200_overlay_planes, DESIGN 4.17) on the host: the 10-bit blend and the 8-bit
4:4:4 blend of export_core.h through a g++ shim against the numpy restatement of tests/overlay_planes_np.py and against
float64, with the zero, opaque and 4:4:4-equals-block identities and the accumulator bounds; the two-pitch overlap test
against brute force; and the refusals and enqueued work of glava_b200_overlay_planes through capi.cu, export.cpp and
overlay_planes.cpp built against the fake runtime of tests/fakecuda (tests/export_fake.py's stubs plus a launcher that
counts its calls and records its OverlayPlanesArgs)."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from tests import export_fake, fakecuda
from tests.overlay_planes_np import cbcr8_np, cbcr10_np, y_np
from tests.test_export_core import CSRC, pack
from tests.test_export_matrix_core import coef_py, kr_kb

NV12, I420, YUV444, P010, YUV420P10, YUV444P10 = 2, 4, 5, 6, 7, 8

SHIM = r"""
#include "export_core.h"
using namespace glb;
template <int E> static void y10(const uint32_t* px, const uint32_t* yd, size_t n, uint32_t* out) {
    for (size_t i = 0; i < n; ++i) out[i] = overlay_y10<E>(px[i], yd[i]);
}
template <int E> static void c10(const uint32_t* s, const uint32_t* sa, const uint32_t* vd, size_t n, uint32_t* out) {
    for (size_t i = 0; i < n; ++i) out[i] = overlay_cbcr10<E>(s[i], sa[i], vd[i] & 0xffffu, vd[i] >> 16);
}
template <int E> static void px10(const uint32_t* px, const uint32_t* vd, size_t n, uint32_t* out) {   // planar samples
    for (size_t i = 0; i < n; ++i) out[i] = overlay_px10<E, false>(px[i], vd[i] & 0xffffu, vd[i] >> 16);
}
template <int E> static void blk10(const uint32_t* q, const uint32_t* vd, size_t n, uint32_t* out) {    // P010 samples
    for (size_t i = 0; i < n; ++i) out[i] = overlay_block10<E, true>(q[4 * i], q[4 * i + 1], q[4 * i + 2], q[4 * i + 3], vd[i], vd[i] >> 16);
}
template <int E> static void q444(const uint32_t* px, const uint32_t* d, size_t n, uint32_t* out) {    // 8-bit 4:4:4 quads
    for (size_t i = 0; i < n; ++i) {
        uint32_t y = d[3 * i], cb = d[3 * i + 1], cr = d[3 * i + 2];
        overlay_444_quad<E>(px + 4 * i, &y, &cb, &cr);
        out[3 * i] = y; out[3 * i + 1] = cb; out[3 * i + 2] = cr;
    }
}
template <int E> static void nv(const uint32_t* q, const uint32_t* d, size_t n, uint32_t* out) {      // NV12 quads
    for (size_t i = 0; i < n; ++i) {
        uint32_t yt = d[3 * i], yb = d[3 * i + 1], uv = d[3 * i + 2];
        overlay_nv12_quad<E>(q + 8 * i, q + 8 * i + 4, &yt, &yb, &uv);
        out[3 * i] = yt; out[3 * i + 1] = yb; out[3 * i + 2] = uv;
    }
}
template <int E> static void i420(const uint32_t* q, const uint32_t* d, size_t n, uint32_t* out) {     // I420 quads
    for (size_t i = 0; i < n; ++i) {
        uint32_t yt = d[4 * i], yb = d[4 * i + 1], cb = d[4 * i + 2], cr = d[4 * i + 3];
        overlay_i420_quad<E>(q + 8 * i, q + 8 * i + 4, &yt, &yb, &cb, &cr);
        out[4 * i] = yt; out[4 * i + 1] = yb; out[4 * i + 2] = cb; out[4 * i + 3] = cr;
    }
}
template <int E, bool Msb> static void p10q(const uint32_t* q, const uint32_t* d, size_t n, uint32_t* out) {  // 10-bit 4:2:0 quads
    for (size_t i = 0; i < n; ++i) {
        uint32_t yt[2] = { d[6 * i], d[6 * i + 1] }, yb[2] = { d[6 * i + 2], d[6 * i + 3] }, uv[2] = { d[6 * i + 4], d[6 * i + 5] };
        overlay_p10_quad<E, Msb>(q + 8 * i, q + 8 * i + 4, yt, yb, uv);
        const uint32_t o[6] = { yt[0], yt[1], yb[0], yb[1], uv[0], uv[1] };
        for (int k = 0; k < 6; ++k) out[6 * i + k] = o[k];
    }
}
"""
for _name, _args, _call in (("y10", "const uint32_t* a, const uint32_t* b, size_t n, uint32_t* out", "y10<E>(a, b, n, out)"),
                            ("c10", "const uint32_t* a, const uint32_t* b, const uint32_t* c, size_t n, uint32_t* out",
                             "c10<E>(a, b, c, n, out)"),
                            ("px10", "const uint32_t* a, const uint32_t* b, size_t n, uint32_t* out", "px10<E>(a, b, n, out)"),
                            ("blk10", "const uint32_t* a, const uint32_t* b, size_t n, uint32_t* out", "blk10<E>(a, b, n, out)"),
                            ("q444", "const uint32_t* a, const uint32_t* b, size_t n, uint32_t* out", "q444<E>(a, b, n, out)"),
                            ("nv", "const uint32_t* a, const uint32_t* b, size_t n, uint32_t* out", "nv<E>(a, b, n, out)"),
                            ("i420", "const uint32_t* a, const uint32_t* b, size_t n, uint32_t* out", "i420<E>(a, b, n, out)"),
                            ("p010q", "const uint32_t* a, const uint32_t* b, size_t n, uint32_t* out", "p10q<E, true>(a, b, n, out)"),
                            ("i010q", "const uint32_t* a, const uint32_t* b, size_t n, uint32_t* out", "p10q<E, false>(a, b, n, out)")):
    SHIM += f'extern "C" void t_{_name}(int e, {_args}) {{\n'
    SHIM += "".join(f"    if (e == {E}) {{ constexpr int E = {E}; {_call}; }}\n" for E in range(4)) + "}\n"


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("overlay_planes_core")
    src, so = d / "shim.cpp", d / "shim.so"
    src.write_text(SHIM)
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I", CSRC,
                    "-I", CSRC + "/../../include", "-include", "cstdint", "-include", "cstddef", "-o", str(so), str(src)], check=True)
    return C.CDLL(str(so))


def call(fn, e, per_out, *arrays):
    arrays = [np.ascontiguousarray(a, np.uint32) for a in arrays]
    n = arrays[-1].size // max(1, per_out) if per_out else arrays[0].size
    out = np.zeros(arrays[-1].size if per_out else arrays[0].size, np.uint32)
    fn(C.c_int(e), *[C.c_void_p(a.ctypes.data) for a in arrays], C.c_size_t(n), C.c_void_p(out.ctypes.data))
    return out


def premult(rng, n):
    """n premultiplied pixels over every alpha, with the extremes 0 and a included"""
    a = np.repeat(np.arange(256), n)
    rgb = np.minimum((rng.random((a.size, 3)) * (a[:, None] + 1)).astype(np.int64), a[:, None])
    rgb[::7] = a[::7, None]
    rgb[3::7] = 0
    return np.concatenate([rgb, a[:, None]], axis=1)


def float10(e, P, VD, chroma, scale=1):
    """the float64 composite at 10 bits of premultiplied P (channels scale times a pixel's) over codes VD"""
    kr, kb = kr_kb(e)
    full = bool(e & 1)
    ys, cs = (1023 / 255, 1023 / 255) if full else (876 / 255, 896 / 255)
    r, g, b, al = tuple(P[:, k] / scale for k in range(3)) + (P[:, 3] / (255.0 * scale),)
    yp = kr * r + (1 - kr - kb) * g + kb * b
    if not chroma:
        return np.clip((0 if full else 64) * al + ys * yp + (1 - al) * VD, 0, 1023)
    return (np.clip(512 * al + cs * (b - yp) / (2 * (1 - kb)) + (1 - al) * VD[:, 0], 0, 1023),
            np.clip(512 * al + cs * (r - yp) / (2 * (1 - kr)) + (1 - al) * VD[:, 1], 0, 1023))


# ---- 10-bit arithmetic -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("e", range(4))
def test_y10_every_alpha_against_numpy_and_float64(shim, e):
    rng = np.random.default_rng(e)
    P = premult(rng, 24)
    vd = rng.integers(0, 1024, P.shape[0])
    vd[::5] = 0; vd[1::5] = 1023
    got = call(shim.t_y10, e, 0, pack(P[:, 0], P[:, 1], P[:, 2], P[:, 3]), vd)
    assert np.array_equal(got, y_np(e, 10, P, vd))
    err = np.abs(got - float10(e, P, vd, False)).max()
    assert err <= 0.506, err


@pytest.mark.parametrize("e", range(4))
def test_420_chroma_of_block_sums_against_numpy_and_float64(shim, e):
    rng = np.random.default_rng(10 + e)
    Q = premult(rng, 64)
    S = np.stack([Q[rng.permutation(Q.shape[0])] for _ in range(4)]).sum(axis=0)   # sums of four premultiplied pixels
    vd = rng.integers(0, 1024, (S.shape[0], 2))
    vd[::5] = 0; vd[1::5] = 1023
    s = S[:, 0] | (S[:, 1] << 10) | (S[:, 2] << 20)
    got = call(shim.t_c10, e, 0, s, S[:, 3], vd[:, 0] | (vd[:, 1] << 16))
    cb, cr = cbcr10_np(e, S, vd[:, 0], vd[:, 1])
    assert np.array_equal(got & 0xffff, cb) and np.array_equal(got >> 16, cr)
    fcb, fcr = float10(e, S, vd, True, scale=4)
    err = max(np.abs((got & 0xffff) - fcb).max(), np.abs((got >> 16) - fcr).max())
    assert err <= 0.506, err


@pytest.mark.parametrize("e", range(4))
def test_zero_opaque_and_block_identities(shim, e):
    rng = np.random.default_rng(20 + e)
    vd = np.arange(1024)
    assert np.array_equal(call(shim.t_y10, e, 0, np.zeros(1024), vd), vd)                    # zero gives V_D
    z = call(shim.t_c10, e, 0, np.zeros(1024), np.zeros(1024), vd | (vd[::-1] << 16))
    assert np.array_equal(z, vd | (vd[::-1] << 16))
    c = rng.integers(0, 256, (4096, 3))
    ky, kcb, kcr, yoff, coff, top, _ = coef_py(e, 10)
    opaque = pack(c[:, 0], c[:, 1], c[:, 2], 255)
    want_y = np.clip((ky[0] * c[:, 0] + ky[1] * c[:, 1] + ky[2] * c[:, 2] + (yoff << 16) + (1 << 15)) >> 16, 0, top)
    assert np.array_equal(call(shim.t_y10, e, 0, opaque, rng.integers(0, 1024, 4096)), want_y)   # opaque: the export's code
    S = 4 * c
    want_cb = np.clip((kcb[0] * S[:, 0] + kcb[1] * S[:, 1] + kcb[2] * S[:, 2] + (coff << 18) + (1 << 17)) >> 18, 0, top)
    got = call(shim.t_c10, e, 0, S[:, 0] | (S[:, 1] << 10) | (S[:, 2] << 20), np.full(4096, 1020), rng.integers(0, 1 << 26, 4096))
    assert np.array_equal(got & 0xffff, want_cb)
    # YUV444P10 chroma of a pixel is P010 chroma of a 2x2 block of that pixel (P010 samples << 6)
    P = premult(rng, 8)
    px = pack(P[:, 0], P[:, 1], P[:, 2], P[:, 3])
    vd = rng.integers(0, 1024, (px.size, 2))
    planar = call(shim.t_px10, e, 0, px, vd[:, 0] | (vd[:, 1] << 16))
    block = call(shim.t_blk10, e, 1, np.repeat(px, 4), (vd[:, 0] << 6) | (vd[:, 1] << 22))
    assert np.array_equal(planar, (block >> 6) & 0x3ff03ff), e
    # YUV444 (8-bit) chroma of a pixel is NV12 chroma of a 2x2 block of that pixel
    q = px[:4 * (px.size // 4)].reshape(-1, 4)
    d = rng.integers(0, 1 << 32, (q.shape[0], 3), dtype=np.uint64).astype(np.uint32)
    y444 = call(shim.t_q444, e, 3, q, d).reshape(-1, 3)
    for k in range(4):
        quad = np.repeat(q[:, k:k + 1], 8, axis=1)          # a 2x2 block of pixel k, twice
        uvd = ((d[:, 1] >> (8 * k)) & 255) | (((d[:, 2] >> (8 * k)) & 255) << 8)
        nvq = call(shim.t_nv, e, 3, quad, np.stack([d[:, 0], d[:, 0], uvd | (uvd << 16)], 1)).reshape(-1, 3)
        assert np.array_equal((y444[:, 1] >> (8 * k)) & 255, nvq[:, 2] & 255), (e, k)
        assert np.array_equal((y444[:, 2] >> (8 * k)) & 255, (nvq[:, 2] >> 8) & 255), (e, k)


def test_accumulators_stay_in_their_documented_bounds():
    for e in range(4):
        ky, kcb, kcr, yoff, coff, top, _ = coef_py(e, 10)
        # Y: |coef c| + F + 2^15, F <= 1023 * 2^16
        assert sum(abs(k) for k in ky) * 255 + 1023 * 65536 + (1 << 15) < 1 << 28
        for k in (kcb, kcr):
            assert sum(abs(v) for v in k) * 1020 + 4 * 1023 * 65536 + (1 << 17) < 1 << 29
    # the exact split keeps every intermediate of F and G in 32 bits
    assert (254 << 16) + 127 < 1 << 32 and (1019 << 16) + 509 < 1 << 32 and 1023 * 255 + 255 * 1023 < 1 << 32


@pytest.mark.parametrize("e", range(4))
def test_quads_equal_the_restatement_and_keep_uncovered_samples(shim, e):
    """I420 is NV12 deinterleaved; YUV420P10 is P010 deinterleaved and >> 6 on the same codes; samples under zero pixels and
    chroma of all-zero blocks keep every bit (garbage padding included)"""
    rng = np.random.default_rng(30 + e)
    n = 4000
    P = premult(rng, 64)[rng.integers(0, 256 * 64, 8 * n)]
    px = pack(P[:, 0], P[:, 1], P[:, 2], P[:, 3])
    px[rng.random(px.size) < 0.4] = 0
    px[8 * rng.integers(0, n, n // 8)[:, None] + np.arange(8)] = 0            # whole zero quads
    q = px.reshape(n, 8)
    d = rng.integers(0, 1 << 32, (n, 3), dtype=np.uint64).astype(np.uint32)
    nvq = call(shim.t_nv, e, 3, q, d).reshape(n, 3)
    cb = (d[:, 2] & 0xff) | ((d[:, 2] >> 8) & 0xff00)
    cr = ((d[:, 2] >> 8) & 0xff) | ((d[:, 2] >> 16) & 0xff00)
    iq = call(shim.t_i420, e, 4, q, np.stack([d[:, 0], d[:, 1], cb, cr], 1)).reshape(n, 4)
    assert np.array_equal(iq[:, :2], nvq[:, :2])
    assert np.array_equal(iq[:, 2], (nvq[:, 2] & 0xff) | ((nvq[:, 2] >> 8) & 0xff00))
    assert np.array_equal(iq[:, 3], ((nvq[:, 2] >> 8) & 0xff) | ((nvq[:, 2] >> 16) & 0xff00))
    codes = rng.integers(0, 1024, (n, 8)).astype(np.uint32)                   # Y top 4, Y bot 4 ... as words below
    cc = rng.integers(0, 1024, (n, 4)).astype(np.uint32)                      # Cb0, Cr0, Cb1, Cr1
    w2 = lambda a, b: a | (b << 16)
    ymsb = [w2(codes[:, 2 * k] << 6, codes[:, 2 * k + 1] << 6) for k in range(4)]
    ylsb = [w2(codes[:, 2 * k], codes[:, 2 * k + 1]) for k in range(4)]
    pm = call(shim.t_p010q, e, 6, q, np.stack(ymsb + [w2(cc[:, 0] << 6, cc[:, 1] << 6), w2(cc[:, 2] << 6, cc[:, 3] << 6)], 1)).reshape(n, 6)
    pl = call(shim.t_i010q, e, 6, q, np.stack(ylsb + [w2(cc[:, 0], cc[:, 2]), w2(cc[:, 1], cc[:, 3])], 1)).reshape(n, 6)
    s = lambda v: (v >> 6) & 0x3ff03ff
    assert np.array_equal(pl[:, :4], s(pm[:, :4]))
    assert np.array_equal(pl[:, 4], (s(pm[:, 4]) & 0xffff) | (s(pm[:, 5]) << 16))
    assert np.array_equal(pl[:, 5], (s(pm[:, 4]) >> 16) | (s(pm[:, 5]) & 0xffff0000))
    # garbage padding bits: kept exactly where no non-zero pixel covers the sample, cleared where one does
    garbage = rng.integers(0, 1 << 32, (n, 6), dtype=np.uint64).astype(np.uint32)
    pg = call(shim.t_p010q, e, 6, q, garbage).reshape(n, 6)
    for k in range(4):
        for half in range(2):
            cov = q[:, 2 * k + half] != 0
            got, was = (pg[:, k] >> (16 * half)) & 0xffff, (garbage[:, k] >> (16 * half)) & 0xffff
            assert np.array_equal(got[~cov], was[~cov]) and not np.any(got[cov] & 63)
    for k in range(2):
        blk = (q[:, [2 * k, 2 * k + 1, 4 + 2 * k, 5 + 2 * k]] != 0).any(axis=1)
        assert np.array_equal(pg[~blk, 4 + k], garbage[~blk, 4 + k]) and not np.any(pg[blk, 4 + k] & 0x003f003f)
    # and the numpy restatement of the 8-bit Y and chroma
    ky = y_np(e, 8, np.stack([(q[:, 0] >> (8 * c)) & 255 for c in range(4)], 1).astype(np.int64), (d[:, 0] & 255).astype(np.int64))
    assert np.array_equal(nvq[:, 0] & 255, ky)
    m = ((np.stack([(q[:, [0, 1, 4, 5]] >> (8 * c)) & 255 for c in range(4)], -1).sum(axis=1) + 2) >> 2).astype(np.int64)
    want = cbcr8_np(e, m, (d[:, 2] & 255).astype(np.int64), ((d[:, 2] >> 8) & 255).astype(np.int64))
    assert np.array_equal(nvq[:, 2] & 255, want[0]) and np.array_equal((nvq[:, 2] >> 8) & 255, want[1])


# ---- the fake runtime ----------------------------------------------------------------------------------------------------------
PLANES_STUBS = r"""
static long g_planes = 0;
static glb::OverlayPlanesArgs g_pl;
extern "C" long planes_fake_launches(void) { return g_planes; }
extern "C" void planes_fake_last(long* out) {
    out[0] = g_pl.count; out[1] = g_pl.band; out[2] = g_pl.native; out[3] = g_pl.format; out[4] = g_pl.enc;
    out[5] = (long) g_pl.pitch; out[6] = (long) g_pl.chroma_pitch; out[7] = g_pl.w; out[8] = g_pl.h;
}
// planes_geometry_check on plain addresses: count entries of `planes` pointers each, one framebuffer range
extern "C" int t_planes_geometry(int w, int h, int count, const uintptr_t* ptrs, int format, size_t pitch, size_t cpitch,
                                 uintptr_t fb, size_t fb_bytes) {
    std::vector<glava_b200_picture> p((size_t) count);
    const int n = format == GLAVA_B200_EXPORT_NV12 || format == GLAVA_B200_EXPORT_P010 ? 2 : 3;
    for (int i = 0; i < count; ++i)
        for (int k = 0; k < 3; ++k) p[i].plane[k] = k < n ? (void*) ptrs[(size_t) i * n + k] : nullptr;
    glava_b200_overlay_planes_desc d = { format, 0, pitch, cpitch };
    const uint8_t* f = (const uint8_t*) fb;
    return glb::planes_geometry_check(w, h, count, p.data(), d, &f, &fb_bytes, 1, "t_planes_geometry");
}
namespace glb {
int launch_overlay_planes(const OverlayPlanesArgs& a, void*) {
    ++g_planes; g_pl = a;
    return a.fb && a.list && a.count > 0 && (!a.band || (a.marks && a.mark_rows > 0 && a.native)) ? 0
                                                                                                : fail(GLAVA_B200_EINVAL, "planes launch: bad arguments");
}
}
"""


@pytest.fixture(scope="module")
def fake():
    inc = fakecuda.cuda_include()
    if inc is None:
        pytest.skip("no CUDA toolkit headers")
    from glava_b200.api import Params
    out = tempfile.mkdtemp(prefix="glava_planes_fake_")
    src, so = os.path.join(out, "planes_fake.cpp"), os.path.join(out, "libplanes_fake.so")
    with open(src, "w") as f:
        f.write("#include <vector>\n" + export_fake.STUBS + PLANES_STUBS)
    subprocess.run(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I", inc,
                    "-I", fakecuda.CSRC, "-x", "c++", "-include", "cuda_runtime.h", "-o", so,
                    *[os.path.join(fakecuda.CSRC, f) for f in ("capi.cu", "export.cpp", "overlay_planes.cpp", "config.cpp")],
                    os.path.join(fakecuda.HERE, "fakecuda.cpp"), src, "-lpthread", "-Wl,-Bsymbolic"], check=True)
    L = C.CDLL(so)
    shutil.rmtree(out)
    vp, i32, P = C.c_void_p, C.c_int, C.POINTER(Params)
    sig = {
        "glava_b200_default_params": (i32, [P, C.c_char_p]), "glava_b200_new": (vp, [P, i32, i32]),
        "glava_b200_destroy": (None, [vp]), "glava_b200_last_error": (C.c_char_p, []), "glava_b200_set_abort_hook": (None, [vp]),
        "glava_b200_overlay_planes": (i32, [vp, vp, i32, vp, vp, vp, vp]),
        "cudaMalloc": (i32, [C.POINTER(vp), C.c_size_t]), "fake_trace": (C.c_char_p, []),
        "export_fake_device": (None, [vp, C.c_size_t]), "planes_fake_launches": (C.c_long, []), "planes_fake_last": (None, [vp]),
        "glava_b200_framebuffer_device": (vp, [vp]),
        "t_planes_geometry": (i32, [i32, i32, i32, vp, i32, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = res, args
    L._quiet = C.CFUNCTYPE(None, C.c_char_p)(lambda msg: None)
    L.glava_b200_set_abort_hook(C.cast(L._quiet, vp))
    return L


def renderer(L, w=64, h=32, batch=2):
    from glava_b200.api import Params
    p = Params()
    assert L.glava_b200_default_params(C.byref(p), b"bars") == 0
    p.n, p.w, p.h = 1024, w, h
    r = L.glava_b200_new(C.byref(p), batch, 0)
    assert r, L.glava_b200_last_error()
    return C.c_void_p(r)


def device_buf(L, nbytes=1 << 18):
    b = C.c_void_p()
    assert L.cudaMalloc(C.byref(b), nbytes) == 0
    L.export_fake_device(b, nbytes)
    return b.value + (-b.value) % 256


def _planes(L, r, streams, pics, fmt, pitch, cpitch, flags=0, null_desc=False):
    from glava_b200.api import OverlayPlanesDesc, Picture
    s = np.asarray(streams, np.int32)
    arr = (Picture * max(len(pics), 1))()
    for i, p in enumerate(pics):
        arr[i].plane = (C.c_void_p * 3)(*p)
    d = OverlayPlanesDesc()
    d.format, d.flags, d.pitch, d.chroma_pitch = fmt, flags, pitch, cpitch
    n0 = L.planes_fake_launches()
    rc = L.glava_b200_overlay_planes(r, s.ctypes.data if len(streams) else None, len(streams), arr, None if null_desc else C.byref(d),
                                     None, None)
    return rc, L.glava_b200_last_error().decode(), L.planes_fake_launches() - n0


def test_refusals_name_the_function_and_launch_nothing(fake):
    L = fake
    r = renderer(L)
    b = device_buf(L)
    i420 = (b, b + 4096, b + 8192)
    rc, msg, n = _planes(L, r, [0], [i420], I420, 64, 32)
    assert rc == 0 and n == 1, msg
    host = np.zeros(1 << 14, np.uint8)
    ha = host.ctypes.data + (-host.ctypes.data) % 16
    bad = [
        ([0], [i420], 0, 64, 32, 0, "overlay_frames"),                      # RGBA
        ([0], [i420], 1, 64, 32, 0, "overlay_frames"),                      # BGRA
        ([0], [i420], 3, 64, 32, 0, "unknown format"),
        ([0], [i420], I420, 64, 32, 1, "flags"),                            # EXPORT_OVER
        ([0], [i420], I420, 64, 32, 0x400, "flags"),
        ([0], [i420], I420, 48, 32, 0, "pitch"),                            # below w
        ([0], [i420], I420, 72, 32, 0, "pitch"),                            # not a multiple of 16
        ([0], [i420], I420, 64, 16, 0, "chroma_pitch"),                     # below w / 2
        ([0], [i420], I420, 64, 40, 0, "chroma_pitch"),
        ([0], [(b, b + 4096, 0)], P010, 128, 128, 0, None),                 # fine: P010 takes two planes
        ([0], [(b, b + 4096, b + 8192)], P010, 128, 128, 0, "plane[2]"),
        ([0], [(b, b + 4096, 0)], P010, 128, 112, 0, "chroma_pitch"),       # P010 chroma rows are 2w bytes
        ([0], [(b, b + 4096, 0)], NV12, 64, 48, 0, "chroma_pitch"),
        ([0], [(b, b + 8192, b + 16384)], YUV444P10, 128, 112, 0, "chroma_pitch"),
        ([0], [(b, b + 8192, b + 16384)], YUV420P10, 128, 48, 0, "chroma_pitch"),   # w bytes: w / 2 samples
        ([0], [(b, b + 4096, 0)], YUV444, 64, 64, 0, "null"),               # Cr missing
        ([0], [(b + 8, b + 4096, b + 8192)], I420, 64, 32, 0, "16-byte"),
        ([0], [(ha, b + 4096, b + 8192)], I420, 64, 32, 0, "device memory"),
        ([2], [i420], I420, 64, 32, 0, "out of range"),
        ([0, 1], [i420, i420], I420, 64, 32, 0, "overlaps"),
        ([0], [(b, b + 64 * 31, b + 8192)], I420, 64, 32, 0, "overlaps"),   # chroma inside the luma's last row
        ([0], [(b, b + 4096, b + 4096 + 32 * 15 + 16)], I420, 64, 32, 0, "overlaps"),   # Cr within Cb's rows
        ([], [], I420, 64, 32, 0, "count"),
    ]
    for streams, pics, fmt, P, CP, flags, what in bad:
        rc, msg, n = _planes(L, r, streams, pics, fmt, P, CP, flags)
        if what is None:
            assert rc == 0 and n == 1, msg
            continue
        assert rc != 0 and n == 0 and "glava_b200_overlay_planes" in msg and what in msg, (fmt, what, msg)
    rc, msg, n = _planes(L, r, [0], [i420], I420, 64, 32, null_desc=True)
    assert rc != 0 and n == 0 and "null" in msg
    odd = renderer(L, w=62, h=33)
    rc, msg, n = _planes(L, odd, [0], [i420], I420, 64, 32)
    assert rc != 0 and n == 0 and "even" in msg
    rc, msg, n = _planes(L, odd, [0], [(b, b + 8192, b + 16384)], YUV444, 64, 64)
    assert rc == 0 and n == 1, msg                                         # 4:4:4 takes any size
    fb = L.glava_b200_framebuffer_device(r)
    L.export_fake_device(fb, 64 * 32 * 4)                                  # the framebuffer is device memory
    rc, msg, n = _planes(L, r, [0], [(b, fb + 256, b + 8192)], I420, 64, 32)
    assert rc != 0 and n == 0 and "framebuffer" in msg


def test_the_launch_gets_format_encoding_pitches_and_item_kind(fake):
    L = fake
    r = renderer(L, w=96, h=48)
    b = device_buf(L)
    last = np.zeros(9, np.int64)
    for fmt, pics, P, CP in ((NV12, (b, b + 8192, 0), 96, 112), (YUV420P10, (b, b + 16384, b + 32768), 192, 96),
                             (YUV444, (b, b + 8192, b + 16384), 96, 128)):
        for flags, e in ((0, 0), (0x100, 1), (0x200, 2), (0x300, 3)):
            rc, msg, n = _planes(L, r, [1, 0, 1][:1], [pics], fmt, P, CP, flags)
            assert rc == 0 and n == 1, msg
            L.planes_fake_last(last.ctypes.data)
            assert list(last) == [1, 0, 1, fmt, e, P, CP, 96, 48], (fmt, e, list(last))   # no raster pass: no marks, row pairs


def brute(rects):
    """rects: (p, rows, P, B) -> whether any two overlap, by bytes"""
    seen = {}
    for i, (p, rows, P, B) in enumerate(rects):
        for r in range(rows):
            for x in range(p + r * P, p + r * P + B):
                if seen.setdefault(x, i) != i:
                    return True
    return False


def test_two_pitch_overlap_against_brute_force(fake):
    L = fake
    rng = np.random.default_rng(3)
    w, h = 32, 8
    for fmt in (I420, NV12, YUV444, P010, YUV420P10, YUV444P10):
        wide = fmt in (P010, YUV420P10, YUV444P10)
        c420 = fmt in (NV12, I420, P010, YUV420P10)
        n = 2 if fmt in (NV12, P010) else 3
        B = w * (2 if wide else 1)
        CB = {NV12: w, I420: w // 2, YUV444: w, P010: 2 * w, YUV420P10: w, YUV444P10: 2 * w}[fmt]
        CH = h // 2 if c420 else h
        for trial in range(150):
            P = B + 16 * int(rng.integers(0, 3))
            CP = CB + (-CB) % 16 + 16 * int(rng.integers(0, 3))
            count = int(rng.integers(1, 4))
            ptrs = (1 << 20) + 16 * rng.integers(0, 96, count * n)
            rects = [(int(ptrs[i * n + k]), h if k == 0 else CH, P if k == 0 else CP, B if k == 0 else CB)
                     for i in range(count) for k in range(n)]
            got = L.t_planes_geometry(w, h, count, np.ascontiguousarray(ptrs, np.uint64).ctypes.data, fmt, P, CP, 1 << 30, 64)
            assert (got != 0) == brute(rects), (fmt, trial, rects)
        # a tight mosaic passes: 4 x 4 tiles side by side, chroma planes of their own
        cols = 4
        P, CP = B * cols, CB * cols + (-(CB * cols)) % 16
        ptrs = []
        for t in range(16):
            ty, tx = divmod(t, cols)
            ptrs.append((1 << 24) + ty * h * P + tx * B)
            for k in range(1, n):
                ptrs.append((1 << 26) * k + ty * CH * CP + tx * CB)
        if all(v % 16 == 0 for v in ptrs):
            assert L.t_planes_geometry(w, h, 16, np.asarray(ptrs, np.uint64).ctypes.data, fmt, P, CP, 1 << 30, 64) == 0, fmt
