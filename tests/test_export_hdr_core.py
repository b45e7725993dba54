"""BT.2020 HDR exports and overlay (DESIGN 4.22) on the host: export_core.h's float32 arithmetic against the float64 definition
of tests/export_hdr_np.py over every colour, seeded blocks and pairs and sampled overlays; the checkpoints; the
linearisation table and matrix constants; the overlay's bit-for-bit invariants; the refusals and encodings through capi.cu,
export.cpp and export_ladder.cpp built against tests/fakecuda's runtime; and the Python keywords."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from tests import export_hdr_np as H
from tests import export_hdr_shim as S
from tests.export_fake import desc_of
from tests.test_export_core import CSRC
from tests.test_export_ladder_core import _ladder, scale_of
from tests.test_export_matrix_core import _call, encs
from tests.test_export_matrix_core import fake  # noqa: F401 (the fake-runtime fixture)

# Largest |code - float64| over all 2^24 colours, Y, Cb and Cr (measured: PQ 0.50318 / 0.50324 / 0.50309, HLG 0.50008 /
# 0.50007 / 0.50009; DESIGN 4.22).  PQ's exponent m2 = 78.8 turns the rounding of its base into up to 0.0033 code values.
BOUND = {H.PQ: 0.504, H.HLG: 0.501}
RGBA, NV12, I420, YUV444 = 0, 2, 4, 5
P010, YUV420P10, YUV444P10, YUV422P10 = S.P010, S.YUV420P10, S.YUV444P10, S.YUV422P10
YUVA420P, YUVA444P10, YUV422P, UYVY = 14, 15, 10, 12
PQF, HLGF, FULL, BT601, STRAIGHT = 0x800, 0x1000, 0x100, 0x200, 0x4


def rgb_of(c):
    c = np.asarray(c, np.uint32)
    return np.stack([c & 255, (c >> 8) & 255, (c >> 16) & 255], -1).astype(np.int64)


def test_the_linearisation_table_is_float64_rounded_to_float32():
    want = H.linear(np.arange(256)).astype(np.float32)
    got = np.array([S.lib().hdr_lin_c(v) for v in range(256)], np.float32)
    assert np.array_equal(got, want)


def test_the_matrix_constants_are_the_float64_derivation():
    assert np.allclose(H.M709_2020, [[0.6274, 0.3293, 0.0433], [0.0691, 0.9195, 0.0114], [0.0164, 0.0880, 0.8956]], atol=5e-5)
    src = open(os.path.join(CSRC, "export_core.h")).read()
    for name, k in (("GLB_HDR_M_PQ", 10000.0), ("GLB_HDR_M_HLG", 1000.0)):
        body = re.search(r"#define %s \{([^}]*)\}" % name, src).group(1)
        vals = np.array([float(v.strip().rstrip("f")) for v in body.replace("\\", "").split(",")], np.float32)
        assert np.array_equal(vals, (H.WHITE * H.M709_2020 / k).astype(np.float32).ravel()), name


@pytest.mark.parametrize("e", [H.PQ, H.HLG])
def test_every_colour_within_its_bound(e):
    worst = np.zeros(3)
    for k in range(0, 1 << 24, 1 << 21):
        c = np.arange(k, k + (1 << 21), dtype=np.uint32)
        y, cb, cr = S.codes(e, c)
        ep = H.rgb_prime(rgb_of(c), e)
        yf, cf = H.y_float(ep), H.cbcr_float(ep)
        worst = np.maximum(worst, [np.abs(y - yf).max(), np.abs(cb - cf[:, 0]).max(), np.abs(cr - cf[:, 1]).max()])
    assert (worst <= BOUND[e]).all(), worst


def test_the_checkpoints():
    table = {H.PQ: {0xffffff: (572.683,), 0: (64.001,), 0x010101: (66.987,), 0xff: (392.212, 438.372, 607.928)},
             H.HLG: {0xffffff: (720.893,), 0: (64.0,), 0x010101: (67.062,), 0xff: (392.107, 395.451, 714.937)}}
    for e, rows in table.items():
        for c, want in rows.items():
            ep = H.rgb_prime(rgb_of(c), e)
            got = (H.y_float(ep),) + tuple(H.cbcr_float(ep)) if len(want) == 3 else (H.y_float(ep),)
            assert np.allclose(got, want, atol=6e-4), (e, hex(c), got)
            y, cb, cr = S.codes(e, [c])
            assert y[0] == H.code(H.y_float(ep)), (e, hex(c))
    # greys: Cb = Cr = 512; black: Y 64; white 58 % PQ and 75 % HLG (BT.2408's levels)
    g = np.arange(256, dtype=np.uint32) * 0x010101
    for e in (H.PQ, H.HLG):
        y, cb, cr = S.codes(e, g)
        assert (cb == 512).all() and (cr == 512).all() and y[0] == 64 and np.all(np.diff(y.astype(int)) >= 0)
    assert S.codes(H.PQ, [0xffffff])[0][0] == 573 and S.codes(H.HLG, [0xffffff])[0][0] == 721


def test_no_channel_passes_graphics_white():
    F = H.WHITE * H.linear(rgb_of(np.arange(0, 1 << 24, 4099, dtype=np.uint32))) @ H.M709_2020.T
    assert F.max() <= H.WHITE * (1 + 1e-12) and F.min() >= 0


@pytest.mark.parametrize("e", [H.PQ, H.HLG])
def test_blocks_and_pairs_are_the_chroma_of_the_mean(e):
    rng = np.random.default_rng(22 + e)
    q = rng.integers(0, 1 << 24, (1_000_000, 4), dtype=np.uint32)
    q[::3] &= 0x3f3f3f                                                    # darker blocks, where PQ is steepest
    pairs = q[:, [0, 1, 0, 1]]
    for blk in (q, pairs):
        cb, cr = S.blocks(e, blk)
        m = H.rgb_prime(rgb_of(blk), e).mean(-2)
        cf = H.cbcr_float(m)
        assert np.abs(cb - cf[:, 0]).max() <= BOUND[e] and np.abs(cr - cf[:, 1]).max() <= BOUND[e]
    # one pixel's block of four is its own chroma, bit for bit
    c = q[:, 0]
    _, cb1, cr1 = S.codes(e, c)
    cb4, cr4 = S.blocks(e, np.repeat(c[:, None], 4, 1))
    assert np.array_equal(cb1, cb4) and np.array_equal(cr1, cr4)


def premultiplied(rng, n):
    a = rng.integers(0, 256, n)
    a[::5] = 255
    a[1::7] = 0
    c = (rng.random((n, 3)) * (a[:, None] + 1)).astype(np.int64)
    return S.pack(np.concatenate([np.minimum(c, a[:, None]), a[:, None]], -1))


@pytest.mark.parametrize("e", [H.PQ, H.HLG])
def test_the_overlay_blend_within_its_bound(e):
    rng = np.random.default_rng(7 + e)
    n = 400_000
    px = premultiplied(rng, n)
    yd = rng.integers(0, 1024, n)
    q = premultiplied(rng, 4 * n).reshape(n, 4)
    cd = rng.integers(0, 1024, (n, 2))
    y, cb, cr = S.over(e, px, yd, q, cd)
    assert np.abs(y - H.overlay_y_float(px, yd, e)).max() <= BOUND[e]
    cf = H.overlay_c_float(q, cd, e)
    assert np.abs(cb - cf[:, 0]).max() <= BOUND[e] and np.abs(cr - cf[:, 1]).max() <= BOUND[e]


@pytest.mark.parametrize("e", [H.PQ, H.HLG])
def test_opaque_pixels_give_the_export_codes_exactly_over_every_destination(e):
    rng = np.random.default_rng(3)
    colours = np.concatenate([rng.integers(0, 1 << 24, 512, dtype=np.uint32), [0, 0xffffff, 0xff, 0xff00, 0xff0000]])
    px = (colours | 0xff000000).astype(np.uint32)
    y0, cb0, cr0 = S.codes(e, colours)
    d = np.arange(1024)
    P, D = np.repeat(px, d.size), np.tile(d, px.size)
    y, _, _ = S.over(e, P, D, np.zeros((0, 4), np.uint32), np.zeros((0, 2)))
    assert np.array_equal(y, np.repeat(y0, d.size))
    q = np.repeat(px, 4).reshape(-1, 4)
    Q, CD = np.repeat(q, d.size, 0), np.stack([np.tile(d, px.size), np.tile(d[::-1], px.size)], -1)
    _, cb, cr = S.over(e, np.zeros(0, np.uint32), np.zeros(0), Q, CD)
    assert np.array_equal(cb, np.repeat(cb0, d.size)) and np.array_equal(cr, np.repeat(cr0, d.size))
    # a zero-alpha pixel whose straight colour is 0 leaves every destination code as it is
    y, cb, cr = S.over(e, np.full(d.size, 0x00000000, np.uint32) | 0x10, d, np.full((d.size, 4), 0x10, np.uint32),
                       np.stack([d, d[::-1]], -1))
    assert np.array_equal(y, d) and np.array_equal(cb, d) and np.array_equal(cr, d[::-1])


@pytest.mark.parametrize("fmt", sorted(S.HDR_FORMATS))
@pytest.mark.parametrize("e", [H.PQ, H.HLG])
def test_the_overlay_walk_keeps_zero_pixels_and_gives_opaque_pixels_the_export(e, fmt):
    """quads of the kernels' overlay functions: every sample no non-zero pixel covers keeps all 16 bits (random high
    bits included), and a picture under an opaque frame becomes exactly the HDR export of that frame"""
    rng = np.random.default_rng(fmt)
    w, h = 24, 6
    pl = S.planes(e, fmt, np.zeros((h, w), np.uint32))
    garbage = tuple(rng.integers(0, 1 << 16, p.shape).astype(np.uint16) for p in pl)
    out = S.overlay(e, fmt, np.zeros((h, w), np.uint32), garbage)
    assert all(np.array_equal(a, b) for a, b in zip(out, garbage))
    opaque = rng.integers(0, 1 << 24, (h, w), dtype=np.uint32) | 0xff000000
    out = S.overlay(e, fmt, opaque, garbage)
    want = S.planes(e, fmt, opaque)
    assert all(np.array_equal(a, b) for a, b in zip(out, want))
    # a picture half covered: the uncovered half keeps its bytes
    half = opaque.copy()
    half[:, w // 2:] = 0
    out = S.overlay(e, fmt, half, garbage)
    assert np.array_equal(out[0][:, w // 2:], garbage[0][:, w // 2:])


# ---- refusals and encodings through the host paths ---------------------------------------------------------------------
def _export(L, h, d, dst, s):
    return _call(L, lambda: L.glava_b200_export_frames(h, s.ctypes.data, 1, dst, C.byref(d), None, None))


def test_refusals_name_the_call_and_enqueue_nothing(fake):
    L = fake
    L.fake_fail_at(-1)
    h, p = L.renderer(n=1024, w=64, h=32)
    buf = L.device_buf(1 << 18)
    s = np.zeros(1, np.int32)
    dst = (C.c_void_p * 1)(buf.value)
    sc = scale_of((32, 16))
    bad = [(P010, 128, PQF | HLGF, "exclude each other"), (P010, 128, PQF | FULL, "limited range"),
           (YUV420P10, 128, HLGF | BT601, "limited range"), (YUV444P10, 128, PQF | FULL | BT601, "limited range"),
           (RGBA, 256, PQF | STRAIGHT, "no alpha"), (RGBA, 256, PQF, "not format 0"), (NV12, 64, HLGF, "not format 2"),
           (I420, 64, PQF, "not format 4"), (YUV444, 64, HLGF, "not format 5"), (YUV422P, 64, PQF, "not format 10"),
           (UYVY, 128, PQF, "not format 12"), (YUVA420P, 64, HLGF, "not format 14"), (YUVA444P10, 128, PQF, "not format 15")]
    for fmt, pitch, flags, why in bad:
        d = desc_of(fmt, pitch, flags=flags)
        rc, msg, trace, launched = _export(L, h, d, dst, s)
        assert rc != 0 and msg.startswith("glava_b200_export_frames") and why in msg and trace == "" and launched == 0, msg
        rc, msg, trace, launched = _call(L, lambda: L.glava_b200_export_scaled(h, s.ctypes.data, 1, dst, None, C.byref(d),
                                                                               C.byref(sc), None, None))
        assert rc != 0 and msg.startswith("glava_b200_export_scaled") and why in msg and launched == 0, msg
        rc, msg, trace, launched = _ladder(L, h, [0], [(d, sc)], [buf.value])
        assert rc != 0 and msg.startswith("glava_b200_export_ladder") and why in msg and launched == 0, msg
        n = C.c_size_t()
        assert L.glava_b200_export_bytes(h, C.byref(d), C.byref(n)) != 0
    # overlay_frames takes neither bit, on any format
    for fmt, pitch in ((NV12, 64), (RGBA, 256)):
        for flags in (PQF, HLGF):
            d = desc_of(fmt, pitch, flags=flags)
            rc, msg, trace, launched = _call(L, lambda: L.glava_b200_overlay_frames(h, s.ctypes.data, 1, dst, None, C.byref(d),
                                                                                    None, None))
            assert rc != 0 and msg.startswith("glava_b200_overlay_frames") and "HDR" in msg and launched == 0, msg
    # 0x400 stays an unknown flag
    rc, msg, _, launched = _export(L, h, desc_of(P010, 128, flags=0x400), dst, s)
    assert rc != 0 and "unknown flags" in msg and launched == 0
    L.glava_b200_destroy(h)
    L.cudaFree(buf)


def test_the_bits_reach_the_launchers_and_the_byte_counts_do_not_change(fake):
    L = fake
    L.fake_fail_at(-1)
    h, p = L.renderer(n=1024, w=64, h=32)
    buf = L.device_buf(1 << 18)
    s = np.zeros(1, np.int32)
    dst = (C.c_void_p * 1)(buf.value)
    sc = scale_of((32, 16))
    for fmt in S.HDR_FORMATS:
        pitch = 128
        base, base_s = C.c_size_t(), C.c_size_t()
        assert L.glava_b200_export_bytes(h, C.byref(desc_of(fmt, pitch)), C.byref(base)) == 0
        assert L.glava_b200_export_scaled_bytes(h, C.byref(desc_of(fmt, pitch)), C.byref(sc), C.byref(base_s)) == 0
        for flags, e in ((PQF, 4), (HLGF, 5)):
            d = desc_of(fmt, pitch, flags=flags)
            n, n_s = C.c_size_t(), C.c_size_t()
            assert L.glava_b200_export_bytes(h, C.byref(d), C.byref(n)) == 0 and n.value == base.value
            assert L.glava_b200_export_scaled_bytes(h, C.byref(d), C.byref(sc), C.byref(n_s)) == 0 and n_s.value == base_s.value
            rc, msg, trace, launched = _export(L, h, d, dst, s)
            assert rc == 0 and launched == 1, msg
            rc, msg, trace, launched = _call(L, lambda: L.glava_b200_export_scaled(h, s.ctypes.data, 1, dst, None, C.byref(d),
                                                                                   C.byref(sc), None, None))
            assert rc == 0 and launched == 1 and encs(L)[0] == e, msg
    # a ladder mixing HDR and SDR rungs: one launch, each rung's encoding
    bufs = [L.device_buf(1 << 16) for _ in range(4)]
    pairs = [(desc_of(P010, 128, flags=PQF), scale_of((64, 32))), (desc_of(NV12, 32), scale_of((32, 16))),
             (desc_of(YUV422P10, 64, flags=HLGF), scale_of((32, 16))), (desc_of(YUV420P10, 64, flags=FULL), scale_of((16, 8)))]
    rc, msg, trace, launched = _ladder(L, h, [0], pairs, [b.value for b in bufs])
    assert rc == 0 and launched == 1, msg
    assert encs(L)[2:6] == [4, 0, 5, 1]
    L.glava_b200_destroy(h)
    L.cudaFree(buf)
    for b in bufs:
        L.cudaFree(b)


def test_python_keywords():
    import glava_b200 as g
    from glava_b200.api import _colour_flags, _export_desc
    assert (g.EXPORT_PQ, g.EXPORT_HLG) == (0x800, 0x1000)
    assert _export_desc("p010", False, (0, 0, 0), "bt2020", transfer="pq").flags == 0x800
    assert _export_desc("yuv422p10", False, (0, 0, 0), "bt2020", transfer="hlg").flags == 0x1000
    assert _colour_flags("bt709", True) == 0x100 and _colour_flags() == 0
    for kw in (dict(matrix="bt2020"), dict(transfer="pq"), dict(matrix="bt601", transfer="hlg"),
               dict(matrix="bt2020", transfer="pq", full_range=True), dict(matrix="bt2020", transfer="gamma")):
        with pytest.raises(ValueError):
            _export_desc("p010", False, (0, 0, 0), **kw)
        with pytest.raises(ValueError):
            _colour_flags(**kw)
    # the library refuses HDR on formats without 10 bits; Python leaves that to it
    assert _export_desc("nv12", False, (0, 0, 0), "bt2020", transfer="pq").flags == 0x800
