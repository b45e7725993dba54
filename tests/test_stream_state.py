"""CPU tier of the per-stream state calls (glava_b200_stream_state_bytes, stream_state_core.h).

The blob size follows the documented formula for every pipeline, averaging depth, module and setbufsize, and the host
build of the layout header moves every average-ring frame to the same age whatever the source and destination cursors
are: checked against a numpy restatement of the blob layout (DESIGN.md §4.8)."""
import ctypes as C
import os
import subprocess
import types

import numpy as np
import pytest

import glava_b200 as g

HERE = os.path.dirname(os.path.abspath(__file__))


class StateLayout(C.Structure):
    """stream_state_core.h StateLayout"""
    _fields_ = [("n", C.c_int), ("n_in", C.c_int), ("F", C.c_int), ("esz", C.c_int), ("chans", C.c_int)]


class StateArrays:
    """host copies of a renderer's per-stream state arrays, laid out as on the device (stream_state_core.h StatePtrs);
    random bit patterns when `rng` is given (the kernels move bytes), else zeros"""

    def __init__(self, L, batch, rng=None):
        dt = np.uint16 if L.esz == 2 else np.uint32
        shapes = [((batch * 2, L.n), dt), ((batch * 2, L.F, L.n), dt), ((batch * 2, L.n), np.uint32),
                  ((batch * 2, L.n), np.uint16), ((batch * 2, L.n), np.uint16), ((batch, L.n_in), np.uint32),
                  ((batch, L.n_in), np.uint32)]
        self.a = [np.zeros(s, d) if rng is None else rng.integers(0, np.iinfo(d).max, size=s, dtype=d) for s, d in shapes]
        self.gravity, self.ring, self.spec, self.tex, self.av, self.fifo_l, self.fifo_r = self.a

    def ptrs(self):
        return (C.c_void_p * 7)(*[x.ctypes.data for x in self.a])


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    """host build of stream_state_core.h (tests/emul/stream_state_emul.cpp), compiled into a temporary directory"""
    so = str(tmp_path_factory.mktemp("state_emul") / "libstate_emul.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul", "stream_state_emul.cpp")],
                   check=True)
    L = C.CDLL(so)
    vp = C.c_void_p
    L.emul_state_segment_bytes.argtypes = [vp]
    L.emul_state_segment_bytes.restype = C.c_size_t
    L.emul_state_pack.argtypes = [vp, vp, C.c_int, C.c_uint32, vp]
    L.emul_state_unpack.argtypes = [vp, vp, C.c_int, C.c_uint32, vp]

    def state_pack(lay, arrays, stream, cursor):
        blob = np.zeros(L.emul_state_segment_bytes(C.byref(lay)), np.uint8)
        L.emul_state_pack(C.byref(lay), arrays.ptrs(), stream, cursor, blob.ctypes.data)
        return blob

    def state_unpack(lay, arrays, stream, cursor, blob):
        L.emul_state_unpack(C.byref(lay), arrays.ptrs(), stream, cursor, None if blob is None else blob.ctypes.data)

    return types.SimpleNamespace(StateLayout=StateLayout, StateArrays=StateArrays, state_pack=state_pack,
                                 state_unpack=state_unpack, lib=L)


def _formula(n_in, bufscale, F, esz, chans):
    n = n_in // bufscale
    return 4096 + chans * ((1 + F) * n * esz + 4 * n + 2 * n + 2 * n + 4 * n_in)


@pytest.mark.parametrize("n", [256, 512, 1024, 2048, 4096, 8192, 16384])
def test_state_bytes_formula_at_every_size(built, n):
    assert g.STATE_HEADER_BYTES == 4096
    for accel, esz in ((1, 2), (0, 4)):
        for F in (1, 3, 5, 7):
            p = g.default_params("bars", n=n, accel_fft=accel, avg_frames=F)
            assert g.stream_state_bytes(p) == _formula(n, 1, F, esz, 2), (n, accel, F)
    assert g.stream_state_bytes(g.default_params("wave", n=n)) == _formula(n, 1, g.default_params("wave").avg_frames,
                                                                          2 if g.default_params("wave").accel_fft else 4, 1)
    if n >= 512:
        p = g.default_params("bars", n=n, bufscale=2)
        assert g.stream_state_bytes(p) == _formula(n, 2, p.avg_frames, 2, 2)


def test_state_bytes_headline_and_smooth_after_fft(built):
    p = g.default_params("bars", n=4096, avg_frames=5)
    assert p.accel_fft == 1
    assert g.stream_state_bytes(p) - 4096 == 192 * 1024                       # 192 KiB of segments per stream
    q = g.default_params("bars", n=4096, avg_frames=5, transform_smooth=1)   # "smooth" after "fft": pipeline A's float state
    assert g.stream_state_bytes(q) == _formula(4096, 1, 5, 4, 2)
    q = g.default_params("bars", n=4096, avg_frames=5, transform_smooth=2)   # before "fft": the R16 passes stay
    assert g.stream_state_bytes(q) == _formula(4096, 1, 5, 2, 2)


def test_state_bytes_reject_interpolation(built):
    p = g.default_params("wave", n=512, w=64, h=32, interpolate=1, fr=400.0)
    with pytest.raises(g.GlavaError, match="interpolation"):
        g.stream_state_bytes(p)
    assert g.lib().glava_b200_stream_state_bytes(p) == 0


def _restated_blob(L, A, s, cursor):
    """numpy restatement of the segments of stream s: per channel gravity, ring by age (newest first), spec, texture,
    pre-smoothing texture, FIFO ring"""
    parts = []
    for ch in range(L.chans):
        pl = 2 * s + ch
        parts.append(A.gravity[pl])
        parts += [A.ring[pl, (cursor - 1 - age) % L.F] for age in range(L.F)]
        parts += [A.spec[pl], A.tex[pl], A.av[pl], (A.fifo_l, A.fifo_r)[ch][s]]
    return np.concatenate([x.view(np.uint8) for x in parts])


def _layout(emul, F, esz=2, chans=2):
    return emul.StateLayout(n=32, n_in=64, F=F, esz=esz, chans=chans)


def test_pack_unpack_keeps_every_frame_at_its_age(emul):
    rng = np.random.default_rng(1)
    for F in range(1, 17):
        L = _layout(emul, F)
        for cs in range(F):
            src = emul.StateArrays(L, 3, rng)
            blob = emul.state_pack(L, src, 2, cs)
            assert np.array_equal(blob, _restated_blob(L, src, 2, cs)), (F, cs)
            for cd in range(F):
                dst = emul.StateArrays(L, 2)
                emul.state_unpack(L, dst, 1, cd, blob)
                for ch in range(2):
                    ps, pd = 4 + ch, 2 + ch
                    for age in range(F):
                        assert np.array_equal(dst.ring[pd, (cd - 1 - age) % F], src.ring[ps, (cs - 1 - age) % F]), (F, cs, cd, age)
                    for a, b in ((dst.gravity, src.gravity), (dst.spec, src.spec), (dst.tex, src.tex), (dst.av, src.av)):
                        assert np.array_equal(a[pd], b[ps])
                assert np.array_equal(dst.fifo_l[1], src.fifo_l[2]) and np.array_equal(dst.fifo_r[1], src.fifo_r[2])
                for x in dst.a:                                             # stream 0 untouched
                    assert not x[:2 if x.shape[0] == 4 else 1].any()
                assert np.array_equal(emul.state_pack(L, dst, 1, cd), blob)


@pytest.mark.parametrize("esz,chans", [(4, 2), (2, 1), (4, 1)])
def test_pack_unpack_other_layouts_and_reset(emul, esz, chans):
    rng = np.random.default_rng(esz * 10 + chans)
    for F in (1, 2, 5, 7, 16):
        L = _layout(emul, F, esz, chans)
        for cs, cd in ((0, F - 1), (F - 1, 0), (F // 2, F // 3)):
            src = emul.StateArrays(L, 2, rng)
            blob = emul.state_pack(L, src, 1, cs)
            assert np.array_equal(blob, _restated_blob(L, src, 1, cs)), (F, cs)
            dst = emul.StateArrays(L, 2, rng)
            keep = [x.copy() for x in dst.a]
            emul.state_unpack(L, dst, 0, cd, blob)
            assert np.array_equal(emul.state_pack(L, dst, 0, cd), blob)
            for x, k in zip(dst.a, keep):                                   # stream 1 untouched; wave: channel 1 untouched
                rows = [2, 3] if x.shape[0] == 4 else [1]
                if chans == 1 and x.shape[0] == 4:
                    rows.append(1)
                assert np.array_equal(x[rows], k[rows])
            if chans == 1:
                assert np.array_equal(dst.fifo_r, keep[6])
            emul.state_unpack(L, dst, 0, cd, None)                          # reset: the same segments, zeroed
            assert not emul.state_pack(L, dst, 0, cd).any()
