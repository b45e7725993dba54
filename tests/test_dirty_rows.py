"""Dirty-row marks of the bars / graph / wave rasters (raster_core.h dirty_pack / dirty_zero_span), on the host build.

A band's mark says which rows [lo, hi) may be non-zero in memory; a kernel stores a zero row only where it lies inside
that interval.  Checked exhaustively for small band heights against a per-row model, and as a sequence of frames: the
memory the policy leaves behind must equal every new frame."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest


SHIM = r"""
#include "raster_core.h"
extern "C" uint32_t t_pack(int lo, int hi) { return glb::dirty_pack(lo, hi); }
extern "C" void t_span(uint32_t old, int za, int zb, int* a, int* b) { glb::dirty_zero_span(old, za, zb, a, b); }
"""


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("dirty_rows")
    src, so = d / "shim.cpp", d / "shim.so"
    src.write_text(SHIM)
    csrc = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "glava_b200", "csrc")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I", csrc,
                    "-o", str(so), str(src)], check=True)
    L = C.CDLL(str(so))
    L.t_pack.restype = C.c_uint32
    L.t_pack.argtypes = [C.c_int, C.c_int]
    L.t_span.argtypes = [C.c_uint32, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    return L


def _span(L, old, za, zb):
    a, b = C.c_int(), C.c_int()
    L.t_span(old, za, zb, C.byref(a), C.byref(b))
    return a.value, b.value


def _intervals(y0, y1):
    """every interval [lo, hi) inside [y0, y1), the empty one once"""
    yield y0, y0
    for lo in range(y0, y1):
        for hi in range(lo + 1, y1 + 1):
            yield lo, hi


@pytest.mark.parametrize("h", range(1, 11))
def test_zero_span_matches_the_per_row_model(shim, h):
    """for a band [y0, y1) of every position in a frame of h rows, every old mark and every zero range: the rows stored are
    exactly the zero rows inside the old dirty interval"""
    for y0 in range(h):
        for y1 in range(y0 + 1, h + 1):
            for lo, hi in _intervals(y0, y1):
                old = shim.t_pack(lo, hi)
                for za in range(y0, y1 + 1):
                    for zb in range(za, y1 + 1):
                        a, b = _span(shim, old, za, zb)
                        want = [y for y in range(za, zb) if lo <= y < hi]
                        assert y0 <= a <= b <= y1 or a == b, (h, y0, y1, lo, hi, za, zb, a, b)
                        assert list(range(a, b)) == want, (h, y0, y1, lo, hi, za, zb, a, b)
            # no valid marks: the whole band counts as dirty, every zero row is stored
            full = shim.t_pack(y0, y1)
            for za in range(y0, y1 + 1):
                for zb in range(za, y1 + 1):
                    assert _span(shim, full, za, zb) == (za, zb)


def test_pack_fields_cover_the_largest_frame(shim):
    """rows up to 16384 (validate_params) fit both 16-bit fields; an empty interval packs to 0, the freshly zeroed word"""
    for lo, hi in ((0, 16384), (16383, 16384), (4095, 8191), (1, 2)):
        m = shim.t_pack(lo, hi)
        assert (m & 0xFFFF, m >> 16) == (lo, hi)
    for lo, hi in ((0, 0), (7, 7), (9, 3)):
        assert shim.t_pack(lo, hi) == 0
    assert _span(shim, 0, 0, 16384)[0] == _span(shim, 0, 0, 16384)[1]


@pytest.mark.parametrize("layout", ["bars", "flip", "wave"])
def test_frame_sequences_leave_memory_equal_to_each_frame(shim, layout):
    """A band of h rows through random frames that rise, fall and go silent.  Each frame is non-zero only in some rows;
    the kernel stores its content rows (bars: the rows below the tallest bar, FLIP: above, wave: around the line), the
    zero rows the old mark says may be dirty, and records the content rows.  Memory must equal the frame every time."""
    rng = np.random.default_rng(7)
    for h in (1, 2, 5, 17, 64):
        y0, y1 = 0, h
        mem = np.zeros(h, np.int64)              # the framebuffer starts zeroed, the marks empty
        mark = 0
        for step in range(200):
            kind = rng.integers(0, 4)
            n = h if kind == 0 else (0 if kind == 1 else int(rng.integers(0, h + 1)))
            if layout == "bars":
                c0, c1 = 0, n
            elif layout == "flip":
                c0, c1 = h - n, h
            else:
                c0 = int(rng.integers(0, h + 1)); c1 = min(h, c0 + n)
            frame = np.zeros(h, np.int64)
            frame[c0:c1] = rng.integers(0, 3, c1 - c0)            # content rows may hold zeros too
            for za, zb in ((y0, c0), (c1, y1)):
                a, b = _span(shim, mark, za, zb)
                mem[a:b] = 0
            mem[c0:c1] = frame[c0:c1]
            mark = shim.t_pack(c0, c1)
            assert np.array_equal(mem, frame), (layout, h, step)
            if step % 50 == 49:                                   # something else writes the band: invalid marks
                mem[:] = rng.integers(0, 3, h)
                frame2 = np.zeros(h, np.int64)
                a, b = _span(shim, shim.t_pack(y0, y1), y0, y1)   # invalid mode stores every zero row
                mem[a:b] = 0
                mark = 0
                assert np.array_equal(mem, frame2)
