"""The overlay onto 4:2:2 pictures through the C ABI (glava_b200_overlay_planes, DESIGN 4.18) on the host: planes_geometry
and the overlap test of YUV422P, YUV422P10 and UYVY rectangles against brute force, every refusal the three formats add
(odd width, the chroma pitch minimums, UYVY's NULL plane[1] / plane[2] and zero chroma_pitch) with nothing launched, and
the launch's arguments, through capi.cu, export.cpp and overlay_planes.cpp built against the fake runtime of
tests/fakecuda (tests/export_fake.py's stubs and tests/test_overlay_planes_core.py's recording launcher)."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from tests import export_fake, fakecuda
from tests.test_overlay_planes_core import PLANES_STUBS, _planes, brute, device_buf, renderer

I420, YUV422P, YUV422P10, UYVY = 4, 10, 11, 12
PLANES = {YUV422P: 3, YUV422P10: 3, UYVY: 1}

# planes_geometry_check on plain addresses with `n` pointers per entry (the rest NULL)
GEOMETRY = r"""
extern "C" int t_planes_geometry_n(int w, int h, int count, int n, const uintptr_t* ptrs, int format, size_t pitch, size_t cpitch,
                                   uintptr_t fb, size_t fb_bytes) {
    std::vector<glava_b200_picture> p((size_t) count);
    for (int i = 0; i < count; ++i)
        for (int k = 0; k < 3; ++k) p[i].plane[k] = k < n ? (void*) ptrs[(size_t) i * n + k] : nullptr;
    glava_b200_overlay_planes_desc d = { format, 0, pitch, cpitch };
    const uint8_t* f = (const uint8_t*) fb;
    return glb::planes_geometry_check(w, h, count, p.data(), d, &f, &fb_bytes, 1, "t_planes_geometry_n");
}
"""


@pytest.fixture(scope="module")
def fake():
    inc = fakecuda.cuda_include()
    if inc is None:
        pytest.skip("no CUDA toolkit headers")
    from glava_b200.api import Params
    out = tempfile.mkdtemp(prefix="glava_planes422_fake_")
    src, so = os.path.join(out, "planes422_fake.cpp"), os.path.join(out, "libplanes422_fake.so")
    with open(src, "w") as f:
        f.write("#include <vector>\n" + export_fake.STUBS + PLANES_STUBS + GEOMETRY)
    subprocess.run(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I", inc,
                    "-I", fakecuda.CSRC, "-x", "c++", "-include", "cuda_runtime.h", "-o", so,
                    *[os.path.join(fakecuda.CSRC, f) for f in ("capi.cu", "export.cpp", "overlay_planes.cpp", "config.cpp")],
                    os.path.join(fakecuda.HERE, "fakecuda.cpp"), src, "-lpthread", "-Wl,-Bsymbolic"], check=True)
    L = C.CDLL(so)
    shutil.rmtree(out)
    vp, i32, sz, P = C.c_void_p, C.c_int, C.c_size_t, C.POINTER(Params)
    sig = {
        "glava_b200_default_params": (i32, [P, C.c_char_p]), "glava_b200_new": (vp, [P, i32, i32]),
        "glava_b200_destroy": (None, [vp]), "glava_b200_last_error": (C.c_char_p, []), "glava_b200_set_abort_hook": (None, [vp]),
        "glava_b200_overlay_planes": (i32, [vp, vp, i32, vp, vp, vp, vp]),
        "cudaMalloc": (i32, [C.POINTER(vp), sz]), "fake_trace": (C.c_char_p, []),
        "export_fake_device": (None, [vp, sz]), "planes_fake_launches": (C.c_long, []), "planes_fake_last": (None, [vp]),
        "glava_b200_framebuffer_device": (vp, [vp]),
        "t_planes_geometry_n": (i32, [i32, i32, i32, i32, vp, i32, sz, sz, sz, sz]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = res, args
    L._quiet = C.CFUNCTYPE(None, C.c_char_p)(lambda msg: None)
    L.glava_b200_set_abort_hook(C.cast(L._quiet, vp))
    return L


def test_refusals_name_the_format_and_launch_nothing(fake):
    L = fake
    r = renderer(L)                                                        # 64 x 32
    b = device_buf(L)
    p422, p10, uyvy = (b, b + 4096, b + 8192), (b, b + 8192, b + 16384), (b, 0, 0)
    cases = [  # (streams, pictures, format, pitch, chroma_pitch, what the message names; None: taken)
        ([0], [p422], YUV422P, 64, 32, None),
        ([0], [p10], YUV422P10, 128, 64, None),
        ([0], [uyvy], UYVY, 128, 0, None),
        ([0], [p422], YUV422P, 64, 48, None),                              # a chroma pitch of its own, above w / 2
        ([0], [p422], YUV422P, 48, 32, "pitch 48 must be a multiple of 16 and at least 64"),
        ([0], [p422], YUV422P, 72, 32, "pitch 72 must be a multiple of 16"),
        ([0], [p422], YUV422P, 64, 16, "YUV422P chroma_pitch 16 must be a multiple of 16 and at least 32"),   # w / 2 bytes
        ([0], [p422], YUV422P, 64, 40, "YUV422P chroma_pitch 40"),
        ([0], [p10], YUV422P10, 112, 64, "pitch 112 must be a multiple of 16 and at least 128"),
        ([0], [p10], YUV422P10, 128, 48, "YUV422P10 chroma_pitch 48 must be a multiple of 16 and at least 64"),   # w bytes
        ([0], [uyvy], UYVY, 112, 0, "pitch 112 must be a multiple of 16 and at least 128"),              # 2 w bytes
        ([0], [uyvy], UYVY, 128, 16, "UYVY chroma_pitch 16 must be 0"),
        ([0], [uyvy], UYVY, 128, 64, "UYVY chroma_pitch 64 must be 0"),
        ([0], [(b, b + 8192, 0)], UYVY, 128, 0, "pics[0].plane[1] must be NULL: UYVY has one packed plane"),
        ([0], [(b, 0, b + 8192)], UYVY, 128, 0, "pics[0].plane[2] must be NULL: UYVY has one packed plane"),
        ([0, 1], [uyvy, (b + 8192, b + 4096, 0)], UYVY, 128, 0, "pics[1].plane[1] must be NULL"),
        ([0], [(0, 0, 0)], UYVY, 128, 0, "null"),
        ([0], [(b + 8, 0, 0)], UYVY, 128, 0, "16-byte"),
        ([0], [(b, b + 4096, 0)], YUV422P, 64, 32, "null"),                 # Cr missing
        ([0], [(b, b + 4096, 0)], YUV422P10, 128, 64, "null"),
        ([2], [uyvy], UYVY, 128, 0, "out of range"),
        ([0, 1], [uyvy, uyvy], UYVY, 128, 0, "the Y rectangle of entry 0 overlaps the Y rectangle of entry 1"),
        ([0, 1], [uyvy, (b + 128 * 31, 0, 0)], UYVY, 128, 0, "overlaps"),   # entry 1 starts in entry 0's last row
        ([0, 1], [uyvy, (b + 128 * 32, 0, 0)], UYVY, 128, 0, None),         # right after it
        ([0], [(b, b + 64 * 31, b + 8192)], YUV422P, 64, 32, "the Y rectangle of entry 0 overlaps the Cb rectangle of entry 0"),
        # 4:2:2 chroma has h rows: Cr 20 rows past Cb meets Cb's rows (it would not for I420's h / 2)
        ([0], [(b, b + 4096, b + 4096 + 32 * 20)], YUV422P, 64, 32, "the Cb rectangle of entry 0 overlaps the Cr rectangle"),
        ([0], [(b, b + 4096, b + 4096 + 32 * 32)], YUV422P, 64, 32, None),
        ([0], [(b, b + 8192, b + 8192 + 64 * 31)], YUV422P10, 128, 64, "overlaps"),
    ]
    for streams, pics, fmt, P, CP, what in cases:
        rc, msg, n = _planes(L, r, streams, pics, fmt, P, CP)
        if what is None:
            assert rc == 0 and n == 1, (fmt, msg)
            continue
        assert rc != 0 and n == 0 and "glava_b200_overlay_planes" in msg and what in msg, (fmt, what, msg)
    assert _planes(L, r, [0], [(b, b + 4096, b + 4096 + 32 * 20)], I420, 64, 32)[0] == 0   # the same planes as I420
    # odd widths are refused by name, odd heights taken
    narrow, odd = renderer(L, w=62, h=32), renderer(L, w=63, h=33)
    for fmt, pics, P, CP in ((YUV422P, p422, 64, 32), (YUV422P10, p10, 128, 64), (UYVY, uyvy, 128, 0)):
        name = {YUV422P: "YUV422P", YUV422P10: "YUV422P10", UYVY: "UYVY"}[fmt]
        rc, msg, n = _planes(L, odd, [0], [pics], fmt, P, CP)
        assert rc != 0 and n == 0 and f"{name} needs an even width, the frame is 63x33" in msg, msg
        rc, msg, n = _planes(L, narrow, [0], [pics], fmt, P, CP)
        assert rc == 0 and n == 1, (fmt, msg)                              # 62 wide: w % 4 == 2
        tall = renderer(L, w=64, h=33)
        rc, msg, n = _planes(L, tall, [0], [pics], fmt, P, CP)
        assert rc == 0 and n == 1, (fmt, msg)                              # any height
        L.glava_b200_destroy(tall)
    # a plane rectangle that meets the framebuffer
    fb = L.glava_b200_framebuffer_device(r)
    L.export_fake_device(fb, 64 * 32 * 4)
    rc, msg, n = _planes(L, r, [0], [(fb + 256, 0, 0)], UYVY, 128, 0)
    assert rc != 0 and n == 0 and "the Y rectangle of entry 0 overlaps the renderer's framebuffer" in msg, msg
    rc, msg, n = _planes(L, r, [0], [(b, fb + 256, b + 8192)], YUV422P, 64, 32)
    assert rc != 0 and n == 0 and "the Cb rectangle of entry 0 overlaps the renderer's framebuffer" in msg, msg
    for h in (r, narrow, odd):
        L.glava_b200_destroy(h)


def test_the_launch_gets_format_encoding_and_pitches(fake):
    L = fake
    r = renderer(L, w=96, h=47)
    b = device_buf(L)
    last = np.zeros(9, np.int64)
    for fmt, pics, P, CP in ((YUV422P, (b, b + 8192, b + 16384), 96, 48), (YUV422P10, (b, b + 16384, b + 32768), 192, 112),
                             (UYVY, (b, 0, 0), 192, 0)):
        for flags, e in ((0, 0), (0x100, 1), (0x200, 2), (0x300, 3)):
            rc, msg, n = _planes(L, r, [1], [pics], fmt, P, CP, flags)
            assert rc == 0 and n == 1, msg
            L.planes_fake_last(last.ctypes.data)
            assert list(last) == [1, 0, 1, fmt, e, P, CP, 96, 47], (fmt, e, list(last))
    L.glava_b200_destroy(r)


def test_planes_geometry_and_overlap_against_brute_force(fake):
    """random 4:2:2 lists: planes_geometry_check refuses exactly the lists whose plane rectangles share a byte (Y rows of w,
    2w or 2w bytes; chroma h rows of w / 2 or w bytes at their own pitch; UYVY one plane)"""
    L = fake
    rng = np.random.default_rng(5)
    w, h = 32, 7
    for fmt in (YUV422P, YUV422P10, UYVY):
        n = PLANES[fmt]
        B = w if fmt == YUV422P else 2 * w
        CB = w // 2 if fmt == YUV422P else w
        for trial in range(200):
            P = B + 16 * int(rng.integers(0, 3))
            CP = 0 if fmt == UYVY else CB + (-CB) % 16 + 16 * int(rng.integers(0, 3))
            count = int(rng.integers(1, 4))
            ptrs = (1 << 20) + 16 * rng.integers(0, 96, count * n)
            rects = [(int(ptrs[i * n + k]), h, P if k == 0 else CP, B if k == 0 else CB) for i in range(count) for k in range(n)]
            got = L.t_planes_geometry_n(w, h, count, n, np.ascontiguousarray(ptrs, np.uint64).ctypes.data, fmt, P, CP, 1 << 30, 64)
            assert (got != 0) == brute(rects), (fmt, trial, rects)
        # a tight mosaic passes: 4 x 4 tiles side by side, chroma planes of their own
        cols = 4
        P, CP = B * cols, 0 if fmt == UYVY else CB * cols + (-(CB * cols)) % 16
        ptrs = []
        for t in range(16):
            ty, tx = divmod(t, cols)
            ptrs.append((1 << 24) + ty * h * P + tx * B)
            for k in range(1, n):
                ptrs.append((1 << 26) * k + ty * h * CP + tx * CB)
        assert all(v % 16 == 0 for v in ptrs), fmt
        assert L.t_planes_geometry_n(w, h, 16, n, np.asarray(ptrs, np.uint64).ctypes.data, fmt, P, CP, 1 << 30, 64) == 0, fmt
        # the geometry's own refusals: odd width, the chroma pitch minimums, UYVY's chroma pitch
        one = np.asarray([1 << 20, 1 << 22, 1 << 23][:n], np.uint64)
        assert L.t_planes_geometry_n(w - 1, h, 1, n, one.ctypes.data, fmt, P, CP, 1 << 30, 64) != 0, fmt
        if fmt == UYVY:
            assert L.t_planes_geometry_n(w, h, 1, n, one.ctypes.data, fmt, P, 16, 1 << 30, 64) != 0
        else:
            assert L.t_planes_geometry_n(w, h, 1, n, one.ctypes.data, fmt, P, CB - 16 if CB > 16 else 0, 1 << 30, 64) != 0, fmt
        assert L.t_planes_geometry_n(w, h, 1, n, one.ctypes.data, fmt, B - 16, CP, 1 << 30, 64) != 0, fmt
