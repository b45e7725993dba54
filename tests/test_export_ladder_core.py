"""Encoder ladder (DESIGN 4.13) on the host: the schedule of ladder_plan.h through a g++ shim (every unit of every rung once,
each rung's units exactly its standalone kernel's items, in non-decreasing order of the first source row they read), and
the refusals and enqueued work of glava_b200_export_ladder through capi.cu, export.cpp and export_ladder.cpp built against
the fake runtime of tests/fakecuda: tests/export_fake.py's stubs plus a ladder launcher that counts its calls and records its
LadderArgs."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from tests import export_fake, fakecuda
from tests.export_fake import desc_of
from tests.test_export_core import BGRA, CSRC, NV12, RGBA

SHIM = r"""
#include "ladder_plan.h"
using namespace glb;
// g: per rung src_x, src_y, src_w, src_h, out_w, out_h (defaults applied), nv12
static LadderGeom geom_of(int w, int h, const int* g) {
    LadderGeom q = { g[0], g[1], g[2], g[3], g[4], g[5], false, g[6] != 0 };
    q.whole = ladder_whole(w, h, q);
    return q;
}
extern "C" int t_whole(int w, int h, const int* g) { return geom_of(w, h, g).whole; }
extern "C" size_t t_schedule(int w, int h, const int* g, int n, uint64_t* out, size_t cap) {
    LadderGeom geom[GLAVA_B200_LADDER_MAX];
    for (int j = 0; j < n; ++j) geom[j] = geom_of(w, h, g + 7 * j);
    const std::vector<uint64_t> s = ladder_schedule(w, h, geom, n);
    for (size_t i = 0; i < s.size() && i < cap; ++i) out[i] = s[i];
    return s.size();
}
"""


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("export_ladder_core")
    src, so = d / "shim.cpp", d / "shim.so"
    src.write_text(SHIM)
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I", CSRC,
                    "-I", CSRC + "/../../include", "-include", "cstdint", "-include", "cstddef", "-o", str(so), str(src)], check=True)
    L = C.CDLL(str(so))
    L.t_whole.argtypes = [C.c_int, C.c_int, C.c_void_p]
    L.t_schedule.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]
    L.t_schedule.restype = C.c_size_t
    return L


def geom(w, h, crop, size, nv12):
    x, y, cw, ch = crop or (0, 0, w, h)
    return [x, y, cw, ch, size[0], size[1], int(nv12)]


def schedule(L, w, h, rungs):
    g = np.asarray([v for r in rungs for v in geom(w, h, *r)], np.int32)
    n = L.t_schedule(w, h, g.ctypes.data, len(rungs), None, 0)
    out = np.zeros(max(n, 1), np.uint64)
    assert L.t_schedule(w, h, g.ctypes.data, len(rungs), out.ctypes.data, n) == n
    whole = [bool(L.t_whole(w, h, np.asarray(geom(w, h, *r), np.int32).ctypes.data)) for r in rungs]
    return out[:n], whole


def decode(u):
    u = int(u)
    return u >> 56, (u >> 28) & 0xFFFFFFF, u & 0xFFFFFFF


def first_row(w, h, rung, whole, row):
    """the top-down index of the first source row a unit reads: export_span(Y).first = floor(Y src_h / out_h)"""
    crop, size, nv12 = rung
    if whole:
        return 2 * row
    y, ch = (crop or (0, 0, w, h))[1], (crop or (0, 0, w, h))[3]
    Y = 2 * row if nv12 else row
    return y + Y * ch // size[1]


LADDERS = [  # (w, h, [(crop, size, nv12)])
    (1920, 1080, [(None, (1920, 1080), True), (None, (1280, 720), True), (None, (640, 360), True), (None, (480, 270), True)]),
    (97, 63, [(None, (97, 63), False), (None, (13, 7), False), ((5, 3, 90, 58), (30, 29), False)]),
    (130, 64, [(None, (130, 64), True), ((2, 4, 64, 32), (64, 32), True), (None, (86, 42), True), (None, (7, 5), False)]),
    (300, 33, [((100, 2, 60, 30), (12, 10), True), (None, (300, 33), False), ((0, 0, 300, 33), (299, 33), False)]),
    (1080, 6, [(None, (1, 2), True), (None, (1080, 6), True), (None, (1080, 3), False), (None, (540, 6), False)] * 2),
    (64, 32, [((0, 0, 32, 32), (32, 32), False), ((32, 0, 32, 32), (32, 32), True)]),
]


@pytest.mark.parametrize("w,h,rungs", LADDERS)
def test_schedule_holds_every_item_of_every_rung_once_in_row_order(shim, w, h, rungs):
    sched, whole = schedule(shim, w, h, rungs)
    units = [decode(u) for u in sched]
    assert len(set(units)) == len(units), "a unit listed twice"
    for j, (crop, size, nv12) in enumerate(rungs):
        assert whole[j] == (crop in (None, (0, 0, w, h)) and size == (w, h)), j
        got = {(r, c) for q, r, c in units if q == j}
        if whole[j]:                                                   # export_kernel: row pairs x 128-pixel strips
            want = {(r, c) for r in range((h + 1) // 2) for c in range((w + 127) // 128)}
        else:                                                          # export_scaled_kernel: rows (pairs) x 32-column runs
            want = {(r, c) for r in range(size[1] // 2 if nv12 else size[1]) for c in range((size[0] + 31) // 32)}
        assert got == want, j
    keys = [(first_row(w, h, rungs[q], whole[q], r), q) for q, r, _ in units]
    assert keys == sorted(keys), "not in (first source row, rung) order"


def test_a_cropped_one_to_one_rung_is_a_scaled_rung(shim):
    sched, whole = schedule(shim, 64, 32, [((0, 0, 32, 32), (32, 32), False), (None, (64, 32), False), ((0, 0, 64, 32), (64, 32), True)])
    assert whole == [False, True, True]
    assert {decode(u)[2] for u in sched if decode(u)[0] == 0} == {0}     # one run of 32 columns, not strips
    assert sum(1 for u in sched if decode(u)[0] == 0) == 32            # one unit per output row


# ---- refusals and enqueued work through the fake runtime -----------------------------------------------------------------
LADDER_STUBS = r"""
static glb::LadderArgs g_ladder;
static long g_ladder_launches = 0;
extern "C" long ladder_fake_launches(void) { return g_ladder_launches; }
// the last ladder's common fields, then per rung: format, over, whole, pitch, crop (4), out size (2), div_mul low / high
// 32 bits, div_shift, bg
extern "C" void ladder_fake_last(long long* out) {
    out[0] = g_ladder.count; out[1] = g_ladder.nrungs; out[2] = g_ladder.units; out[3] = g_ladder.native;
    for (int j = 0; j < GLAVA_B200_LADDER_MAX; ++j) {
        const glb::LadderRung& g = g_ladder.rung[j];
        long long* o = out + 4 + 14 * j;
        o[0] = g.format; o[1] = g.over; o[2] = g.whole; o[3] = (long long) g.pitch; o[4] = g.src_x; o[5] = g.src_y; o[6] = g.src_w;
        o[7] = g.src_h; o[8] = g.out_w; o[9] = g.out_h; o[10] = (long long) (g.div_mul & 0xffffffffu); o[11] = (long long) (g.div_mul >> 32);
        o[12] = g.div_shift; o[13] = g.bg;
    }
}
namespace glb {
int launch_export_ladder(const LadderArgs& a, void*) {
    ++g_launches; ++g_ladder_launches; g_ladder = a;
    return a.fb && a.list && a.sched && a.count > 0 && a.units > 0 && a.nrungs > 0 && (!a.marks || a.mark_rows > 0)
               ? 0 : fail(GLAVA_B200_EINVAL, "ladder launch: bad arguments");
}
}
"""


@pytest.fixture(scope="module")
def fake():
    """export_fake.lib()'s library with export_ladder.cpp and the ladder launcher added"""
    inc = fakecuda.cuda_include()
    if inc is None:
        pytest.skip("no CUDA toolkit headers")
    from glava_b200.api import Params
    out = tempfile.mkdtemp(prefix="glava_ladder_fake_")
    src, so = os.path.join(out, "ladder_fake.cpp"), os.path.join(out, "libladder_fake.so")
    with open(src, "w") as f:
        f.write(export_fake.STUBS + LADDER_STUBS)
    subprocess.run(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I", inc,
                    "-I", fakecuda.CSRC, "-x", "c++", "-include", "cuda_runtime.h", "-o", so,
                    *[os.path.join(fakecuda.CSRC, f) for f in ("capi.cu", "export.cpp", "export_ladder.cpp", "config.cpp")],
                    os.path.join(fakecuda.HERE, "fakecuda.cpp"), src, "-lpthread", "-Wl,-Bsymbolic"], check=True)
    L = C.CDLL(so)
    shutil.rmtree(out)                                                # stays mapped
    vp, i32, P = C.c_void_p, C.c_int, C.POINTER(Params)
    sig = {
        "glava_b200_default_params": (i32, [P, C.c_char_p]), "glava_b200_new": (vp, [P, i32, i32]),
        "glava_b200_destroy": (None, [vp]), "glava_b200_update": (i32, [vp, vp, vp, C.c_size_t, i32]),
        "glava_b200_last_error": (C.c_char_p, []), "glava_b200_set_abort_hook": (None, [vp]),
        "glava_b200_export_ladder": (i32, [vp, vp, i32, vp, i32, vp, vp, vp, vp]),
        "cudaMalloc": (i32, [C.POINTER(vp), C.c_size_t]), "cudaFree": (i32, [vp]), "cudaEventCreate": (i32, [C.POINTER(vp)]),
        "cudaEventDestroy": (i32, [vp]), "fake_trace": (C.c_char_p, []), "fake_fail_at": (None, [C.c_long]),
        "fake_live": (C.c_long, [i32]), "export_fake_device": (None, [vp, C.c_size_t]), "export_fake_forget": (None, [vp]),
        "export_fake_launches": (C.c_long, []), "ladder_fake_launches": (C.c_long, []), "ladder_fake_last": (None, [vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = res, args
    L._quiet = C.CFUNCTYPE(None, C.c_char_p)(lambda msg: None)
    L.glava_b200_set_abort_hook(C.cast(L._quiet, vp))

    def renderer(module="bars", batch=2, **kw):
        p = Params()
        assert L.glava_b200_default_params(C.byref(p), module.encode()) == 0
        for k, v in kw.items():
            setattr(p, k, v)
        h = L.glava_b200_new(C.byref(p), batch, 0)
        assert h, L.glava_b200_last_error()
        return C.c_void_p(h), p

    def device_buf(nbytes=1 << 16):
        b = C.c_void_p()
        assert L.cudaMalloc(C.byref(b), nbytes) == 0
        L.export_fake_device(b, nbytes)
        return b

    free = L.cudaFree

    def cuda_free(p):
        L.export_fake_forget(p)
        return free(p)

    L.renderer, L.device_buf, L.cudaFree = renderer, device_buf, cuda_free
    return L


def scale_of(out, crop=(0, 0, 0, 0)):
    from glava_b200.api import ExportScale
    s = ExportScale()
    s.src_x, s.src_y, s.src_w, s.src_h = crop
    s.out_w, s.out_h = out
    return s


def rungs_of(pairs):
    from glava_b200.api import ExportRung
    arr = (ExportRung * max(len(pairs), 1))()
    for j, (d, s) in enumerate(pairs):
        arr[j].desc, arr[j].scale = d, s
    return arr


def _ladder(L, h, streams, pairs, dsts, uvs=None, nrungs=None, null_rungs=False, after=None, done=None):
    s = np.asarray(streams, np.int32)
    arr = (C.c_void_p * max(len(dsts), 1))(*dsts)
    uv = None if uvs is None else (C.c_void_p * max(len(uvs), 1))(*uvs)
    n0 = L.export_fake_launches()
    L.fake_trace_begin()
    rc = L.glava_b200_export_ladder(h, s.ctypes.data, len(streams), None if null_rungs else rungs_of(pairs),
                                    len(pairs) if nrungs is None else nrungs, arr, uv, after, done)
    L.fake_trace_end()
    return rc, L.glava_b200_last_error().decode(), L.fake_trace().decode(), L.export_fake_launches() - n0


def memcpys(trace):
    """the byte counts of the host-to-device copies of a trace"""
    return [int(x.split()[-2]) for x in trace.splitlines() if x.split()[0] == "memcpy"]


def recip(d):
    if d < 2:
        return 0, 0
    s = (d - 1).bit_length() - 1
    return -(-(1 << (64 + s)) // d), s


def test_refusals_name_the_rung_and_enqueue_nothing(fake):
    L = fake
    L.fake_fail_at(-1)
    h, p = L.renderer(n=1024, w=64, h=32)
    buf, buf2 = L.device_buf(), L.device_buf()
    host = np.zeros(1 << 16, np.uint8)
    aligned_host = host.ctypes.data + (-host.ctypes.data) % 16
    good = [(desc_of(NV12, 64), scale_of((64, 32))), (desc_of(RGBA, 64), scale_of((16, 8), (4, 2, 40, 20))),
            (desc_of(BGRA, 16, flags=1), scale_of((4, 2)))]
    two = [buf.value, buf2.value, buf2.value, buf.value, buf2.value, buf.value]     # [2 entries][3 rungs]
    rc, msg, trace, launched = _ladder(L, h, [0, 1], good, two)
    assert rc == 0 and launched == 1, msg
    ok = scale_of((16, 8), (4, 2, 40, 20))
    bad_rung = [  # (desc, scale, what): every refusal of glava_b200_export_scaled's descriptor and rectangle
        (desc_of(3, 64), ok, "unknown format"),
        (desc_of(RGBA, 64, flags=2), ok, "unknown flags"),
        (desc_of(RGBA, 48), ok, "pitch"),
        (desc_of(RGBA, 72), ok, "pitch"),
        (desc_of(NV12, 16, uv=8), ok, "uv_offset"),
        (desc_of(NV12, 16, uv=16 * 4), ok, "uv_offset"),
        (desc_of(RGBA, 64), scale_of((16, 8), (30, 0, 40, 20)), "leaves"),
        (desc_of(RGBA, 64), scale_of((16, 8), (-1, 0, 40, 20)), "leaves"),
        (desc_of(RGBA, 64), scale_of((16, 8), (0, 0, 40, 0)), "empty"),
        (desc_of(RGBA, 256), scale_of((41, 8), (0, 0, 40, 20)), "upscaling"),
        (desc_of(RGBA, 256), scale_of((0, 8)), "upscaling"),
        (desc_of(NV12, 16), scale_of((15, 8)), "even"),
    ]
    for j in (0, 2):
        for d, sc, what in bad_rung:
            pairs = list(good)
            pairs[j] = (d, sc)
            rc, msg, trace, launched = _ladder(L, h, [0, 1], pairs, two)
            assert rc != 0 and f"glava_b200_export_ladder: rung {j}:" in msg and what in msg, (j, what, msg)
            assert trace == "" and launched == 0, (j, what, trace)
        # destinations of rung j: entry 1's pointer at index 3 + j
        for bad, what in ((buf.value + 8, "aligned"), (None, "null"), (aligned_host, "not device memory")):
            dsts = list(two)
            dsts[3 + j] = bad
            rc, msg, trace, launched = _ladder(L, h, [0, 1], good, dsts)
            assert rc != 0 and f"glava_b200_export_ladder: rung {j}:" in msg and what in msg and "dst[1]" in msg, (j, what, msg)
            assert trace == "" and launched == 0
    uvs = [buf2.value, None, None, buf2.value, None, None]              # chroma of the NV12 rung only
    rc, msg, trace, launched = _ladder(L, h, [0, 1], good, two, uvs)
    assert rc == 0 and launched == 1, msg
    cases = [
        (dict(uvs=[buf2.value, None, buf2.value, buf2.value, None, None]), "rung 2: dst_uv[2] is for NV12 only"),
        (dict(uvs=[buf2.value, buf2.value, None, buf2.value, None, None]), "rung 1: dst_uv[1] is for NV12 only"),
        (dict(uvs=[buf2.value, None, None, buf2.value + 8, None, None]), "rung 0: dst_uv[1]"),
        (dict(uvs=[buf2.value, None, None, None, None, None]), "rung 0: dst_uv[1]"),
        (dict(nrungs=0), "nrungs 0"),
        (dict(nrungs=9), "nrungs 9"),
        (dict(null_rungs=True), "null rungs"),
    ]
    for kw, what in cases:
        rc, msg, trace, launched = _ladder(L, h, [0, 1], good, two, **kw)
        assert rc != 0 and "glava_b200_export_ladder" in msg and what in msg, (what, msg)
        assert trace == "" and launched == 0, (what, trace)
    rc, msg, trace, launched = _ladder(L, h, [0, 2], good, two)
    assert rc != 0 and "rung 0: stream 2 out of range" in msg and trace == "" and launched == 0, msg
    rc, msg, trace, launched = _ladder(L, h, [], good, [])
    assert rc != 0 and "count 0" in msg and trace == "" and launched == 0, msg
    L.glava_b200_destroy(h)
    assert L.cudaFree(buf) == 0 and L.cudaFree(buf2) == 0


def test_one_list_copy_one_launch_and_the_schedule_uploaded_per_geometry(fake):
    L = fake
    L.fake_fail_at(-1)
    live0 = [L.fake_live(k) for k in range(4)]
    h, p = L.renderer(n=1024, w=200, h=100)
    buf = L.device_buf(1 << 20)
    a, d = C.c_void_p(), C.c_void_p()
    assert L.cudaEventCreate(C.byref(a)) == 0 and L.cudaEventCreate(C.byref(d)) == 0
    pcm = np.zeros((2, 1024), np.float32)
    assert L.glava_b200_update(h, pcm.ctypes.data, pcm.ctypes.data, 1024, 1) == 0
    ladder_a = [(desc_of(NV12, 208), scale_of((200, 100))), (desc_of(NV12, 144), scale_of((134, 66))),
                (desc_of(RGBA, 256, flags=1), scale_of((50, 30), (10, 20, 100, 60))), (desc_of(BGRA, 64), scale_of((13, 7)))]
    ladder_b = ladder_a[:2]
    units_a = 50 * 2 + 33 * 5 + 30 * 2 + 7 * 1
    entry = 24                                                       # sizeof(ExportEntryUV)
    for pairs, count, sched_units in ((ladder_a, 3, units_a), (ladder_a, 5, 0), (ladder_a, 1, 0), (ladder_b, 2, 50 * 2 + 33 * 5),
                                      (ladder_b, 2, 0), (ladder_a, 2, units_a)):
        n0 = L.ladder_fake_launches()
        rc, msg, trace, launched = _ladder(L, h, [1] * count, pairs, [buf.value] * (count * len(pairs)), after=a, done=d)
        assert rc == 0 and launched == 1 and L.ladder_fake_launches() == n0 + 1, msg
        want = ([sched_units * 8] if sched_units else []) + [count * len(pairs) * entry]
        assert memcpys(trace) == want, (count, trace)
        kinds = [x.split()[0] for x in trace.splitlines()]
        assert kinds[-4:] == ["wait", "memcpy", "record", "record"], trace
        last = (C.c_longlong * (4 + 14 * 8))()
        L.ladder_fake_last(last)
        assert list(last[:2]) == [count, len(pairs)] and (not sched_units or last[2] == sched_units)
    # the per-rung fields of the last call (ladder_a)
    L.ladder_fake_last(last)
    assert last[2] == units_a
    want = [  # format, over, whole, pitch, crop, out, reciprocal of src_w * src_h
        (NV12, 1, 1, 208, (0, 0, 200, 100), (200, 100)),
        (NV12, 1, 0, 144, (0, 0, 200, 100), (134, 66)),
        (RGBA, 1, 0, 256, (10, 20, 100, 60), (50, 30)),
        (BGRA, 0, 0, 64, (0, 0, 200, 100), (13, 7)),
    ]
    for j, (fmt, over, whole, pitch, crop, out) in enumerate(want):
        o = list(last[4 + 14 * j:4 + 14 * (j + 1)])
        mul, shift = recip(crop[2] * crop[3])
        assert o[:13] == [fmt, over, whole, pitch, *crop, *out, mul & 0xFFFFFFFF, mul >> 32, shift], (j, o)
    L.glava_b200_destroy(h)
    L.cudaEventDestroy(a); L.cudaEventDestroy(d); L.cudaFree(buf)
    assert [L.fake_live(k) for k in range(4)] == live0
