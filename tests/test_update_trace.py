"""The stream and event traffic of the update paths, without a GPU: capi.cu built against the fake runtime of tests/fakecuda,
which writes one line per launch, copy, fill, event record, event wait and synchronisation, with its stream and event
numbered in creation order.

For every configuration of test_handle_lifetime, a fixed walk (creation; plain, silent, masked, device-pointer, FIFO-ring
and raster-only updates; a resize; timed updates; asynchronous input; destruction) must produce the recorded trace in
tests/golden/update_trace.json line for line: no copy, launch, record or wait of an update may move, appear or vanish
without this file changing with it.

    python -m tests.test_update_trace     # rewrites the golden file from the current tree
"""
import ctypes as C
import json
import os

import numpy as np
import pytest

from tests import fakecuda
from tests.test_handle_lifetime import BATCH, CONFIGS, Fake

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "update_trace.json")


def aligned(shape, dtype):
    """a zeroed array whose data starts on a 64-byte boundary (device PCM pointers must be 16-byte aligned)"""
    n = int(np.prod(shape)) * np.dtype(dtype).itemsize
    raw = np.zeros(n + 64, np.uint8)
    off = (-raw.ctypes.data) % 64
    return raw[off:off + n].view(dtype).reshape(shape)


def walk(fake, p):
    """the calls whose trace is recorded; every one of them must succeed"""
    L = fake.L
    n = p.n // p.bufscale
    pcm = aligned((BATCH, p.n), np.float32)
    tex = np.zeros((BATCH, n), np.uint16)
    one, both, none = (np.array(m, np.uint8) for m in ([0, 1], [1, 1], [0, 0]))
    uneven = both if p.interpolate else one                # keyframe interpolation refuses uneven masks
    chunks = np.zeros((BATCH, 64, 2), np.int16)
    ready = C.c_void_p()
    assert L.cudaEventCreate(C.byref(ready)) == 0
    h = fake.new(p)
    assert h
    d = pcm.ctypes.data
    calls = [
        lambda: L.glava_b200_update(h, d, d, p.n, 1),
        lambda: L.glava_b200_update(h, d, d, p.n, 0),
        lambda: L.glava_b200_update_masked(h, d, d, p.n, uneven.ctypes.data),
        lambda: L.glava_b200_update_masked(h, d, d, p.n, both.ctypes.data),
        lambda: L.glava_b200_update_masked(h, d, d, p.n, none.ctypes.data),
        lambda: L.glava_b200_update_device(h, d, d, p.n, 1),
        lambda: L.glava_b200_update_device(h, d, d, p.n, 0),
        lambda: L.glava_b200_update_device_masked(h, d, d, p.n, uneven.ctypes.data),
        lambda: L.glava_b200_update_device_after(h, d, d, p.n, 1, ready),
        lambda: L.glava_b200_ingest_fifo(h, chunks.ctypes.data, 64),
        lambda: L.glava_b200_update_rings(h, 1),
        lambda: L.glava_b200_update_rings_masked(h, uneven.ctypes.data),
        lambda: L.glava_b200_update_rings(h, 0),
        lambda: L.glava_b200_raster_textures(h, tex.ctypes.data, tex.ctypes.data),
        lambda: L.glava_b200_raster_textures(h, tex.ctypes.data, None),
        lambda: L.glava_b200_sizereq(h, 80, 40),
        lambda: L.glava_b200_update(h, d, d, p.n, 1),
        lambda: L.glava_b200_set_timing(h, 1),
        lambda: L.glava_b200_update(h, d, d, p.n, 1),
        lambda: L.glava_b200_update_masked(h, d, d, p.n, uneven.ctypes.data),
        lambda: L.glava_b200_update_rings(h, 0),
        lambda: L.glava_b200_kernel_times(h, None, None, None, None),
        lambda: L.glava_b200_set_async_input(h, 1),
        lambda: L.glava_b200_update(h, d, d, p.n, 1),
        lambda: L.glava_b200_update(h, d, d, p.n, 1),
        lambda: L.glava_b200_wait_input(h),
    ]
    for i, call in enumerate(calls):
        assert call() == 0, (i, L.glava_b200_last_error())
    L.glava_b200_destroy(h)
    assert L.cudaEventDestroy(ready) == 0


def trace(fake, name):
    module, kw, env, _ = CONFIGS[name]
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        fake.L.fake_fail_at(-1)
        fake.L.fake_clear()
        fake.L.fake_trace_begin()
        try:
            walk(fake, fake.params(module, **kw))
        finally:
            fake.L.fake_trace_end()
        assert fake.L.fake_violations() == 0, fake.L.fake_first_violation()
        return fake.L.fake_trace().decode().splitlines()
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


@pytest.fixture(scope="module")
def fake():
    if fakecuda.cuda_include() is None:
        pytest.skip("no CUDA toolkit headers")
    return Fake()


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_update_trace_matches_the_recorded_one(fake, name):
    with open(GOLDEN) as f:
        want = json.load(f)[name]
    got = trace(fake, name)
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"line {i}: {g!r} != {w!r}"


if __name__ == "__main__":
    if fakecuda.cuda_include() is None:
        raise SystemExit("no CUDA toolkit headers")
    fk = Fake()
    out = {name: trace(fk, name) for name in sorted(CONFIGS)}
    with open(GOLDEN, "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
