"""The renderer handle's CUDA resources and its rebuild path, without a GPU: capi.cu and config.cpp built against the fake
runtime of tests/fakecuda, which counts live resources, fails the k-th creation on request and checks in every launcher
that the tables the launch structure names exist.

- A creation that fails at any resource returns null and leaves nothing behind.
- A reconfigure or resize that fails at any resource reports it, keeps the parameters of the last successful build and
  leaves the renderer refusing updates without launching anything, until a retry succeeds; no launcher reports the
  injected error later.
- A walk through the whole API, then destroy, leaves nothing behind, also with a failure at any resource it creates."""
import ctypes as C

import numpy as np
import pytest

from glava_b200.api import Params
from tests import fakecuda

R_NEED, R_TAPS, R_FULL, R_NEED_SMEM, R_NEED_L2, R_GEO, R_CTILE, R_COLTAB, R_TSMOOTH = (1 << i for i in range(9))
BATCH = 2

# name: (module, parameters, environment, tables the updates must reach)
CONFIGS = {
    "bars1024": ("bars", dict(n=1024, w=64, h=32, lazy_smooth=1), {}, R_NEED | R_TAPS),
    "bars4096_need_smem": ("bars", dict(n=4096, w=64, h=32, lazy_smooth=1), {}, R_NEED | R_TAPS | R_NEED_SMEM),
    "bars4096_need_l2": ("bars", dict(n=4096, w=64, h=32, lazy_smooth=1), {"GLAVA_B200_K5N_SMEM": "0"}, R_NEED | R_NEED_L2),
    "full_table": ("bars", dict(n=1024, w=64, h=32, lazy_smooth=0), {}, R_FULL),
    "radial": ("radial", dict(n=1024, w=64, h=64), {}, R_GEO),
    "circle_tiles": ("circle", dict(n=1024, w=64, h=64), {"GLAVA_B200_CTILE": "1"}, R_GEO | R_CTILE),
    "graph": ("graph", dict(n=1024, w=64, h=32), {}, R_COLTAB),
    "post_chain": ("bars", dict(n=1024, w=64, h=32, transform_smooth=1, interpolate=1, ur=30.0, fr=60.0), {}, R_TSMOOTH),
}
NOTHING = (0, 0, 0, 0)


class Fake:
    def __init__(self):
        L = self.L = fakecuda.lib()
        vp, i32 = C.c_void_p, C.c_int
        P = C.POINTER(Params)
        sig = {
            "glava_b200_default_params": (i32, [P, C.c_char_p]), "glava_b200_new": (vp, [P, i32, i32]),
            "glava_b200_destroy": (None, [vp]), "glava_b200_reconfigure": (i32, [vp, P]), "glava_b200_get_params": (i32, [vp, P]),
            "glava_b200_update": (i32, [vp, vp, vp, C.c_size_t, i32]), "glava_b200_update_masked": (i32, [vp, vp, vp, C.c_size_t, vp]),
            "glava_b200_update_device": (i32, [vp, vp, vp, C.c_size_t, i32]),
            "glava_b200_update_device_masked": (i32, [vp, vp, vp, C.c_size_t, vp]),
            "glava_b200_update_device_after": (i32, [vp, vp, vp, C.c_size_t, i32, vp]),
            "glava_b200_update_rings_masked": (i32, [vp, vp]),
            "glava_b200_set_async_input": (i32, [vp, i32]), "glava_b200_wait_input": (i32, [vp]),
            "glava_b200_ingest_fifo": (i32, [vp, vp, i32]), "glava_b200_update_rings": (i32, [vp, i32]),
            "glava_b200_reset_streams": (i32, [vp, vp]), "glava_b200_save_streams": (i32, [vp, vp, i32, vp]),
            "glava_b200_load_streams": (i32, [vp, vp, i32, vp]), "glava_b200_stream_state_bytes": (C.c_size_t, [P]),
            "glava_b200_readback_async": (i32, [vp, i32, vp]), "glava_b200_readback_fence": (i32, [vp]),
            "glava_b200_set_timing": (i32, [vp, i32]), "glava_b200_kernel_times": (i32, [vp, vp, vp, vp, vp]),
            "glava_b200_smooth_pass": (i32, [vp, vp, vp, i32]), "glava_b200_transform_smooth": (i32, [vp, vp, i32]),
            "glava_b200_raster_textures": (i32, [vp, vp, vp]), "glava_b200_input_event": (vp, [vp]),
            "glava_b200_sizereq": (i32, [vp, i32, i32]), "glava_b200_sync": (i32, [vp]), "glava_b200_last_error": (C.c_char_p, []),
            "glava_b200_set_abort_hook": (None, [vp]),
        }
        for name, (res, args) in sig.items():
            f = getattr(L, name)
            f.restype, f.argtypes = res, args
        self._quiet = C.CFUNCTYPE(None, C.c_char_p)(lambda msg: None)
        L.glava_b200_set_abort_hook(C.cast(self._quiet, vp))

    def params(self, module, **kw):
        p = Params()
        assert self.L.glava_b200_default_params(C.byref(p), module.encode()) == 0
        for k, v in kw.items():
            setattr(p, k, v)
        return p

    def new(self, p):
        h = self.L.glava_b200_new(C.byref(p), BATCH, 0)
        return C.c_void_p(h) if h else None

    def get_params(self, h):
        q = Params()
        assert self.L.glava_b200_get_params(h, C.byref(q)) == 0
        return q

    def update(self, h, p):
        pcm = np.zeros((BATCH, p.n), np.float32)
        return self.L.glava_b200_update(h, pcm.ctypes.data, pcm.ctypes.data, p.n, 1)

    def live(self):
        """live resources beyond those of the test's start (a failed test may leave its renderer behind)"""
        return tuple(a - b for a, b in zip(fakecuda.live(self.L), self.base))


@pytest.fixture(scope="module")
def fake():
    if fakecuda.cuda_include() is None:
        pytest.skip("no CUDA toolkit headers")
    return Fake()


@pytest.fixture(params=sorted(CONFIGS))
def config(request, fake, monkeypatch):
    module, kw, env, reach = CONFIGS[request.param]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    fake.L.fake_fail_at(-1)
    fake.L.fake_clear()
    fake.base = fakecuda.live(fake.L)
    yield fake.params(module, **kw), reach
    fake.L.fake_fail_at(-1)


def test_failed_creation_leaves_nothing(fake, config):
    p, _ = config
    L = fake.L
    h = fake.new(p)
    total = L.fake_creations()
    assert h and total > 0
    L.glava_b200_destroy(h)
    assert fake.live() == NOTHING
    for k in range(total):
        L.fake_fail_at(k)
        assert fake.new(p) is None, k
        assert fake.live() == NOTHING, k
    assert L.fake_stale() == 0


def _other(fake, how, q):
    """the parameters a reconfigure / resize of a renderer that now has q moves to (and back from)"""
    t = Params.from_buffer_copy(bytes(q))
    if how == "resize":
        t.w, t.h = (80, 40) if q.w == 64 else (64, 32)
    else:
        t.smooth_factor = 0.02 if q.smooth_factor != 0.02 else 0.03
    return t


def _rebuild(fake, how, h, t):
    if how == "reconfigure":
        return fake.L.glava_b200_reconfigure(h, C.byref(t))
    assert fake.L.glava_b200_sizereq(h, t.w, t.h) == 0
    return fake.update(h, t)                                          # applied at the start of the update


@pytest.mark.parametrize("how", ["reconfigure", "resize"])
def test_failed_rebuild_leaves_the_renderer_unbuilt_until_a_retry_succeeds(fake, config, how):
    p, reach = config
    L = fake.L
    h = fake.new(p)
    for _ in range(2):
        assert fake.update(h, p) == 0
    counts = []
    for _ in range(2):                                                # creations of a rebuild, there and back
        L.fake_fail_at(-1)
        assert _rebuild(fake, how, h, _other(fake, how, fake.get_params(h))) == 0
        counts.append(L.fake_creations())
    assert counts[0] == counts[1] and counts[0] > 0
    n = p.n // p.bufscale
    tex = np.zeros((BATCH, n), np.uint16)
    for k in range(counts[0]):
        cur = fake.get_params(h)
        t = _other(fake, how, cur)
        L.fake_fail_at(k)
        rc = _rebuild(fake, how, h, t)
        L.fake_fail_at(-1)
        assert rc != 0, k
        assert bytes(fake.get_params(h)) == bytes(cur), k
        launches = L.fake_launches()
        assert fake.update(h, cur) != 0, k
        assert L.glava_b200_raster_textures(h, tex.ctypes.data, tex.ctypes.data) != 0, k
        assert L.glava_b200_smooth_pass(h, tex.ctypes.data, tex.ctypes.data, 1) != 0, k
        assert b"failed" in L.glava_b200_last_error(), k
        assert L.fake_launches() == launches, k
        assert _rebuild(fake, how, h, t) == 0, k
        assert fake.update(h, t) == 0, k
        assert L.fake_violations() == 0, (k, L.fake_first_violation())
        assert L.fake_stale() == 0, k
    L.glava_b200_destroy(h)
    assert fake.live() == NOTHING
    assert L.fake_reached() & reach == reach


def _walk(fake, h, p):
    """every entry point that creates something lazily, return codes ignored"""
    L = fake.L
    n = p.n // p.bufscale
    pcm = np.zeros((BATCH, p.n), np.float32)
    mask = np.array([1, 0], np.uint8)
    fake.update(h, p)
    L.glava_b200_update_masked(h, pcm.ctypes.data, pcm.ctypes.data, p.n, mask.ctypes.data)
    chunks = np.zeros((BATCH, 64, 2), np.int16)
    L.glava_b200_ingest_fifo(h, chunks.ctypes.data, 64)
    L.glava_b200_update_rings(h, 1)
    L.glava_b200_reset_streams(h, mask.ctypes.data)
    size = L.glava_b200_stream_state_bytes(C.byref(p))
    if size:
        streams = np.arange(BATCH, dtype=np.int32)
        blobs = np.zeros(BATCH * size, np.uint8)
        L.glava_b200_save_streams(h, streams.ctypes.data, BATCH, blobs.ctypes.data)
        L.glava_b200_load_streams(h, streams.ctypes.data, BATCH, blobs.ctypes.data)
    frame = np.zeros(2 * 80 * 64 * 4, np.uint8)
    L.glava_b200_readback_async(h, 0, frame.ctypes.data)
    L.glava_b200_readback_fence(h)
    L.glava_b200_set_timing(h, 1)
    fake.update(h, p)
    L.glava_b200_kernel_times(h, None, None, None, None)
    tex = np.zeros((1, n), np.uint16)
    L.glava_b200_smooth_pass(h, tex.ctypes.data, tex.ctypes.data, 1)
    planes = np.zeros((1, n), np.float32)
    L.glava_b200_transform_smooth(h, planes.ctypes.data, 1)
    L.glava_b200_input_event(h)
    L.glava_b200_sizereq(h, 80, 40)
    fake.update(h, p)
    L.glava_b200_readback_async(h, 1, frame.ctypes.data)
    L.glava_b200_sync(h)


def test_api_walk_leaves_nothing(fake, config):
    p, _ = config
    L = fake.L
    h = fake.new(p)
    L.fake_fail_at(-1)
    _walk(fake, h, p)
    total = L.fake_creations()
    L.glava_b200_destroy(h)
    assert fake.live() == NOTHING
    assert L.fake_violations() == 0, L.fake_first_violation()
    assert L.fake_stale() == 0
    for k in range(total):
        h = fake.new(p)
        L.fake_fail_at(k)
        _walk(fake, h, p)
        L.fake_fail_at(-1)
        L.glava_b200_destroy(h)
        assert fake.live() == NOTHING, k
        assert L.fake_violations() == 0, (k, L.fake_first_violation())
