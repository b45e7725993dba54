"""-m gpu: a resize whose framebuffer cannot be allocated leaves the renderer unbuilt — it keeps its parameters and refuses
updates without launching anything — and the next resize that succeeds makes it usable again, as if it had been created at
that size."""
import numpy as np
import pytest

import glava_b200 as g

pytestmark = pytest.mark.gpu

ECUDA = -3                                                            # GLAVA_B200_ECUDA


def test_failed_resize_leaves_the_renderer_unbuilt_until_a_resize_succeeds(built):
    n, batch = 1024, 256
    rings = g.StreamRings(batch, n)
    feed = []

    def step():
        rings.advance()
        feed.append((rings.lb.copy(), rings.rb.copy()))
        return feed[-1]

    with g.Renderer(g.default_params("bars", n=n, w=64, h=32), batch=batch) as r:
        for _ in range(2):
            r.update(*step(), True)
        r.sync()
        r.sizereq(16384, 16384)              # 256 frames of 16384 x 16384 RGBA8 = 256 GiB: the cudaMalloc fails at once
        lb, rb = rings.lb, rings.rb
        assert r._L.glava_b200_update(r._h, lb.ctypes.data, rb.ctypes.data, n, 1) == ECUDA
        launches = r.launch_count
        with pytest.raises(g.GlavaError, match="resize"):
            r.update(lb, rb, True)
        assert r.launch_count == launches
        q = r.refresh_params()
        assert (q.w, q.h) == (64, 32)
        r.sizereq(96, 48)
        for _ in range(2):
            r.update(*step(), True)
        assert (r.params.w, r.params.h) == (96, 48)
        got_spec = r.spectrum()
        got = [r.readback(s) for s in range(batch)]

    with g.Renderer(g.default_params("bars", n=n, w=96, h=48), batch=batch) as f:
        for lb, rb in feed:
            f.update(lb, rb, True)
        want_spec = f.spectrum()
        for s in range(batch):
            assert np.array_equal(got[s], f.readback(s)), s
    for a, b in zip(got_spec, want_spec):
        assert np.array_equal(a, b)
