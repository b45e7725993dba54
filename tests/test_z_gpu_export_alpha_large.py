"""-m gpu: the transparent exports at the headline size (DESIGN 4.19): 1024 streams of 1080p bars exported in YUVA420P,
YUVA444P10 and straight RGBA in one call each.  A strided sample of entries equals the numpy restatement of
tests/export_alpha_np.py bit for bit."""
import numpy as np
import pytest

import glava_b200 as g
from tests.export_alpha_np import frame_alpha_np
from tests.test_gpu_export_alpha import feed

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


def test_a_thousand_1080p_streams_in_every_alpha_format(built):
    p = g.default_params("bars", n=4096, w=1920, h=1080)
    p.lazy_smooth = 1
    count = 1024
    sample = list(range(0, count, 97)) + [count - 1]
    with g.Renderer(p, batch=count) as r:
        feed(r, 2, seed=3, scale=0.2)
        for fmt, kw, e in (("yuva420p", dict(matrix="bt601"), 2), ("yuva444p10", dict(full_range=True), 1),
                           ("rgba", dict(straight=True), 0)):
            l0 = r.launch_count
            got = r.export_frames(range(count), fmt, **kw)
            assert r.launch_count == l0 + 1
            planes = got if isinstance(got, tuple) else (got,)
            for i in sample:
                want = frame_alpha_np(r.readback(i), fmt, e)
                want = want if isinstance(want, tuple) else (want,)
                for k, t in enumerate(planes):
                    assert np.array_equal(t[i].cpu().numpy(), want[k]), (fmt, i, k)
            del got, planes
            torch.cuda.empty_cache()
