"""-m gpu: the 4:2:2 formats at the headline size (DESIGN 4.18): 1024 streams of 1080p bars exported in YUV422P, YUV422P10
and UYVY in one call each, and overlaid onto 1024 pictures of random samples in one call each.  A strided sample of entries
equals the numpy restatement of tests/export_422_np.py bit for bit; the overlay's batched and per-entry forms agree
everywhere."""
import numpy as np
import pytest

import glava_b200 as g
from tests.export_422_np import FORMATS, export422_np, overlay422_np
from tests.test_export_core import over_np
from tests.test_gpu_overlay_422 import crop, feed

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


def test_a_thousand_1080p_streams_in_every_format(built):
    p = g.default_params("bars", n=4096, w=1920, h=1080)
    p.lazy_smooth = 1
    count = 1024
    sample = list(range(0, count, 97)) + [count - 1]
    with g.Renderer(p, batch=count) as r:
        feed(r, 2, seed=3, scale=0.2)
        for fmt in FORMATS:
            got = r.export_frames(range(count), fmt, matrix="bt601")
            planes = (got,) if fmt == "uyvy" else got
            for i in sample:
                want = export422_np(over_np(r.readback(i)[::-1], (0, 0, 0), True), fmt, 2)
                want = (want,) if fmt == "uyvy" else want
                for k, t in enumerate(planes):
                    assert np.array_equal(t[i].cpu().numpy(), want[k]), (fmt, i, k)
            gen = torch.Generator(device="cuda").manual_seed(7)
            for t in planes:
                for c in range(0, count, 64):
                    t[c:c + 64].copy_(torch.randint(0, 1 << (8 * t.element_size()), t[c:c + 64].shape, dtype=torch.int32,
                                                    device="cuda", generator=gen).to(t.dtype))
            before = {i: [t[i].cpu().numpy() for t in planes] for i in sample}
            twin = tuple(t.clone() for t in planes)
            streams = list(range(count))[::-1]
            r.overlay_planes(streams, planes, None, fmt)
            r.overlay_planes(streams, [tuple(t[i] for t in twin) for i in range(count)], None, fmt)
            torch.cuda.synchronize()
            for a, b in zip(planes, twin):                          # batched and per-entry tuples agree everywhere
                assert torch.equal(a.view(torch.int16) if a.dtype == torch.uint16 else a,
                                   b.view(torch.int16) if b.dtype == torch.uint16 else b), fmt
            for i in sample:
                want = overlay422_np(r.readback(streams[i]), crop(before[i], fmt, 0, 0, 1920, 1080), fmt, 0, True)
                for k, t in enumerate(planes):
                    assert np.array_equal(t[i].cpu().numpy(), want[k]), (fmt, i, k)
            del got, planes, twin
            torch.cuda.empty_cache()
