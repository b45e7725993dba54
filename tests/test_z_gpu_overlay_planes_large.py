"""-m gpu: glava_b200_overlay_planes at the headline size, 1024 streams of 1080p bars in one call per format (DESIGN 4.17):
a strided sample of entries equals the numpy restatement of tests/overlay_planes_np.py bit for bit, and every picture's
bytes outside the sample are checked against a second call onto a copy."""
import numpy as np
import pytest

import glava_b200 as g
from tests.overlay_planes_np import FORMATS, planes_np
from tests.test_gpu_overlay_planes import crop, feed

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


def test_a_thousand_1080p_streams_in_every_format(built):
    p = g.default_params("bars", n=4096, w=1920, h=1080)
    p.lazy_smooth = 1
    count = 1024
    with g.Renderer(p, batch=count) as r:
        feed(r, 2, seed=3, scale=0.2)
        for fmt in FORMATS:
            planes = r.export_frames(range(count), fmt)
            planes = planes if isinstance(planes, tuple) else (planes[:, :1080], planes[:, 1080:])
            gen = torch.Generator(device="cuda").manual_seed(7)
            for t in planes:
                t.copy_(torch.randint(0, 1 << (8 * t.element_size()), t.shape, dtype=torch.int32, device="cuda", generator=gen).to(t.dtype))
            sample = list(range(0, count, 97)) + [count - 1]
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
                want = planes_np(r.readback(streams[i]), crop(before[i], fmt, 0, 0, 1920, 1080), fmt, 0, True)
                for k, t in enumerate(planes):
                    assert np.array_equal(t[i].cpu().numpy(), want[k]), (fmt, i, k)
            del planes, twin
            torch.cuda.empty_cache()
