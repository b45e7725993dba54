"""-m gpu, large: the scaled overlay (glava_b200_overlay_scaled, DESIGN 4.21) of 3840 x 2160 frames shrunk to small rectangles,
against the restatement of tests/test_gpu_overlay_scaled.py, under native opacity and any other."""
import pytest

import glava_b200 as g
from tests.test_gpu_overlay_opacity import feed
from tests.test_gpu_overlay_scaled import check
from tests.test_overlay_opacity_core import NV12, P010, RGBA, YUV444

pytestmark = pytest.mark.gpu
pytest.importorskip("torch")


@pytest.mark.parametrize("native", [True, False], ids=["native", "blended"])
def test_4k_frames_to_small_rectangles(built, native):
    kw0 = {} if native else dict(premultiply_alpha=0)
    p = g.default_params("bars", n=1024, w=3840, h=2160, **kw0)
    with g.Renderer(p, batch=2) as r:
        feed(r, 2)
        for fmt, planes, size, crop in ((RGBA, False, (160, 90), None), (NV12, False, (214, 120), (100, 60, 3700, 2080)),
                                        (P010, True, (96, 54), None), (YUV444, True, (37, 23), (0, 0, 3840, 2160))):
            check(r, [1, 0], fmt, [255, 128], {}, 0, planes, size, crop, what="4K")
