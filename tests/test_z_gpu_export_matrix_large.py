"""-m gpu: the Y'CbCr encodings (DESIGN 4.15) at the headline size, 1920x1080 bars: whole frames in every format and
encoding under live, stale and absent dirty-row marks, so that rows the marks skip still encode as the background; and a
1080p ladder that mixes encodings and formats per rung, each rung equal to its standalone call."""
import pytest

import glava_b200 as g
from tests.test_gpu_export_matrix import BG, FORMATS, NEW, check, check_identities, feed, ladder_vs_standalone

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


def test_bars_1080p_live_stale_and_absent_marks(built):
    p = g.default_params("bars", n=4096, w=1920, h=1080)
    p.lazy_smooth = 1
    with g.Renderer(p, batch=3) as r:
        for step in range(3):                                          # marks valid from the second pass on
            feed(r, 1, seed=step, scale=0.1 + 0.3 * step)
            for kw, e in NEW:
                for fmt in FORMATS:
                    check(r, [2, 0], fmt, kw, e, bg=BG if step else (0, 0, 0), what=step)
        for kw, _ in NEW:
            check_identities(r, [0, 1, 2], kw)
        q = r.params.copy(); q.bars_mirror_yx = 1                      # the generic kernel keeps no marks
        r.reconfigure(q)
        feed(r, 1, seed=9)
        for kw, e in NEW:
            for fmt in FORMATS:
                check(r, [1], fmt, kw, e, what="no marks")


def test_1080p_ladder_mixing_encodings_and_formats(built):
    p = g.default_params("bars", n=4096, w=1920, h=1080)
    p.lazy_smooth = 1
    rungs = [dict(size=None, fmt="nv12"), dict(size=None, fmt="nv12", full_range=True),
             dict(size=(1280, 720), fmt="i420", matrix="bt601", full_range=True), dict(size=(640, 360), fmt="p010", full_range=True),
             dict(size=(480, 270), fmt="nv12", matrix="bt601"), dict(size=(321, 181), fmt="yuv444", matrix="bt601", full_range=True),
             dict(size=None, fmt="p010", matrix="bt601", background=BG), dict(size=(96, 54), fmt="rgba", over=True)]
    with g.Renderer(p, batch=3) as r:
        for step in range(2):
            feed(r, 1, seed=step, scale=0.2 + 0.3 * step)
            ladder_vs_standalone(r, [2, 0], rungs)
