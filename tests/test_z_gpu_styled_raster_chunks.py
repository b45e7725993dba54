"""-m gpu: styled raster launches past the 32768-stream chunk (DESIGN 4.9).

A styled kernel finds its stream's style slot through style_of[stream0 + blockIdx.z], so a launch that starts at
stream0 > 0 must look up the global stream, as the column table, the texture min / max and the framebuffer slot already
do (tests/test_z_gpu_raster_chunks.py).  The probe streams on both sides of the chunk boundary each get a style of their
own; the others are a mix of styled and unstyled streams.  Every probe must equal the oracle at its styled parameters, and
the pass must issue the plain plan's launches.  With the tiny frames of the plain test, device memory sampled every 0.5 s
on an H100 80GB HBM3 (700 W limit) peaked between 0.55 and 1.3 GiB over two runs of this file, CUDA context included."""
import numpy as np
import pytest

import glava_b200 as g
from oracle.oracle import params_from
from tests import test_z_gpu_raster_chunks as rc

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

AMP = dict(radial="radial_amplify", circle="circle_amplify", graph="graph_vscale", wave="wave_amplify")


def _probe_styles(module, a):
    """six distinct styles for the probes 0, 1, 32767, 32768, 32769 and batch - 1"""
    fg = [(0.9, 0.2, 0.1, 1.0), (0.1, 0.9, 0.3, 0.7), (0.3, 0.3, 1.0, 1.0)]
    bg = None if module == "circle" else (0.25, 0.2, 0.15, 1.0)
    out = [{"amplify": 1.7 * a}, {"fg": fg[0]}, {"amplify": 0.5 * a, "fg": fg[1]}, {"amplify": 1.3 * a},
           {"amplify": -a} if module in ("radial", "circle") else {"amplify": 0.8 * a, "fg": fg[2]},
           {"fg": fg[2], "bg": bg} if bg else {"amplify": 1.2 * a, "fg": fg[2]}]
    return out


@pytest.mark.parametrize("module", ["graph", "wave", "radial", "circle"])
def test_styled_raster_past_the_stream_chunk(orc_pm, module, built):
    n, batch = 256, 32771
    p = g.default_params(module, n=n, w=32, h=24, **rc.SMALL_PARAMS[module])
    a = getattr(p, AMP[module])
    tl, tr = rc._textures(n, batch, 11, wave=module == "wave")
    probes = (0, 1, 32767, 32768, 32769, batch - 1)
    own = _probe_styles(module, a)
    mix = [None, {"amplify": 1.5 * a}, None, {"fg": (0.6, 0.6, 0.1, 1.0)}, {"amplify": 0.7 * a}]
    styles = [mix[s % len(mix)] for s in range(batch)]
    for s, st in zip(probes, own):
        styles[s] = st
    with g.Renderer(p, batch=batch) as r:
        r.set_stream_styles(range(batch), styles)
        rc._raster(r, p, batch, batch, tl, tr)
        for s in probes + (2, 32770 - 5):
            got = r.readback(s)
            want = orc_pm.raster(params_from(g.style_params(p, styles[s])), tl[s], tr[s])
            assert got.any() or not want.any(), (module, s)
            assert np.array_equal(got, want), (module, s, styles[s])
        assert sum(orc_pm.raster(params_from(g.style_params(p, styles[s])), tl[s], tr[s]).any() for s in probes) >= 5, module
