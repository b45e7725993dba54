"""-m gpu: the largest shapes of BASELINE.json — 7680x4320 frames, setbufsize 16384 — and the largest sides the renderer
takes (16384 x 256, 256 x 16384), checked against the oracle on row bands (the oracle renders only the requested rows, so 33 M-pixel frames stay cheap): bottom rows, the rows around the
tallest bars, the vertical centre and the top rows, bit-exact."""
import numpy as np
import pytest

import glava_b200 as g
from oracle.oracle import params_from

pytestmark = pytest.mark.gpu


def _tex(orc, op, n, seed):
    rng = np.random.default_rng(seed)
    tl = orc.smooth_pass(op, (rng.random(n) ** 2 * 65535).astype(np.uint16))
    tr = orc.smooth_pass(op, (rng.random(n) ** 3 * 65535).astype(np.uint16))
    return tl, tr


@pytest.mark.parametrize("module,n,w,h", [("bars", 16384, 7680, 4320), ("radial", 8192, 3840, 2160), ("graph", 16384, 7680, 4320),
                                          ("wave", 4096, 7680, 4320), ("circle", 4096, 3840, 2160),
                                          # the largest sides the renderer takes: 128 strips of 128 pixels, 16384 rows
                                          ("bars", 4096, 16384, 256), ("graph", 4096, 16384, 256), ("wave", 4096, 16384, 256),
                                          ("bars", 4096, 256, 16384), ("graph", 4096, 256, 16384), ("wave", 4096, 256, 16384)])
def test_largest_frames_row_bands_bit_exact(orc_pm, module, n, w, h, built):
    p = g.default_params(module, n=n, w=w, h=h)
    op = params_from(p)
    tl, tr = _tex(orc_pm, op, n, 3)
    if module == "wave":
        tl = np.clip(tl.astype(int) // 4 + 24576, 0, 65535).astype(np.uint16)
    bands = [(0, 6), (h // 2 - 3, h // 2 + 3), (h - 5, h)]
    if module in ("bars", "graph"):
        bands += [(96, 104), (188, 200)]                          # where most bars / the graph line end for these textures
    if module in ("radial", "circle"):
        bands.append((h // 2 + 120, h // 2 + 134))                # through the ring at C_RADIUS = 128
    with g.Renderer(p, batch=2) as r:
        r.raster_textures(np.stack([tl, tr]), np.stack([tr, tl]))
        a, b = r.readback(0), r.readback(1)
    for y0, y1 in bands:
        want = orc_pm.raster(op, tl, tr, rows=(y0, y1))
        assert np.array_equal(a[y0:y1], want[y0:y1]), (module, y0, y1, int((a[y0:y1] != want[y0:y1]).any(axis=2).sum()))
        want = orc_pm.raster(op, tr, tl, rows=(y0, y1))
        assert np.array_equal(b[y0:y1], want[y0:y1]), (module, "swapped", y0, y1)
    assert a.any() and not np.array_equal(a, b)
