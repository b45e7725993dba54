"""-m gpu: reset, save and load of streams above index 65535 (the state kernels flatten streams onto grid.x).

A bars renderer of 65537 streams at setbufsize 256 resets, saves and loads streams past 65535; a three-stream renderer
fed the same rows mirrors those streams and must stay equal bit for bit."""
import numpy as np
import pytest

import glava_b200 as g

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]


def test_stream_state_past_65535_streams(built):
    n, batch = 256, 65537
    probes = [65534, 65535, 65536]
    p = g.default_params("bars", n=n, w=64, h=16)
    rng = np.random.default_rng(12)
    base = (rng.random((11, n), np.float32) - 0.5) * 0.8
    gain = (0.2 + 0.8 * rng.random(batch)).astype(np.float32)

    def rows(t):
        return base[(np.arange(batch) + t) % base.shape[0]] * gain[:, None], base[(np.arange(batch) + 3 * t) % base.shape[0]] * gain[:, None]

    def step(big, small, t, mask=None):
        lb, rb = rows(t)
        if mask is None:
            big.update(lb, rb, True); small.update(lb[probes], rb[probes], True)
        else:
            big.update_masked(lb, rb, mask); small.update_masked(lb[probes], rb[probes], mask[probes])

    def same(big, small):
        (bl, br), (tl, tr) = big.spectrum(), big.textures()
        (sl, sr), (ul, ur) = small.spectrum(), small.textures()
        for i, s in enumerate(probes):
            assert np.array_equal(bl[s], sl[i]) and np.array_equal(br[s], sr[i]), s
            assert np.array_equal(tl[s], ul[i]) and np.array_equal(tr[s], ur[i]), s
            assert np.array_equal(big.readback(s), small.readback(i)), s

    with g.Renderer(p, batch=batch) as big, g.Renderer(p, batch=len(probes)) as small:
        mask = np.ones(batch, bool); mask[65535] = False
        for t in range(4):
            step(big, small, t, mask if t == 2 else None)
        m = np.zeros(batch, bool); m[65536] = True
        big.reset_streams(m); small.reset_streams([0, 0, 1])
        blobs = big.save_streams([65535, 65536, 65534])
        assert np.array_equal(blobs[:, 4096:], small.save_streams([1, 2, 0])[:, 4096:])
        big.load_streams([65536, 65534], blobs[[0, 1]]); small.load_streams([2, 0], blobs[[0, 1]])
        for t in range(4, 7):
            step(big, small, t)
        same(big, small)
        assert big.textures()[0][65536].any()
