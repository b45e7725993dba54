"""-m gpu: batches past CUDA's grid-y limit of 65535.

glava_b200_new takes any batch >= 1.  The launchers whose grid y axis counts planes, streams or groups of planes
(epilogue_b_kernel: 2 * batch planes; fifo_ingest_kernel: batch streams; k5_table_kernel / k5_planes_kernel: 2 * batch / S
plane groups) launch slices of at most 65535 rows.  Probe streams on both sides of the slice boundaries must equal the same
rows run through a small renderer fed the same history.  Tiny frames and cheap rows (a few base rows times a per-stream
gain) keep the host side small; device memory is that of the batch (about 10 GB for the FFT-4096 case)."""
import numpy as np
import pytest

import glava_b200 as g

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]


def _probes(batch):
    """streams on both sides of every slice boundary: plane 65535 (stream 32767 / 32768), stream 65535, and the plane group
    65535 of 8 planes (stream 262140)"""
    return sorted(s for s in {0, 1, 32767, 32768, 32769, 65535, 65536, 262139, 262140, batch - 2, batch - 1} if s < batch)


def _gain(batch):
    s = np.arange(batch, dtype=np.uint64)
    return (0.15 + 0.85 * ((s * np.uint64(2654435761)) % np.uint64(1009)).astype(np.float32) / np.float32(1009)).astype(np.float32)


def _rows(base, gain, t, batch):
    """[batch][n] float32: base row (s + t) % len(base) times the stream's gain"""
    idx = (np.arange(batch) + t) % base.shape[0]
    return base[idx] * gain[:, None]


def _compare(big, small, probes):
    (bl, br), (tl, tr) = big.spectrum(), big.textures()
    (sl, sr), (ul, ur) = small.spectrum(), small.textures()
    assert tl.any()
    for i, s in enumerate(probes):
        assert np.array_equal(bl[s], sl[i]) and np.array_equal(br[s], sr[i]), s
        assert np.array_equal(tl[s], ul[i]) and np.array_equal(tr[s], ur[i]), s
        assert np.array_equal(big.readback(s), small.readback(i)), s


@pytest.mark.parametrize("n,batch,over", [(4096, 32771, dict(lazy_smooth=1)),           # epilogue_b_kernel: 65542 planes
                                          (256, 262147, dict()),                         # k5_table_kernel: 65537 groups of 8 planes
                                          (256, 262147, dict(k5_planes=1))],             # k5_planes_kernel (no tap table)
                         ids=["bars-4096-lazy-epilogue", "bars-256-k5-table", "bars-256-k5-planes"])
def test_update_past_the_grid_y_limit(built, monkeypatch, n, batch, over):
    over = dict(over)
    if over.pop("k5_planes", 0):
        monkeypatch.setenv("GLAVA_B200_NO_K5_TABLE", "1")
    p = g.default_params("bars", n=n, w=64, h=16, **over)
    rng = np.random.default_rng(batch)
    base_l = ((rng.random((7, n), np.float32) - 0.5) * 0.8); base_r = ((rng.random((5, n), np.float32) - 0.5) * 0.8)
    gain = _gain(batch)
    probes = _probes(batch)
    with g.Renderer(p, batch=batch) as big, g.Renderer(p, batch=len(probes)) as small:
        for t in range(3):
            lb = _rows(base_l, gain, t, batch); rb = _rows(base_r, gain, 2 * t, batch)
            big.update(lb, rb, True)
            small.update(lb[probes], rb[probes], True)
            del lb, rb
        _compare(big, small, probes)


def test_fifo_ingest_past_the_grid_y_limit(built):
    """fifo_ingest_kernel: one grid row per stream; ingest_fifo + update_rings at 65537 streams"""
    n, batch, hop = 256, 65537, 96
    p = g.default_params("bars", n=n, w=64, h=16)
    rng = np.random.default_rng(11)
    base = rng.integers(-30000, 30000, size=(9, hop * 2)).astype(np.float32)
    gain = _gain(batch)
    probes = _probes(batch)
    with g.Renderer(p, batch=batch) as big, g.Renderer(p, batch=len(probes)) as small:
        for t in range(5):                                            # 5 * 96 frames: the rings wrap
            chunks = _rows(base, gain, t, batch).astype(np.int16)
            big.ingest_fifo(chunks)
            small.ingest_fifo(chunks[probes])
            if t >= 2:
                big.update_rings(True)
                small.update_rings(True)
        _compare(big, small, probes)
