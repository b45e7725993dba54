"""Bytes the bars / graph / wave raster stores per step at a bench.py workload, with and without the dirty-row marks, from the
host build (CPU only, no GPU needed).

    python tools/stored_bytes.py [--config headline|graph720|wave720] [--streams 24] [--steps 20] [--raster-ms MS]

The inputs are bench.py's: the first --streams streams of synth_batch_int16, its 4-snapshot cycle and its warm-up updates, run
through the host build of the spectrum path (tests/emul Channel.update) and rastered by the host build (emul.raster).  Per
frame and 128-pixel warp strip, the kernel stores the rows that can hold content (bars / graph: from the base line to the
first all-zero row; wave: the rows between the first and last non-zero one) and, of the other rows, those that held content
in the previous frame of that slot (raster_core.h dirty_zero_span); every other row is a zero row that is already zero.  The
kernels bound the content rows from the column data rather than the frame, a few rows wider for graph's and wave's
3x3 stencil, so this slightly undercounts those two.  Without the marks every row is stored: W * H * 4 bytes per frame.

--raster-ms: a raster kernel time measured at the same workload; prints the stored bytes over it as achieved bandwidth."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import HOP, workload            # noqa: E402  (stdlib only at import time)
import glava_b200 as g                     # noqa: E402
from glava_b200.synth import synth_batch_int16   # noqa: E402
from tests import emul                     # noqa: E402

STRIP = 128


def content_rows(frame, module, flip):
    """[strips] (lo, hi): rows the kernel stores as content for each 128-pixel strip of one frame ([h][w][4], row 0 = bottom)"""
    h, w = frame.shape[:2]
    nstrip = (w + STRIP - 1) // STRIP
    pad = np.zeros((h, nstrip * STRIP, 4), np.uint8); pad[:, :w] = frame
    nz = pad.reshape(h, nstrip, STRIP * 4).any(axis=2)                  # [row][strip]
    anyrow = nz.any(axis=0)
    first = np.where(anyrow, np.argmax(nz, axis=0), 0)
    last = np.where(anyrow, h - np.argmax(nz[::-1], axis=0), 0)          # one past the last non-zero row
    if module == "wave":
        return first, last
    if flip:
        return np.where(anyrow, first, h), np.full(nstrip, h)
    return np.zeros(nstrip, int), last


def union_rows(a, b):
    """rows of [a0, a1) u [b0, b1), per strip"""
    (a0, a1), (b0, b1) = a, b
    la, lb = np.maximum(a1 - a0, 0), np.maximum(b1 - b0, 0)
    overlap = np.maximum(np.minimum(a1, b1) - np.maximum(a0, b0), 0)
    return la + lb - np.where((la > 0) & (lb > 0), overlap, 0)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--config", default="headline")
    ap.add_argument("--streams", type=int, default=24, help="streams sampled (the first of the bench's batch)")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--raster-ms", type=float, default=None)
    args = ap.parse_args()
    wl = workload(args.config)
    module, n, w, h, batch = wl["module"], wl["n"], wl["w"], wl["h"], wl["batch"]
    if module not in ("bars", "graph", "wave"):
        raise SystemExit("dirty-row marks are kept by the bars, graph and wave rasters only")
    p = g.default_params(module, n=n, w=w, h=h)
    p.lazy_smooth = 1
    flip = module == "bars" and bool(p.bars_flip)
    is_fft = module != "wave"
    nsnap = 4
    pcm = synth_batch_int16(0, args.streams, 0, n + nsnap * HOP)
    pcm_f = pcm.astype(np.float32) / np.float32(65535)
    strip_w = np.minimum(STRIP, w - STRIP * np.arange((w + STRIP - 1) // STRIP))
    full = marked = 0
    per_stream = []
    for s in range(args.streams):
        cl, cr = emul.Channel(p), emul.Channel(p)
        prev = None
        fs = ms = 0
        for i in range(args.warmup + args.steps):
            k = (i % nsnap + 1) * HOP
            _, tl = cl.update(pcm_f[s, k:k + n, 0], is_fft)
            _, tr = cr.update(pcm_f[s, k:k + n, 1], is_fft)
            if i < args.warmup - 1:
                continue                                                 # only the frame before the first timed one matters
            cur = content_rows(emul.raster(p, tl, tr if is_fft else tl, fast=True), module, flip)
            if i >= args.warmup:
                fs += w * h * 4
                ms += int((union_rows(cur, prev) * strip_w).sum()) * 4
            prev = cur
        full += fs; marked += ms
        per_stream.append(ms / fs)
    frac = marked / full
    out = {"config": args.config, "module": module, "w": w, "h": h, "batch": batch, "streams_sampled": args.streams,
           "steps": args.steps, "warmup": args.warmup,
           "bytes_per_step_full_store": batch * w * h * 4, "bytes_per_step": batch * w * h * 4 * frac,
           "fraction_stored": frac, "per_stream_fraction": [round(v, 4) for v in per_stream]}
    if args.raster_ms:
        out["raster_ms"] = args.raster_ms
        out["stored_GB_per_s"] = out["bytes_per_step"] / (args.raster_ms / 1e3) / 1e9
    print(json.dumps(out))


if __name__ == "__main__":
    main()
