"""Worst case of the dirty-row marks: every bar at full height, so no zero row can be skipped and the marks only cost their
word per warp.  Rasters saturated textures (glava_b200_raster_textures) at the headline geometry and times the raster kernel
(CUDA events around each launch) with GLAVA_B200_FULL_STORE=1 and without, alternated in one process.

    python tools/full_height_ab.py [--reps 3] [--launches 50] [--batch 1024] [--amplify 4000]

Prints one JSON line: per arm the median raster kernel time of each repetition, and the card it ran on."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np          # noqa: E402
import glava_b200 as g      # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--amplify", type=float, default=4000.0, help="bars AMPLIFY: saturated texels reach past the top row")
    args = ap.parse_args()
    p = g.default_params("bars", n=4096, w=1920, h=1080)
    p.lazy_smooth = 1
    p.bars_amplify = args.amplify
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    res = {"full": [], "marks": []}
    with g.Renderer(p, batch=args.batch) as r:
        tex = np.full((args.batch, r.nsz), 65535, np.uint16)
        for _ in range(3):
            r.raster_textures(tex, tex)
        r.sync()
        for rep in range(args.reps):
            for arm in ("full", "marks"):
                if arm == "full":
                    os.environ["GLAVA_B200_FULL_STORE"] = "1"
                else:
                    os.environ.pop("GLAVA_B200_FULL_STORE", None)
                r.raster_textures(tex, tex)                  # one untimed launch in this arm
                r.sync()
                r.set_timing(True)
                for _ in range(args.launches):
                    r.raster_textures(tex, tex)
                r.sync()
                kt = r.kernel_times()
                r.set_timing(False)
                res[arm].append(kt["raster_ms"] / max(kt["raster_launches"], 1))
        os.environ.pop("GLAVA_B200_FULL_STORE", None)
        frame = r.readback(0)
    rows_lit = int((frame != 0).any(axis=(1, 2)).sum())
    out = {"card": card, "module": "bars", "amplify": args.amplify, "rows": os.environ.get("GLAVA_B200_ROWS", "default"),
           "batch": args.batch, "w": 1920, "h": 1080, "launches_per_rep": args.launches,
           "rows_with_content_stream0": rows_lit,
           "raster_ms": {k: [round(v, 5) for v in vs] for k, vs in res.items()},
           "median_ms": {k: statistics.median(vs) for k, vs in res.items()},
           "algorithmic_GB_per_s": {k: args.batch * 1920 * 1080 * 4 / (statistics.median(vs) / 1e3) / 1e9 for k, vs in res.items()}}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
