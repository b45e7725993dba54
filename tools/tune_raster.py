"""Sweep rows-per-CTA / block width of the bars raster kernel at the headline (development aid).

Each point is one bench.py run (spectrum and raster co-running, the bench's own inputs) with GLAVA_B200_ROWS / _BX set.  With
the dirty-row marks the raster of an unchanged texture stores almost nothing, so an isolated re-raster of one texture is no
longer representative: the step is what is timed.

    python tools/tune_raster.py [--steps 200] [--rows 68,135,270,540,1080] [--bx 96,160,256] [--bx-rows ROWS]

The --bx widths are swept at --bx-rows (default: the launch default); prints one line per point."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run(steps, rows=None, bx=None):
    env = dict(os.environ)
    if rows:
        env["GLAVA_B200_ROWS"] = str(rows)
    if bx:
        env["GLAVA_B200_BX"] = str(bx)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", str(steps), "--no-cpu-baseline", "--no-extras"],
                         env=env, capture_output=True, text=True, cwd=ROOT)
    try:
        d = json.loads(out.stdout.strip().splitlines()[-1])
    except Exception:
        return f"failed: {out.stderr.strip()[-300:]}"
    r = d["roofline"]
    return (f"value {d['value']:10.0f}  ms/step {d['ms_per_step']:.4f}  raster ms {r['kernel_ms']:.4f}  "
            f"isolated {r['kernel_ms_isolated']:.4f}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rows", default="68,135,270,540,1080")
    ap.add_argument("--bx", default="96,160,256")
    ap.add_argument("--bx-rows", default=None)
    args = ap.parse_args()
    for rows in args.rows.split(","):
        print(f"rows={rows:>5s} bx=auto: {run(args.steps, rows=rows)}", flush=True)
    for bx in args.bx.split(","):
        print(f"rows={args.bx_rows or 'auto':>5s} bx={bx:>4s}: {run(args.steps, rows=args.bx_rows, bx=bx)}", flush=True)


if __name__ == "__main__":
    main()
