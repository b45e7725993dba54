"""Scaled export rates (glava_b200_export_scaled, DESIGN 4.11) on one GPU, with the card and its power limit read in the same
run.  Per workload (bench.py's inputs and warm-up), CUDA-event time of: 1024 streams to 480x270 and 192x108 NV12, the same
streams as one 32x32 NV12 mosaic of 128x72 tiles (4096x2304), and the full-size NV12 export_frames for comparison, legs
alternated over rounds.  Bytes per call = the source rows the marks let through (counted from the read-back frames of a
stream sample as tools/export_bench.py counts them; every row for modules without marks) plus the bytes written, over the
median time, against the data sheet's 3.35 TB/s unless MEASURED_PEAKS.json gives a peak.

    python tools/export_scaled_bench.py --out profiles/h100_export_scaled.json [--configs headline,radial1080 --reps 20 --rounds 3]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import HOP, hbm_peak, workload      # noqa: E402  (stdlib only at import time)
from tools.export_bench import read_fraction   # noqa: E402
from tools.style_bench import card             # noqa: E402

# (name, kind, size): kind "scaled" (one destination per stream), "mosaic" (32 columns of tiles), "full" (export_frames)
LEGS = (("nv12_480x270", "scaled", (480, 270)), ("nv12_192x108", "scaled", (192, 108)),
        ("nv12_mosaic_32x32_128x72", "mosaic", (128, 72)), ("nv12_full", "full", None))
COUNT = 1024


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--configs", default="headline,radial1080")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import torch
    import glava_b200 as g
    from glava_b200.synth import synth_batch_int16

    name, limit = card()
    peak, peak_src = hbm_peak()
    result = {"gpu": name, "power_limit": limit, "peak_gbs": peak, "peak_source": peak_src, "reps": args.reps,
              "rounds": args.rounds, "count": COUNT, "workloads": {}}
    for cfg in args.configs.split(","):
        wl = workload(cfg)
        module, n, w, h, batch = wl["module"], wl["n"], wl["w"], wl["h"], wl["batch"]
        assert batch >= COUNT, (cfg, batch)
        p = g.default_params(module, n=n, w=w, h=h)
        p.lazy_smooth = 1
        nsnap = 4
        pcm = synth_batch_int16(0, batch, 0, n + nsnap * HOP).astype(np.float32) / np.float32(65535)
        dev_l = [torch.from_numpy(np.ascontiguousarray(pcm[:, (i + 1) * HOP:(i + 1) * HOP + n, 0])).cuda() for i in range(nsnap)]
        dev_r = [torch.from_numpy(np.ascontiguousarray(pcm[:, (i + 1) * HOP:(i + 1) * HOP + n, 1])).cuda() for i in range(nsnap)]
        with g.Renderer(p, batch=batch) as r:
            st = torch.cuda.ExternalStream(r.cuda_stream)
            for i in range(5):
                r.update_device(dev_l[i % nsnap].data_ptr(), dev_r[i % nsnap].data_ptr(), True)
            r.sync()
            streams = list(range(COUNT))
            outs = {}

            def run(leg):
                key, kind, size = leg
                if kind == "scaled":
                    outs[key] = r.export_scaled(streams, size, fmt="nv12", out=outs.get(key))
                elif kind == "mosaic":
                    outs[key] = r.export_mosaic(streams, 32, size, "nv12", out=outs.get(key))
                else:
                    outs[key] = r.export_frames(streams, "nv12", out=outs.get(key))

            for leg in LEGS:                                  # allocates, warms the list buffers and the kernels
                run(leg)
            torch.cuda.synchronize()
            frac = read_fraction(g, r, p, module, np.linspace(0, batch - 1, 32).astype(int))
            times = {leg[0]: [] for leg in LEGS}
            for _ in range(args.rounds):
                for leg in LEGS:
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    r.sync()
                    a.record(st)
                    for _ in range(args.reps):
                        run(leg)
                    b.record(st)
                    b.synchronize()
                    times[leg[0]].append(a.elapsed_time(b) / args.reps)
            legs = {}
            for key, kind, size in LEGS:
                ms = float(np.median(times[key]))
                ow, oh = size or (w, h)
                wbytes = COUNT * ow * oh * 1.5
                rbytes = COUNT * w * h * 4.0 * frac           # every crop here is the whole frame
                gbs = (wbytes + rbytes) / (ms / 1e3) / 1e9
                legs[key] = {"ms": ms, "ms_all": times[key], "write_bytes": wbytes, "read_bytes": rbytes, "gbs": gbs,
                             "frac_of_peak": gbs / peak, "frames_per_s": COUNT / (ms / 1e3)}
        result["workloads"][cfg] = {"module": module, "n": n, "w": w, "h": h, "batch": batch, "read_fraction": frac, "legs": legs}
        print(cfg, json.dumps({k: [round(v["ms"], 4), round(v["frac_of_peak"], 3)] for k, v in legs.items()}), flush=True)
    text = json.dumps(result, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
