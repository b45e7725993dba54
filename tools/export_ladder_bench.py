"""Encoder ladder rates (glava_b200_export_ladder, DESIGN 4.13) on one GPU, with the card and its power limit read in the same
run.  Per workload (bench.py's inputs and warm-up), 1024 streams, the NV12 ladder {1920x1080, 1280x720, 640x360, 480x270}
as one ladder call against the same four standalone calls back to back (export_frames + 3 x export_scaled); legs
alternated, medians of rounds x reps calls in CUDA-event time.  Bytes per call = the source rows the marks let through
(tools/export_bench.py read_fraction), counted once for the ladder and once per call for the four calls, plus the bytes
written, against the data sheet's 3.35 TB/s unless MEASURED_PEAKS.json gives a peak.

    python tools/export_ladder_bench.py --out profiles/h100_export_ladder.json [--configs headline,radial1080 --reps 20 --rounds 3]
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

SIZES = ((1920, 1080), (1280, 720), (640, 360), (480, 270))
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
              "rounds": args.rounds, "count": COUNT, "ladder": [list(s) for s in SIZES], "workloads": {}}
    for cfg in args.configs.split(","):
        wl = workload(cfg)
        module, n, w, h, batch = wl["module"], wl["n"], wl["w"], wl["h"], wl["batch"]
        assert batch >= COUNT and (w, h) == SIZES[0], (cfg, batch, w, h)
        p = g.default_params(module, n=n, w=w, h=h)
        p.lazy_smooth = 1
        nsnap = 4
        pcm = synth_batch_int16(0, batch, 0, n + nsnap * HOP).astype(np.float32) / np.float32(65535)
        dev_l = [torch.from_numpy(np.ascontiguousarray(pcm[:, (i + 1) * HOP:(i + 1) * HOP + n, 0])).cuda() for i in range(nsnap)]
        dev_r = [torch.from_numpy(np.ascontiguousarray(pcm[:, (i + 1) * HOP:(i + 1) * HOP + n, 1])).cuda() for i in range(nsnap)]
        rungs = [dict(size=s) for s in SIZES]
        with g.Renderer(p, batch=batch) as r:
            st = torch.cuda.ExternalStream(r.cuda_stream)
            for i in range(5):
                r.update_device(dev_l[i % nsnap].data_ptr(), dev_r[i % nsnap].data_ptr(), True)
            r.sync()
            streams = list(range(COUNT))
            outs = {}

            def run(leg):
                if leg == "ladder":
                    outs[leg] = r.export_ladder(streams, rungs, out=outs.get(leg))
                else:
                    prev = outs.get(leg) or [None] * len(SIZES)
                    outs[leg] = [r.export_frames(streams, "nv12", out=prev[0])] + \
                                [r.export_scaled(streams, s, fmt="nv12", out=prev[j]) for j, s in enumerate(SIZES) if j]

            legs_order = ("ladder", "four_calls")
            for leg in legs_order:                            # allocates, warms the list buffers, the schedule and the kernels
                run(leg)
            torch.cuda.synchronize()
            for j in range(len(SIZES)):                       # the same bytes either way
                assert torch.equal(outs["ladder"][j], outs["four_calls"][j]), (cfg, j)
            frac = read_fraction(g, r, p, module, np.linspace(0, batch - 1, 32).astype(int))
            times = {leg: [] for leg in legs_order}
            for _ in range(args.rounds):
                for leg in legs_order:
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    r.sync()
                    a.record(st)
                    for _ in range(args.reps):
                        run(leg)
                    b.record(st)
                    b.synchronize()
                    times[leg].append(a.elapsed_time(b) / args.reps)
            wbytes = COUNT * sum(ow * oh * 1.5 for ow, oh in SIZES)
            rframe = COUNT * w * h * 4.0 * frac
            legs = {}
            for leg in legs_order:
                ms = float(np.median(times[leg]))
                rbytes = rframe * (1 if leg == "ladder" else len(SIZES))
                gbs = (wbytes + rbytes) / (ms / 1e3) / 1e9
                legs[leg] = {"ms": ms, "ms_all": times[leg], "write_bytes": wbytes, "read_bytes": rbytes, "gbs": gbs,
                             "frac_of_peak": gbs / peak, "floor_ms": (wbytes + rbytes) / (peak * 1e9) * 1e3}
            legs["speedup"] = legs["four_calls"]["ms"] / legs["ladder"]["ms"]
        result["workloads"][cfg] = {"module": module, "n": n, "w": w, "h": h, "batch": batch, "read_fraction": frac, "legs": legs}
        print(cfg, json.dumps({k: (round(v["ms"], 4) if isinstance(v, dict) else round(v, 3)) for k, v in legs.items()}), flush=True)
    text = json.dumps(result, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
