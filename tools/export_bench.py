"""Frame export rates (glava_b200_export_frames, DESIGN 4.10) on one GPU, with the card and its power limit read in the same
run.  Per workload (bench.py's inputs and warm-up), CUDA-event time of exporting 1024 and 64 streams to NV12 and to RGBA
and one composited RGBA leg, legs alternated over rounds; the bytes the export moves (writes, plus the rows the dirty-row
marks let it read, counted from the read-back frames of a stream sample as tools/stored_bytes.py counts content rows) over
kernel time against MEASURED_PEAKS.json hbm_gbs; and the step time of a device-resident update loop with and without an
NV12 export of 64 streams per step, alternated.

    python tools/export_bench.py --out profiles/h100_export.json [--configs headline,radial1080 --reps 20 --rounds 3]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import HOP, hbm_peak, workload      # noqa: E402  (stdlib only at import time)
from tools.stored_bytes import content_rows, STRIP   # noqa: E402
from tools.style_bench import card             # noqa: E402

LEGS = (("nv12", False, 1024), ("nv12", False, 64), ("rgba", False, 1024), ("rgba", False, 64), ("rgba", True, 1024))


def read_fraction(g, r, p, module, sample):
    """share of the framebuffer rows the export reads: the content rows of each strip (bars / graph / wave keep marks),
    else every row"""
    import numpy as np
    if module not in ("bars", "graph", "wave"):
        return 1.0
    flip = module == "bars" and bool(p.bars_flip)
    w, h = p.w, p.h
    strip_w = np.minimum(STRIP, w - STRIP * np.arange((w + STRIP - 1) // STRIP))
    rows = 0
    for s in sample:
        lo, hi = content_rows(r.readback(int(s)), module, flip)
        rows += int((np.maximum(hi - lo, 0) * strip_w).sum())
    return rows / (len(sample) * w * h)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--configs", default="headline,radial1080")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import torch
    import glava_b200 as g
    from glava_b200.synth import synth_batch_int16

    name, limit = card()
    peak, peak_src = hbm_peak()
    result = {"gpu": name, "power_limit": limit, "peak_gbs": peak, "peak_source": peak_src, "reps": args.reps,
              "rounds": args.rounds, "workloads": {}}
    for cfg in args.configs.split(","):
        wl = workload(cfg)
        module, n, w, h, batch = wl["module"], wl["n"], wl["w"], wl["h"], wl["batch"]
        p = g.default_params(module, n=n, w=w, h=h)
        p.lazy_smooth = 1
        nsnap = 4
        pcm = synth_batch_int16(0, batch, 0, n + nsnap * HOP).astype(np.float32) / np.float32(65535)
        dev_l = [torch.from_numpy(np.ascontiguousarray(pcm[:, (i + 1) * HOP:(i + 1) * HOP + n, 0])).cuda() for i in range(nsnap)]
        dev_r = [torch.from_numpy(np.ascontiguousarray(pcm[:, (i + 1) * HOP:(i + 1) * HOP + n, 1])).cuda() for i in range(nsnap)]
        with g.Renderer(p, batch=batch) as r:
            st = torch.cuda.ExternalStream(r.cuda_stream)
            step = [0]

            def update():
                i = step[0] % nsnap
                r.update_device(dev_l[i].data_ptr(), dev_r[i].data_ptr(), True)
                step[0] += 1

            for _ in range(5):
                update()
            r.sync()
            outs = {}
            for fmt, over, count in LEGS:
                key = (fmt, count)
                if key not in outs:
                    outs[key] = r.export_frames(range(count), fmt)        # allocates, warms the list buffers and the kernel
            torch.cuda.synchronize()
            frac = read_fraction(g, r, p, module, np.linspace(0, batch - 1, 32).astype(int))
            times = {f"{fmt}{'_over' if over else ''}_{count}": [] for fmt, over, count in LEGS}
            for _ in range(args.rounds):
                for fmt, over, count in LEGS:
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    out = outs[(fmt, count)]
                    r.sync()
                    a.record(st)
                    for _ in range(args.reps):
                        r.export_frames(range(count), fmt, over=over, out=out)
                    b.record(st)
                    b.synchronize()
                    times[f"{fmt}{'_over' if over else ''}_{count}"].append(a.elapsed_time(b) / args.reps)
            legs = {}
            for fmt, over, count in LEGS:
                k = f"{fmt}{'_over' if over else ''}_{count}"
                ms = float(np.median(times[k]))
                wbytes = count * w * h * (1.5 if fmt == "nv12" else 4.0)
                rbytes = count * w * h * 4.0 * frac
                legs[k] = {"ms": ms, "ms_all": times[k], "write_bytes": wbytes, "read_bytes": rbytes,
                           "gbs": (wbytes + rbytes) / (ms / 1e3) / 1e9, "frac_of_peak": (wbytes + rbytes) / (ms / 1e3) / 1e9 / peak,
                           "frames_per_s": count / (ms / 1e3)}
            # step time of the update loop with and without an NV12 export of 64 streams per step, alternated
            out64 = outs[("nv12", 64)]
            loop = {"updates": [], "updates_plus_export64": []}
            for _ in range(args.rounds):
                for leg in loop:
                    for _ in range(3):
                        update()
                    r.sync()
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record(st)
                    for _ in range(args.steps):
                        update()
                        if leg != "updates":
                            r.export_frames(range(64), "nv12", out=out64)
                    b.record(st)
                    b.synchronize()
                    loop[leg].append(a.elapsed_time(b) / args.steps)
            med = {k: float(np.median(v)) for k, v in loop.items()}
        result["workloads"][cfg] = {"module": module, "n": n, "w": w, "h": h, "batch": batch,
                                    "read_fraction": frac, "legs": legs,
                                    "step_ms": {"all": loop, "median": med,
                                                "export64_added_ms": med["updates_plus_export64"] - med["updates"]}}
        print(cfg, json.dumps({k: round(v["ms"], 4) for k, v in legs.items()}), json.dumps(med), flush=True)
    text = json.dumps(result, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
