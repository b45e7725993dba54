"""Frame export rates per output format (glava_b200_export_frames and _export_scaled, DESIGN 4.14) on one GPU, with the card
and its power limit read in the same run.  Per workload (bench.py's inputs and warm-up), CUDA-event time of exporting 1024
streams whole-frame to NV12, I420, YUV444, P010 and RGBA, and scaled to 480x270 in the four YUV formats, legs alternated over
rounds; bytes written per call computed from the formats' layouts.  Before timing it checks on the device that I420's planes
are the deinterleaved NV12 CbCr plane and YUV444's Y plane NV12's.

    python tools/export_formats_bench.py --out profiles/h100_export_formats.json [--configs headline,radial1080]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import HOP, workload                # noqa: E402  (stdlib only at import time)
from tools.style_bench import card             # noqa: E402

COUNT = 1024
WHOLE = ("nv12", "i420", "yuv444", "p010", "rgba")
SCALED = ("nv12", "i420", "yuv444", "p010")
THUMB = (480, 270)
BYTES_PER_PIXEL = {"nv12": 1.5, "i420": 1.5, "yuv444": 3.0, "p010": 3.0, "rgba": 4.0}


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
    result = {"gpu": name, "power_limit": limit, "count": COUNT, "reps": args.reps, "rounds": args.rounds, "workloads": {}}
    for cfg in args.configs.split(","):
        wl = workload(cfg)
        module, n, w, h, batch = wl["module"], wl["n"], wl["w"], wl["h"], wl["batch"]
        p = g.default_params(module, n=n, w=w, h=h)
        p.lazy_smooth = 1
        pcm = synth_batch_int16(0, batch, 0, n + HOP).astype(np.float32) / np.float32(65535)
        dl = torch.from_numpy(np.ascontiguousarray(pcm[:, HOP:HOP + n, 0])).cuda()
        dr = torch.from_numpy(np.ascontiguousarray(pcm[:, HOP:HOP + n, 1])).cuda()
        count = min(COUNT, batch)
        with g.Renderer(p, batch=batch) as r:
            st = torch.cuda.ExternalStream(r.cuda_stream)
            for _ in range(5):
                r.update_device(dl.data_ptr(), dr.data_ptr(), True)
            r.sync()
            legs = [("whole", f) for f in WHOLE] + [("scaled", f) for f in SCALED]
            outs = {}
            for kind, fmt in legs:                           # one [count, rows, pitch] buffer per leg, as _export_plan lays it out
                ow, oh = (w, h) if kind == "whole" else THUMB
                rows, row_bytes, align = g.api._export_layout(fmt, ow, oh)
                outs[(kind, fmt)] = torch.empty((count, rows, (row_bytes + align - 1) // align * align), dtype=torch.uint8,
                                                device=f"cuda:{r.device}")

            def run(kind, fmt):
                if kind == "whole":
                    r.export_frames(range(count), fmt, out=outs[(kind, fmt)])
                else:
                    r.export_scaled(range(count), THUMB, fmt=fmt, out=outs[(kind, fmt)])

            for kind, fmt in legs:                           # warms the list buffers and the kernels
                run(kind, fmt)
            torch.cuda.synchronize()
            view = lambda fmt: g.api._export_views(fmt, outs[("whole", fmt)], w, h)
            nv12, (yp, cb, cr), y4 = view("nv12"), view("i420"), view("yuv444")[0]
            assert torch.equal(yp, nv12[:, :h]) and torch.equal(y4, nv12[:, :h])
            assert torch.equal(cb, nv12[:, h:, 0::2]) and torch.equal(cr, nv12[:, h:, 1::2])
            times = {f"{k}_{f}": [] for k, f in legs}
            for _ in range(args.rounds):
                for kind, fmt in legs:
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    r.sync()
                    a.record(st)
                    for _ in range(args.reps):
                        run(kind, fmt)
                    b.record(st)
                    b.synchronize()
                    times[f"{kind}_{fmt}"].append(a.elapsed_time(b) / args.reps)
            res = {}
            for kind, fmt in legs:
                k = f"{kind}_{fmt}"
                ms = float(np.median(times[k]))
                ow, oh = (w, h) if kind == "whole" else THUMB
                wbytes = count * ow * oh * BYTES_PER_PIXEL[fmt]
                res[k] = {"ms": ms, "ms_all": times[k], "write_bytes": wbytes, "write_gbs": wbytes / (ms / 1e3) / 1e9}
        result["workloads"][cfg] = {"module": module, "n": n, "w": w, "h": h, "batch": batch, "count": count, "legs": res}
        print(cfg, json.dumps({k: round(v["ms"], 4) for k, v in res.items()}), flush=True)
    text = json.dumps(result, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
