"""Planar 10-bit export rates (glava_b200_export_frames and _export_scaled in YUV420P10 / YUV444P10, DESIGN 4.16) on one GPU,
with the card and its power limit read in the same run.  Per workload (bench.py's inputs and warm-up), CUDA-event time of
exporting 1024 streams whole-frame and scaled to 480x270 in YUV420P10, YUV444P10, P010 and YUV444, and of what a caller does
without the new formats: a P010 export followed by a torch shift-and-deinterleave into a yuv420p10le buffer.  Legs are
alternated over rounds and every time is the median of the rounds.  Before timing it checks on the device that YUV420P10 is
P010 deinterleaved and >> 6, that YUV444P10's Y is the same, and that the caller-side conversion gives the same bytes.

    python tools/export_p10_bench.py --out profiles/h100_export_p10.json [--configs headline,radial1080]
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
FORMATS = ("yuv420p10", "yuv444p10", "p010", "yuv444")
THUMB = (480, 270)
BYTES_PER_PIXEL = {"yuv420p10": 3.0, "yuv444p10": 6.0, "p010": 3.0, "yuv444": 3.0}


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
            for _ in range(5):
                r.update_device(dl.data_ptr(), dr.data_ptr(), True)
            r.sync()
            legs = [(k, f) for k in ("whole", "scaled") for f in FORMATS] + [("whole", "caller"), ("scaled", "caller")]
            outs = {}
            for kind, fmt in legs:                           # one [count, rows, pitch] buffer per leg, as _export_plan lays it out
                ow, oh = (w, h) if kind == "whole" else THUMB
                rows, row_bytes, align = g.api._export_layout("yuv420p10" if fmt == "caller" else fmt, ow, oh)
                outs[(kind, fmt)] = torch.empty((count, rows, (row_bytes + align - 1) // align * align), dtype=torch.uint8,
                                                device=f"cuda:{r.device}")

            def run(kind, fmt):
                ow, oh = (w, h) if kind == "whole" else THUMB
                if fmt == "caller":                          # P010, then shift and deinterleave into yuv420p10le planes
                    run(kind, "p010")
                    q = g.api._export_views("p010", outs[(kind, "p010")], ow, oh).view(torch.int16)
                    # int16 views (torch has no uint16 shifts): shift, then clear the sign bits the shift copies in
                    for src, dst in zip((q[:, :oh], q[:, oh:, 0::2], q[:, oh:, 1::2]),
                                        g.api._export_views("yuv420p10", outs[(kind, fmt)], ow, oh)):
                        d = dst.view(torch.int16)
                        torch.bitwise_right_shift(src, 6, out=d)
                        d.bitwise_and_(1023)
                elif kind == "whole":
                    r.export_frames(range(count), fmt, out=outs[(kind, fmt)])
                else:
                    r.export_scaled(range(count), THUMB, fmt=fmt, out=outs[(kind, fmt)])

            for kind, fmt in legs:                           # warms the list buffers and the kernels
                run(kind, fmt)
            torch.cuda.synchronize()
            for kind in ("whole", "scaled"):
                ow, oh = (w, h) if kind == "whole" else THUMB
                view = lambda fmt: g.api._export_views(fmt, outs[(kind, fmt)], ow, oh)
                s16 = lambda t: t.view(torch.int16)
                code = lambda t: (s16(t) >> 6) & 1023
                q, (y, cb, cr), y4 = view("p010"), view("yuv420p10"), view("yuv444p10")[0]
                assert torch.equal(s16(y), code(q[:, :oh])) and torch.equal(s16(y4), s16(y)), kind
                assert torch.equal(s16(cb), code(q[:, oh:, 0::2])) and torch.equal(s16(cr), code(q[:, oh:, 1::2])), kind
                assert all(torch.equal(s16(a), s16(b)) for a, b in
                           zip(g.api._export_views("yuv420p10", outs[(kind, "caller")], ow, oh), (y, cb, cr))), kind
            times = {f"{k}_{f}": [] for k, f in legs}
            cur = torch.cuda.current_stream()
            for _ in range(args.rounds):
                for kind, fmt in legs:
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    r.sync()
                    torch.cuda.synchronize()
                    a.record(cur)                            # every export is ordered against torch's current stream
                    for _ in range(args.reps):
                        run(kind, fmt)
                    b.record(cur)
                    b.synchronize()
                    times[f"{kind}_{fmt}"].append(a.elapsed_time(b) / args.reps)
            res = {}
            for kind, fmt in legs:
                k = f"{kind}_{fmt}"
                ms = float(np.median(times[k]))
                ow, oh = (w, h) if kind == "whole" else THUMB
                wbytes = count * ow * oh * BYTES_PER_PIXEL["yuv420p10" if fmt == "caller" else fmt]
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
