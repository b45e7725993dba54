"""Transparent export rates (YUVA420P, YUVA444P10 and straight RGBA, DESIGN 4.19) on one GPU, with the card and its power
limit read in the same run.  Per workload (bench.py's inputs and warm-up), CUDA-event time of exporting 1024 streams
whole-frame and scaled to 480x270 in YUVA420P, YUVA444P10 and straight RGBA beside I420, YUV444P10 and RGBA (stored
channels, no composite).  Every whole-frame leg writes into one shared buffer (the legs never run at once), so that the
six fit beside a 1024-stream 1080p framebuffer.  Legs are alternated over rounds and every time is the median of the
rounds.  Before timing it checks on the device that straight RGBA of an opaque pixel is the pixel and that YUVA's A
plane is the stored alpha.

    python tools/export_alpha_bench.py --out profiles/h100_export_alpha.json [--configs headline,radial1080]
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
# (leg name, format, export keywords, written bytes per pixel)
LEGS = (("yuva420p", "yuva420p", {}, 2.5), ("yuva444p10", "yuva444p10", {}, 8.0), ("rgba_straight", "rgba", {"straight": True}, 4.0),
        ("i420", "i420", {}, 1.5), ("yuv444p10", "yuv444p10", {}, 6.0), ("rgba", "rgba", {}, 4.0))
THUMB = (480, 270)


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
        streams = list(range(count))
        with g.Renderer(p, batch=batch) as r:
            for _ in range(5):
                r.update_device(dl.data_ptr(), dr.data_ptr(), True)
            r.sync()
            shapes = {}
            for kind in ("whole", "scaled"):
                ow, oh = (w, h) if kind == "whole" else THUMB
                for leg, fmt, _, _ in LEGS:
                    rows, row_bytes, align = g.api._export_layout(fmt, ow, oh)
                    shapes[(kind, leg)] = (count, rows, (row_bytes + align - 1) // align * align)
            bufs = {k: torch.empty(max(int(np.prod(s)) for (kk, _), s in shapes.items() if kk == k), dtype=torch.uint8,
                                   device=f"cuda:{r.device}") for k in ("whole", "scaled")}
            outs = {key: bufs[key[0]][:int(np.prod(s))].view(s) for key, s in shapes.items()}
            calls = {}
            for leg, fmt, kw, _ in LEGS:
                calls[f"whole_{leg}"] = (lambda o, f, k: lambda: r.export_frames(streams, f, out=o, **k))(outs[("whole", leg)], fmt, kw)
                calls[f"scaled_{leg}"] = (lambda o, f, k: lambda: r.export_scaled(streams, THUMB, fmt=f, out=o, **k))(
                    outs[("scaled", leg)], fmt, kw)
            for f in calls.values():                         # warms the list buffers and the kernels
                f()
            torch.cuda.synchronize()
            # on the device: A is the stored alpha, and straight RGBA keeps opaque pixels and every alpha byte
            rgba = r.export_frames(streams[:8], "rgba")
            st = r.export_frames(streams[:8], "rgba", straight=True)
            a = r.export_frames(streams[:8], "yuva420p")[3]
            assert torch.equal(a, rgba[..., 3]) and torch.equal(st[..., 3], rgba[..., 3])
            opaque = rgba[..., 3] == 255
            assert torch.equal(st[opaque], rgba[opaque]), cfg
            del rgba, st, a
            times = {k: [] for k in calls}
            cur = torch.cuda.current_stream()
            for _ in range(args.rounds):
                for key, f in calls.items():
                    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    r.sync()
                    torch.cuda.synchronize()
                    t0.record(cur)
                    for _ in range(args.reps):
                        f()
                    t1.record(cur)
                    t1.synchronize()
                    times[key].append(t0.elapsed_time(t1) / args.reps)
            res = {}
            bpp = {leg: b for leg, _, _, b in LEGS}
            for key in calls:
                ms = float(np.median(times[key]))
                kind, leg = key.split("_", 1)
                ow, oh = (w, h) if kind == "whole" else THUMB
                wbytes = count * ow * oh * bpp[leg]
                res[key] = {"ms": ms, "ms_all": times[key], "write_bytes": wbytes, "write_gbs": wbytes / (ms / 1e3) / 1e9}
            del outs, bufs
            torch.cuda.empty_cache()
        result["workloads"][cfg] = {"module": module, "n": n, "w": w, "h": h, "batch": batch, "count": count, "legs": res}
        print(cfg, json.dumps({k: round(v["ms"], 4) for k, v in res.items()}), flush=True)
    text = json.dumps(result, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
