"""Scaled overlay rates (glava_b200_overlay_scaled, DESIGN 4.21) on one GPU, with the card and its power limit read in the
same run.  Per workload (bench.py's inputs and warm-up), device time (torch.profiler: every kernel and copy a leg enqueues,
per call; the CUDA-event wall time beside it) of 1024 streams onto 1080p pictures, legs alternated over rounds: the scaled
overlay of the whole frame at a third of its size (both workloads render 1920x1080, so 640x360) at the bottom right of each
picture, NV12 and RGBA, under native opacity at K = 255 and K = 128 and under any other opacity (a second
renderer of the workload with premultiply_alpha = 0); export_scaled of the same rectangle to NV12 and RGBA; and the plain
full-size overlay (glava_b200_overlay_frames) of the frame into the same pictures.

    python tools/overlay_scaled_bench.py --out profiles/h100_overlay_scaled.json [--configs headline,radial1080 --reps 20]
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import HOP, workload               # noqa: E402  (stdlib only at import time)
from tools.style_bench import card            # noqa: E402

# (name, kind, renderer, format, K)
LEGS = tuple([(f"scaled_{op}_k{k}_{fmt}", "scaled", op, fmt, k) for fmt in ("nv12", "rgba")
              for op, k in (("native", 255), ("native", 128), ("opaque", 255))]
             + [(f"export_scaled_{fmt}", "export", "native", fmt, None) for fmt in ("nv12", "rgba")]
             + [(f"plain_overlay_{fmt}", "plain", "native", fmt, None) for fmt in ("nv12", "rgba")])
COUNT = 1024
PW, PH = 1920, 1080                           # the pictures


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
    result = {"gpu": name, "power_limit": limit, "reps": args.reps, "rounds": args.rounds, "count": COUNT,
              "picture": [PW, PH], "workloads": {}}
    for cfg in args.configs.split(","):
        wl = workload(cfg)
        module, n, w, h, batch = wl["module"], wl["n"], wl["w"], wl["h"], wl["batch"]
        assert batch >= COUNT, (cfg, batch)
        ow, oh = w // 3 // 2 * 2, h // 3 // 2 * 2
        nsnap = 4
        pcm = synth_batch_int16(0, batch, 0, n + nsnap * HOP).astype(np.float32) / np.float32(65535)
        dev_l = [torch.from_numpy(np.ascontiguousarray(pcm[:, (i + 1) * HOP:(i + 1) * HOP + n, 0])).cuda() for i in range(nsnap)]
        dev_r = [torch.from_numpy(np.ascontiguousarray(pcm[:, (i + 1) * HOP:(i + 1) * HOP + n, 1])).cuda() for i in range(nsnap)]
        rs = {}
        for op in ("native", "opaque"):
            p = g.default_params(module, n=n, w=w, h=h)
            p.lazy_smooth = 1
            if op == "opaque":
                p.premultiply_alpha = 0
            rs[op] = g.Renderer(p, batch=batch)
            for i in range(5):
                rs[op].update_device(dev_l[i % nsnap].data_ptr(), dev_r[i % nsnap].data_ptr(), True)
            rs[op].sync()
        try:
            streams = list(range(COUNT))
            imgs = {"nv12": torch.randint(0, 256, (COUNT, PH * 3 // 2, PW), dtype=torch.uint8, device="cuda"),
                    "rgba": torch.randint(0, 256, (COUNT, PH, PW, 4), dtype=torch.uint8, device="cuda")}
            imgs["rgba"][..., 3] = 255
            at_small = [((PW - ow) // 16 * 16, (PH - oh) // 2 * 2)] * COUNT
            at_full = [((PW - w) // 16 * 16, (PH - h) // 2 * 2)] * COUNT
            outs = {"nv12": torch.empty((COUNT, oh * 3 // 2, ow), dtype=torch.uint8, device="cuda"),
                    "rgba": torch.empty((COUNT, oh, ow, 4), dtype=torch.uint8, device="cuda")}
            sc = g.api._export_scale((ow, oh), None)

            def plan(leg):
                """the leg as one call with everything Python decides computed once (host time then stays off the clock)"""
                _, kind, op, fmt, k = leg
                r = rs[op]
                s = np.arange(COUNT, dtype=np.int32)
                if kind == "export":
                    s, desc, dst, _ = r._export_plan(streams, fmt, False, (0, 0, 0), outs[fmt], lambda st: r.device, (ow, oh))
                    return lambda: g.api._check(r._L.glava_b200_export_scaled(r._h, s.ctypes.data, COUNT, dst, None, C.byref(desc),
                                                                               C.byref(sc), None, None))
                if kind == "plain":
                    s, desc, dst, uv = r._overlay_plan(streams, imgs[fmt], at_full, fmt)
                    return lambda: g.api._check(r._L.glava_b200_overlay_frames(r._h, s.ctypes.data, COUNT, dst, uv, C.byref(desc),
                                                                                None, None))
                s, desc, dst, uv = r._overlay_plan(streams, imgs[fmt], at_small, fmt, size=(ow, oh))
                pd, arr = r._frames_pictures(desc, dst, uv, COUNT)
                K = np.full(COUNT, k, np.uint8)
                return lambda: g.api._check(r._L.glava_b200_overlay_scaled(r._h, s.ctypes.data, COUNT, arr, C.byref(pd), C.byref(sc),
                                                                            K.ctypes.data, None, None))

            calls = {}
            for leg in LEGS:                                  # allocates, warms the list buffers and the kernels
                calls[leg[0]] = plan(leg)
                calls[leg[0]]()
            torch.cuda.synchronize()
            times = {leg[0]: [] for leg in LEGS}
            walls = {leg[0]: [] for leg in LEGS}
            for _ in range(args.rounds):
                for leg in LEGS:
                    st = torch.cuda.ExternalStream(rs[leg[2]].cuda_stream)
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    for r in rs.values():
                        r.sync()
                    torch.cuda.synchronize()
                    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                        a.record(st)
                        for _ in range(args.reps):
                            calls[leg[0]]()
                        b.record(st)
                        b.synchronize()
                    dev_us = sum(getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0)
                                 for e in prof.key_averages())
                    times[leg[0]].append(dev_us / 1e3 / args.reps)
                    walls[leg[0]].append(a.elapsed_time(b) / args.reps)
            legs = {}
            for key, kind, op, fmt, k in LEGS:
                ms = float(np.median(times[key]))
                legs[key] = {"ms": ms, "ms_all": times[key], "wall_ms": float(np.median(walls[key])), "kind": kind, "opacity": op,
                             "format": fmt, "K": k, "frames_per_s": COUNT / (ms / 1e3)}
        finally:
            for r in rs.values():
                r.close()
        result["workloads"][cfg] = {"module": module, "n": n, "w": w, "h": h, "batch": batch, "out": [ow, oh], "legs": legs}
        print(cfg, json.dumps({k: round(v["ms"], 4) for k, v in legs.items()}), flush=True)
    text = json.dumps(result, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
