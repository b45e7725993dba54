"""Overlay rates (glava_b200_overlay_frames, DESIGN 4.12) on one GPU, with the card and its power limit read in the same run.
Per workload (bench.py's inputs and warm-up), device time (torch.profiler: every kernel and copy a leg enqueues, per call;
the CUDA-event wall time beside it) of 1024 streams composited onto same-size images, legs
alternated over rounds: the overlay in NV12 and RGBA, export_frames of the same streams in NV12 and RGBA, and the
caller-side baseline: an RGBA export into scratch followed by a torch blend onto the images.  Bytes per call = the framebuffer rows the marks let through
(counted from read-back frames of a stream sample as tools/export_bench.py counts them; every row for modules without
marks) plus the destination bytes read and written, over the median time, against the data sheet's 3.35 TB/s unless
MEASURED_PEAKS.json gives a peak.  Overlay legs count the destination bytes under non-zero quads twice (read and written).

    python tools/overlay_bench.py --out profiles/h100_overlay.json [--configs headline,radial1080 --reps 20 --rounds 3]
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import HOP, hbm_peak, workload      # noqa: E402  (stdlib only at import time)
from tools.export_bench import read_fraction   # noqa: E402
from tools.style_bench import card             # noqa: E402

# (name, kind, format): kind "overlay", "export" (export_frames), "baseline"
LEGS = (("overlay_nv12", "overlay", "nv12"), ("export_nv12", "export", "nv12"), ("overlay_rgba", "overlay", "rgba"),
        ("export_rgba", "export", "rgba"), ("baseline_rgba", "baseline", "rgba"))
COUNT = 1024


def touched_fraction(r, sample):
    """the share of the destination an overlay reads and writes under native opacity: RGBA / BGRA, the 4-pixel quads of a
    row that hold a non-zero pixel; NV12, the quads of a row pair (eight pixels) that do, from read-back frames"""
    import numpy as np
    rgba = nv12 = 0.0
    for s in sample:
        f = r.readback(int(s)).view(np.uint32)[..., 0]                 # [h][w] words
        h, w = f.shape
        q = np.pad(f, ((0, h % 2), (0, -w % 4))).reshape(h + h % 2, -1, 4).any(axis=-1)
        rgba += q[:h].mean()
        nv12 += (q[0::2] | q[1::2]).mean()
    return {"rgba": rgba / len(sample), "nv12": nv12 / len(sample)}


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
            imgs = {"nv12": torch.randint(0, 256, (COUNT, h * 3 // 2, w), dtype=torch.uint8, device="cuda"),
                    "rgba": torch.randint(0, 256, (COUNT, h, w, 4), dtype=torch.uint8, device="cuda")}
            imgs["rgba"][..., 3] = 255
            calls = {}

            def plan(leg):
                """the leg as one call with everything Python decides computed once (host time then stays off the clock)"""
                key, kind, fmt = leg
                if kind == "overlay":
                    s, desc, dst, uv = r._overlay_plan(streams, imgs[fmt], None, fmt)

                    def call():
                        g.api._check(r._L.glava_b200_overlay_frames(r._h, s.ctypes.data, COUNT, dst, uv, C.byref(desc), None, None))
                    return call
                out = r.export_frames(streams, "rgba" if kind == "baseline" else fmt)
                s, desc, dst, _ = r._export_plan(streams, "rgba" if kind == "baseline" else fmt, False, (0, 0, 0), out, lambda x: r.device)

                def export():
                    g.api._check(r._L.glava_b200_export_frames(r._h, s.ctypes.data, COUNT, dst, C.byref(desc), None, None))
                if kind == "export":
                    return export

                def baseline():                                # RGBA scratch, then premultiplied "over" in torch
                    export()
                    with torch.cuda.stream(st):
                        for c in range(0, COUNT, 64):         # 64 frames at a time bound the int32 temporaries
                            d, sc = imgs["rgba"][c:c + 64], out[c:c + 64]
                            ia = 255 - sc[..., 3:].to(torch.int32)
                            d.copy_(torch.clamp(sc.to(torch.int32) + (2 * d.to(torch.int32) * ia + 255) // 510, max=255).to(torch.uint8))
                return baseline

            for leg in LEGS:                                  # allocates, warms the list buffers and the kernels
                calls[leg[0]] = plan(leg)
                calls[leg[0]]()
            torch.cuda.synchronize()
            sample = np.linspace(0, batch - 1, 32).astype(int)
            frac = read_fraction(g, r, p, module, sample)
            touch = touched_fraction(r, sample)
            times = {leg[0]: [] for leg in LEGS}
            walls = {leg[0]: [] for leg in LEGS}
            for _ in range(args.rounds):
                for leg in LEGS:
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
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
            for key, kind, fmt in LEGS:
                ms = float(np.median(times[key]))
                fb = COUNT * w * h * 4.0 * frac                # framebuffer rows the marks let through
                img = COUNT * w * h * (1.5 if fmt == "nv12" else 4.0)
                if kind == "export":
                    nbytes = fb + img
                elif kind == "baseline":                      # export into scratch, then read scratch and image, write image
                    nbytes = fb + img + 3 * img
                else:                                          # destination bytes under non-zero quads, read and written
                    nbytes = fb + 2 * img * touch[fmt]
                gbs = nbytes / (ms / 1e3) / 1e9
                legs[key] = {"ms": ms, "ms_all": times[key], "wall_ms": float(np.median(walls[key])), "bytes": nbytes, "gbs": gbs, "frac_of_peak": gbs / peak,
                             "frames_per_s": COUNT / (ms / 1e3)}
        result["workloads"][cfg] = {"module": module, "n": n, "w": w, "h": h, "batch": batch, "read_fraction": frac,
                                    "touched_fraction": touch, "legs": legs}
        print(cfg, json.dumps({k: [round(v["ms"], 4), round(v["frac_of_peak"], 3)] for k, v in legs.items()}), flush=True)
    text = json.dumps(result, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
