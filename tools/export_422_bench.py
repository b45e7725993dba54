"""4:2:2 export and overlay rates (YUV422P, YUV422P10 and UYVY, DESIGN 4.18) on one GPU, with the card and its power limit
read in the same run.  Per workload (bench.py's inputs and warm-up), CUDA-event time of exporting 1024 streams whole-frame
and scaled to 480x270 in YUV422P, YUV422P10 and UYVY beside I420, YUV420P10 and YUV444; of overlay_planes onto 1024 pictures
in YUV422P10 beside YUV420P10 (the pictures are the whole-frame export buffers); and of what a caller does without the new formats: an RGBA export (composited) followed by a
torch conversion to yuv422p, whose bytes differ from the library's and which is reported as a time only.  Legs are
alternated over rounds and every time is the median of the rounds.  Before timing it checks on the device that UYVY is
YUV422P interleaved and that YUV422P's Y is I420's.

    python tools/export_422_bench.py --out profiles/h100_export_422.json [--configs headline,radial1080]
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import HOP, workload                # noqa: E402  (stdlib only at import time)
from tools.style_bench import card             # noqa: E402

COUNT = 1024
FORMATS = ("yuv422p", "yuv422p10", "uyvy", "i420", "yuv420p10", "yuv444")
OVERLAY = ("yuv422p10", "yuv420p10")
THUMB = (480, 270)
BYTES_PER_PIXEL = {"yuv422p": 2.0, "yuv422p10": 4.0, "uyvy": 2.0, "i420": 1.5, "yuv420p10": 3.0, "yuv444": 3.0}


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
            legs = [(k, f) for k in ("whole", "scaled") for f in FORMATS]
            outs = {}
            for kind, fmt in legs:                           # one [count, rows, pitch] buffer per leg, as _export_plan lays it out
                ow, oh = (w, h) if kind == "whole" else THUMB
                rows, row_bytes, align = g.api._export_layout(fmt, ow, oh)
                outs[(kind, fmt)] = torch.empty((count, rows, (row_bytes + align - 1) // align * align), dtype=torch.uint8,
                                                device=f"cuda:{r.device}")
            calls = {}
            for kind, fmt in legs:
                if kind == "whole":
                    calls[f"whole_{fmt}"] = (lambda o: lambda: r.export_frames(streams, o[1], out=outs[o]))((kind, fmt))
                else:
                    calls[f"scaled_{fmt}"] = (lambda o: lambda: r.export_scaled(streams, THUMB, fmt=o[1], out=outs[o]))((kind, fmt))
            # the caller's workaround: RGBA composited over black, then BT.709 limited-range yuv422p in torch, 32 frames at a time
            rgba = torch.empty((count, h, w * 4), dtype=torch.uint8, device=f"cuda:{r.device}")
            dst = g.api._export_views("yuv422p", outs[("whole", "yuv422p")], w, h)
            kr, kb = 0.2126, 0.0722
            ky = torch.tensor([kr, 1 - kr - kb, kb], device="cuda") * (219 / 255)

            def caller():
                r.export_frames(streams, "rgba", over=True, out=rgba)
                for c in range(0, count, 32):
                    src = rgba[c:c + 32].view(-1, h, w, 4)[..., :3].float()
                    dst[0][c:c + 32].copy_((src @ ky + 16).round().clamp(0, 255).to(torch.uint8))
                    m = (src[:, :, 0::2] + src[:, :, 1::2]) * 0.5
                    yp = m @ (ky * (255 / 219))
                    dst[1][c:c + 32].copy_((128 + (m[..., 2] - yp) * (224 / 255) / (2 * (1 - kb))).round().clamp(0, 255).to(torch.uint8))
                    dst[2][c:c + 32].copy_((128 + (m[..., 0] - yp) * (224 / 255) / (2 * (1 - kr))).round().clamp(0, 255).to(torch.uint8))
            calls["whole_caller_rgba_torch_yuv422p"] = caller
            # overlay_planes onto pictures of random samples (padding bits included), one [count, ...] set per format
            pics = {}
            for fmt in OVERLAY:                              # the whole-frame export buffers, refilled (exports overwrite them)
                planes = g.api._export_views(fmt, outs[("whole", fmt)], w, h)
                for t in planes:
                    for c in range(0, count, 64):
                        t[c:c + 64].copy_(torch.randint(0, 1 << 16, t[c:c + 64].shape, dtype=torch.int32, device="cuda").to(t.dtype))
                s, desc, arr = r._planes_plan(streams, planes, None, fmt)
                pics[fmt] = (planes, s, desc, arr)
                calls[f"overlay_{fmt}"] = (lambda f: lambda: g.api._check(r._L.glava_b200_overlay_planes(
                    r._h, pics[f][1].ctypes.data, count, pics[f][3], C.byref(pics[f][2]), None, None)))(fmt)
            for f in calls.values():                         # warms the list buffers and the kernels
                f()
            torch.cuda.synchronize()
            for kind in ("whole", "scaled"):
                ow, oh = (w, h) if kind == "whole" else THUMB
                y, cb, cr = g.api._export_views("yuv422p", outs[(kind, "yuv422p")], ow, oh)
                if kind == "whole":                          # the caller leg wrote this buffer: export it again
                    r.export_frames(streams, "yuv422p", out=outs[(kind, "yuv422p")])
                    torch.cuda.synchronize()
                u = g.api._export_views("uyvy", outs[(kind, "uyvy")], ow, oh)
                assert torch.equal(u[..., 1::2], y) and torch.equal(u[..., 0::4], cb) and torch.equal(u[..., 2::4], cr), kind
                assert torch.equal(y, g.api._export_views("i420", outs[(kind, "i420")], ow, oh)[0]), kind
            times = {k: [] for k in calls}
            cur = torch.cuda.current_stream()
            st = torch.cuda.ExternalStream(r.cuda_stream)
            for _ in range(args.rounds):
                for key, f in calls.items():
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    r.sync()
                    torch.cuda.synchronize()
                    s = st if key.startswith("overlay") else cur   # the raw overlay call is not ordered against torch's stream
                    a.record(s)
                    for _ in range(args.reps):
                        f()
                    b.record(s)
                    b.synchronize()
                    times[key].append(a.elapsed_time(b) / args.reps)
            res = {}
            for key in calls:
                ms = float(np.median(times[key]))
                res[key] = {"ms": ms, "ms_all": times[key]}
                kind, fmt = key.split("_", 1)
                # written bytes of the exports only: the overlay writes only the quads that are not zero
                if kind in ("whole", "scaled") and fmt in BYTES_PER_PIXEL:
                    ow, oh = (w, h) if kind == "whole" else THUMB
                    wbytes = count * ow * oh * BYTES_PER_PIXEL[fmt]
                    res[key].update(write_bytes=wbytes, write_gbs=wbytes / (ms / 1e3) / 1e9)
            del pics, outs, rgba
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
