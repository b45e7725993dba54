"""Overlay rates onto decoded pictures (glava_b200_overlay_planes, DESIGN 4.17) on one GPU, with the card and its power limit
read in the same run.  Per workload (bench.py's inputs and warm-up) and format, 1024 streams composited onto same-size
pictures of that format, one batched tensor per plane; device time (torch.profiler, per call) with the CUDA-event wall
time beside it, medians of `rounds` alternated rounds of `reps` calls.  Legs per format: the overlay, export_frames of the
same streams in the same format, for NV12 also glava_b200_overlay_frames (after checking both calls write the same bytes),
and for I420 and P010 the caller-side baseline: an RGBA export into scratch followed by a torch blend onto the planes.
Bytes as tools/overlay_bench.py counts them: the framebuffer rows the marks let through plus the picture bytes under
non-zero quads, read and written (the export: every picture byte written), against the data sheet's 3.35 TB/s unless
MEASURED_PEAKS.json gives a peak.

    python tools/overlay_planes_bench.py --out profiles/h100_overlay_planes.json [--configs headline,radial1080 --reps 20]
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
from tools.overlay_bench import touched_fraction   # noqa: E402
from tools.style_bench import card             # noqa: E402

FORMATS = ("nv12", "i420", "yuv444", "p010", "yuv420p10", "yuv444p10")
WIDE = ("p010", "yuv420p10", "yuv444p10")
COUNT = 1024


def picture_bytes(fmt, w, h):
    """bytes of one w x h picture"""
    return w * h * (2 if fmt in WIDE else 1) * (3 if fmt in ("yuv444", "yuv444p10") else 1.5)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--configs", default="headline,radial1080")
    ap.add_argument("--formats", default=",".join(FORMATS))
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
        p = g.default_params(module, n=n, w=w, h=h)
        p.lazy_smooth = 1
        nsnap = 4
        pcm = synth_batch_int16(0, batch, 0, n + nsnap * HOP).astype(np.float32) / np.float32(65535)
        dev_l = [torch.from_numpy(np.ascontiguousarray(pcm[:, (i + 1) * HOP:(i + 1) * HOP + n, 0])).cuda() for i in range(nsnap)]
        dev_r = [torch.from_numpy(np.ascontiguousarray(pcm[:, (i + 1) * HOP:(i + 1) * HOP + n, 1])).cuda() for i in range(nsnap)]
        out = {"module": module, "n": n, "w": w, "h": h, "batch": batch, "formats": {}}
        with g.Renderer(p, batch=batch) as r:
            st = torch.cuda.ExternalStream(r.cuda_stream)
            for i in range(5):
                r.update_device(dev_l[i % nsnap].data_ptr(), dev_r[i % nsnap].data_ptr(), True)
            r.sync()
            streams = list(range(COUNT))
            sample = np.linspace(0, batch - 1, 32).astype(int)
            frac = read_fraction(g, r, p, module, sample)
            touch = touched_fraction(r, sample)
            out["read_fraction"], out["touched_fraction"] = frac, touch
            for fmt in args.formats.split(","):
                planes = r.export_frames(streams, fmt)          # [COUNT, ...] planes of the format, refilled below
                planes = planes if isinstance(planes, tuple) else (planes[:, :h], planes[:, h:])
                for t in planes:                                 # random samples, padding bits included
                    t.copy_(torch.randint(0, 1 << (8 * t.element_size()), t.shape, dtype=torch.int32, device="cuda").to(t.dtype))
                s, desc, arr = r._planes_plan(streams, planes, None, fmt)
                legs = {}

                def planes_call():
                    g.api._check(r._L.glava_b200_overlay_planes(r._h, s.ctypes.data, COUNT, arr, C.byref(desc), None, None))
                legs["planes_" + fmt] = planes_call
                es, edesc, edst, ex = r._export_plan(streams, fmt, False, (0, 0, 0), None, lambda x: r.device)

                def export_call():
                    g.api._check(r._L.glava_b200_export_frames(r._h, es.ctypes.data, COUNT, edst, C.byref(edesc), None, None))
                legs["export_" + fmt] = export_call
                if fmt == "nv12":
                    img = torch.empty((COUNT, h * 3 // 2, w), dtype=torch.uint8, device="cuda")
                    twin = torch.cat([planes[0], planes[1]], dim=1).contiguous()
                    img.copy_(twin)
                    fs, fdesc, fdst, fuv = r._overlay_plan(streams, img, None, "nv12")
                    planes_call()
                    g.api._check(r._L.glava_b200_overlay_frames(r._h, fs.ctypes.data, COUNT, fdst, fuv, C.byref(fdesc), None, None))
                    r.sync()
                    same = bool(torch.equal(img, torch.cat([planes[0], planes[1]], dim=1)))
                    out.setdefault("nv12_both_calls_identical", same)
                    assert same, "overlay_frames and overlay_planes wrote different NV12 bytes"

                    def frames_call():
                        g.api._check(r._L.glava_b200_overlay_frames(r._h, fs.ctypes.data, COUNT, fdst, fuv, C.byref(fdesc), None, None))
                    legs["frames_nv12"] = frames_call
                if fmt in ("i420", "p010"):
                    scratch = r.export_frames(streams, "rgba")
                    ss, sdesc, sdst, _ = r._export_plan(streams, "rgba", False, (0, 0, 0), scratch, lambda x: r.device)
                    ky = torch.tensor([0.2126 * 219 / 255, 0.7152 * 219 / 255, 0.0722 * 219 / 255], device="cuda")

                    def baseline():                            # RGBA scratch, then a float blend of Y and 2x2 chroma in torch
                        g.api._check(r._L.glava_b200_export_frames(r._h, ss.ctypes.data, COUNT, sdst, C.byref(sdesc), None, None))
                        unit, off = (64.0, 4.0) if fmt == "p010" else (1.0, 1.0)      # sample per code, 10-bit codes per 8-bit
                        with torch.cuda.stream(st):
                            for c in range(0, COUNT, 32):
                                src = scratch[c:c + 32].float()
                                al = src[..., 3:] / 255
                                yd = planes[0][c:c + 32]
                                yp = (src[..., :3] * ky).sum(-1, keepdim=True)
                                yn = off * (yp + 16 * al) + (1 - al) * yd.float().unsqueeze(-1) / unit
                                yd.copy_((yn[..., 0] * unit).round().clamp(0, 65535).to(torch.int32).to(yd.dtype))
                                blk = torch.nn.functional.avg_pool2d(src.permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1)
                                ab = blk[..., 3] / 255
                                ypb = (blk[..., :3] * ky).sum(-1)
                                chroma = ((planes[1][c:c + 32, :, 0::2], 2), (planes[1][c:c + 32, :, 1::2], 0)) if fmt == "p010" else \
                                    ((planes[1][c:c + 32], 2), (planes[2][c:c + 32], 0))
                                for d, k in chroma:
                                    v = off * (128 * ab + 0.5 * (blk[..., k] - ypb)) + (1 - ab) * d.float() / unit
                                    d.copy_((v * unit).round().clamp(0, 65535).to(torch.int32).to(d.dtype))
                    legs["baseline_" + fmt] = baseline
                for f in legs.values():                          # warm every leg
                    f()
                r.sync()
                torch.cuda.synchronize()
                times = {k: [] for k in legs}
                walls = {k: [] for k in legs}
                for _ in range(args.rounds):
                    for key, f in legs.items():
                        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        r.sync()
                        torch.cuda.synchronize()
                        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                            a.record(st)
                            for _ in range(args.reps):
                                f()
                            b.record(st)
                            b.synchronize()
                        dev_us = sum(getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0)
                                     for e in prof.key_averages())
                        times[key].append(dev_us / 1e3 / args.reps)
                        walls[key].append(a.elapsed_time(b) / args.reps)
                res = {}
                fb = COUNT * w * h * 4.0 * frac
                img = COUNT * picture_bytes(fmt, w, h)
                for key in legs:
                    ms = float(np.median(times[key]))
                    if key.startswith("export"):
                        nbytes = fb + img
                    elif key.startswith("baseline"):
                        nbytes = fb + COUNT * w * h * 4.0 * 2 + 2 * img
                    else:
                        nbytes = fb + 2 * img * touch["nv12" if fmt not in ("yuv444", "yuv444p10") else "rgba"]
                    gbs = nbytes / (ms / 1e3) / 1e9
                    res[key] = {"ms": ms, "ms_all": times[key], "wall_ms": float(np.median(walls[key])), "bytes": nbytes, "gbs": gbs,
                                "frac_of_peak": gbs / peak}
                out["formats"][fmt] = res
                print(cfg, fmt, json.dumps({k: [round(v["ms"], 4), round(v["frac_of_peak"], 3)] for k, v in res.items()}), flush=True)
                del planes, ex, legs
                torch.cuda.empty_cache()
        result["workloads"][cfg] = out
    text = json.dumps(result, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
