"""Frame export rates per Y'CbCr encoding (DESIGN 4.15) on one GPU, with the card and its power limit read in the same run.
Per workload (bench.py's inputs and warm-up), CUDA-event time of exporting 1024 streams whole-frame and scaled to 480x270 in
NV12, I420 and P010, each in BT.709 limited range (the encoding every call without a colour flag writes), BT.709 full range,
BT.601 limited and BT.601 full range; all legs alternated within each round, so that every encoding is measured beside
BT.709 limited in the same run.  Before timing it checks, per encoding, sampled streams of every leg bit for bit against the
numpy restatement of tests/test_gpu_export_matrix.py and I420 against the deinterleaved NV12 planes.

    python tools/export_matrix_bench.py --out profiles/h100_export_matrix.json [--configs headline,radial1080]
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
FORMATS = ("nv12", "i420", "p010")
THUMB = (480, 270)
ENCODINGS = {"bt709_limited": ({}, 0), "bt709_full": (dict(full_range=True), 1), "bt601_limited": (dict(matrix="bt601"), 2),
             "bt601_full": (dict(matrix="bt601", full_range=True), 3)}
BYTES_PER_PIXEL = {"nv12": 1.5, "i420": 1.5, "p010": 3.0}


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
    from tests.test_export_scaled_core import scaled_np
    from tests.test_export_core import RGBA
    from tests.test_gpu_export_matrix import frame_np, ycbcr_np

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
            legs = [(kind, fmt, enc) for kind in ("whole", "scaled") for fmt in FORMATS for enc in ENCODINGS]
            outs = {}
            for kind in ("whole", "scaled"):                 # one [count, rows, pitch] buffer per (kind, format), shared by the encodings
                for fmt in FORMATS:
                    ow, oh = (w, h) if kind == "whole" else THUMB
                    rows, row_bytes, align = g.api._export_layout(fmt, ow, oh)
                    outs[(kind, fmt)] = torch.empty((count, rows, (row_bytes + align - 1) // align * align), dtype=torch.uint8,
                                                    device=f"cuda:{r.device}")

            def run(kind, fmt, enc):
                kw = ENCODINGS[enc][0]
                if kind == "whole":
                    r.export_frames(range(count), fmt, out=outs[(kind, fmt)], **kw)
                else:
                    r.export_scaled(range(count), THUMB, fmt=fmt, out=outs[(kind, fmt)], **kw)

            # the bytes first: every leg on sampled streams against the restatement, and the I420 / NV12 identity
            samples = [0, count // 2, count - 1]
            frames = {s: r.readback(s) for s in samples}
            thumbs = {s: scaled_np(frames[s], RGBA, True, (0, 0, 0), True, THUMB) for s in samples}
            for enc, (kw, e) in ENCODINGS.items():
                for kind in ("whole", "scaled"):
                    ow, oh = (w, h) if kind == "whole" else THUMB
                    views = {}
                    for fmt in FORMATS:
                        run(kind, fmt, enc)
                        torch.cuda.synchronize()
                        views[fmt] = g.api._export_views(fmt, outs[(kind, fmt)], ow, oh)
                        for s in samples:
                            got = views[fmt]
                            got = tuple(x[s].cpu().numpy() for x in got) if isinstance(got, tuple) else got[s].cpu().numpy()
                            want = frame_np(frames[s], fmt, e, (0, 0, 0), True) if kind == "whole" else ycbcr_np(thumbs[s], fmt, e)
                            ok = (all(np.array_equal(a, b) for a, b in zip(got, want)) if isinstance(want, tuple)
                                  else np.array_equal(got, want))
                            assert ok, (cfg, enc, kind, fmt, s)
                    yp, cb, cr = views["i420"]
                    nv12 = views["nv12"]
                    assert torch.equal(yp, nv12[:, :oh]) and torch.equal(cb, nv12[:, oh:, 0::2]) and torch.equal(cr, nv12[:, oh:, 1::2])
            for leg in legs:                                 # warms the list buffers and every kernel
                run(*leg)
            torch.cuda.synchronize()
            times = {"_".join(leg): [] for leg in legs}
            for _ in range(args.rounds):
                for leg in legs:
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    r.sync()
                    a.record(st)
                    for _ in range(args.reps):
                        run(*leg)
                    b.record(st)
                    b.synchronize()
                    times["_".join(leg)].append(a.elapsed_time(b) / args.reps)
            res = {}
            for kind, fmt, enc in legs:
                k = f"{kind}_{fmt}_{enc}"
                ms = float(np.median(times[k]))
                ow, oh = (w, h) if kind == "whole" else THUMB
                wbytes = count * ow * oh * BYTES_PER_PIXEL[fmt]
                base = float(np.median(times[f"{kind}_{fmt}_bt709_limited"]))
                res[k] = {"ms": ms, "ms_all": times[k], "write_bytes": wbytes, "write_gbs": wbytes / (ms / 1e3) / 1e9,
                          "vs_bt709_limited": ms / base}
        result["workloads"][cfg] = {"module": module, "n": n, "w": w, "h": h, "batch": batch, "count": count, "legs": res}
        print(cfg, json.dumps({k: round(v["ms"], 4) for k, v in res.items()}), flush=True)
    text = json.dumps(result, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
