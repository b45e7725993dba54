"""Frame export and overlay rates of the BT.2020 HDR encodings (DESIGN 4.22) on one GPU, with the card and its power limit
read in the same run.  Per workload (bench.py's inputs and warm-up), CUDA-event time of exporting 1024 streams whole-frame
and scaled to 480x270 in P010, YUV420P10, YUV444P10 and YUV422P10, each in BT.709 limited range, PQ and HLG, and of
overlay_planes onto 1024 P010 pictures in BT.709 limited range, PQ and HLG; all legs alternated within each round.  Before
timing it checks sampled streams of every HDR leg bit for bit against the host build of export_core.h
(tests/export_hdr_shim.py) applied to glava_b200_readback.

    python tools/export_hdr_bench.py --out profiles/h100_export_hdr.json [--configs headline,radial1080]
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
FORMATS = ("p010", "yuv420p10", "yuv444p10", "yuv422p10")
THUMB = (480, 270)
ENCODINGS = {"bt709_limited": {}, "pq": dict(matrix="bt2020", transfer="pq"), "hlg": dict(matrix="bt2020", transfer="hlg")}
BYTES_PER_PIXEL = {"p010": 3.0, "yuv420p10": 3.0, "yuv444p10": 6.0, "yuv422p10": 4.0}


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
    from tests import export_hdr_shim as S
    from tests.export_hdr_np import HLG, PQ
    from tests.test_export_core import RGBA, over_np
    from tests.test_export_scaled_core import scaled_np

    E = {"pq": PQ, "hlg": HLG}
    F = {"p010": S.P010, "yuv420p10": S.YUV420P10, "yuv444p10": S.YUV444P10, "yuv422p10": S.YUV422P10}
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
            legs += [("overlay", "p010", enc) for enc in ENCODINGS]
            outs = {}
            for kind in ("whole", "scaled"):                 # one [count, rows, pitch] buffer per (kind, format), shared by the encodings
                for fmt in FORMATS:
                    ow, oh = (w, h) if kind == "whole" else THUMB
                    rows, row_bytes, align = g.api._export_layout(fmt, ow, oh)
                    outs[(kind, fmt)] = torch.empty((count, rows, (row_bytes + align - 1) // align * align), dtype=torch.uint8,
                                                    device=f"cuda:{r.device}")
            # the overlay's pictures: mid-grey P010 (Y 512, C 512), one [h * 3 / 2, w] tensor per stream in one allocation
            pics = torch.from_numpy(np.full((count, h * 3 // 2, w), 512 << 6, np.uint16)).to(f"cuda:{r.device}")
            pic_list = [(pics[i, :h], pics[i, h:]) for i in range(count)]

            def run(kind, fmt, enc):
                kw = ENCODINGS[enc]
                if kind == "whole":
                    r.export_frames(range(count), fmt, out=outs[(kind, fmt)], **kw)
                elif kind == "scaled":
                    r.export_scaled(range(count), THUMB, fmt=fmt, out=outs[(kind, fmt)], **kw)
                else:
                    r.overlay_planes(range(count), pic_list, None, fmt, **kw)

            # the bytes first: every HDR leg on sampled streams against the host build
            samples = [0, count // 2, count - 1]
            frames = {s: r.readback(s) for s in samples}
            for enc in ("pq", "hlg"):
                for kind in ("whole", "scaled"):
                    ow, oh = (w, h) if kind == "whole" else THUMB
                    for fmt in FORMATS:
                        run(kind, fmt, enc)
                        torch.cuda.synchronize()
                        views = g.api._export_views(fmt, outs[(kind, fmt)], ow, oh)
                        for s in samples:
                            img = (over_np(frames[s][::-1], (0, 0, 0), True) if kind == "whole"
                                   else scaled_np(frames[s], RGBA, True, (0, 0, 0), True, THUMB))
                            want = S.planes(E[enc], F[fmt], S.pack(img))
                            got = (views[s].cpu().numpy()[:oh], views[s].cpu().numpy()[oh:]) if fmt == "p010" else \
                                tuple(x[s].cpu().numpy() for x in views)
                            assert all(np.array_equal(a, b) for a, b in zip(got, want)), (cfg, enc, kind, fmt, s)
                before = [(pics[s, :h].cpu().numpy(), pics[s, h:].cpu().numpy()) for s in samples]
                run("overlay", "p010", enc)
                torch.cuda.synchronize()
                for s, b in zip(samples, before):
                    want = S.overlay(E[enc], S.P010, S.pack(frames[s][::-1]), b)
                    got = (pics[s, :h].cpu().numpy(), pics[s, h:].cpu().numpy())
                    assert all(np.array_equal(x, y) for x, y in zip(got, want)), (cfg, enc, "overlay", s)
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
                ow, oh = (w, h) if kind != "scaled" else THUMB
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
