"""Measure the per-stream state calls at the headline configuration (bars, setbufsize 4096, setavgframes 5, pipeline B,
lazy K5, 1920x1080, 1024 streams) and write profiles/<out>.json:

  - device time of the pack kernel (state_pack_kernel, every launch of a whole-batch save, from torch.profiler's CUDA
    activity) and its rate: bytes read + written over that time, against the measured copy peak of 3.03 TB/s;
  - wall time of glava_b200_save_streams and glava_b200_load_streams for the whole batch, into / from pinned
    (glava_b200_host_alloc) and pageable host memory;
  - step time of the device-resident update loop with one stream reset every step against no resets, alternated.

    python tools/stream_state_probe.py [--out h100_stream_state] [--out-dir profiles] [--steps 200] [--reps 3]
Needs a GPU; reads the card's name and power limit in the same run.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

COPY_PEAK = 3.03e12


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="h100_stream_state")
    ap.add_argument("--out-dir", default="profiles")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batch", type=int, default=1024)
    args = ap.parse_args()
    import torch
    import glava_b200 as g
    from glava_b200.synth import synth_batch_int16

    n, w, h, batch = 4096, 1920, 1080, args.batch
    p = g.default_params("bars", n=n, w=w, h=h, avg_frames=5)
    p.lazy_smooth = 1
    res = {"gpu": gpu_info(), "config": f"bars n={n} F=5 pipeline B lazy K5 {w}x{h}, batch {batch}"}
    r = g.Renderer(p, batch=batch)
    L, hnd = r._L, r._h
    pcm = synth_batch_int16(0, batch, 0, n + 4 * 256).astype(np.float32) / np.float32(65535)
    dev = [(torch.from_numpy(np.ascontiguousarray(pcm[:, i * 256:i * 256 + n, 0])).cuda(),
            torch.from_numpy(np.ascontiguousarray(pcm[:, i * 256:i * 256 + n, 1])).cuda()) for i in range(4)]
    for i in range(8):
        r.update_device(dev[i % 4][0].data_ptr(), dev[i % 4][1].data_ptr(), True)
    r.sync()
    bytes_ = g.stream_state_bytes(p)
    seg = bytes_ - g.STATE_HEADER_BYTES
    res["blob_bytes_per_stream"] = bytes_
    res["segment_bytes_per_stream"] = seg
    streams = (C.c_int * batch)(*range(batch))
    pinned = g.pinned_empty((batch, bytes_), np.uint8)
    pageable = np.empty((batch, bytes_), np.uint8)
    pageable[:] = 1                                                   # fault the pages in before timing

    def check(rc):
        if rc != 0:
            raise g.GlavaError(L.glava_b200_last_error().decode())

    # ---- pack kernel device time (profiler), whole-batch save -----------------------------------------------------------
    check(L.glava_b200_save_streams(hnd, streams, batch, pinned.ctypes.data))          # warm-up: staging allocated
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            check(L.glava_b200_save_streams(hnd, streams, batch, pinned.ctypes.data))
        torch.cuda.synchronize()
    ks = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "state_pack_kernel" in e.name]
    us = sum(e.device_time for e in ks) / 5
    res["pack_kernel"] = {"launches_per_save": len(ks) // 5, "device_us_per_save": us,
                          "bytes_moved": 2 * seg * batch, "rate_TBps": 2 * seg * batch / (us * 1e-6) / 1e12,
                          "of_copy_peak_3.03TBps": 2 * seg * batch / (us * 1e-6) / COPY_PEAK}

    # ---- wall time of save and load ------------------------------------------------------------------------------------
    def wall(fn, reps=5):
        out = []
        for _ in range(reps):
            r.sync()
            t0 = time.perf_counter(); fn(); t1 = time.perf_counter(); r.sync(); t2 = time.perf_counter()
            out.append(((t1 - t0) * 1e3, (t2 - t0) * 1e3))
        return {"call_ms_median": float(np.median([a for a, _ in out])), "call_plus_sync_ms_median": float(np.median([b for _, b in out])),
                "GBps_call": bytes_ * batch / (np.median([a for a, _ in out]) * 1e-3) / 1e9}

    res["save_pinned"] = wall(lambda: check(L.glava_b200_save_streams(hnd, streams, batch, pinned.ctypes.data)))
    res["save_pageable"] = wall(lambda: check(L.glava_b200_save_streams(hnd, streams, batch, pageable.ctypes.data)))
    res["load_pinned"] = wall(lambda: check(L.glava_b200_load_streams(hnd, streams, batch, pinned.ctypes.data)))
    res["load_pageable"] = wall(lambda: check(L.glava_b200_load_streams(hnd, streams, batch, pageable.ctypes.data)))
    assert np.array_equal(pinned[:, g.STATE_HEADER_BYTES:], pageable[:, g.STATE_HEADER_BYTES:])

    # ---- step time with one reset per step ------------------------------------------------------------------------------
    st = torch.cuda.ExternalStream(r.cuda_stream)
    masks = [np.zeros(batch, np.uint8) for _ in range(batch)]
    for s in range(batch):
        masks[s][s] = 1

    def leg(reset):
        for i in range(3):
            r.update_device(dev[i % 4][0].data_ptr(), dev[i % 4][1].data_ptr(), True)
        r.sync()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(st)
        for i in range(args.steps):
            r.update_device(dev[i % 4][0].data_ptr(), dev[i % 4][1].data_ptr(), True)
            if reset:
                check(L.glava_b200_reset_streams(hnd, masks[i % batch].ctypes.data))
        b.record(st)
        r.sync()
        return a.elapsed_time(b) / args.steps

    plain, resets = [], []
    for _ in range(args.reps):
        plain.append(leg(False)); resets.append(leg(True))
    res["step_ms"] = {"no_reset": plain, "one_reset_per_step": resets,
                      "median_no_reset": float(np.median(plain)), "median_one_reset": float(np.median(resets)),
                      "change_pct": (float(np.median(resets)) / float(np.median(plain)) - 1) * 100}
    r.close()
    out = os.path.join(ROOT, args.out_dir, args.out + ".json")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    with open(out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
