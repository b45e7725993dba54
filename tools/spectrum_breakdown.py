"""Where one spectrum update's time and bytes go (development aid): device time of every spectrum-stream and raster kernel of
a bench.py workload, from torch.profiler CUDA activity, in two legs of one run:

  corun     bench.py's device-resident loop: the spectrum kernels of update i+1 co-run with the raster kernel of update i
  spectrum  the same spectrum (module, n, frame width, batch) with a 16-row frame: the spectrum chain alone

and the bytes each kernel of the chain moves per update, computed from the shapes (not measured).  The card's name, power
limit and maximum SM clock come from nvidia-smi in the same run.

    python tools/spectrum_breakdown.py [--config headline] [--steps 50] [--out FILE.json]
    python tools/spectrum_breakdown.py --bytes-only        # the byte table only (no GPU)
"""
import argparse
import collections
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload shapes only)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except (OSError, subprocess.SubprocessError):
        return None


def params(wl, h=None):
    import glava_b200 as g
    p = g.default_params(wl["module"], n=wl["n"], w=wl["w"], h=h or wl["h"])
    p.lazy_smooth = 1
    return p


def byte_table(wl, batch, sm_count=132):
    """MB one update moves per kernel of the spectrum chain, from the shapes and the launch structure plan_spectrum chooses
    (tests/emul: the same decision compiled for the host)"""
    from tests import emul
    p = params(wl)
    pl = emul.spectrum_plan(p, False, batch, sm_count, {})
    n, F = wl["n"], int(p.avg_frames)
    fft = wl["module"] != "wave"
    planes = batch * 2 if fft else batch
    epi = pl["epi_n"] if 0 < pl["epi_n"] < n else n
    mb = lambda b: round(b / 1e6, 2)
    rows = [("spectrum_kernel", "PCM read (TMA)", planes * n * 4)]
    if fft and pl["split_epilogue"]:
        rows += [("spectrum_kernel", "spec write (epi_n bins)", planes * epi * 4),
                 ("spectrum_kernel", "state prefetch (none in the FFT-only form)", 0),
                 ("spectrum_kernel", "[whole-plane state prefetch, the form before it was limited to the in-kernel epilogue]",
                  planes * n * 2 * (1 + F)),
                 ("epilogue_b_kernel", "spec read", planes * epi * 4),
                 ("epilogue_b_kernel", "gr_store read + write", planes * epi * 2 * 2),
                 ("epilogue_b_kernel", f"{F - 1} ring slots read + 1 written", planes * epi * 2 * F if F > 1 else 0),
                 ("epilogue_b_kernel", "av_out write", planes * epi * 2)]
    elif fft and p.accel_fft:
        rows += [("spectrum_kernel", "spec write", planes * epi * 4),
                 ("spectrum_kernel", f"state prefetch + epilogue: gr_store r/w, {F - 1} ring slots read, 1 written",
                  planes * epi * 2 * (2 + F))]
    if pl["k5"] == "need_smem":
        rows.append(("k5_need_smem_kernel", "av_out read (leading av_t_len bins; sparse tex writes not counted)",
                     planes * pl["av_t_len"] * 2))
    return {"plan": {k: pl[k] for k in ("split_epilogue", "epi_n", "av_t_len", "k5", "fft_oop", "fft_t", "spec_grid")},
            "rows": [{"kernel": k, "traffic": t, "MB": mb(b)} for k, t, b in rows],
            "note": "per update, computed from the shapes and the plan, not measured; the bracketed row is not moved by this tree"}


def short(name):
    """kernel name without the namespace, argument list and return type"""
    s = name.split("(")[0]
    for pre in ("void ", "glb::"):
        s = s.replace(pre, "")
    return s


def profile_leg(r, dev_l, dev_r, updates, warmup, modified=True):
    import torch
    from torch.profiler import ProfilerActivity, profile
    for i in range(warmup):
        r.update_device(dev_l[i % len(dev_l)].data_ptr(), dev_r[i % len(dev_r)].data_ptr(), modified)
    r.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(updates):
            r.update_device(dev_l[i % len(dev_l)].data_ptr(), dev_r[i % len(dev_r)].data_ptr(), modified)
        r.sync()
        torch.cuda.synchronize()
    per = collections.defaultdict(lambda: [0, 0.0])
    for ev in prof.events():
        if ev.device_type.name != "CUDA":
            continue
        k = short(ev.name)
        if k.startswith("Memcpy") or k.startswith("Memset"):
            continue
        per[k][0] += 1
        per[k][1] += ev.time_range.elapsed_us()
    rows = [{"kernel": k, "launches_per_update": c / updates, "us_per_launch": round(t / c, 2),
             "us_per_update": round(t / updates, 2)} for k, (c, t) in per.items()]
    rows.sort(key=lambda d: -d["us_per_update"])
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="headline", help="a bench.py --config")
    ap.add_argument("--batch", type=int, default=0)
    ap.add_argument("--steps", type=int, default=50, help="profiled updates per leg")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--bytes-only", action="store_true")
    ap.add_argument("--out", default=None, help="write the result as JSON here")
    a = ap.parse_args()
    wl = bench.workload(a.config)
    batch = a.batch or wl["batch"]
    res = {"config": a.config, "workload": {k: wl[k] for k in ("module", "n", "w", "h")}, "batch": batch}
    if not a.bytes_only:
        import numpy as np
        import torch
        import glava_b200 as g
        from glava_b200.synth import synth_batch_int16
        res["card"] = card()
        sm = torch.cuda.get_device_properties(0).multi_processor_count
        res["bytes"] = byte_table(wl, batch, sm)
        n = wl["n"]
        pcm = synth_batch_int16(0, batch, 0, n + 4 * bench.HOP).astype(np.float32) / np.float32(65535)
        dev_l = [torch.from_numpy(np.ascontiguousarray(pcm[:, (i + 1) * bench.HOP:(i + 1) * bench.HOP + n, 0])).cuda() for i in range(3)]
        dev_r = [torch.from_numpy(np.ascontiguousarray(pcm[:, (i + 1) * bench.HOP:(i + 1) * bench.HOP + n, 1])).cuda() for i in range(3)]
        legs = {}
        p = params(wl)
        frame_bytes = wl["w"] * wl["h"] * 4
        if batch * frame_bytes > bench.FB_BUDGET:
            p.fb_slots = max(1, int(bench.FB_BUDGET // frame_bytes))
        with g.Renderer(p, batch=batch) as r:
            legs["corun"] = profile_leg(r, dev_l, dev_r, a.steps, a.warmup)
        with g.Renderer(params(wl, h=16), batch=batch) as r:
            legs["spectrum"] = profile_leg(r, dev_l, dev_r, a.steps, a.warmup)
        res["legs"] = legs
        res["method"] = (f"torch.profiler CUDA activity over {a.steps} updates per leg after {a.warmup} warm-up updates; "
                         "corun = the bench workload, spectrum = the same spectrum with a 16-row frame")
    else:
        res["bytes"] = byte_table(wl, batch)
    print(f"# {a.config}: {wl['module']} n {wl['n']} {wl['w']}x{wl['h']} batch {batch}" + (f"   [{res['card']}]" if res.get("card") else ""))
    for leg, rows in res.get("legs", {}).items():
        print(f"## {leg}")
        for d in rows:
            print(f"  {d['kernel'][:60]:60s} {d['launches_per_update']:5.2f} x {d['us_per_launch']:9.2f} us = {d['us_per_update']:9.2f} us/update")
    print("## bytes per update (from shapes)", json.dumps(res["bytes"]["plan"]))
    for d in res["bytes"]["rows"]:
        print(f"  {d['kernel']:22s} {d['MB']:9.2f} MB  {d['traffic']}")
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
