"""Frames/s of styled batches (DESIGN 4.9, 6): one process, one renderer per workload, update_device from HBM, alternating
unstyled / 8 shared styles / one style per stream so that clocks and thermals affect the three alike.  Records the card
and its power limit with the numbers, and the wall time of each set_stream_styles call (a table rebuild).

    python tools/style_bench.py --out profiles/h100_stream_styles.json [--steps 100 --rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = {"headline": ("bars", 4096, 1920, 1080, 1024), "graph720": ("graph", 2048, 1280, 720, 256),
             "wave720": ("wave", 2048, 1280, 720, 256), "circle1080": ("circle", 4096, 1920, 1080, 1024),
             "radial1080": ("radial", 4096, 1920, 1080, 1024)}
AMP = dict(bars="bars_amplify", radial="radial_amplify", circle="circle_amplify", graph="graph_vscale", wave="wave_amplify")


def styles(g, p, count):
    """`count` distinct looks: amplify, fg and (but circle) bg all vary"""
    m = g.MODULES[p.module]
    a = getattr(p, AMP[m])
    out = []
    for k in range(count):
        t = k / max(count - 1, 1)
        s = {"amplify": a * (0.6 + 0.8 * t), "fg": (t, 1.0 - t, 0.5, 1.0)}
        if m != "circle":
            s["bg"] = (0.2, 0.2 * t, 0.3, 1.0)
        out.append(s)
    return out


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (x.strip() for x in q.split(","))
        return name, limit
    except Exception:
        return "unknown", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--configs", default=",".join(WORKLOADS))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import torch
    import glava_b200 as g

    name, limit = card()
    result = {"gpu": name, "power_limit": limit, "steps": args.steps, "rounds": args.rounds, "workloads": {}}
    for cfg in args.configs.split(","):
        module, n, w, h, batch = WORKLOADS[cfg]
        p = g.default_params(module, n=n, w=w, h=h)
        rng = np.random.default_rng(0)
        dev = [torch.from_numpy((rng.standard_normal((batch, n)) * 0.3).astype(np.float32)).cuda() for _ in range(4)]
        legs = {"unstyled": None, "8_styles": styles(g, p, 8), "per_stream": styles(g, p, batch)}
        rates = {k: [] for k in legs}
        set_ms = {k: [] for k in legs}
        with g.Renderer(p, batch=batch) as r:
            st = torch.cuda.ExternalStream(r.cuda_stream)
            for _ in range(args.rounds):
                for leg, looks in legs.items():
                    want = [None] * batch if looks is None else [looks[s % len(looks)] for s in range(batch)]
                    t0 = time.perf_counter()
                    r.set_stream_styles(range(batch), want)          # rebuilds the tables and waits for them
                    set_ms[leg].append((time.perf_counter() - t0) * 1e3)
                    for i in range(args.warmup):
                        r.update_device(dev[i % 2].data_ptr(), dev[i % 2 + 2].data_ptr(), True)
                    r.sync()
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record(st)
                    for i in range(args.steps):
                        r.update_device(dev[i % 2].data_ptr(), dev[i % 2 + 2].data_ptr(), True)
                    b.record(st)
                    r.sync(); b.synchronize()
                    rates[leg].append(batch * args.steps / (a.elapsed_time(b) / 1e3))
        med = {k: float(np.median(v)) for k, v in rates.items()}
        result["workloads"][cfg] = {"module": module, "n": n, "w": w, "h": h, "batch": batch, "frames_per_s": rates,
                                    "median": med, "styled_vs_unstyled": {k: med[k] / med["unstyled"] for k in med},
                                    "set_stream_styles_ms": set_ms}
        print(cfg, json.dumps(result["workloads"][cfg]["median"]), flush=True)
    text = json.dumps(result, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
