#!/usr/bin/env python
"""step_trace.py -- where the time of bench.py's headline step goes between the K5 kernels.

    python benchmarks/step_trace.py --out DIR [--steps 50]

Runs bench.py's hot loop (1e8 f64 rows, c = a + b with sum(c) fused, one step in flight) under torch.profiler with CUDA
activities, once with the library's launch records on (as bench.py's timed loop runs) and once with them off, and writes
DIR/step_<records>.pt.trace.json plus one JSON summary line per run:
  k5_ms        duration of each k_binary launch (median)
  gap_us       idle time between the end of one k_binary and the start of the next (median, p90)
  finish_us    k_finish duration, and how much of it overlaps the next k_binary
  step_ms      start-to-start period of consecutive k_binary launches (median)
  copies       memcpy / memset activities per step
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def summarize(trace_path: str, steps: int) -> dict:
    with open(trace_path) as f:
        ev = json.load(f)["traceEvents"]
    kern = sorted((e for e in ev if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    k5 = [e for e in kern if "k_binary" in e["name"]]
    fin = [e for e in kern if "k_finish" in e["name"]]
    gaps = [k5[i + 1]["ts"] - (k5[i]["ts"] + k5[i]["dur"]) for i in range(len(k5) - 1)]
    period = [k5[i + 1]["ts"] - k5[i]["ts"] for i in range(len(k5) - 1)]
    overlap = []
    for f in fin:
        # the K5 this k_finish folds is the last one that ended before it started; measure the overlap with the one after it
        done = [i for i, k in enumerate(k5) if k["ts"] + k["dur"] <= f["ts"]]
        if done and done[-1] + 1 < len(k5):
            k = k5[done[-1] + 1]
            overlap.append(max(0.0, min(f["ts"] + f["dur"], k["ts"] + k["dur"]) - max(f["ts"], k["ts"])))
    copies = [e for e in ev if e.get("cat") in ("gpu_memcpy", "gpu_memset")]
    pct = lambda x, q: float(np.percentile(x, q)) if x else None
    return {"k5_launches": len(k5), "k5_ms_median": pct([k["dur"] / 1e3 for k in k5], 50),
            "gap_us_median": pct(gaps, 50), "gap_us_p90": pct(gaps, 90), "gap_us_min": min(gaps) if gaps else None,
            "step_ms_median": pct([p / 1e3 for p in period], 50),
            "finish_us_median": pct([f["dur"] for f in fin], 50), "finish_overlap_us_median": pct(overlap, 50),
            "copies_per_step": len(copies) / max(1, steps), "copy_kinds": sorted({e["name"] for e in copies})}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=50)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)

    import torch
    from torch.profiler import ProfilerActivity, profile

    import bench
    import rust_dataframe_b200 as rdf
    from rust_dataframe_b200 import native as N

    torch.cuda.init()
    ctx = rdf.Context(0)
    a, b, _ = bench.make_inputs(rdf, ctx, 0, 1, "weak")
    loop = bench.HotLoop(N, a, b, 1)
    for _ in range(5):
        loop.step()
    loop.drain()
    for records in (True, False):
        ctx.profile_enable(records)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                loop.step()
            loop.drain()
        ctx.profile_enable(False)
        ctx.profile_read()
        path = os.path.join(args.out, f"step_records_{'on' if records else 'off'}.pt.trace.json")
        prof.export_chrome_trace(path)
        line = {"launch_records": records, "steps": args.steps, **summarize(path, args.steps)}
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
