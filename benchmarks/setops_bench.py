#!/usr/bin/env python
"""Distinct rows and set operations at 1e8 rows in 25 chunks of 4e6: duplicated on group-by's two-key row of DESIGN §8 (Int32 with
10 % nulls x Int8) beside group_by(keys, [count]) on the same keys; drop_duplicates of a four-column frame; intersect_all and
except_all of 1e8 x 1e7 rows; and union of two 1e8-row Float64 frames beside a device-to-device copy of the same bytes.

Every row is the sum of the call's per-launch CUDA-event records (bdf_profile_read) and, beside it, the wall time of the call ending
in a synchronise; each is the median of three calls after a warm-up call.  The card's name and power limit are read in the same run.

    python benchmarks/setops_bench.py [--json out.json] [--rows 100000000]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from collections import OrderedDict

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import rust_dataframe_b200 as rdf  # noqa: E402


def card() -> str:
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def free_all(x):
    if isinstance(x, rdf.DeviceFrame):
        x = list(x.columns.values())
    if isinstance(x, (list, tuple)):
        for y in x:
            free_all(y)
    elif x is not None:
        x.free()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--json")
    args = ap.parse_args()
    ctx = rdf.default_context()
    G = rdf.Column.generate
    chunk = 4_000_000
    lens = [chunk] * (args.rows // chunk)
    rows = sum(lens)
    out_rows = []
    print(f"card: {card()}; {rows} rows in {len(lens)} chunks", flush=True)

    def timed(what, fn, **meta):
        free_all(fn())   # warm-up
        ctx.synchronize()
        ctx.profile_read()
        walls, events, parts = [], [], []
        for _ in range(3):
            ctx.profile_enable(True)
            t0 = time.perf_counter()
            res = fn()
            ctx.synchronize()
            walls.append((time.perf_counter() - t0) * 1e3)
            ctx.profile_enable(False)
            recs = ctx.profile_read()
            free_all(res)
            events.append(sum(r["ms"] for r in recs))
            by_kernel = OrderedDict()
            for r in recs:
                by_kernel[r["kernel"]] = by_kernel.get(r["kernel"], 0.0) + r["ms"]
            parts.append({k: round(v, 3) for k, v in by_kernel.items()})
        med = int(np.argsort(events)[1])
        print(f"{what:66s} events {events[med]:8.2f} ms   wall {float(np.median(walls)):8.2f} ms   parts: {parts[med]}", flush=True)
        out_rows.append({"case": what, "ms": events[med], "events_ms": events, "wall_ms": walls, "parts": parts[med], **meta})
        return events[med]

    # 1. duplicated against group-by on the same two keys
    i32n = G(rdf.I32, lens, 2, col_id=53, null_mod=10)
    kf = G(rdf.F64, lens, 0, -100.0, 100.0, col_id=54)
    i8 = kf.cast(rdf.I8)
    kf.free()
    gb = timed("group_by(i32 10% nulls, i8; count)", lambda: rdf.group_by([i32n, i8], [(i8, "count")]), op="group_by")
    dup = timed("duplicated(i32 10% nulls, i8)", lambda: rdf.duplicated([i32n, i8]), op="duplicated")
    print(f"{'':66s} duplicated / group_by = {dup / gb:.3f}", flush=True)

    # 2. drop_duplicates of a four-column frame (about 30 % of the rows repeat an earlier one)
    small = G(rdf.F64, lens, 0, 0.0, 0.7 * rows, col_id=55)
    a = small.cast(rdf.I64)
    b = G(rdf.F64, lens, 0, 0.0, 1.0, col_id=56)
    frame = rdf.DeviceFrame(OrderedDict([("a", a), ("i8", i8), ("i32", i32n), ("x", b)]))
    timed("drop_duplicates(subset=[a, i8]) of (i64, i8, i32, f64)", lambda: frame.drop_duplicates(["a", "i8"]), op="drop_duplicates")

    # 3. intersect_all / except_all, 1e8 x 1e7 rows, keys (i64 over 0.7 x rows, i8)
    rl = [chunk] * (len(lens) // 10) or [rows // 10]
    rf = G(rdf.F64, rl, 0, 0.0, 0.7 * rows, col_id=57)
    ra = rf.cast(rdf.I64)
    rf.free()
    kf = G(rdf.F64, rl, 0, -100.0, 100.0, col_id=58)
    r8 = kf.cast(rdf.I8)
    kf.free()
    for op in ("intersect_all", "except_all"):
        timed(f"{op}((i64, i8) x 1e8, (i64, i8) x 1e7) mask", lambda: rdf.set_op_mask([a, i8], [ra, r8], op), op=op)

    # 4. union of two f64 frames against a device-to-device copy of the same bytes
    x = G(rdf.F64, lens, 0, -1.0, 1.0, col_id=59)
    y = G(rdf.F64, lens, 0, -1.0, 1.0, col_id=60)
    fx, fy = rdf.DeviceFrame(OrderedDict([("v", x)])), rdf.DeviceFrame(OrderedDict([("v", y)]))
    un = timed("union of two 1e8-row f64 frames", lambda: fx.union(fy), op="union")
    import torch

    src = torch.empty(2 * rows * 8, dtype=torch.uint8, device=f"cuda:{ctx.device}")
    dst = torch.empty_like(src)
    dst.copy_(src)
    torch.cuda.synchronize()
    copies = []
    for _ in range(3):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        dst.copy_(src)
        e1.record()
        torch.cuda.synchronize()
        copies.append(e0.elapsed_time(e1))
    cp = float(np.median(copies))
    gbps = 2 * src.numel() / cp / 1e6
    print(f"{'device-to-device copy of the same bytes (torch)':66s} events {cp:8.2f} ms   ({gbps:.0f} GB/s read + write)   "
          f"union / copy = {un / cp:.3f}", flush=True)
    out_rows.append({"case": "d2d copy of 2 x 1e8 x 8 bytes", "ms": cp, "events_ms": copies, "op": "copy"})
    for c in (i32n, i8, a, b, ra, r8, x, y):
        c.free()
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": card(), "rows": out_rows}, f, indent=1)


if __name__ == "__main__":
    main()
