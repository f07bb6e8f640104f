#!/usr/bin/env python
"""Top-k against sort + limit at 1e8 rows in 25 chunks of 4e6.

Rows: one Float64 key with four payload columns (frame.top_k against frame.sort(...).limit(...)) at k = 10 / 1e3 / 1e6; one Int32
key with 10 % nulls; two keys (Int8 with about 200 values, then Float64), so ties reach the second round; an all-equal first key (every
row ties in round 0, the worst case).  Then the index step alone at growing k / n, beside one full sort, to place the crossover
(bdf_top_k_indices_dev runs the full sort above k = 5n / 8): the rows at k = 5n / 8 and 5n / 8 + 1 are on either side of it.

Every row is the sum of the call's per-launch CUDA-event records (bdf_profile_read) and, beside it, the wall time of the call ending
in a synchronise; each is the median of three calls after a warm-up call, top-k and sort + limit alternating.  The card's name and
power limit are read in the same run.

    python benchmarks/topk_bench.py [--json out.json] [--rows 100000000]
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
    chunk = min(4_000_000, args.rows)
    lens = [chunk] * (args.rows // chunk)
    n = sum(lens)
    out_rows = []
    print(f"card: {card()}; {n} rows in {len(lens)} chunks", flush=True)

    def run(fn):
        ctx.profile_enable(True)
        t0 = time.perf_counter()
        res = fn()
        ctx.synchronize()
        wall = (time.perf_counter() - t0) * 1e3
        ctx.profile_enable(False)
        recs = ctx.profile_read()
        free_all(res)
        parts = OrderedDict()
        for r in recs:
            parts[r["kernel"]] = parts.get(r["kernel"], 0.0) + r["ms"]
        return sum(r["ms"] for r in recs), wall, {k: round(v, 3) for k, v in parts.items()}

    def pair(what, fast, slow, **meta):
        """fast and slow alternating: warm-up of both, then three calls of each."""
        free_all(fast())
        free_all(slow())
        ctx.synchronize()
        ctx.profile_read()
        res = {"top_k": [], "sort_limit": []}
        for _ in range(3):
            res["top_k"].append(run(fast))
            res["sort_limit"].append(run(slow))
        line = {"case": what, **meta}
        for name, rs in res.items():
            ev = [r[0] for r in rs]
            med = int(np.argsort(ev)[1])
            line[name] = {"ms": ev[med], "events_ms": ev, "wall_ms": [r[1] for r in rs], "parts": rs[med][2]}
            print(f"  {what:58s} {name:10s} events {ev[med]:8.2f} ms   wall {float(np.median([r[1] for r in rs])):8.2f} ms   parts: {rs[med][2]}",
                  flush=True)
        line["speedup"] = line["sort_limit"]["ms"] / line["top_k"]["ms"]
        print(f"  {'':58s} sort + limit / top_k = {line['speedup']:.2f}", flush=True)
        out_rows.append(line)

    # 1. one Float64 key with four payload columns
    key = G(rdf.F64, lens, 0, -1.0, 1.0, col_id=71)
    pay = OrderedDict([("key", key)] + [(f"p{i}", G(rdf.F64, lens, 0, 0.0, 1.0, col_id=72 + i)) for i in range(4)])
    frame = rdf.DeviceFrame(pay)
    for k in (10, 1000, 1_000_000):
        crit = [("key", True)]
        pair(f"f64 key + 4 f64 payload, k = {k}", lambda: frame.top_k(crit, k), lambda: frame.sort(crit).limit(k), k=k, keys="f64")

    # 2. one Int32 key with 10 % nulls
    i32 = G(rdf.I32, lens, 2, col_id=80, null_mod=10)
    f32 = rdf.DeviceFrame(OrderedDict([("key", i32)]))
    pair("i32 key, 10 % nulls, k = 1000", lambda: f32.top_k([("key", False)], 1000), lambda: f32.sort([("key", False)]).limit(1000),
         k=1000, keys="i32 nulls")

    # 3. two keys: Int8 with about 200 values, then Float64 (ties reach the second round)
    kf = G(rdf.F64, lens, 0, -100.0, 100.0, col_id=81)
    i8 = kf.cast(rdf.I8)
    kf.free()
    f2 = rdf.DeviceFrame(OrderedDict([("a", i8), ("b", key)]))
    crit2 = [("a", False), ("b", True)]
    pair("(i8 ~200 values, f64), k = 1000", lambda: f2.top_k(crit2, 1000), lambda: f2.sort(crit2).limit(1000), k=1000, keys="i8,f64")

    # 4. an all-equal first key: every row ties in round 0
    kz = G(rdf.F64, lens, 0, 0.0, 1.0, col_id=82)
    zero = kz.cast(rdf.I8)
    kz.free()
    f3 = rdf.DeviceFrame(OrderedDict([("z", zero), ("b", key)]))
    crit3 = [("z", False), ("b", False)]
    pair("(all-equal i8, f64), k = 1000", lambda: f3.top_k(crit3, 1000), lambda: f3.sort(crit3).limit(1000), k=1000, keys="equal,f64")

    # 5. the index step across k / n: the fast path up to 5n / 8, the full sort above
    for name, col in (("f64", key), ("i32 nulls", i32)):
        for frac in (0.01, 0.1, 0.25, 0.5, 0.6, 0.625, 0.625 + 1 / n):
            k = int(round(frac * n))
            pair(f"indices of {name}, k = {k} ({k / n:.4f} n)", lambda: rdf.top_k_indices([(col, False)], k),
                 lambda: rdf.sort_indices([(col, False)]), k=k, keys=name, indices_only=True)
    for c in list(pay.values()) + [i32, i8, zero]:
        c.free()
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": card(), "rows": out_rows}, f, indent=1)


if __name__ == "__main__":
    main()
