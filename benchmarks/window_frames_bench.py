#!/usr/bin/env python
"""Bounded window frames over 1e8 Float64 rows in 25 chunks of 4e6 (bdf_window_dev with ROWS / RANGE BETWEEN and the value
functions), next to the existing running-sum "rows" row measured in the same session as the yardstick.  Every row prints the
device time of one call (the sum of its launch records, median of the runs) and its parts by launch.

    python benchmarks/window_frames_bench.py [--rows 100000000] [--json out.json]
"""
from __future__ import annotations

import argparse
import datetime
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import rust_dataframe_b200 as rdf  # noqa: E402


def card() -> str:
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json")
    args = ap.parse_args()
    ctx = rdf.default_context()
    chunk = min(4_000_000, args.rows)
    lens = [chunk] * (args.rows // chunk)
    rows = sum(lens)
    G = rdf.Column.generate
    out_rows = []
    print(f"card: {card()}; {rows} rows in {len(lens)} chunks", flush=True)

    def run(what, part, order, calls):
        for _ in range(2):   # warm-up
            for c in rdf.window(part, order, calls):
                c.free()
        ctx.synchronize()
        ctx.profile_read()
        totals, parts = [], []
        for _ in range(args.reps):
            ctx.profile_enable(True)
            res = rdf.window(part, order, calls)
            ctx.profile_enable(False)
            recs = ctx.profile_read()
            for c in res:
                c.free()
            totals.append(sum(r["ms"] for r in recs))
            parts.append([(r["kernel"], round(r["ms"], 3)) for r in recs])
        med = int(np.argsort(totals)[len(totals) // 2])
        print(f"{what:64s} {totals[med]:9.3f} ms   parts: " + ", ".join(f"{k} {v}" for k, v in parts[med]), flush=True)
        out_rows.append({"case": what, "ms": totals[med], "runs_ms": totals, "rows": rows, "parts": parts[med]})

    x = G(rdf.F64, lens, 0, -1e3, 1e3, col_id=60)
    run("running sum f64, frame 'rows' (existing scan: the yardstick)", [], [], [("sum", x, "rows")])
    w100 = ("rows", -99, 0)
    run("moving sum ROWS -99..0, no keys", [], [], [("sum", x, w100)])
    run("moving sum, avg, max ROWS -99..0, no keys (one hierarchy)", [], [], [("sum", x, w100), ("avg", x, w100), ("max", x, w100)])
    w1e5 = ("rows", -99_999, 0)
    run("moving sum ROWS -99999..0, no keys", [], [], [("sum", x, w1e5)])
    run("moving sum, avg, max ROWS -99999..0, no keys (one hierarchy)", [], [], [("sum", x, w1e5), ("avg", x, w1e5), ("max", x, w1e5)])
    kf = G(rdf.F64, lens, 0, 0.0, rows / 100.0, col_id=61)
    key = kf.cast(rdf.I32)   # ~1e6 partitions of ~100 rows
    kf.free()
    run("partition i32 (~1e6): sum ROWS -2..+2", [key], [], [("sum", x, ("rows", -2, 2))])
    key.free()
    tf = G(rdf.F64, lens, 0, 0.0, 365 * 86_400_000.0, col_id=62)
    ts = tf.cast(rdf.I64).with_temporal(rdf.TemporalType(rdf.arrays.TIMESTAMP, "ms"))   # one year of ms timestamps
    tf.free()
    run("order i64 timestamp: sum RANGE -7 days..0", [], [(ts, False)], [("sum", x, ("range", datetime.timedelta(days=-7), 0))])
    ts.free()
    xn = G(rdf.F64, lens, 0, -1e3, 1e3, col_id=63, null_mod=7)
    run("forward fill: last_value IGNORE NULLS ROWS unbounded..0", [], [], [("last_value", xn, ("rows", None, 0), True)])
    xn.free()
    x.free()
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": card(), "rows": out_rows}, f, indent=1)


if __name__ == "__main__":
    main()
