#!/usr/bin/env python
"""The as-of join (bdf_join_asof_dev) beside the sort of its right side (bdf_sort_indices_dev by (by, on), the sort the as-of join
starts with), and LEFT SEMI / ANTI beside INNER on the same keys (bdf_join_indices_dev), at 1e8 left x 1e6 right and 1e7 x 1e7 rows,
with Int64 and Timestamp(ms) `on` keys, without and with one Int32 `by` key.  Every row is the wall time of one call that ends in a
device synchronise, the median of three calls after a warm-up call; the card's name and power limit are read in the same run.

    python benchmarks/join_asof_bench.py [--json out.json] [--sizes 1e8x1e6,1e7x1e7]
"""
from __future__ import annotations

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

import rust_dataframe_b200 as rdf  # noqa: E402


def card() -> str:
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1e8x1e6,1e7x1e7")
    ap.add_argument("--json")
    args = ap.parse_args()
    ctx = rdf.default_context()
    G = rdf.Column.generate
    out_rows = []
    print(f"card: {card()}", flush=True)

    def timed(what, fn, free, **meta):
        free(fn())   # warm-up
        ctx.synchronize()
        runs = []
        for _ in range(3):
            t0 = time.perf_counter()
            res = fn()
            ctx.synchronize()
            runs.append((time.perf_counter() - t0) * 1e3)
            free(res)
        ms = float(np.median(runs))
        print(f"{what:72s} {ms:9.2f} ms   runs: {', '.join(f'{r:.2f}' for r in runs)}", flush=True)
        out_rows.append({"case": what, "ms": ms, "runs_ms": runs, **meta})

    def int_col(dtype, n, lo, hi, col_id):
        chunk = 4_000_000
        lens = [chunk] * (n // chunk) + ([n % chunk] if n % chunk else [])
        f = G(rdf.F64, lens, 0, lo, hi, col_id=col_id)
        c = f.cast(dtype)
        f.free()
        return c

    free_one = lambda c: c.free()
    free_pair = lambda p: [c.free() for c in p if c is not None]
    TS = rdf.TemporalType.timestamp("ms")
    for size in args.sizes.split(","):
        nl, nr = (int(float(x)) for x in size.split("x"))
        span = 365 * 86_400_000.0   # one year of milliseconds
        lon, ron = int_col(rdf.I64, nl, 0.0, span, 70), int_col(rdf.I64, nr, 0.0, span, 71)
        lby, rby = int_col(rdf.I32, nl, 0.0, 5000.0, 72), int_col(rdf.I32, nr, 0.0, 5000.0, 73)   # ~5000 symbols
        for by in (False, True):
            tag = f"{nl:.0e} x {nr:.0e}, {'one i32 by key' if by else 'no by key'}"
            keys = [rdf.native.SortKeyC(c.handle.value, 0) for c in ([rby] if by else []) + [ron]]
            arr = (rdf.native.SortKeyC * len(keys))(*keys)

            def sort_right():
                h = C.c_void_p()
                rdf.native.raise_for_status(rdf.native.lib().bdf_sort_indices_dev(ctx.handle, len(keys), arr, C.byref(h)))
                return rdf.Column(ctx, h)

            timed(f"sort right side by ({'by, ' if by else ''}on)   [{tag}]", sort_right, free_one, left=nl, right=nr, by=by, op="sort")
            for kind in ("i64", "timestamp"):
                for c in (lon, ron):
                    c.with_temporal(TS if kind == "timestamp" else None)
                timed(f"as-of backward, {kind} on   [{tag}]",
                      lambda: rdf.join_asof_indices(lon, ron, [lby] if by else [], [rby] if by else []), free_one, left=nl, right=nr, by=by,
                      op=f"asof_{kind}")
            for c in (lon, ron):
                c.with_temporal(None)
            # equi-joins on the same sizes: keys drawn from 2 x the right side's row count, so about 40 % of left rows match once
            lk, rk = int_col(rdf.I64, nl, 0.0, 2.0 * nr, 74), int_col(rdf.I64, nr, 0.0, 2.0 * nr, 75)
            crit_l, crit_r = ([lby] if by else []) + [lk], ([rby] if by else []) + [rk]
            for how in ("inner", "left_semi", "left_anti"):
                timed(f"join {how:9s}   [{tag}]", lambda: rdf.join_indices(crit_l, crit_r, how), free_pair, left=nl, right=nr, by=by, op=how)
            lk.free()
            rk.free()
        for c in (lon, ron, lby, rby):
            c.free()
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": card(), "rows": out_rows}, f, indent=1)


if __name__ == "__main__":
    main()
