#!/usr/bin/env python
"""Per-kernel roofline table for the SURVEY 8(d) configurations (device-resident data, CUDA-event timing on
the library's compute stream via its launch records).  Not the headline benchmark (that is bench.py); this
is the evidence that every kernel of the path, not only f64 add, runs near the HBM roofline.

    python benchmarks/kernels_bench.py [--rows 100000000] [--json kernels.json]
    python benchmarks/kernels_bench.py --csv [--csv-rows 50000000] [--json csv.json]   # the CSV reader rows instead (a 2.55 GB temporary file)
    python benchmarks/kernels_bench.py --window [--rows 100000000]                      # only the window-function rows
    python benchmarks/kernels_bench.py --math [--rows 100000000]                        # only the float-function rows
    python benchmarks/kernels_bench.py --stats [--rows 100000000]                       # only the statistical-aggregate rows
    python benchmarks/kernels_bench.py --csv-write [--csv-rows 50000000]                # the CSV writer rows (the reader's table written back)
    python benchmarks/kernels_bench.py --json-write [--csv-rows 50000000]               # the JSON writer rows (that table and a List<Float64>)
    python benchmarks/kernels_bench.py --lists [--rows 100000000]                       # the list-function rows (ArrayFunctions)
    python benchmarks/kernels_bench.py --temporal [--rows 100000000]                    # the date / timestamp function rows
    python benchmarks/kernels_bench.py --ndjson [--csv-rows 50000000]                   # the line-delimited JSON reader rows (a 4.85 GB temporary file)
    python benchmarks/kernels_bench.py --parquet [--csv-rows 50000000]                  # the Parquet reader rows (two temporary files: snappy, none)
    python benchmarks/kernels_bench.py --parquet-write [--csv-rows 50000000]            # the Parquet writer rows (none/PLAIN, none/dictionary, snappy/dictionary)
    python benchmarks/kernels_bench.py --distribution [--rows 100000000]                # median, hist, uniques, mode next to k_reduce and the sort
    python benchmarks/kernels_bench.py --nulls [--rows 100000000]                       # coalesce, case_when, greatest, nanvl, is_null ... against ADD, then bench.py
"""
from __future__ import annotations

import argparse
from collections import OrderedDict
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import rust_dataframe_b200 as rdf  # noqa: E402
from rust_dataframe_b200 import native as N  # noqa: E402
from benchmarks import configs_bench  # noqa: E402


def timed(ctx, fn, reps=12):
    """Run fn() reps times with profiling on; return per-kernel-kind (median ms, bytes, rows)."""
    for _ in range(3):
        out = fn()
        for o in out if isinstance(out, (list, tuple)) else [out]:
            if isinstance(o, rdf.Column):
                o.free()
    ctx.synchronize()
    ctx.profile_read()
    ctx.profile_enable(True)
    for _ in range(reps):
        out = fn()
        for o in out if isinstance(out, (list, tuple)) else [out]:
            if isinstance(o, rdf.Column):
                o.free()
    ctx.profile_enable(False)
    recs = ctx.profile_read()
    per_call = max(1, len(recs) // reps)
    by = {}
    for i, r in enumerate(recs):   # several launches of the same kind per call (filter: count+scan, scatter) stay separate
        key = r["kernel"] if per_call == 1 or sum(1 for q in recs[:per_call] if q["kernel"] == r["kernel"]) == 1 else f'{r["kernel"]}#{i % per_call}'
        by.setdefault(key, []).append(r)
    return {k: (float(np.median([r["ms"] for r in v])), v[0]["bytes"], v[0]["rows"]) for k, v in by.items()}


def _digits(v, width):
    """uint8 [len(v), width]: the non-negative integers v as zero-padded ASCII."""
    p = 10 ** np.arange(width - 1, -1, -1, dtype=np.int64)
    return ((v[:, None] // p[None, :]) % 10 + 48).astype(np.uint8)


def write_csv(path, rows, seed=11, block=5_000_000):
    """rows x (Int64 id, lat and lng with 6 decimals, Boolean, a quoted city with a comma): 51 bytes per row, fixed width."""
    rng = np.random.default_rng(seed)
    with open(path, "wb") as f:
        f.write(b"id,lat,lng,flag,city\n")
        for r0 in range(0, rows, block):
            n = min(block, rows - r0)
            m = np.empty((n, 51), np.uint8)
            m[:, 0:10] = _digits(np.arange(r0, r0 + n, dtype=np.int64) * 7 % 10 ** 10, 10)
            lat, lng = rng.integers(-90_000_000, 90_000_000, n), rng.integers(-180_000_000, 180_000_000, n)
            m[:, 10] = 44
            m[:, 11] = np.where(lat < 0, 45, 43)
            d = _digits(np.abs(lat), 8)
            m[:, 12:14], m[:, 14], m[:, 15:21] = d[:, :2], 46, d[:, 2:]
            m[:, 21] = 44
            m[:, 22] = np.where(lng < 0, 45, 43)
            d = _digits(np.abs(lng), 9)
            m[:, 23:26], m[:, 26], m[:, 27:33] = d[:, :3], 46, d[:, 3:]
            m[:, 33] = 44
            flag = rng.random(n) < 0.5
            m[:, 34:50] = np.where(flag[:, None], np.frombuffer(b'true,"Leeds, UK"', np.uint8), np.frombuffer(b'false,"Leed, UK"', np.uint8))
            m[:, 50] = 10
            f.write(m.tobytes())


def csv_bench(ctx, rows, rows_out, reps=3):
    """File -> device columns: the upload, the tokenizer and parse kernels (launch records), end to end; Arrow C++ on the host."""
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "bench.csv")
        write_csv(path, rows)
        nbytes = os.path.getsize(path)
        schema = [rdf.I64, rdf.F64, rdf.F64, N.BOOL, N.UTF8]
        e2e, up, tok, parse = [], [], [], []
        for _ in range(reps + 1):
            ctx.synchronize()
            ctx.profile_read()
            ctx.profile_enable(True)
            t0 = time.perf_counter()
            with rdf.CsvFile(path, schema=schema, ctx=ctx) as f:
                cols = f.read(["id", "lat", "lng", "flag"])
                ctx.synchronize()
                t1 = time.perf_counter()
                st = f.stats()
            ctx.profile_enable(False)
            recs = [r for r in ctx.profile_read() if r["kernel"] == "csv"]
            for c in cols.values():
                c.free()
            e2e.append((t1 - t0) * 1e3)
            up.append(st["upload_ms"])
            tok.append(sum(r["ms"] for r in recs[:3]))   # tokenize (4 kernels), field index, record check
            parse.append(sum(r["ms"] for r in recs[3:]))
        med = lambda v: float(np.median(v[1:]))   # the first run warms up
        for name, ms in (("csv upload (page cache -> HBM)", med(up)), ("csv tokenize + index + check", med(tok)),
                         ("csv parse 4 columns", med(parse)), ("csv file -> device columns, end to end", med(e2e))):
            gbs = nbytes / ms / 1e6
            rows_out.append({"case": name, "config": "csv", "kernel": "csv", "ms": ms, "rows": rows, "file_bytes": nbytes, "GBs_of_file": gbs})
            print(f"{name:44s} {ms:9.2f} ms  {gbs:7.2f} GB/s of file bytes ({nbytes / 1e9:.2f} GB, {rows:.1e} rows)", flush=True)
        try:
            import pyarrow as pa
            import pyarrow.csv as pacsv
        except ImportError:
            return
        types = {"id": pa.int64(), "lat": pa.float64(), "lng": pa.float64(), "flag": pa.bool_(), "city": pa.string()}
        ts = []
        for _ in range(2):
            t0 = time.perf_counter()
            pacsv.read_csv(path, convert_options=pacsv.ConvertOptions(column_types=types))
            ts.append((time.perf_counter() - t0) * 1e3)
        ms = min(ts)
        name = f"Arrow C++ (not the reference) read_csv, {os.cpu_count()} cores"
        rows_out.append({"case": name, "config": "csv", "kernel": "host", "ms": ms, "rows": rows, "file_bytes": nbytes, "GBs_of_file": nbytes / ms / 1e6})
        print(f"{name:44s} {ms:9.2f} ms  {nbytes / ms / 1e6:7.2f} GB/s of file bytes", flush=True)


def write_ndjson(path, rows, seed=13, block=2_000_000):
    """rows x {"id": Int64, "a", "b": Float64 with 7 significant digits, "ok": Boolean, "tags": 0..4 two-digit Int32, "s": a string}:
    97 bytes per line, fixed width (the unused places of a value are JSON whitespace)."""
    rng = np.random.default_rng(seed)
    parts = [b'{"id":', 10, b',"a":', 13, b',"b":', 13, b',"ok":', 5, b',"tags":', 14, b',"s":"abc"}\n']
    width = sum(len(x) if isinstance(x, bytes) else x for x in parts)
    with open(path, "wb") as f:
        for r0 in range(0, rows, block):
            n = min(block, rows - r0)
            m = np.empty((n, width), np.uint8)
            at, fields = 0, []
            for x in parts:
                if isinstance(x, bytes):
                    m[:, at:at + len(x)] = np.frombuffer(x, np.uint8)
                    at += len(x)
                else:
                    fields.append((at, x))
                    at += x
            (pi, _), (pa_, _), (pb, _), (po, _), (pt, _) = fields
            m[:, pi:pi + 10] = _digits(1_000_000_000 + np.arange(r0, r0 + n, dtype=np.int64) * 7 % 9_000_000_000, 10)
            for p in (pa_, pb):   # [-]d.dddddde[+-]dd
                mant, ex = rng.integers(1_000_000, 10_000_000, n), rng.integers(-30, 31, n)
                m[:, p] = np.where(rng.random(n) < 0.5, 45, 32)
                d = _digits(mant, 7)
                m[:, p + 1], m[:, p + 2], m[:, p + 3:p + 9] = d[:, 0], 46, d[:, 1:]
                m[:, p + 9], m[:, p + 10] = 101, np.where(ex < 0, 45, 43)
                m[:, p + 11:p + 13] = _digits(np.abs(ex), 2)
            ok = rng.random(n) < 0.5
            m[:, po:po + 5] = np.where(ok[:, None], np.frombuffer(b"true ", np.uint8), np.frombuffer(b"false", np.uint8))
            k = rng.integers(0, 5, n)
            m[:, pt:pt + 14] = 32
            m[:, pt], m[:, pt + 13] = 91, 93
            for i in range(4):
                has = k > i
                d = _digits(rng.integers(10, 100, n), 2)
                c = pt + 1 + 3 * i
                m[:, c] = np.where(has & (i > 0), 44, 32)
                m[:, c + 1] = np.where(has, d[:, 0], 32)
                m[:, c + 2] = np.where(has, d[:, 1], 32)
            f.write(m.tobytes())


def write_parquet_table(path, rows, compression, seed=17, block=5_000_000):
    """Int64 id, two Float64 (b: 10 % nulls, values on a grid of 1/64 so that it dictionary-encodes), Boolean, Date32, Timestamp(us),
    written by pyarrow with its defaults (snappy + dictionary) or uncompressed."""
    import pyarrow as pa
    import pyarrow.parquet as pq

    rng = np.random.default_rng(seed)
    schema = pa.schema([("id", pa.int64()), ("a", pa.float64()), ("b", pa.float64()), ("ok", pa.bool_()), ("d", pa.date32()),
                        ("ts", pa.timestamp("us"))])
    with pq.ParquetWriter(path, schema, compression=compression) as w:
        for s in range(0, rows, block):
            n = min(block, rows - s)
            w.write_table(pa.table({
                "id": pa.array(np.arange(s, s + n, dtype=np.int64)),
                "a": pa.array(rng.standard_normal(n)),
                "b": pa.array(rng.integers(0, 4096, n) / 64.0, mask=rng.random(n) < 0.1),
                "ok": pa.array(rng.random(n) < 0.5),
                "d": pa.array(rng.integers(0, 20000, n).astype(np.int32), pa.date32()),
                "ts": pa.array(1_600_000_000_000_000 + np.sort(rng.integers(0, 10 ** 13, n)), pa.timestamp("us")),
            }, schema=schema))


def parquet_bench(ctx, rows, rows_out, reps=3):
    """Parquet -> device columns, for a file written with pyarrow's defaults and one written uncompressed: the upload of the column
    chunks, snappy, the run walk + levels and the values (launch records), end to end (open + read + synchronise); pyarrow's
    read_table on the host for comparison."""
    import pyarrow.parquet as pq

    names = ["id", "a", "b", "ok", "d", "ts"]
    with tempfile.TemporaryDirectory() as td:
        for label, comp in (("snappy", "snappy"), ("none", "none")):
            path = os.path.join(td, f"bench-{label}.parquet")
            write_parquet_table(path, rows, comp)
            fbytes = os.path.getsize(path)
            e2e, up, sn, lv, va, ub, sb, ob = [], [], [], [], [], 0, 0, 0
            for _ in range(reps + 1):
                ctx.synchronize()
                ctx.profile_read()
                ctx.profile_enable(True)
                t0 = time.perf_counter()
                with rdf.ParquetFile(path) as f:
                    cols = f.read(names, ctx=ctx)
                    ctx.synchronize()
                    t1 = time.perf_counter()
                    st = f.stats()
                ctx.profile_enable(False)
                recs = [r for r in ctx.profile_read() if r["kernel"] == "parquet"]
                assert len(recs) == 4, recs
                for c in cols.values():
                    c.free()
                e2e.append((t1 - t0) * 1e3)
                up.append(st["upload_ms"])
                sn.append(recs[0]["ms"]); lv.append(recs[1]["ms"] + recs[2]["ms"]); va.append(recs[3]["ms"])
                ub, sb, ob = st["uploaded_bytes"], recs[0]["bytes"] - st["uploaded_bytes"], recs[3]["bytes"]
            med = lambda v: float(np.median(v[1:]))   # the first run warms up
            for name, ms, nbytes in ((f"parquet[{label}] upload (page cache -> HBM)", med(up), ub),
                                     (f"parquet[{label}] snappy", med(sn), ub + sb),
                                     (f"parquet[{label}] runs + levels", med(lv), ub + sb),
                                     (f"parquet[{label}] values", med(va), ub + sb + ob),
                                     (f"parquet[{label}] file -> device columns, end to end", med(e2e), fbytes)):
                rows_out.append({"case": name, "config": "parquet", "kernel": "parquet", "ms": ms, "rows": rows, "bytes": nbytes,
                                 "file_bytes": fbytes, "uploaded_bytes": ub, "scratch_bytes": sb, "output_bytes": ob})
                print(f"{name:52s} {ms:9.2f} ms  {nbytes / 1e9:6.2f} GB  {nbytes / ms / 1e6:8.1f} GB/s", flush=True)
            ts = []
            for _ in range(2):
                t0 = time.perf_counter()
                pq.read_table(path, columns=names)
                ts.append((time.perf_counter() - t0) * 1e3)
            ms = min(ts)
            name = f"parquet[{label}] pyarrow read_table (not the reference), {os.cpu_count()} cores"
            rows_out.append({"case": name, "config": "parquet", "kernel": "host", "ms": ms, "rows": rows, "file_bytes": fbytes})
            print(f"{name:52s} {ms:9.2f} ms  {fbytes / 1e9:6.2f} GB of file", flush=True)


def parquet_write_bench(ctx, rows, rows_out, reps=3):
    """The reader benchmark's table on the device in 2^20-row chunks, written back with bdf_parquet_write three ways (none / PLAIN,
    none / dictionary, snappy / dictionary): the dictionary step (the sorted_runs kernels and the id scatter), the encode and the snappy
    steps from the launch records, end to end to /dev/null and to a file; a D2H copy of one column for the link's rate; pyarrow's
    write_table with the same options on the host for comparison.  Medians of `reps` runs after a warm-up."""
    import pyarrow as pa
    import pyarrow.parquet as pq

    names = ["id", "a", "b", "ok", "d", "ts"]
    with tempfile.TemporaryDirectory() as td:
        src = os.path.join(td, "src.parquet")
        write_parquet_table(src, rows, "none")
        with rdf.ParquetFile(src, batch_size=1 << 20) as f:
            cols = f.read(names, ctx=ctx)
        host = pq.read_table(src)
        os.unlink(src)
        import torch   # the link's device -> pinned host rate, for the end-to-end rows to be read against

        dev = torch.empty(rows * 8, dtype=torch.uint8, device="cuda")
        pin = torch.empty(rows * 8, dtype=torch.uint8, pin_memory=True)
        d2h = []
        for _ in range(reps + 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pin.copy_(dev)
            torch.cuda.synchronize()
            d2h.append((time.perf_counter() - t0) * 1e3)
        del dev, pin
        d2h_ms = float(np.median(d2h[1:]))
        name = f"parquet write: D2H into pinned memory ({rows * 8 / 1e9:.2f} GB)"
        rows_out.append({"case": name, "config": "parquet-write", "kernel": "d2h", "ms": d2h_ms, "rows": rows, "GBs": rows * 8 / d2h_ms / 1e6})
        print(f"{name:58s} {d2h_ms:9.2f} ms  {rows * 8 / d2h_ms / 1e6:7.2f} GB/s", flush=True)
        out = os.path.join(td, "out.parquet")
        for label, kw in (("none/PLAIN", {"dictionary": False}), ("none/dictionary", {}), ("snappy/dictionary", {"compression": "snappy"})):
            rdf.write_parquet(out, cols, **kw)
            fbytes = os.path.getsize(out)
            res = {"dictionary": [], "encode": [], "snappy": [], "end to end, /dev/null": [], "end to end, file": []}
            for i in range(reps + 1):
                for target, key in (("/dev/null", "end to end, /dev/null"), (out, "end to end, file")):
                    ctx.synchronize()
                    ctx.profile_read()
                    ctx.profile_enable(True)
                    t0 = time.perf_counter()
                    rdf.write_parquet(target, cols, **kw)
                    t1 = time.perf_counter()
                    ctx.profile_enable(False)
                    recs = ctx.profile_read()
                    if i == 0:
                        continue
                    res[key].append((t1 - t0) * 1e3)
                    if target == "/dev/null":
                        pw = [r for r in recs if r["kernel"] == "parquet_write"]
                        res["encode"].append(sum(r["ms"] for r in pw if r["dtype"] == -1))
                        res["snappy"].append(sum(r["ms"] for r in pw if r["dtype"] == rdf.U8))
                        res["dictionary"].append(sum(r["ms"] for r in recs if not (r["kernel"] == "parquet_write" and r["dtype"] in (-1, rdf.U8))))
            for key, v in res.items():
                ms = float(np.median(v))
                if (key == "snappy" and "snappy" not in label) or (key == "dictionary" and "PLAIN" in label):
                    continue
                name = f"parquet write [{label}] {key}"
                rows_out.append({"case": name, "config": "parquet-write", "kernel": "parquet_write", "ms": ms, "rows": rows, "file_bytes": fbytes,
                                 "Mrows_per_s": rows / ms / 1e3, "GBs_of_file": fbytes / ms / 1e6})
                print(f"{name:58s} {ms:9.2f} ms  {rows / ms / 1e3:9.1f} Mrows/s  {fbytes / ms / 1e6:7.2f} GB/s of file ({fbytes / 1e9:.2f} GB)",
                      flush=True)
            ts = []
            for _ in range(2):
                t0 = time.perf_counter()
                pq.write_table(host, out, compression="snappy" if "snappy" in label else "none", use_dictionary="PLAIN" not in label,
                               data_page_version="1.0", row_group_size=1 << 20)
                ts.append((time.perf_counter() - t0) * 1e3)
            ms = min(ts)
            name = f"parquet write [{label}] pyarrow write_table (not the reference), {os.cpu_count()} cores"
            rows_out.append({"case": name, "config": "parquet-write", "kernel": "host", "ms": ms, "rows": rows, "file_bytes": os.path.getsize(out)})
            print(f"{name:58s} {ms:9.2f} ms  {rows / ms / 1e3:9.1f} Mrows/s", flush=True)
        for c in cols.values():
            c.free()


def ndjson_bench(ctx, rows, rows_out, reps=3):
    """Line-delimited JSON -> device columns: the upload, the record index, key resolution + inference and the conversions (launch
    records), end to end; pyarrow's read_json on the host for comparison."""
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "bench.json")
        write_ndjson(path, rows)
        nbytes = os.path.getsize(path)
        e2e, up, tok, keys, parse = [], [], [], [], []
        for _ in range(reps + 1):
            ctx.synchronize()
            ctx.profile_read()
            ctx.profile_enable(True)
            t0 = time.perf_counter()
            with rdf.JsonFile(path, ctx=ctx) as f:
                cols = f.read(["id", "a", "b", "ok"])
                tags = f.read_list("tags")
                ctx.synchronize()
                t1 = time.perf_counter()
                st = f.stats()
                schema = f.schema
            ctx.profile_enable(False)
            recs = [r for r in ctx.profile_read() if r["kernel"] == "json"]
            for c in cols.values():
                c.free()
            tags.free()
            e2e.append((t1 - t0) * 1e3)
            up.append(st["upload_ms"])
            tok.append(sum(r["ms"] for r in recs[:5]))     # newline count + index, record check, the two scans, the member list
            keys.append(sum(r["ms"] for r in recs[5:8]))   # key table, resolution, inference
            parse.append(sum(r["ms"] for r in recs[8:]))   # four scalar columns, the List<Int64> column
        assert [n for n, _, _ in schema] == ["id", "a", "b", "ok", "tags", "s"], schema
        med = lambda v: float(np.median(v[1:]))   # the first run warms up
        for name, ms in (("json upload (page cache -> HBM)", med(up)), ("json tokenize + index", med(tok)),
                         ("json key resolution + inference", med(keys)), ("json parse 4 columns + 1 list", med(parse)),
                         ("json file -> device columns, end to end", med(e2e))):
            gbs = nbytes / ms / 1e6
            rows_out.append({"case": name, "config": "ndjson", "kernel": "json", "ms": ms, "rows": rows, "file_bytes": nbytes, "GBs_of_file": gbs})
            print(f"{name:44s} {ms:9.2f} ms  {gbs:7.2f} GB/s of file bytes ({nbytes / 1e9:.2f} GB, {rows:.1e} records)", flush=True)
        try:
            import pyarrow.json as pajson
        except ImportError:
            return
        ts = []
        for _ in range(2):
            t0 = time.perf_counter()
            pajson.read_json(path)
            ts.append((time.perf_counter() - t0) * 1e3)
        ms = min(ts)
        name = f"pyarrow read_json (not the reference), {os.cpu_count()} cores"
        rows_out.append({"case": name, "config": "ndjson", "kernel": "host", "ms": ms, "rows": rows, "file_bytes": nbytes, "GBs_of_file": nbytes / ms / 1e6})
        print(f"{name:44s} {ms:9.2f} ms  {nbytes / ms / 1e6:7.2f} GB/s of file bytes", flush=True)


def csv_write_bench(ctx, rows, rows_out, reps=3):
    """The reader benchmark's table (Int64, two Float64, Boolean) read onto the device, then written back: the measure + scan and
    emit kernels (launch records) in GB/s of text, end to end to /dev/null (D2H and the pipeline without a file system) and to a file;
    pyarrow's write_csv on the host cores.  Medians of `reps` runs after a warm-up."""
    print("card:", _card(), flush=True)
    with tempfile.TemporaryDirectory() as td:
        src = os.path.join(td, "bench.csv")
        write_csv(src, rows)
        with rdf.CsvFile(src, schema=[rdf.I64, rdf.F64, rdf.F64, N.BOOL, N.UTF8], batch_size=1 << 20, ctx=ctx) as f:
            cols = f.read(["id", "lat", "lng", "flag"])
        os.unlink(src)
        out = os.path.join(td, "out.csv")
        rdf.write_csv(out, cols)
        text = os.path.getsize(out)
        res = {"measure + scan": [], "emit": [], "end to end, /dev/null": [], "end to end, file": []}
        for i in range(reps + 1):
            for target, key in (("/dev/null", "end to end, /dev/null"), (out, "end to end, file")):
                ctx.synchronize()
                ctx.profile_read()
                ctx.profile_enable(True)
                t0 = time.perf_counter()
                rdf.write_csv(target, cols)
                t1 = time.perf_counter()
                ctx.profile_enable(False)
                recs = [r for r in ctx.profile_read() if r["kernel"] == "csv_write"]
                if i == 0:
                    continue
                res[key].append((t1 - t0) * 1e3)
                if target == "/dev/null":
                    res["measure + scan"].append(sum(r["ms"] for r in recs if r["dtype"] == rdf.U64))
                    res["emit"].append(sum(r["ms"] for r in recs if r["dtype"] == rdf.U8))
        for key, v in res.items():
            ms = float(np.median(v))
            rows_out.append({"case": f"csv write {key}", "config": "csv-write", "kernel": "csv_write", "ms": ms, "rows": rows, "text_bytes": text,
                             "GBs_of_text": text / ms / 1e6})
            print(f"{'csv write ' + key:44s} {ms:9.2f} ms  {text / ms / 1e6:7.2f} GB/s of text ({text / 1e9:.2f} GB, {rows:.1e} rows)", flush=True)
        try:
            import pyarrow as pa
            import pyarrow.csv as pacsv
        except ImportError:
            return
        host = {n: np.concatenate([a.value_bits() if n == "flag" else a.value_slice() for a in c.download()]) for n, c in cols.items()}
        table = pa.table(host)
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            pacsv.write_csv(table, out)
            ts.append((time.perf_counter() - t0) * 1e3)
        ms = float(np.median(ts))
        name = f"pyarrow write_csv (not the reference), {os.cpu_count()} cores"
        rows_out.append({"case": name, "config": "csv-write", "kernel": "host", "ms": ms, "rows": rows, "text_bytes": os.path.getsize(out)})
        print(f"{name:44s} {ms:9.2f} ms  {os.path.getsize(out) / ms / 1e6:7.2f} GB/s of its text", flush=True)
        for c in cols.values():
            c.free()


def json_write_bench(ctx, rows, rows_out, reps=3, pandas_rows=1_000_000):
    """The CSV writer benchmark's table (Int64, two Float64, Boolean) plus a List<Float64> of mean length 4 (0..8 elements per row),
    written as line-delimited JSON: the measure, scan and emit launches (launch records) in GB/s of text, end to end to /dev/null and
    to a file, the CSV writer on the same numeric columns in the same session, and pandas' to_json(orient="records", lines=True) on
    the host over the first `pandas_rows` rows.  Medians of `reps` runs after a warm-up."""
    print("card:", _card(), flush=True)
    with tempfile.TemporaryDirectory() as td:
        src = os.path.join(td, "bench.csv")
        write_csv(src, rows)
        with rdf.CsvFile(src, schema=[rdf.I64, rdf.F64, rdf.F64, N.BOOL, N.UTF8], batch_size=1 << 20, ctx=ctx) as f:
            cols = f.read(["id", "lat", "lng", "flag"])
        os.unlink(src)
        rng = np.random.default_rng(20261019)
        chunks = []
        for a in cols["id"].download():
            offs = np.concatenate([[0], np.cumsum(rng.integers(0, 9, a.length))]).astype(np.int32)
            chunks.append(rdf.ListArray(rdf.F64, offs, None, 0, a.length, 0, rdf.PrimitiveArray.from_numpy(rng.normal(size=int(offs[-1])) * 100.0)))
        tags = rdf.ListColumn.upload(chunks, ctx=ctx, dtype=rdf.F64)
        del chunks
        frame = OrderedDict(list(cols.items()) + [("tags", tags)])
        out = os.path.join(td, "out.json")
        rdf.write_json(out, frame)
        text = os.path.getsize(out)
        rdf.write_csv(out, cols)
        csv_text = os.path.getsize(out)
        res = {"measure": [], "scan": [], "emit": [], "plan": [], "end to end, /dev/null": [], "end to end, file": [], "csv, /dev/null": []}
        for i in range(reps + 1):
            for target, key in (("/dev/null", "end to end, /dev/null"), (out, "end to end, file"), ("/dev/null", "csv, /dev/null")):
                ctx.synchronize()
                ctx.profile_read()
                ctx.profile_enable(True)
                t0 = time.perf_counter()
                if key.startswith("csv"):
                    rdf.write_csv(target, cols)
                else:
                    rdf.write_json(target, frame)
                t1 = time.perf_counter()
                ctx.profile_enable(False)
                recs = [r for r in ctx.profile_read() if r["kernel"] == "json_write"]
                if i == 0:
                    continue
                res[key].append((t1 - t0) * 1e3)
                if key == "end to end, /dev/null":
                    for part, dt in (("measure", rdf.U64), ("scan", rdf.U32), ("emit", rdf.U8), ("plan", -1)):
                        res[part].append(sum(r["ms"] for r in recs if r["dtype"] == dt))
        for key, v in res.items():
            ms = float(np.median(v))
            nb = csv_text if key.startswith("csv") else text
            name = "csv write (same numeric columns) /dev/null" if key.startswith("csv") else f"json write {key}"
            rows_out.append({"case": name, "config": "json-write", "kernel": "csv_write" if key.startswith("csv") else "json_write", "ms": ms,
                             "rows": rows, "text_bytes": nb, "GBs_of_text": nb / ms / 1e6})
            print(f"{name:44s} {ms:9.2f} ms  {nb / ms / 1e6:7.2f} GB/s of text ({nb / 1e9:.2f} GB, {rows:.1e} rows)", flush=True)
        try:
            import pandas as pd
        except ImportError:
            return
        m = min(pandas_rows, rows)
        host = {n: np.concatenate([a.value_bits() if n == "flag" else a.value_slice() for a in c.download()])[:m] for n, c in cols.items()}
        lists = [x for a in tags.download() for x in a.to_pylist()][:m] if m <= 2_000_000 else None
        df = pd.DataFrame(dict(host, tags=lists))
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            df.to_json(out, orient="records", lines=True)
            ts.append((time.perf_counter() - t0) * 1e3)
        ms = float(np.median(ts))
        nb = os.path.getsize(out)
        name = f"pandas to_json lines (not the reference), {m:.0e} rows"
        rows_out.append({"case": name, "config": "json-write", "kernel": "host", "ms": ms, "rows": m, "text_bytes": nb, "GBs_of_text": nb / ms / 1e6})
        print(f"{name:44s} {ms:9.2f} ms  {nb / ms / 1e6:7.2f} GB/s of its text", flush=True)
        for c in cols.values():
            c.free()
        tags.free()


def window_parts(recs, value_calls):
    """Label the launch records of ONE bdf_window_dev call by step, in launch order: the sort, the gathers of the sorted keys, the
    head bitmaps (k_group_heads, the boolean OR), the runs (popcount scan and run-start compactions), the ranks, then per value call
    (``value_calls``: "shift" or "scan" in call order) the gather of x in sorted order, the kernel itself and the gather back to row
    order."""
    parts, k, seen_rank, back = {}, 0, False, False
    for r in recs:
        kind = r["kernel"]
        if kind == "sort":
            label = "sort"
        elif kind == "compare" or (kind == "window" and r["dtype"] == N.BOOL):
            label = "heads"
        elif kind == "filter" or (kind == "window" and r["dtype"] == rdf.U64):
            label = "runs"
        elif kind == "window" and r["dtype"] == rdf.U32 and not seen_rank:
            label, seen_rank = "rank", True
        elif kind == "window":
            label, k, back = value_calls[k], k + 1, True
        elif kind == "take":
            label = "key gathers" if not seen_rank else "return gathers" if back else "value gathers"
            back = False if seen_rank else back
        else:
            label = kind
        parts[label] = parts.get(label, 0.0) + r["ms"]
    return parts


def window_bench(ctx, rows, lens, rows_out, reps=3):
    """Window functions over 1e8 rows (bdf_window_dev): every row prints its total and its parts."""
    G = rdf.Column.generate

    def run(what, part, order, calls, value_calls):
        for _ in range(2):   # warm-up
            for c in rdf.window(part, order, calls):
                c.free()
        ctx.synchronize()
        ctx.profile_read()
        totals, per_run = [], []
        for _ in range(reps):
            ctx.profile_enable(True)
            out = rdf.window(part, order, calls)
            ctx.profile_enable(False)
            recs = ctx.profile_read()
            for c in out:
                c.free()
            p = window_parts(recs, value_calls)
            per_run.append(p)
            totals.append(sum(p.values()))
        med = int(np.argsort(totals)[len(totals) // 2])
        parts = per_run[med]
        print(f"{what:60s} {totals[med]:8.3f} ms  (" + ", ".join(f"{k} {v:.3f}" for k, v in parts.items()) + ")", flush=True)
        rows_out.append({"case": what, "config": "window", "ms": totals[med], "runs_ms": totals, "rows": rows, "parts": parts})
        return parts

    x = G(rdf.F64, lens, 0, -1e3, 1e3, col_id=60)
    p = run(f"running sum f64 over {rows:.0e} rows (no keys: the scan alone)", [], [], [("sum", x, "rows")], ["scan"])
    pk, pk_src = configs_bench._peak()
    scan_bytes = rows * 16   # 8 B read + 8 B written per row
    print(f"{'':60s} scan: {scan_bytes / p['scan'] / 1e6:8.1f} GB/s algorithmic = {scan_bytes / p['scan'] / 1e6 / pk:5.3f} of the "
          f"{pk:.0f} GB/s ceiling ({pk_src})", flush=True)
    kf = G(rdf.F64, lens, 0, 0.0, rows / 100.0, col_id=61)
    key = kf.cast(rdf.I32)                                  # ~1e6 partitions of ~100 rows
    kf.free()
    run("partition i32 (~1e6) order f64 desc: row_number, rank, lag, sum RANGE", [key], [(x, True)],
        [("row_number",), ("rank",), ("lag", x, 1), ("sum", x, "range")], ["shift", "scan"])
    key.free()
    o = G(rdf.I64, lens, 3, col_id=62)
    run("one partition, order i64: rank, cume_dist (hot partition)", [], [(o, False)], [("rank",), ("cume_dist",)], [])
    o.free()
    kf = G(rdf.F64, lens, 0, -100.0, 100.0, col_id=63)
    small = kf.cast(rdf.I8)                                 # 200 partitions, no order
    kf.free()
    run("partition i8 (200), no order: sum PARTITION (totals on every row)", [small], [], [("sum", x, "partition")], ["scan"])
    small.free()
    x.free()


def math_bench(ctx, lens, report):
    """The float function library: trig, the functions with an exact-result step (log2 f64, log10 f32, hypot f64) next to
    their siblings without one, and the same functions in the fused kernel."""
    G = rdf.Column.generate
    x = G(rdf.F64, lens, 0, 1e-3, 1e3, col_id=30)
    y = G(rdf.F64, lens, 0, 1e-3, 1e3, col_id=31)
    x32 = G(rdf.F32, lens, 0, 1e-3, 1e3, col_id=32)
    for name in ("sin", "exp", "log2", "log10"):
        report(f"{name} f64", "math", timed(ctx, lambda: x.unary(getattr(N, name.upper()))), "unary")
    for name in ("sin", "log2", "log10"):
        report(f"{name} f32", "math", timed(ctx, lambda: x32.unary(getattr(N, name.upper()))), "unary")
    for name in ("atan2", "hypot", "log"):
        report(f"{name} f64", "math", timed(ctx, lambda: getattr(x, name)(y)), "binary")
    report("N3 fused log2(a) + b", "math", timed(ctx, lambda: rdf.eval_expr([x, y], [("log2", 0), (N.ADD, 2, 1)])), "expr")
    report("N3 fused hypot(a, b)", "math", timed(ctx, lambda: rdf.eval_expr([x, y], [(N.HYPOT, 0, 1)])), "expr")
    for col in (x, y, x32):
        col.free()


def _card():
    import subprocess

    try:   # read-only query: the card and its power limit belong beside every number of the run
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def stats_bench(ctx, lens, report, rows_out):
    """The statistical aggregates: k_moments against k_reduce on the same columns (old and new rows alternating, the median of
    three medians), group-by variance against avg (fold part apart from sort and takes), whole-column count_distinct."""
    G = rdf.Column.generate
    print("card:", _card(), flush=True)
    cols = [("f64", G(rdf.F64, lens, 0, -1e3, 1e3, col_id=50)), ("f64 10% nulls", G(rdf.F64, lens, 0, -1e3, 1e3, col_id=51, null_mod=10)),
            ("i32", G(rdf.I32, lens, 2, col_id=52))]
    for what, col in cols:
        old, new = [], []
        for _ in range(3):
            old.append(timed(ctx, lambda: col.aggregate_all())["reduce"])
            new.append(timed(ctx, lambda: col.moments())["moments"])
        med = lambda runs: (float(np.median([r[0] for r in runs])), runs[0][1], runs[0][2])
        report(f"aggregate_all {what} (k_reduce)", "stats", {"reduce": med(old)}, "reduce")
        report(f"moments {what} (k_moments)", "stats", {"moments": med(new)}, "moments")
        print(f"{'':44s} ratio moments / reduce = {med(new)[0] / med(old)[0]:.3f}", flush=True)
    a = cols[0][1]
    i32n = G(rdf.I32, lens, 2, col_id=53, null_mod=10)
    kf = G(rdf.F64, lens, 0, -100.0, 100.0, col_id=54)
    small = kf.cast(rdf.I8)
    kf.free()
    for fn in ("avg", "variance", "avg", "variance"):
        res = timed(ctx, lambda: [c.free() for part in rdf.group_by([i32n, small], [(a, fn)]) for c in part] and None, reps=3)
        total = sum(v[0] for v in res.values())
        print(f"group-by i32 (nulls) x i8, {fn} f64{'':14s} {total:8.4f} ms  (" + ", ".join(f"{k} {v[0]:.3f}" for k, v in sorted(res.items())) + ")",
              flush=True)
        rows_out.append({"case": f"group-by i32 (nulls) x i8 keys, {fn} f64", "config": "stats", "kernel": "sort + take + filter + group",
                         "ms": total, "parts": {k: v[0] for k, v in res.items()}})
    res = timed(ctx, lambda: cols[2][1].count_distinct(), reps=3)
    total = sum(v[0] for v in res.values())
    print(f"{'count_distinct i32 (whole column)':44s} {total:8.4f} ms  (" + ", ".join(f"{k} {v[0]:.3f}" for k, v in sorted(res.items())) + ")",
          flush=True)
    rows_out.append({"case": "count_distinct i32 (whole column)", "config": "stats", "kernel": "sort + take + filter + group", "ms": total,
                     "parts": {k: v[0] for k, v in res.items()}})
    for col in [c for _, c in cols] + [i32n, small]:
        col.free()


def _wall3(ctx, fn):
    """The median of three timed calls after one warm-up call (each call ends in a device synchronise), in ms."""
    def once():
        out = fn()
        ctx.synchronize()
        for o in out if isinstance(out, (list, tuple)) else [out]:
            if isinstance(o, rdf.Column):
                o.free()
    once()
    t = []
    for _ in range(3):
        t0 = time.perf_counter()
        once()
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def distribution_bench(ctx, lens, rows_out):
    """The column distributions: whole-column median (radix select), hist, uniques and mode, each next to k_reduce and
    bdf_sort_indices_dev on the same column in the same session; per-group median and mode next to avg.  Times are the median of three
    calls after a warm-up call, host clock around calls that end in a synchronise."""
    G = rdf.Column.generate
    card = _card()
    print("card:", card, flush=True)

    def row(case, col, fn):
        ms = _wall3(ctx, fn)
        red = _wall3(ctx, lambda: col.aggregate_all())
        srt = _wall3(ctx, lambda: rdf.sort_indices([(col, False)]))
        rows_out.append({"case": case, "ms": ms, "k_reduce_ms": red, "sort_indices_ms": srt, "card": card})
        print(f"{case:44s} {ms:9.3f} ms   k_reduce {red:8.3f} ms   sort_indices {srt:9.3f} ms   {'faster' if ms < srt else 'SLOWER'} than the sort",
              flush=True)

    f64 = G(rdf.F64, lens, 0, -1e3, 1e3, col_id=60)
    f64n = G(rdf.F64, lens, 0, -1e3, 1e3, col_id=61, null_mod=10)
    eq = G(rdf.F64, lens, 0, 5.0, 5.0, col_id=62)
    i32 = G(rdf.I32, lens, 2, col_id=63)
    i32n = G(rdf.I32, lens, 2, col_id=64, null_mod=10)
    kf = G(rdf.F64, lens, 0, -100.0, 100.0, col_id=65)
    i8 = kf.cast(rdf.I8)
    kf.free()
    eq_i32 = eq.cast(rdf.I32)
    for what, col in (("f64", f64), ("f64 10% nulls", f64n), ("f64 all equal", eq), ("i32", i32), ("i32 10% nulls", i32n),
                      ("i32 all equal", eq_i32)):
        row(f"median {what}", col, lambda: col.median())
    row("hist f64, 10 bins", f64, lambda: f64.hist(10))
    row("hist f64, 2^20 bins", f64, lambda: f64.hist(2 ** 20))
    row("uniques i8 (200 values)", i8, lambda: i8.uniques())
    row("mode i8 (200 values)", i8, lambda: i8.mode())
    row("uniques i32 (~1e8 values)", i32, lambda: i32.uniques())
    row("mode i32 (~1e8 values)", i32, lambda: i32.mode())
    for fn in ("avg", "exact_median", "mode"):
        ms = _wall3(ctx, lambda: [c for part in rdf.group_by([i32n, i8], [(f64, fn)]) for c in part])
        rows_out.append({"case": f"group-by i32 (nulls) x i8 keys, {fn} f64", "ms": ms, "card": card})
        print(f"{'group-by i32 (nulls) x i8 keys, ' + fn + ' f64':44s} {ms:9.3f} ms", flush=True)
    for col in (f64, f64n, eq, i32, i32n, i8, eq_i32):
        col.free()


def _stream_rates(rows):
    """The HBM rates of benchmarks/tune_stream.cu (best of each class), built into a temporary directory and run here:
    {"read": read-only sum, "copy": copy 1 read + 1 write} in GB/s."""
    import re
    import subprocess

    src = os.path.join(ROOT, "benchmarks", "tune_stream.cu")
    with tempfile.TemporaryDirectory() as td:
        exe = os.path.join(td, "tune_stream")
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", src, "-o", exe], check=True, capture_output=True)
        out = subprocess.run([exe, str(rows)], check=True, capture_output=True, text=True).stdout
    m = re.search(r"CEILING read-only ([0-9.]+) GB/s, copy 1R1W ([0-9.]+) GB/s", out)
    return {"read": float(m.group(1)), "copy": float(m.group(2))}


def _card():
    import subprocess

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return q.strip().splitlines()[0] if q.strip() else "unknown"


def _timed_calls(ctx, fn, reps=3):
    """Median over `reps` calls (after one warm-up) of the sum of the library's per-launch CUDA-event records of one call."""
    out = fn()
    del out
    ctx.synchronize()
    ctx.profile_read()
    sums = []
    for _ in range(reps):
        ctx.profile_enable(True)
        out = fn()
        ctx.profile_enable(False)
        sums.append(sum(r["ms"] for r in ctx.profile_read()))
        last = out
        del out
    return float(np.median(sums)), last


def lists_bench(ctx, rows, rows_out):
    """ArrayFunctions over rows elements of Int64 and Float64 in 25 chunks at mean list lengths 4, 32 and 1000 (lengths uniform in
    [1, 2 * mean - 1]: no empty list, so max / min are defined), plus one hot list of rows / 10 elements among about rows one-element lists.
    Algorithmic bytes: offsets and elements read once, plus what is written.  Then list take by a random permutation of the lists beside
    the flat take of the elements by a random permutation of the same count, list filter keeping 50 %, and collect_list / collect_set
    of rows Float64 values by an Int32 key of about 1e6 groups beside group-by count of the same columns."""
    card = _card()
    stream = _stream_rates(rows)["read"]
    print(f"card: {card}; tune_stream read-only rate {stream:.1f} GB/s", flush=True)
    rows_out.append({"case": "tune_stream read-only", "GBs": stream, "card": card})
    rng = np.random.default_rng(20261015)
    n_chunks = 25
    per = rows // n_chunks
    for dt in (rdf.I64, rdf.F64):
        npdt = rdf.NP_DTYPES[dt]
        w = npdt.itemsize
        shapes = [("mean 4", 4), ("mean 32", 32), ("mean 1000", 1000), ("hot list", 0)]
        for label, mean in shapes:
            chunks = []
            for k in range(n_chunks):
                if mean:
                    lens = rng.integers(1, 2 * mean, max(per // mean, 1))
                else:   # chunk 0 is one list of rows / 10 elements, every other element is a one-element list
                    lens = np.ones(per, dtype=np.int64) if k else np.array([rows // 10], dtype=np.int64)
                off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
                vals = rng.integers(0, 1 << 20, int(off[-1])).astype(npdt)
                chunks.append(rdf.ListArray(dt, off, None, 0, len(lens), 0, rdf.PrimitiveArray.from_numpy(vals)))
            c = rdf.ListColumn.upload(chunks, ctx)
            E = sum(len(ch.values) for ch in chunks)
            N_ = sum(len(ch) for ch in chunks)
            del chunks
            off_b = 4 * (N_ + n_chunks)
            cases = [("array_contains", lambda: c.array_contains(5), lambda o: E * w + off_b + N_ / 8, True),
                     ("array_position", lambda: c.array_position(5), lambda o: E * w + off_b + 4 * N_, True),
                     ("array_max", lambda: c.array_max(), lambda o: E * w + off_b + N_ * w + N_ / 8, True),
                     ("array_min", lambda: c.array_min(), lambda o: E * w + off_b + N_ * w + N_ / 8, True),
                     ("size", lambda: c.size(), lambda o: off_b + 4 * N_, True),
                     ("array_sort (lexsort path)", lambda: c.array_sort(), lambda o: 2 * (E * w + off_b), False),
                     ("array_distinct", lambda: c.array_distinct(), lambda o: E * w + off_b + len(o.values()) * w + 4 * (N_ + 1), False),
                     ("array_remove", lambda: c.array_remove(5), lambda o: E * w + off_b + len(o.values()) * w + 4 * (N_ + 1), False),
                     ("array_repeat(2)", lambda: c.array_repeat(2), lambda o: E * w + off_b + 2 * E * w + 4 * (N_ + 1), False),
                     ("array_union(self)", lambda: c.array_union(c), lambda o: 2 * (E * w + off_b) + len(o.values()) * w + 4 * (N_ + 1), False),
                     ("explode", lambda: c.explode(), lambda o: E * w + off_b + E * (w + 4), False)]
            # whole lists moved between rows (frames: sort / join / filter), beside the flat take of the same element count
            perm = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(rng.permutation(N_).astype(np.uint32))], ctx)
            eperm = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(rng.permutation(E).astype(np.uint32))], ctx)
            flat = c.values()
            mask = rdf.Column.upload([rdf.BooleanArray.from_numpy(rng.random(c.chunk_info(k)["len"]) < 0.5) for k in range(n_chunks)], ctx)
            cases += [("take, flat elements (yardstick)", lambda: flat.take(eperm), lambda o: E * (4 + 2 * w), False),
                      ("list take (random permutation)", lambda: c.take(perm), lambda o: E * (4 + 2 * w) + 4 * N_ + 2 * off_b + 20 * N_, False),
                      ("list filter 50 %", lambda: c.filter(mask), lambda o: len(o) * 24 + len(o.values()) * (4 + 2 * w) + N_ / 8, False)]
            for name, fn, nbytes, single in cases:
                ms, out = _timed_calls(ctx, fn)
                b = nbytes(out)
                gbs = b / ms / 1e6
                rows_out.append({"case": f"{name} {rdf.DTYPE_NAMES[dt]} {label}", "ms": ms, "elements": E, "lists": N_, "bytes": b, "GBs": gbs,
                                 "frac_of_stream_read": gbs / stream if single else None, "card": card})
                frac = f"  {gbs / stream:5.3f} of read rate" if single else ""
                print(f"{name:28s} {rdf.DTYPE_NAMES[dt]:8s} {label:10s} {ms:9.3f} ms {gbs:8.1f} GB/s{frac}", flush=True)
                del out
            c.free()
    # lists built per group, beside group-by count of the same shape: Float64 values by an Int32 key of about 1e6 groups
    keys = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(rng.integers(0, 1_000_000, per).astype(np.int32)) for _ in range(n_chunks)], ctx)
    x = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(rng.normal(size=per), rng.random(per) > 0.1) for _ in range(n_chunks)], ctx)
    for fn in ("count", "collect_list", "collect_set"):
        ms, out = _timed_calls(ctx, lambda: rdf.group_by([keys], [(x, fn)]))
        rows_out.append({"case": f"group-by {fn} Float64 by Int32, 1e6 groups", "ms": ms, "rows": per * n_chunks, "card": card})
        print(f"group-by {fn:26s} Float64 1e6 groups {ms:9.3f} ms", flush=True)
        del out


def temporal_bench(ctx, rows, rows_out):
    """Date / timestamp functions over rows values in 25 chunks: Timestamp(us) spread over 1900..2100 with 10 % nulls, and Date32 (the
    to_date of it).  Each row: the median of three calls (after a warm-up) of the summed per-launch CUDA-event records, its GB/s at the
    algorithmic bytes (values in + values out + the bitmaps read and written) and the fraction of tune_stream's copy rate."""
    card = _card()
    copy = _stream_rates(rows)["copy"]
    print(f"card: {card}; tune_stream copy (1R1W) rate {copy:.1f} GB/s", flush=True)
    rows_out.append({"case": "tune_stream copy 1R1W", "GBs": copy, "card": card})
    n_chunks = 25
    per = rows // n_chunks
    lo, hi = -2208988800 * 10 ** 6, 4102444800 * 10 ** 6   # 1900-01-01 .. 2100-01-01 in microseconds
    rng = np.random.default_rng(20261016)
    chunks = []
    for _ in range(n_chunks):
        v = rng.integers(lo, hi, per)
        chunks.append(rdf.PrimitiveArray.from_numpy(v, rng.random(per) >= 0.1))
    T = rdf.TemporalType
    ts = rdf.Column.upload(chunks, ctx).with_temporal(T.timestamp("us"))
    del chunks
    d32 = ts.to_date()
    # distinct second operands for the two-column rows (a column paired with itself would read its second side from cache)
    ts2 = ts.date_trunc("hour")   # Timestamp(us)
    d32b = ts2.add_months(1)      # Date32
    assert ts2.dtype == rdf.I64 and ts2.temporal == T.timestamp("us") and d32b.dtype == rdf.I32 and d32b.temporal == T.date32()
    N_ = len(ts)
    bm = N_ / 8
    cases = [("year Timestamp(us) -> Int32", lambda: ts.year(), N_ * (8 + 4) + 2 * bm),
             ("day_of_week Timestamp(us) -> Int32", lambda: ts.day_of_week(), N_ * (8 + 4) + 2 * bm),
             ("hour Timestamp(us) -> Int32", lambda: ts.hour(), N_ * (8 + 4) + 2 * bm),
             ("date_trunc(day) Timestamp(us)", lambda: ts.date_trunc("day"), N_ * (8 + 8) + 2 * bm),
             ("to_date Timestamp(us) -> Date32", lambda: ts.to_date(), N_ * (8 + 4) + 2 * bm),
             ("add_months(1) Timestamp(us) -> Date32", lambda: ts.add_months(1), N_ * (8 + 4) + 2 * bm),
             ("year Date32 -> Int32", lambda: d32.year(), N_ * (4 + 4) + 2 * bm),
             ("day_of_week Date32 -> Int32", lambda: d32.day_of_week(), N_ * (4 + 4) + 2 * bm),
             ("add_months(1) Date32", lambda: d32.add_months(1), N_ * (4 + 4) + 2 * bm),
             ("months_between(Timestamp(us), Timestamp(us))", lambda: ts.months_between(ts2), N_ * (8 + 8 + 8) + 3 * bm),
             ("months_between(Date32, Date32)", lambda: d32.months_between(d32b), N_ * (4 + 4 + 8) + 3 * bm)]
    for name, fn, b in cases:
        ms, out = _timed_calls(ctx, fn)
        gbs = b / ms / 1e6
        rows_out.append({"case": name, "ms": ms, "rows": N_, "bytes": b, "GBs": gbs, "frac_of_copy": gbs / copy, "card": card})
        print(f"{name:48s} {ms:9.3f} ms {gbs:8.1f} GB/s  {gbs / copy:5.3f} of copy rate", flush=True)
        del out


def nulls_bench(ctx, rows, rows_out):
    """Null handling and conditional selection over rows values in 25 chunks, Float64 and Int32, 10 % nulls.  Each row: the median of
    three calls (after a warm-up) of the summed per-launch CUDA-event records, its GB/s at the bytes a two-argument selection
    moves (two value columns read, one written, and their bitmaps), and its time over the time of bdf_binary_dev ADD of the same two
    columns -- the yardstick: the same rows and the same bytes."""
    card = _card()
    print(f"card: {card}", flush=True)
    n_chunks = 25
    per = rows // n_chunks
    rng = np.random.default_rng(20261017)

    def column(npdt, null_frac, nan_frac=0.0):
        chunks = []
        for _ in range(n_chunks):
            v = rng.uniform(-1e3, 1e3, per).astype(npdt) if np.dtype(npdt).kind == "f" else rng.integers(-10 ** 6, 10 ** 6, per).astype(npdt)
            if nan_frac:
                v[rng.random(per) < nan_frac] = np.nan
            chunks.append(rdf.PrimitiveArray.from_numpy(v, rng.random(per) >= null_frac) if null_frac else rdf.PrimitiveArray.from_numpy(v, np.ones(per, bool)))
        return rdf.Column.upload(chunks, ctx)

    def bools(p_true):
        return rdf.Column.upload([rdf.BooleanArray.from_numpy(rng.random(per) < p_true, rng.random(per) >= 0.1) for _ in range(n_chunks)], ctx,
                                 dtype=rdf.native.BOOL)

    for name, npdt in (("Float64", np.float64), ("Int32", np.int32)):
        w = np.dtype(npdt).itemsize
        a, b, a0 = column(npdt, 0.1, 0.05 if w == 8 else 0.0), column(npdt, 0.1), column(npdt, 0.0)
        c, d = column(npdt, 0.1), column(npdt, 0.1)
        conds = [bools(0.25) for _ in range(4)]
        n = len(a)
        two = n * 3 * w + 3 * n / 8
        cases = [("ADD (yardstick)", lambda: a.add(b), two),
                 ("coalesce(a, b), 10 % nulls in a", lambda: rdf.coalesce(a, b), two),
                 ("coalesce(a, b), 0 % nulls in a", lambda: rdf.coalesce(a0, b), two),
                 ("coalesce(a, 0)", lambda: rdf.coalesce(a, 0), n * 2 * w + 2 * n / 8),
                 ("case_when 1 branch", lambda: rdf.when(conds[0], a).otherwise(b), two + 2 * n / 8),
                 ("case_when 4 branches", lambda: rdf.when(conds[0], a).when(conds[1], b).when(conds[2], c).when(conds[3], d).otherwise(a0),
                  two + 8 * n / 8 + 3 * n / 8),
                 ("greatest of 2", lambda: rdf.greatest(a, b), two),
                 ("greatest of 4", lambda: rdf.greatest(a, b, c, d), n * 5 * w + 5 * n / 8)]
        if w == 8:
            cases.append(("nanvl(a, b)", lambda: a.nanvl(b), two))
        # is_nan of an integer column reads no values (it is all false): only the result bitmap is written
        cases += [("is_null(a)", lambda: a.is_null(), 2 * n / 8),
                  ("is_nan(a)", lambda: a.is_nan(), n * w + 2 * n / 8 if w == 8 else n / 8)]
        base = None
        for case, fn, b_ in cases:
            ms, out = _timed_calls(ctx, fn)
            base = base or ms
            gbs = b_ / ms / 1e6
            rows_out.append({"case": f"{name} {case}", "ms": ms, "rows": n, "bytes": b_, "GBs": gbs, "vs_add": ms / base, "card": card})
            print(f"{name} {case:36s} {ms:9.3f} ms {gbs:8.1f} GB/s  {ms / base:5.2f} x ADD", flush=True)
            del out
        frame = rdf.DeviceFrame(OrderedDict([("a", a), ("b", b), ("c", c), ("d", d)]))
        ms, out = _timed_calls(ctx, lambda: frame.drop_nulls())
        rows_out.append({"case": f"{name} drop_nulls over 4 columns", "ms": ms, "rows": n, "card": card})
        print(f"{name} {'drop_nulls over 4 columns':36s} {ms:9.3f} ms", flush=True)
        del out, frame
        for col in (a, b, a0, c, d, *conds):
            col.free()
    # the headline step in the same call, to show it unchanged
    import subprocess

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--gpus", "1", "--steps", "50", "--warmup", "10"],
                       capture_output=True, text=True, check=True)
    head = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("{")][-1])
    rows_out.append({"case": "bench.py --gpus 1 (headline add+sum)", "ms": head["ms_per_step"], "rows_per_s": head["value"], "card": card})
    print(f"bench.py --gpus 1: {head['ms_per_step']:.3f} ms per step, {head['value']:.4g} rows/s", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--json", default=None)
    ap.add_argument("--csv-rows", type=int, default=50_000_000)
    ap.add_argument("--csv", action="store_true", help="run the CSV reader rows instead of the kernel table")
    ap.add_argument("--window", action="store_true", help="run only the window-function rows")
    ap.add_argument("--math", action="store_true", help="run only the float-function rows (unary, atan2/hypot/log, fused)")
    ap.add_argument("--stats", action="store_true", help="run only the statistical-aggregate rows (moments, group variance, count_distinct)")
    ap.add_argument("--csv-write", action="store_true", help="run only the CSV writer rows")
    ap.add_argument("--json-write", action="store_true", help="run only the JSON writer rows (--csv-rows rows)")
    ap.add_argument("--lists", action="store_true", help="run only the list-function rows (ArrayFunctions)")
    ap.add_argument("--temporal", action="store_true", help="run only the date / timestamp function rows")
    ap.add_argument("--ndjson", action="store_true", help="run the line-delimited JSON reader rows (--csv-rows records)")
    ap.add_argument("--parquet", action="store_true", help="run the Parquet reader rows (--csv-rows rows, snappy and uncompressed)")
    ap.add_argument("--parquet-write", action="store_true", help="run the Parquet writer rows (--csv-rows rows, three encodings)")
    ap.add_argument("--distribution", action="store_true", help="run only the distribution rows (median, hist, uniques, mode)")
    ap.add_argument("--nulls", action="store_true", help="run only the null-handling and conditional rows (coalesce, case_when, ...)")
    args = ap.parse_args()
    ctx = rdf.default_context()
    if args.nulls:
        rows_out = []
        nulls_bench(ctx, args.rows, rows_out)
        if args.json:
            with open(args.json, "w") as f:
                json.dump({"results": rows_out}, f, indent=1)
        return
    if args.parquet_write:
        import subprocess

        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
        print(f"card: {q.strip()}", flush=True)
        rows_out = []
        parquet_write_bench(ctx, args.csv_rows, rows_out)
        if args.json:
            with open(args.json, "w") as f:
                json.dump({"card": q.strip(), "results": rows_out}, f, indent=1)
        return
    if args.parquet:
        import subprocess

        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
        print(f"card: {q.strip()}", flush=True)
        rows_out = []
        parquet_bench(ctx, args.csv_rows, rows_out)
        if args.json:
            with open(args.json, "w") as f:
                json.dump({"card": q.strip(), "results": rows_out}, f, indent=1)
        return
    if args.ndjson:
        import subprocess

        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
        print(f"card: {q.strip()}", flush=True)
        rows_out = []
        ndjson_bench(ctx, args.csv_rows, rows_out)
        if args.json:
            with open(args.json, "w") as f:
                json.dump({"card": q.strip(), "results": rows_out}, f, indent=1)
        return
    if args.temporal:
        rows_out = []
        temporal_bench(ctx, args.rows, rows_out)
        if args.json:
            with open(args.json, "w") as f:
                json.dump({"results": rows_out}, f, indent=1)
        return
    if args.lists:
        rows_out = []
        lists_bench(ctx, args.rows, rows_out)
        if args.json:
            with open(args.json, "w") as f:
                json.dump({"results": rows_out}, f, indent=1)
        return
    if args.json_write:
        rows_out = []
        json_write_bench(ctx, args.csv_rows, rows_out)
        if args.json:
            with open(args.json, "w") as f:
                json.dump({"card": _card(), "results": rows_out}, f, indent=1)
        return
    if args.csv_write:
        rows_out = []
        csv_write_bench(ctx, args.csv_rows, rows_out)
        if args.json:
            with open(args.json, "w") as f:
                json.dump({"results": rows_out}, f, indent=1)
        return
    if args.window:
        rows_out = []
        window_bench(ctx, args.rows, [4_000_000] * (args.rows // 4_000_000), rows_out)
        if args.json:
            with open(args.json, "w") as f:
                json.dump({"results": rows_out}, f, indent=1)
        return
    if args.csv:
        rows_out = []
        csv_bench(ctx, args.csv_rows, rows_out)
        if args.json:
            with open(args.json, "w") as f:
                json.dump({"results": rows_out}, f, indent=1)
        return
    chunk = 4_000_000
    lens = [chunk] * (args.rows // chunk)
    G = rdf.Column.generate
    pk, pk_src = configs_bench._peak()
    rows_out = []

    def report(name, config, res, kind):
        ms, nbytes, rows = res[kind]
        gbs = nbytes / ms / 1e6
        rows_out.append({"case": name, "config": config, "kernel": kind, "ms": ms, "rows": rows, "bytes_per_row": nbytes / rows,
                         "GBs": gbs, "frac_of_peak": gbs / pk, "rows_per_s": rows / ms * 1e3})
        print(f"{name:44s} {ms:8.4f} ms  {nbytes / rows:7.3f} B/row  {gbs:8.1f} GB/s  {gbs / pk:5.3f} of peak  {rows / ms * 1e3:10.3e} rows/s", flush=True)

    if args.distribution:
        distribution_bench(ctx, lens, rows_out)
        if args.json:
            with open(args.json, "w") as f:
                json.dump({"results": rows_out}, f, indent=1)
        return
    if args.math or args.stats:
        (math_bench(ctx, lens, report) if args.math else stats_bench(ctx, lens, report, rows_out))
        if args.json:
            with open(args.json, "w") as f:
                json.dump({"results": rows_out}, f, indent=1)
        return

    # ---- config 1/metric: f64 add, sum ----
    a = G(rdf.F64, lens, 0, -1e3, 1e3, col_id=0)
    b = G(rdf.F64, lens, 0, -1e3, 1e3, col_id=1)
    c3 = G(rdf.F64, lens, 0, -1e3, 1e3, col_id=2)
    d = G(rdf.F64, lens, 1, col_id=3)
    report("add f64 (no nulls)", "metric", timed(ctx, lambda: a.add(b)), "binary")
    report("add f64 + fused sum (K5)", "metric", timed(ctx, lambda: a.binary_agg(N.ADD, b)[0]), "binary")
    report("sum f64 (no nulls)", "metric", timed(ctx, lambda: a.sum()), "reduce")
    # ---- config 2: chain add, mul, div, sin ----
    report("multiply f64", "cfg2", timed(ctx, lambda: a.multiply(c3)), "binary")
    report("divide f64 (zero check fused)", "cfg2", timed(ctx, lambda: a.divide(d)), "binary")
    g = a.divide(d)
    report("sin f64, |x| <~ 1e3", "cfg2", timed(ctx, lambda: g.sin()), "unary")
    report("cos f64", "cfg2", timed(ctx, lambda: g.cos()), "unary")
    report("tan f64", "cfg2", timed(ctx, lambda: g.tan()), "unary")
    report("abs f64", "cfg2", timed(ctx, lambda: g.abs()), "unary")
    g.free()
    # config 2, second run (SURVEY 8(d)): |g| up to 1e12 -- beyond the fast path of the trig argument reduction
    big = G(rdf.F64, lens, 0, -1e12, 1e12, col_id=14)
    report("sin f64, |x| up to 1e12 (slow-path reduction)", "cfg2-slow", timed(ctx, lambda: big.sin()), "unary")
    report("cos f64, |x| up to 1e12", "cfg2-slow", timed(ctx, lambda: big.cos()), "unary")
    report("tan f64, |x| up to 1e12", "cfg2-slow", timed(ctx, lambda: big.tan()), "unary")
    big.free()
    bn = G(rdf.F64, lens, 0, -1e3, 1e3, col_id=4, null_mod=10)
    dn = G(rdf.F64, lens, 1, col_id=5, null_mod=10)
    report("add f64, 10% nulls on one input", "cfg2-nulls", timed(ctx, lambda: a.add(bn)), "binary")
    report("add f64, 10% nulls on both inputs", "cfg2-nulls", timed(ctx, lambda: bn.add(dn)), "binary")
    report("divide f64, 10% nulls on divisor only", "cfg2-nulls", timed(ctx, lambda: a.divide(dn)), "binary")
    report("divide f64, 10% nulls on both", "cfg2-nulls", timed(ctx, lambda: bn.divide(dn)), "binary")
    report("sin f64, 10% nulls", "cfg2-nulls", timed(ctx, lambda: bn.sin()), "unary")
    # ---- N3: the whole config-2 chain in one pass (40 B/row) vs the four materialising launches (88 B/row) ----
    prog = [(N.ADD, 0, 1), (N.MUL, 4, 2), (N.DIV, 5, 3), ("sin", 6)]
    report("N3 fused sin(((a+b)*c)/d)", "cfg2-fused", timed(ctx, lambda: rdf.eval_expr([a, b, c3, d], prog)), "expr")
    report("N3 fused ((a+b)*c)/d (arithmetic only)", "cfg2-fused", timed(ctx, lambda: rdf.eval_expr([a, b, c3, d], prog[:3])), "expr")
    report("N3 fused chain + sum/count of h (one pass)", "cfg2-fused", timed(ctx, lambda: rdf.eval_expr_agg([a, b, c3, d], prog)[0]), "expr")
    report("N3 sum(sin(((a+b)*c)/d)), h never written", "cfg2-fused", timed(ctx, lambda: rdf.eval_expr_agg([a, b, c3, d], prog, materialise=False)[1] and None), "expr")
    report("N3 fused chain, 10% nulls on b and d", "cfg2-fused", timed(ctx, lambda: rdf.eval_expr([a, bn, c3, dn], prog)), "expr")

    def unfused():
        e = a.add(b); f = e.multiply(c3); e.free(); g2 = f.divide(d); f.free(); h = g2.sin(); g2.free()
        return h
    res = timed(ctx, unfused)
    total = sum(v[0] for v in res.values())
    print(f"{'N3 reference: same chain, 4 launches':44s} {total:8.4f} ms  (sum of {sorted(res)})", flush=True)
    rows_out.append({"case": "cfg2 chain unfused (4 launches)", "config": "cfg2-fused", "kernel": "binary x3 + unary", "ms": total, "rows": args.rows})
    for col in (c3, d, bn, dn):
        col.free()
    # f32 trig
    f32 = G(rdf.F32, lens, 0, -1e3, 1e3, col_id=6)
    report("sin f32", "extra", timed(ctx, lambda: f32.sin()), "unary")
    f32b = G(rdf.F32, lens, 0, -1e3, 1e3, col_id=16)   # two DISTINCT inputs: a column added to itself moves 2w, not 3w, bytes per row
    report("add f32", "extra", timed(ctx, lambda: f32.add(f32b)), "binary")
    f32.free(); f32b.free()
    # ---- config 3: int64 aggregates with 10% nulls ----
    i64n = G(rdf.I64, lens, 3, col_id=7, null_mod=10)
    i64 = G(rdf.I64, lens, 3, col_id=8)
    report("sum/min/max/count i64, 10% nulls (4-in-1)", "cfg3", timed(ctx, lambda: i64n.aggregate_all()), "reduce")
    report("sum/min/max/count i64, no nulls", "cfg3", timed(ctx, lambda: i64.aggregate_all()), "reduce")
    report("add i64, 10% nulls", "cfg5", timed(ctx, lambda: i64n.add(i64)), "binary")
    report("add i64 + fused 4-in-1 aggregate", "cfg5", timed(ctx, lambda: i64n.binary_agg(N.ADD, i64)[0]), "binary")
    # ---- config 4: cast chain ----
    i32n = G(rdf.I32, lens, 2, col_id=9, null_mod=10)
    report("cast i32 -> f64, 10% nulls", "cfg4", timed(ctx, lambda: i32n.cast(rdf.F64)), "cast")
    report("cast i64 -> f64", "cfg5", timed(ctx, lambda: i64.cast(rdf.F64)), "cast")
    report("cast f64 -> i32 (fallible)", "cfg4", timed(ctx, lambda: a.cast(rdf.I32)), "cast")
    report("cast f64 -> f32", "extra", timed(ctx, lambda: a.cast(rdf.F32)), "cast")
    report("cast i64 -> i8 (fallible, narrow out)", "extra", timed(ctx, lambda: i64.cast(rdf.I8)), "cast")
    i8 = i64.cast(rdf.I8)
    i8b = i64n.cast(rdf.I8)
    report("add i8", "extra", timed(ctx, lambda: i8.add(i8b)), "binary")
    report("sum/min/max/count i8", "extra", timed(ctx, lambda: i8.aggregate_all()), "reduce")
    i8v = G(rdf.I8, lens, 2, col_id=17, null_mod=10)
    i16v = G(rdf.I16, lens, 2, col_id=18, null_mod=10)
    u16 = G(rdf.U16, lens, 2, col_id=19)
    report("sum/min/max/count i8 full range, 10% nulls", "extra", timed(ctx, lambda: i8v.aggregate_all()), "reduce")
    report("sum/min/max/count i16 full range, 10% nulls", "extra", timed(ctx, lambda: i16v.aggregate_all()), "reduce")
    report("sum/min/max/count u16, no nulls", "extra", timed(ctx, lambda: u16.aggregate_all()), "reduce")
    # the same kernels over as many BYTES as the f64 rows move (1e8 i8 rows are 0.11 GB: tens of us, launch-sized)
    big_lens = [32_000_000] * max(1, args.rows * 8 // 32_000_000)
    i8big = G(rdf.I8, big_lens, 2, col_id=27, null_mod=10)
    report("sum/min/max/count i8 10% nulls, 8x the rows", "extra", timed(ctx, lambda: i8big.aggregate_all()), "reduce")
    i8big.free()
    i16big = G(rdf.I16, big_lens[: len(big_lens) // 2], 2, col_id=28, null_mod=10)
    report("sum/min/max/count i16 10% nulls, 4x the rows", "extra", timed(ctx, lambda: i16big.aggregate_all()), "reduce")
    i16big.free()
    report("sum/min/max/count i32 full range, 10% nulls", "extra", timed(ctx, lambda: i32n.aggregate_all()), "reduce")
    for col in (i8b, i8v, i16v, u16):
        col.free()
    # ---- N2 (next row): BooleanFilter compare + ChunkedArray::filter ----
    report("compare f64 > scalar", "N2", timed(ctx, lambda: a.gt(0.0)), "compare")
    report("compare f64 > f64", "N2", timed(ctx, lambda: a.gt(b)), "compare")
    report("compare i32 (10% nulls) > scalar, cast fused", "N2", timed(ctx, lambda: i32n.gt(0.0)), "compare")
    report("compare i64 > f64 column, cast fused", "N2", timed(ctx, lambda: i64.gt(a)), "compare")
    m_half = a.gt(0.0)
    m_rare = a.gt(980.0)
    an = G(rdf.F64, lens, 0, -1e3, 1e3, col_id=11, null_mod=10)
    for name, fn in (("filter f64, 50% kept", lambda: a.filter(m_half)), ("filter f64, 1% kept", lambda: a.filter(m_rare)),
                     ("filter f64 10% nulls, 50% kept", lambda: an.filter(m_half)), ("filter i32 10% nulls, 50% kept", lambda: i32n.filter(m_half))):
        res = timed(ctx, fn)
        keys = sorted(k for k in res if k.startswith("filter"))
        report(name + ": count+scan", "N2", res, keys[0])
        report(name + ": scatter", "N2", res, keys[1])
    # ---- DataFrame::sort: lexsort_to_indices (stable LSD radix, 32 B/row per executed pass) + take ----
    report("sort indices f64 (8 passes)", "sort", timed(ctx, lambda: rdf.sort_indices([(a, False)]), reps=4), "sort")
    report("sort indices i64 10% nulls, |x| < 2^40 (6+1 passes)", "sort", timed(ctx, lambda: rdf.sort_indices([(i64n, True)]), reps=4), "sort")
    report("sort indices i32 10% nulls (4+1 passes)", "sort", timed(ctx, lambda: rdf.sort_indices([(i32n, False)]), reps=4), "sort")
    report("sort indices i8 then f64 (two criteria)", "sort", timed(ctx, lambda: rdf.sort_indices([(i8, False), (a, True)]), reps=4), "sort")
    sidx = rdf.sort_indices([(a, False)])
    report("take f64 by the sort indices (random gather)", "sort", timed(ctx, lambda: b.take(sidx), reps=4), "take")
    report("take i32 10% nulls by the sort indices", "sort", timed(ctx, lambda: i32n.take(sidx), reps=4), "take")
    # ---- group-by aggregate: sort the key, gather key and value, head bitmap, two compactions, one warp per group ----
    def group_total(key, val, what):
        res = timed(ctx, lambda: _free_group(rdf.group_aggregate(key, [val])), reps=3)
        total = sum(v[0] for v in res.values())
        print(f"{what:44s} {total:8.4f} ms  (" + ", ".join(f"{k} {v[0]:.3f}" for k, v in sorted(res.items())) + ")", flush=True)
        rows_out.append({"case": what, "config": "group", "kernel": "sort + take + filter + group", "ms": total, "rows": args.rows, "parts": {k: v[0] for k, v in res.items()}})

    def _free_group(r):
        keys, res = r
        keys.free()
        for d in res:
            for c in d.values():
                if c is not None:
                    c.free()
        return None

    kf = G(rdf.F64, lens, 0, -100.0, 100.0, col_id=22)
    small = kf.cast(rdf.I8)                                        # 200 distinct keys: every group is a hot key (k_group_big)
    kf.free()
    group_total(small, a, "group-by i8 key (200 groups), sum f64")
    group_total(i32n, i64n, "group-by i32 key (~1e8 groups), i64 4-in-1")

    def group_by_total(keys, aggs, what):   # bdf_group_by_dev: several keys, a flat list of (column, function)
        res = timed(ctx, lambda: [c.free() for part in rdf.group_by(keys, aggs) for c in part] and None, reps=3)
        total = sum(v[0] for v in res.values())
        print(f"{what:44s} {total:8.4f} ms  (" + ", ".join(f"{k} {v[0]:.3f}" for k, v in sorted(res.items())) + ")", flush=True)
        rows_out.append({"case": what, "config": "group", "kernel": "sort + take + filter + group", "ms": total, "rows": args.rows, "parts": {k: v[0] for k, v in res.items()}})

    group_by_total([i32n, small], [(a, f) for f in ("sum", "avg", "min", "max")], "group-by i32 (nulls) x i8 keys, sum/avg/min/max f64")
    i32 = i64n.cast(rdf.I32)
    group_by_total([small], [(i32, "count_distinct")], "group-by i8 key, count_distinct i32")
    group_by_total([small], [(a, "first"), (a, "last")], "group-by i8 key, first/last f64")
    i32.free()
    small.free()

    # ---- equi-join: build-side sort, gathers of its keys, heads + compactions, count (binary search), scan, emit, the takes ----
    def join_total(lk, rk, how, what, payload=None):
        def once():
            li, ri = rdf.join_indices(lk, rk, how)
            out = [li, ri]
            if payload is not None:   # DataFrame::join then takes the columns of both sides
                out += [payload[0].take(li), payload[1].take(ri)]
            return out
        res = timed(ctx, once, reps=3)
        total = sum(v[0] for v in res.values())
        print(f"{what:44s} {total:8.4f} ms  (" + ", ".join(f"{k} {v[0]:.3f}" for k, v in sorted(res.items())) + ")", flush=True)
        rows_out.append({"case": what, "config": "join", "kernel": "sort + take + filter + join", "ms": total, "rows": args.rows,
                         "parts": {k: v[0] for k, v in res.items()}})

    def keys(dtype, n_rows, hi, col_id):   # integer keys uniform in [0, hi)
        n_lens = [chunk] * (n_rows // chunk) if n_rows >= chunk else [n_rows]
        f = G(rdf.F64, n_lens, 0, 0.0, float(hi), col_id=col_id)
        k = f.cast(dtype)
        f.free()
        return k

    P = rdf.PrimitiveArray
    dim = rdf.Column.upload([P.from_numpy(np.random.default_rng(1).permutation(1_000_000).astype(np.int32))])   # unique keys
    dim_val = G(rdf.F64, [1_000_000], 0, -1.0, 1.0, col_id=40)
    fact = keys(rdf.I32, args.rows, 1_000_000, 41)
    join_total([fact], [dim], "left", f"left join {args.rows:.0e} x 1e6 unique i32 keys + takes", (a, dim_val))
    fact.free()
    l64, r64 = keys(rdf.I64, 10_000_000, 1_000_000, 42), keys(rdf.I64, 10_000_000, 1_000_000, 43)
    join_total([l64], [r64], "inner", "inner join 1e7 x 1e7 i64, ~10 matches per row")
    l64.free(); r64.free()
    la, lb = keys(rdf.I32, 10_000_000, 1000, 44), keys(rdf.I8, 10_000_000, 100, 45)
    ra, rb = keys(rdf.I32, 1_000_000, 1000, 46), keys(rdf.I8, 1_000_000, 100, 47)
    join_total([la, lb], [ra, rb], "inner", "inner join 1e7 x 1e6 on (i32, i8), ~10 matches")
    for col in (la, lb, ra, rb, dim, dim_val):
        col.free()
    hot_l = rdf.Column.upload([P.from_numpy(np.zeros(100_000, np.int64))])
    hot_r = rdf.Column.upload([P.from_numpy(np.zeros(1_000, np.int64))])
    join_total([hot_l], [hot_r], "inner", "hot key: 1e5 x 1e3 rows of one key (1e8 out)")
    hot_l.free(); hot_r.free()
    # ---- window functions: sort, key gathers, heads, runs, ranks, the value gather, shift / scan, the gathers back to row order ----
    window_bench(ctx, args.rows, lens, rows_out)
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"rows": args.rows, "peak_GBs": pk, "peak_source": pk_src, "results": rows_out}, f, indent=1)


if __name__ == "__main__":
    main()
