"""Small ragged shapes through every kernel once (for compute-sanitizer memcheck / racecheck / initcheck)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import rust_dataframe_b200 as rdf
from rust_dataframe_b200 import native as N

rng = np.random.default_rng(1)
lens = [0, 1, 33, 2047, 2049, 5000]
P = rdf.PrimitiveArray
for dtype in (rdf.I8, rdf.I16, rdf.I32, rdf.I64, rdf.U8, rdf.U16, rdf.U32, rdf.U64, rdf.F32, rdf.F64):
    npdt = rdf.NP_DTYPES[dtype]
    def col(nulls, nz=False):
        out = []
        for k, n in enumerate(lens):
            v = (rng.uniform(1, 100, n + 9) if npdt.kind == "f" else rng.integers(1, 100, n + 9)).astype(npdt)
            a = P.from_numpy(v, rng.random(n + 9) > 0.2) if nulls else P.from_numpy(v)
            a.null_count = -1 if nulls else 0
            out.append(a.slice(3 + k, n))
        return out
    a, b = col(True), col(False)
    for fn in (rdf.ScalarFunctions.add, rdf.ScalarFunctions.multiply, rdf.ScalarFunctions.divide):
        fn(a, b)
    rdf.AggregateFunctions.all([c for c in a if c.length])
    rdf.AggregateFunctions.count(a)
    for to in (rdf.I8, rdf.U32, rdf.F64, rdf.I64):
        rdf.cast(a, to)
    if dtype in (rdf.F32, rdf.F64):
        rdf.ScalarFunctions.sin(a); rdf.ScalarFunctions.tan(b); rdf.ScalarFunctions.atan2(a[3], b[3])
    ca, cb = rdf.Column.upload_many([a, b], asynchronous=True)
    cc, fut = ca.binary_agg_async(N.ADD, cb)
    fut.result(); cc.download(); ca.download()
    g = rdf.Column.generate(dtype, lens, kind=2 if npdt.kind != "f" else 0, null_mod=3)
    g.download(); g.aggregate_all()
    if dtype == rdf.F64:   # N3: fused expression with both temporaries, a shared node, a divide and a libm node
        prog = [(N.ADD, 0, 1), (N.SUB, 0, 1), (N.MUL, 2, 3), (N.MUL, 2, 2), (N.ADD, 4, 5), (N.DIV, 6, 1), ("sin", 7)]
        rdf.eval_expr([ca, cb], prog).download()
    if dtype in (rdf.F64, rdf.I16):   # DataFrame::sort: two criteria (nullable + dense), take of a numeric and a boolean column
        idx = rdf.sort_indices([(ca, True), (cb, False)])
        ca.take(idx).download(); cb.gt(50.0).take(idx).download()
    if dtype not in (rdf.I64, rdf.U64):
        rdf.AggregateFunctions.avg([c for c in a if c.length])
    # round 2: comparisons against a scalar (integer columns take k_compare_int) and a column, filter, batched multi-column reduce
    m = ca.gt(50.0); m2 = ca.le(cb)
    ca.filter(m).download(); cb.filter(m2).download()
    rdf.Column.aggregate_all_many([ca, cb, g])
    # group-by: short groups (one lane per group), medium (8 lanes), long (a warp) and one hot key (> 64 Ki rows: k_group_big)
    for n_rows, card in ((3000, 2500), (6000, 300), (9000, 7)):
        k = rdf.Column.upload([P.from_numpy(rng.integers(0, card, n_rows).astype(np.int32), rng.random(n_rows) > 0.1)])
        v = rdf.Column.upload([P.from_numpy((rng.uniform(1, 100, n_rows) if npdt.kind == "f" else rng.integers(1, 100, n_rows)).astype(npdt), rng.random(n_rows) > 0.2)])
        keys, res = rdf.group_aggregate(k, [v])
        keys.download(); res[0]["sum"].download(); res[0]["count"].download()
        if res[0]["min"] is not None:
            res[0]["min"].download(); res[0]["max"].download()
    if dtype in (rdf.I64, rdf.F64, rdf.U8):
        n_rows = 150_000
        kk = rng.integers(0, 50_000, n_rows).astype(np.int64); kk[rng.random(n_rows) < 0.6] = 7
        k = rdf.Column.upload([P.from_numpy(kk)])
        v = rdf.Column.upload([P.from_numpy((rng.uniform(1, 100, n_rows) if npdt.kind == "f" else rng.integers(1, 100, n_rows)).astype(npdt), rng.random(n_rows) > 0.2)])
        keys, res = rdf.group_aggregate(k, [v])
        keys.download(); res[0]["sum"].download()
    # group-by over two keys: multi-key heads, every fold accumulator (one hot key: k_group_big), first / last, count_distinct
    n_rows = 150_000 if dtype in (rdf.I32, rdf.F64) else 5000
    k1 = rdf.Column.upload([P.from_numpy(rng.integers(0, 3000, n_rows).astype(np.int16), rng.random(n_rows) > 0.1)])
    k2 = rdf.Column.upload([P.from_numpy(np.where(rng.random(n_rows) < 0.6, 0.0, rng.uniform(-1, 1, n_rows)))])
    v = rdf.Column.upload([P.from_numpy((rng.uniform(1, 100, n_rows) if npdt.kind == "f" else rng.integers(1, 100, n_rows)).astype(npdt), rng.random(n_rows) > 0.2)])
    fns = [f for f in rdf.native.GROUP_FNS if not (f == "avg" and dtype in (rdf.I64, rdf.U64))]
    keys, res = rdf.group_by([k2, k1], [(v, f) for f in fns])
    for c in keys + res:
        c.download()
    # equi-join: every join type (count, scan, emit; full: the unmatched rows), two criteria over ragged, sliced chunks
    jl, jr = col(True), col(False)[2:]
    lk2 = rdf.Column.upload([P.from_numpy(rng.integers(0, 3, sum(c.length for c in jl)).astype(np.int16))])
    rk2 = rdf.Column.upload([P.from_numpy(rng.integers(0, 3, sum(c.length for c in jr)).astype(np.int16), rng.random(sum(c.length for c in jr)) > 0.1)])
    for how in rdf.native.JOIN_TYPES:
        li, ri = rdf.join_indices([rdf.Column.upload(jl), lk2], [rdf.Column.upload(jr), rk2], how)
        li.download(); ri.download()
    # window functions over the ragged, sliced chunks: heads, runs, ranks, shifts and the three-kernel scan, with and without keys
    wx = rdf.Column.upload(jl)
    wk = rdf.Column.upload([P.from_numpy(rng.integers(0, 4, len(wx)).astype(np.int8), rng.random(len(wx)) > 0.1)])
    wo = rdf.Column.upload([P.from_numpy(rng.integers(0, 9, len(wx)).astype(np.int32))])
    wcalls = [("row_number",), ("rank",), ("dense_rank",), ("percent_rank",), ("cume_dist",), ("lag", wx, 2), ("lead", wx, 1, 0)] + \
             [(f, wx, fr) for f in ("sum", "count", "min", "max") for fr in ("rows", "range", "partition")]
    for part, order in (([wk], [(wo, True)]), ([], []), ([wk], []), ([], [(wo, False)])):
        for c in rdf.window(part, order, wcalls):
            c.download()
# CSV reader: tokenizer scan, field index, record check, inference, parse of every type (exact fallback included), scatter
import tempfile
with tempfile.TemporaryDirectory() as td:
    path = os.path.join(td, "s.csv")
    with open(path, "w") as fh:
        fh.write("a,b,c,d,e\n")
        for r in range(20000):
            fh.write(f'{r},"x, ""{r}""",{"" if r % 7 == 0 else r * 0.25},{"true" if r % 2 else "False"},1.00000000000000011102230246251565404236316680908203125\n')
    with rdf.CsvFile(path, batch_size=1000) as f:
        for c in f.read().values():
            c.download()
    with rdf.CsvFile(path, batch_size=7, schema=[rdf.U16, -1, rdf.F32, 10, rdf.F32]) as f:
        for c in f.read().values():
            c.download()
    # CSV writer: measure, scan and emit over ragged sliced chunks with an empty one; one nullable column (""); rows too long for the
    # emit window (direct stores)
    def wcol(dtype, scale=1.0):
        out = []
        for k, n in enumerate(lens):
            v = (rng.uniform(-1, 1, n + 9) * scale).astype(rdf.NP_DTYPES[dtype])
            a = P.from_numpy(v, rng.random(n + 9) > 0.2)
            a.null_count = -1
            out.append(a.slice(3 + k, n))
        return rdf.Column.upload(out)
    bits = [rdf.BooleanArray.from_numpy(rng.random(n + 5) > 0.5).slice(5, n) for n in lens]
    for b in bits:
        b.null_count = 0
    rdf.write_csv(os.path.join(td, "w.csv"), {"d": wcol(rdf.F64), "f": wcol(rdf.F32), "i": wcol(rdf.I16, 3e4), "b": rdf.Column.upload(bits)},
                  delimiter="|")
    rdf.write_csv(os.path.join(td, "w1.csv"), {"d": wcol(rdf.F64)})
    rdf.write_csv(os.path.join(td, "w2.csv"), {f"t{j}": wcol(rdf.F64, 1e-300) for j in range(8)})
# list functions: ragged list chunks (null lists spanning elements, empty lists, null elements, a sliced list array and a sliced child),
# lists past the lane rounds of the search (the long-list work list and its grid-stride pass), every function once
for dtype in (rdf.I8, rdf.U16, rdf.I64, rdf.F32, rdf.F64):
    npdt = rdf.NP_DTYPES[dtype]
    def lchunk(n, long_every=0):
        lens = rng.integers(0, 9, n)
        if long_every:
            lens[::long_every] = 20000
        off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32) + 3
        m = int(off[-1]) + 5
        child = P.from_numpy(rng.integers(0, 6, m).astype(npdt), rng.random(m) > 0.2).slice(2, m - 2)
        child.null_count = -1
        valid = rng.random(n + 2) > 0.1
        return rdf.ListArray(dtype, np.concatenate([[0], off]).astype(np.int32), rdf.arrays.pack_validity(valid), 1, n, int((~valid[1:n + 1]).sum()), child)
    la = rdf.ListColumn.upload([lchunk(n) for n in (0, 1, 33, 2049)] + [lchunk(300, 7)])
    lb = rdf.ListColumn.upload([lchunk(n) for n in (0, 1, 33, 2049)] + [lchunk(300, 11)])
    for col in (la.array_contains(3), la.array_position(3), la.size()):
        col.download()
    for res in (la.array_remove(3), la.array_sort(), la.array_distinct(), la.array_repeat(2), la.array_except(lb), la.array_intersect(lb), la.array_union(lb)):
        res.download()
    for col in la.explode():
        col.download()
    nonempty = rdf.ListColumn.upload([rdf.ListArray.from_pylist(dtype, [[1, None], [None], None, [k % 100 for k in range(70000)]])])
    nonempty.array_max().download(); nonempty.array_min().download()
    # whole lists between rows: take with null and repeated indices (the hot 20000-element lists several times), filter per chunk
    n_l = len(la)
    idx = rng.integers(0, n_l, 3 * n_l).astype(np.uint32)
    idx[:40] = (np.arange(40) * 7) % n_l
    la.take(rdf.Column.upload([P.from_numpy(idx, rng.random(idx.shape[0]) > 0.1)])).download()
    lens_la = [la.chunk_info(k)["len"] for k in range(la.n_chunks)]
    la.filter(rdf.Column.upload([rdf.BooleanArray.from_numpy(rng.random(n) < 0.5, rng.random(n) > 0.1) for n in lens_la])).download()
# collect_list / collect_set over groups whose values are all null, a null key group, one-row groups
ck = rdf.Column.upload([P.from_numpy(rng.integers(0, 50, n).astype(np.int32), rng.random(n) > 0.05) for n in lens])
cx = rdf.Column.upload([P.from_numpy(rng.integers(0, 9, n).astype(np.float64), rng.random(n) > 0.5) for n in lens])
cn = rdf.Column.upload([P.from_numpy(np.zeros(n), np.zeros(n, dtype=bool)) for n in lens])
for r in rdf.group_by([ck], [(cx, "collect_list"), (cx, "collect_set"), (cn, "collect_list"), (cn, "collect_set")])[1]:
    r.download()
# the Parquet writer: ragged and offset chunks, nulls, every encoding path (PLAIN, dictionary, Boolean bits), snappy fragments, row
# groups cut across chunks, and a frame without rows
import tempfile
with tempfile.TemporaryDirectory() as td:
    pw = {"i8": rdf.Column.upload([P.from_numpy(rng.integers(-100, 100, n + 5).astype(np.int8), rng.random(n + 5) > 0.2).slice(3, n) for n in lens]),
          "f64": rdf.Column.upload([P.from_numpy(rng.integers(0, 40, n + 5) / 4.0, rng.random(n + 5) > 0.1).slice(1, n) for n in lens]),
          "u64": rdf.Column.upload([P.from_numpy(rng.integers(0, 2 ** 63, n, dtype=np.uint64)) for n in lens]),
          "ok": rdf.Column.upload([rdf.BooleanArray.from_numpy(rng.random(n) < 0.5, rng.random(n) > 0.3) for n in lens], dtype=10)}
    for kw in ({}, {"compression": "snappy"}, {"dictionary": False}, {"row_group_rows": 700, "compression": "snappy"}):
        rdf.write_parquet(os.path.join(td, "w.parquet"), pw, **kw)
    rdf.write_parquet(os.path.join(td, "e.parquet"), {"x": rdf.Column.upload([P.from_numpy(np.zeros(0, dtype=np.int32))])})
# the distributions: select levels from the column and from compacted scratch (many prefixes), the all-equal column, the histogram on
# both bin paths over ragged, offset chunks with nulls, uniques with counts and mode
for npdt in (np.int8, np.int64, np.float32, np.float64):
    dc = rdf.Column.upload([P.from_numpy(rng.integers(-1000, 1000, n + 3).astype(npdt), rng.random(n + 3) > 0.2).slice(3, n) for n in lens])
    dc.percentile(list(np.linspace(0, 1, 300))); dc.median(); dc.mode(); dc.hist(10); dc.hist(5000, range=(-10.0, 10.0))
    vals, cnts = dc.value_counts()
    vals.download(); cnts.download()
rdf.Column.upload([P.from_numpy(np.full(70000, 2.5))]).median()
# null handling and conditional selection: every kernel of k_cond.cu over ragged, offset chunks with nulls, scalars and NULL literals
for npdt in (np.int8, np.uint16, np.int32, np.float32, np.float64, np.uint64):
    nc = [rdf.Column.upload([P.from_numpy(rng.integers(-9, 9, n + 5).astype(npdt), rng.random(n + 5) > 0.3).slice(2 + j, n) for n in lens])
          for j in range(3)]
    conds = [rdf.Column.upload([rdf.BooleanArray.from_numpy(rng.random(n + 5) < 0.5, rng.random(n + 5) > 0.2).slice(1 + j, n) for n in lens], dtype=10)
             for j in range(2)]
    rdf.coalesce(nc[0], nc[1], 1).download(); rdf.greatest(*nc).download(); rdf.least(nc[0], None, nc[2]).download()
    rdf.when(conds[0], nc[0]).when(conds[1], 2).end().download()
    nc[0].is_null().download(); nc[1].is_not_null().download(); nc[2].is_nan().download()
    if npdt in (np.float32, np.float64):
        nc[0].nanvl(nc[1]).download()
rdf.coalesce(conds[0], conds[1], False).download()
rdf.when(conds[0], conds[1]).otherwise(True).download()
# round 2: the fleet code path on one GPU, and a single-rank communicator (pack -> combine -> unpack on the stream)
fleet = rdf.Context.multi(1)
fa = [P.from_numpy(rng.integers(-100, 100, n).astype(np.int64), rng.random(n) > 0.3) for n in (1000, 0, 77)]
rdf.ScalarFunctions.add(fa, fa, ctx=fleet); rdf.AggregateFunctions.all([c for c in fa if c.length], ctx=fleet)
fleet.close()
solo = rdf.Context(0)
solo.comm_attach(rdf.Context.comm_unique_id(), 0, 1)
rdf.AggregateFunctions.all([c for c in fa if c.length], ctx=solo)
solo.close()
print("sanitize cases done")
