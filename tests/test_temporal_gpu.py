"""Dates and timestamps on the GPU (include/b200df.h "dates and timestamps"), bit for bit against tests/temporal_oracle.py: every function
over every valid kind / unit on ragged, sliced chunks with nulls and edge values; the host-in form; a multi-GPU context; an IPC round
trip through pyarrow; a frame pipeline against pandas; refusals without leaks; one call at 1e8 rows."""
import ctypes as C
import datetime as dt

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pyarrow.ipc as pai
import pytest

import temporal_oracle as O
from helpers import pool_used

pytestmark = pytest.mark.gpu

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1


EDGE_DATES = [(1900, 2, 28), (1900, 3, 1), (2000, 2, 29), (2100, 2, 28), (0, 1, 1), (-1, 6, 15), (2019, 1, 31), (2019, 2, 28),
              (2016, 2, 29), (2016, 8, 31), (2015, 1, 14), (1969, 12, 31), (1677, 9, 21), (2262, 4, 11), (-262144, 1, 1), (262143, 12, 31)]


def edge_values(kind, unit):
    upd, ups = O.per_day(kind, unit)
    lo, hi = (I32_MIN, I32_MAX) if kind in (O.DATE32, O.TIME32) else (I64_MIN, I64_MAX)
    days = [int(O.days_from_civil(y, m, d)) for y, m, d in EDGE_DATES] + [O.MIN_DAY - 1, O.MAX_DAY + 1, I32_MIN // 2, I32_MAX // 2]
    vals = [0, -1, 1, upd, -upd, upd - 1, upd + 1, -upd - 1, -upd + 1, lo, hi, lo + 1, hi - 1]
    for d in days:
        for tod in ([0] if upd == 1 else [0, 1, upd - 1, upd // 2 + 7 * ups]):
            vals.append(d * upd + tod)
    return [v for v in vals if lo <= v <= hi]


def random_values(rng, kind, unit, n):
    upd, ups = O.per_day(kind, unit)
    if kind in (O.TIME32, O.TIME64):
        return rng.integers(-upd // 10, upd + upd // 10, n)
    y0, y1 = (1680, 2260) if upd == 86400 * 10 ** 9 else (1500, 2500)   # nanoseconds span 1677..2262
    days = rng.integers(int(O.days_from_civil(y0, 1, 1)), int(O.days_from_civil(y1, 1, 1)), n)
    v = days * upd + (rng.integers(0, upd, n) if upd > 1 else 0)
    wide = rng.integers(I32_MIN, I32_MAX, n) if kind in (O.DATE32, O.TIME32) else rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64)
    return np.where(rng.random(n) < 0.1, wide, v)


def make_chunks(rdf, rng, t, lens=(1000, 0, 37, 4099, 1)):
    """Ragged chunks, sliced (offset into a bigger buffer), 15 % nulls, edge values mixed in.  Returns (chunks, values, valid)."""
    edges = np.array(edge_values(t.kind, t.unit), dtype=np.int64)
    npdt = np.int32 if t.dtype == rdf.I32 else np.int64
    chunks, allv, allm = [], [], []
    for k, n in enumerate(lens):
        v = random_values(rng, t.kind, t.unit, n + 5)
        if n:
            idx = rng.integers(0, n + 5, min(len(edges), n))
            v[idx] = edges[: len(idx)]
        m = rng.random(n + 5) >= 0.15
        arr = rdf.PrimitiveArray.from_numpy(v.astype(npdt), m).slice(3, n)
        arr.temporal = t
        chunks.append(arr)
        allv.append(v[3:3 + n])
        allm.append(m[3:3 + n])
    return chunks, np.concatenate(allv).astype(np.int64), np.concatenate(allm)


def concat(chunks):
    vals = np.concatenate([c.value_slice() for c in chunks]) if chunks else np.zeros(0)
    mask = np.concatenate([c.valid_mask() for c in chunks]) if chunks else np.zeros(0, bool)
    return vals, mask


def check(got_chunks, want_v, want_ok, what):
    gv, gm = concat(got_chunks)
    assert gm.tolist() == want_ok.tolist() or (gm == want_ok).all(), f"{what}: validity differs at {np.nonzero(gm != want_ok)[0][:8]}"
    assert gv.dtype == want_v.dtype, f"{what}: dtype {gv.dtype} != {want_v.dtype}"
    bad = np.nonzero(gv.view(f"u{gv.dtype.itemsize}") != want_v.view(f"u{want_v.dtype.itemsize}"))[0]
    assert bad.size == 0, f"{what}: {bad.size} values differ, first at {bad[:5]}: got {gv[bad[:5]]}, want {want_v[bad[:5]]}"
    for c in got_chunks:
        assert c.null_count == c.length - int(c.valid_mask().sum()), what


def calls_for(kind):
    if kind in (O.TIME32, O.TIME64):
        return [("hour", 0), ("minute", 0), ("second", 0)]
    calls = [(f, 0) for f in ("year", "quarter", "month", "day_of_month", "day_of_year", "day_of_week", "hour", "minute", "second", "to_date",
                              "last_day", "unix_timestamp")]
    calls += [("date_add", a) for a in (5, -100000, I32_MAX, I32_MIN)] + [("date_sub", a) for a in (7, I32_MIN)]
    calls += [("add_months", a) for a in (1, -13, 12 * 1000, I32_MAX, I32_MIN)] + [("next_day", a) for a in (1, 3, 7)]
    calls += [("date_trunc", a) for a in range(8)] + [("to_timestamp", a) for a in range(4)]
    return calls


def types(rdf):
    T = rdf.TemporalType
    return [T.date32(), T.date64(), T.timestamp("s"), T.timestamp("ms"), T.timestamp("us"), T.timestamp("ns"), T.timestamp("us", "+05:30"),
            T.timestamp("ns", "-08:00"), T.timestamp("s", "UTC"), T.time32("s"), T.time32("ms"), T.time64("us"), T.time64("ns")]


def test_every_function_every_type_against_the_oracle(rdf, ctx):
    for ti, t in enumerate(types(rdf)):
        rng = np.random.default_rng(100 + ti)
        chunks, v, m = make_chunks(rdf, rng, t)
        col = rdf.Column.upload(chunks, ctx, dtype=t.dtype).with_temporal(t)
        for fn, arg in calls_for(t.kind):
            out = col._temporal_fn(rdf.native.TEMPORAL_FNS[fn], arg)
            got = out.download()
            want_v, want_ok = O.unary(fn, t.kind, t.unit, t.tz, v, m, arg)
            check(got, want_v, want_ok, f"{t!r} {fn}({arg})")
            assert [c.length for c in got] == [c.length for c in chunks]
            assert out.temporal == rdf.temporal_result(fn, t, arg)[1]


def test_two_column_functions_against_the_oracle(rdf, ctx):
    T = rdf.TemporalType
    pairs = [(T.timestamp("us"), T.date32()), (T.date32(), T.date32()), (T.timestamp("ns", "+01:00"), T.timestamp("s")),
             (T.date64(), T.timestamp("ms", "-08:00")), (T.timestamp("s"), T.timestamp("us", "+05:30"))]
    for k, (ta, tb) in enumerate(pairs):
        rng = np.random.default_rng(200 + k)
        ca, va, ma = make_chunks(rdf, rng, ta)
        cb, vb, mb = make_chunks(rdf, rng, tb)
        A = rdf.Column.upload(ca, ctx, dtype=ta.dtype).with_temporal(ta)
        B = rdf.Column.upload(cb, ctx, dtype=tb.dtype).with_temporal(tb)
        for fn in ("date_diff", "months_between"):
            got = getattr(A, fn)(B).download()
            want_v, want_ok = O.binary(fn, (ta.kind, ta.unit, ta.tz), va, ma, (tb.kind, tb.unit, tb.tz), vb, mb)
            check(got, want_v, want_ok, f"{fn}({ta!r}, {tb!r})")
    # the documented example, and zip / length rules
    t1 = int(dt.datetime(1997, 2, 28, 10, 30, tzinfo=dt.timezone.utc).timestamp())
    a = rdf.PrimitiveArray.from_numpy(np.array([t1], np.int64))
    b = rdf.PrimitiveArray.from_numpy(np.array([int(O.days_from_civil(1996, 10, 30))], np.int32))
    r = rdf.ScalarFunctions.months_between([a], [b], T.timestamp("s"), T.date32(), ctx=ctx)
    assert r[0].value(0) == 3.94959677
    with pytest.raises(rdf.ComputeError):
        A2 = rdf.Column.upload([a, a], ctx).with_temporal(T.timestamp("s"))
        B2 = rdf.Column.upload([b, rdf.PrimitiveArray.from_numpy(np.array([1, 2], np.int32))], ctx).with_temporal(T.date32())
        A2.date_diff(B2)


def test_host_in_equals_device(rdf, ctx):
    T = rdf.TemporalType
    for t in (T.timestamp("us", "+02:00"), T.date32(), T.time64("ns")):
        rng = np.random.default_rng(7)
        chunks, v, m = make_chunks(rdf, rng, t)
        col = rdf.Column.upload(chunks, ctx, dtype=t.dtype).with_temporal(t)
        for fn, arg in calls_for(t.kind)[:12] + ([("date_trunc", 3), ("add_months", 1), ("to_timestamp", 3)] if t.kind != O.TIME64 else []):
            dev = col._temporal_fn(rdf.native.TEMPORAL_FNS[fn], arg).download()
            f = getattr(rdf.ScalarFunctions, fn)
            host = f(chunks, arg, ctx=ctx) if fn in ("date_trunc", "add_months", "to_timestamp") else f(chunks, ctx=ctx)
            assert len(host) == len(dev)
            for h, d in zip(host, dev):
                assert h.temporal == d.temporal
                assert (h.valid_mask() == d.valid_mask()).all() and (h.value_slice() == d.value_slice()).all(), fn


def test_multi_gpu_context_gives_one_gpu_bits(rdf, ctx):
    T = rdf.TemporalType
    fleet = rdf.Context.multi(0)
    try:
        t = T.timestamp("ns", "+09:00")
        rng = np.random.default_rng(9)
        chunks, v, m = make_chunks(rdf, rng, t, lens=(100000, 0, 3, 77777))
        dchunks, dv, dm = make_chunks(rdf, rng, T.date32(), lens=(100000, 0, 3, 77777))
        one = rdf.Column.upload(chunks, ctx).with_temporal(t)
        many, dmany = rdf.Column.upload_many([chunks, dchunks], fleet)
        many.with_temporal(t)
        dmany.with_temporal(T.date32())
        for fn, arg in [("hour", 0), ("day_of_week", 0), ("date_trunc", 3), ("add_months", 13), ("to_timestamp", 0)]:
            a = one._temporal_fn(rdf.native.TEMPORAL_FNS[fn], arg).download()
            b = many._temporal_fn(rdf.native.TEMPORAL_FNS[fn], arg).download()
            f = getattr(rdf.ScalarFunctions, fn)
            c = f(chunks, arg, ctx=fleet) if fn in ("date_trunc", "add_months", "to_timestamp") else f(chunks, ctx=fleet)
            for x, y, z in zip(a, b, c):
                assert (x.valid_mask() == y.valid_mask()).all() and (x.value_slice() == y.value_slice()).all(), fn
                assert (x.valid_mask() == z.valid_mask()).all() and (x.value_slice() == z.value_slice()).all(), fn
                assert x.null_count == y.null_count == z.null_count
        d1 = one.months_between(rdf.Column.upload(dchunks, ctx).with_temporal(T.date32())).download()
        d2 = many.months_between(dmany).download()
        for x, y in zip(d1, d2):
            assert (x.valid_mask() == y.valid_mask()).all() and (x.value_slice().view(np.uint64) == y.value_slice().view(np.uint64)).all()
    finally:
        fleet.close()


def test_ipc_round_trip_through_pyarrow(rdf, ctx, tmp_path):
    rng = np.random.default_rng(5)
    n = 5000
    us = rng.integers(-2208988800 * 10 ** 6, 4102444800 * 10 ** 6, n)
    batches = []
    for lo, hi in ((0, 1000), (1000, 1000), (1000, n)):
        mask = rng.random(hi - lo) < 0.1
        batches.append(pa.record_batch([pa.array(us[lo:hi], pa.int64(), mask=mask).view(pa.timestamp("us", tz="+02:00")),
                                        pa.array((us[lo:hi] // 86400000000).astype(np.int32), pa.int32(), mask=mask[::-1]).view(pa.date32()),
                                        pa.array(us[lo:hi] % 86400000000 * 1000, pa.int64()).view(pa.time64("ns"))], names=["ts", "d", "t"]))
    path, out = str(tmp_path / "in.arrow"), str(tmp_path / "out.arrow")
    with pai.new_file(path, batches[0].schema) as w:
        for b in batches:
            w.write_batch(b)
    f = rdf.IpcFile(path)
    assert f.read() == {} and [d for _, d, _ in f.schema] == [-1, -1, -1]   # unnamed reads are unchanged
    cols = f.read(["ts", "d", "t"], ctx=ctx)
    trunc, am, hr = cols["ts"].date_trunc("day"), cols["d"].add_months(1), cols["t"].hour()
    rdf.write_ipc(out, {"ts": cols["ts"], "trunc": trunc, "am": am, "d": cols["d"], "t": cols["t"], "hour": hr})
    f.close()
    src = pa.ipc.open_file(path).read_all()
    got = pa.ipc.open_file(out).read_all()
    assert got.schema.field("ts").type == pa.timestamp("us", tz="+02:00") and got.schema.field("trunc").type == pa.timestamp("us", tz="+02:00")
    assert got.schema.field("d").type == pa.date32() and got.schema.field("am").type == pa.date32()
    assert got.schema.field("t").type == pa.time64("ns") and got.schema.field("hour").type == pa.int32()
    assert got.column("ts").equals(src.column("ts")) and got.column("d").equals(src.column("d")) and got.column("t").equals(src.column("t"))
    want_trunc = pc.floor_temporal(src.column("ts"), unit="day")
    assert got.column("trunc").to_pylist() == want_trunc.to_pylist()
    assert got.column("hour").to_pylist() == pc.hour(src.column("t")).to_pylist()
    v, m = concat(cols["d"].download())
    want_v, want_ok = O.unary("add_months", O.DATE32, 0, None, v, m, 1)
    assert got.column("am").to_pylist() == [dt.date(1970, 1, 1) + dt.timedelta(days=int(x)) if ok else None for x, ok in zip(want_v, want_ok)]


def us_of(series):
    """Microseconds since the epoch of a pandas datetime Series, whatever unit pandas keeps it in."""
    return series.astype("datetime64[us]").astype("int64")


def test_frame_pipeline_against_pandas(rdf, ctx, tmp_path):
    import pandas as pd

    rng = np.random.default_rng(6)
    n = 20000
    us = rng.integers(0, 40 * 86400 * 10 ** 6, n) + 1600000000 * 10 ** 6
    ts = pa.array(us, pa.int64()).view(pa.timestamp("us"))
    d = pa.array(rng.integers(19000, 19030, n).astype(np.int32)).view(pa.date32())
    x = pa.array(rng.permutation(n).astype(np.int64))
    tb = pa.table({"ts": ts, "d": d, "x": x})
    path = str(tmp_path / "f.arrow")
    with pai.new_file(path, tb.schema) as w:
        w.write_table(tb, max_chunksize=7000)
    assert list(rdf.DeviceFrame.from_arrow(path, ctx=ctx).columns) == ["x"]   # unnamed: as before
    fr = rdf.DeviceFrame.from_arrow(path, columns=["ts", "d", "x"], ctx=ctx)
    assert fr.column("ts").temporal == rdf.TemporalType.timestamp("us") and fr.column("d").temporal == rdf.TemporalType.date32()
    df = tb.to_pandas()
    # sort by the timestamp, then a filter through to_date
    s = fr.sort([("ts", False)])
    s = s.with_column("day", s.column("ts").to_date())
    cut = int(O.days_from_civil(2020, 9, 25))
    s = s.filter(("ge", ("col", "day"), ("scalar", cut)))
    host = {k: v for k, v in s.to_host().items()}
    pdf = df.sort_values("ts", kind="stable")
    pdf = pdf[pdf.ts.dt.normalize() >= pd.Timestamp("2020-09-25")]
    assert np.concatenate([c.value_slice() for c in host["x"]]).tolist() == pdf.x.tolist()
    assert np.concatenate([c.value_slice() for c in host["ts"]]).tolist() == us_of(pdf.ts).tolist()
    # group-by on to_date with min / max / first / last / count_distinct of the timestamp
    g = fr.with_column("day", fr.column("ts").to_date())
    keys, res = rdf.group_by([g.column("day")], [(g.column("ts"), "min"), (g.column("ts"), "max"), (g.column("ts"), "first"),
                                                 (g.column("ts"), "last"), (g.column("ts"), "count_distinct"), (g.column("ts"), "count")])
    assert keys[0].temporal == rdf.TemporalType.date32() and all(r.temporal == fr.column("ts").temporal for r in res[:4])
    assert res[4].temporal is None and res[5].temporal is None
    want = df.assign(day=df.ts.dt.normalize()).groupby("day").ts.agg(["min", "max", "first", "last", "nunique", "count"])
    kv = keys[0].download()[0].value_slice()
    assert kv.tolist() == [(t - pd.Timestamp(0)).days for t in want.index]
    for r, name in zip(res, ["min", "max", "first", "last", "nunique", "count"]):
        got = r.download()[0].value_slice()
        w = want[name]
        w = us_of(w) if name in ("min", "max", "first", "last") else w
        assert got.tolist() == w.tolist(), name
    # join on Date32 keys
    other = rdf.DeviceFrame.from_host({"k": [rdf.PrimitiveArray.from_numpy(np.arange(19000, 19010, dtype=np.int32))],
                                       "v": [rdf.PrimitiveArray.from_numpy(np.arange(10, dtype=np.int64))]}, ctx=ctx)
    other.column("k").with_temporal(rdf.TemporalType.date32())
    j = fr.join(other, [("d", "k")], "inner")
    assert j.column("d").temporal == rdf.TemporalType.date32() and j.column("ts").temporal == fr.column("ts").temporal
    merged = df.assign(di=(df.d - pd.Timestamp(0).date()).map(lambda t: t.days)).merge(pd.DataFrame({"k": np.arange(19000, 19010), "v": np.arange(10)}),
                                                                                       left_on="di", right_on="k")
    assert len(j.column("x")) == len(merged)
    assert sorted(np.concatenate([c.value_slice() for c in j.column("x").download()]).tolist()) == sorted(merged.x.tolist())
    # window lag of the timestamp (ordered by x)
    w = fr.window([], [("x", False)], [("prev", "lag", "ts", 1)])
    assert w.column("prev").temporal == fr.column("ts").temporal
    order = df.sort_values("x")
    lag = order.ts.shift(1)
    got_v, got_m = concat(w.column("prev").download())
    want_prev = pd.Series(lag.values, index=order.index).reindex(df.index)
    assert (got_m == want_prev.notna().values).all()
    assert (got_v[got_m] == us_of(want_prev[want_prev.notna()]).values).all()
    # to_arrow round-trips the types
    out = str(tmp_path / "o.arrow")
    s.to_arrow(out)
    back = pa.ipc.open_file(out).read_all()
    assert back.schema.field("ts").type == pa.timestamp("us") and back.schema.field("d").type == pa.date32() and back.schema.field("day").type == pa.date32()


def test_refusals_leak_nothing(rdf, ctx, tmp_path):
    T = rdf.TemporalType
    ts = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.arange(10, dtype=np.int64))], ctx).with_temporal(T.timestamp("us"))
    paris = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.arange(10, dtype=np.int64))], ctx).with_temporal(T.timestamp("us", "Europe/Paris"))
    d32 = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.arange(10, dtype=np.int32))], ctx).with_temporal(T.date32())
    plain32 = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.arange(10, dtype=np.int32))], ctx)
    ctx.synchronize()
    before = pool_used(ctx)
    N = rdf.native
    for f in (lambda: ts.sum(), lambda: ts.avg(), lambda: ts.add(ts), lambda: ts.gt(5), lambda: ts.variance(), lambda: ts.sum_distinct(),
              lambda: ts.cast(rdf.F64), lambda: rdf.group_by([d32], [(ts, "sum")]), lambda: rdf.window([], [(d32, False)], [("avg", ts)]),
              lambda: rdf.DeviceFrame({"ts": ts}).to_csv(str(tmp_path / "x.csv")), lambda: paris.hour(), lambda: paris.date_trunc("day")):
        with pytest.raises(rdf.UnsupportedType):
            f()
    for f in (lambda: d32.next_day(0), lambda: d32.next_day(8), lambda: d32.date_add(1 << 31)):
        with pytest.raises(rdf.ComputeError):
            f()
    # a wrong physical dtype: the device entry refuses it
    h = C.c_void_p()
    tc = N.TemporalTypeC(N.TIMESTAMP, 2, None)
    assert N.lib().bdf_temporal_dev(ctx.handle, N.T_HOUR, C.byref(tc), 0, plain32.handle, C.byref(h)) == N.INVALID
    with pytest.raises(rdf.ComputeError):
        plain32.with_temporal(T.timestamp("us"))
    ctx.synchronize()
    assert pool_used(ctx) == before
    assert paris.unix_timestamp().download()[0].value_slice().tolist() == [0] * 10   # instants accept any tz
    # the one-key group-by: sum of a tagged column is not returned, min / max carry the tag, and the frame refuses sum first
    keys, res = rdf.group_aggregate(d32, [ts])
    assert res[0]["sum"] is None and res[0]["min"].temporal == ts.temporal and res[0]["max"].temporal == ts.temporal
    assert res[0]["min"].download()[0].value_slice().tolist() == list(range(10)) and keys.temporal == T.date32()
    fr = rdf.DeviceFrame({"d": d32, "ts": ts})
    g = fr.group_aggregate("d", [("ts", "min"), ("ts", "count")])
    assert g.column("min(ts)").temporal == ts.temporal and g.column("count(ts)").temporal is None
    with pytest.raises(rdf.UnsupportedType):
        fr.group_aggregate("d", [("ts", "sum")])
    # chunks that carry one temporal type tag the uploaded column
    up = rdf.Column.upload(ts.download(), ctx)
    assert up.temporal == ts.temporal
    assert ts.count() == 10 and ts.count_distinct() == 10 and ts.min() == 0 and ts.max() == 9


def test_one_call_at_1e8_rows(rdf, ctx):
    n_chunks, per = 25, 4_000_000
    t = rdf.TemporalType.timestamp("us")
    col = rdf.Column.generate(rdf.I64, [per] * n_chunks, kind=2, null_mod=10, ctx=ctx).with_temporal(t)
    out = col.hour()
    assert out.n_chunks == n_chunks and len(out) == n_chunks * per
    rng = np.random.default_rng(12)
    src, got = col.download(), out.download()
    for c in rng.choice(n_chunks, 5, replace=False):
        rows = rng.choice(per, 20000, replace=False)
        v, m = src[c].value_slice()[rows], src[c].valid_mask()[rows]
        want_v, want_ok = O.unary("hour", O.TIMESTAMP, 2, None, v, m)
        assert (got[c].valid_mask()[rows] == want_ok).all() and (got[c].value_slice()[rows] == want_v).all()
        assert got[c].null_count == per - int(got[c].valid_mask().sum())
