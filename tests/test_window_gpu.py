"""Window functions (bdf_window_dev) on the GPU, element for element against the numpy restatement in tests/window_oracle.py (itself
checked against SQLite in tests/test_window.py)."""
import ctypes as C
import os

import numpy as np
import pytest

import window_oracle as W
from helpers import pool_used

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALL = ["row_number", "rank", "dense_rank", "percent_rank", "cume_dist", "lag", "lead", "sum", "count", "min", "max", "avg"]


def _chunks(rdf, values, mask, lens):
    out, row = [], 0
    for n in lens:
        out.append(rdf.PrimitiveArray.from_numpy(values[row:row + n], None if mask is None else mask[row:row + n]))
        row += n
    return out


def _one(col):
    arrs = col.download()
    assert len(arrs) == 1
    return arrs[0].value_slice(), arrs[0].valid_mask()


def _values(rng, n, dt, null=0.1, card=None):
    dt = np.dtype(dt)
    if dt.kind == "f":
        v = (rng.integers(-card, card + 1, n) * 0.5).astype(dt) if card else rng.uniform(-1e3, 1e3, n).astype(dt)
        v[rng.random(n) < 0.01] = np.nan
        v[rng.random(n) < 0.01] = -0.0
    else:
        info = np.iinfo(dt)
        lo, hi = (max(info.min, -card), min(info.max, card)) if card else (info.min, info.max)
        v = rng.integers(lo, hi, n, dtype=dt, endpoint=True)
    return v, (rng.random(n) >= null if null else None)


def _check(got_cols, want, calls):
    for col, w, call in zip(got_cols, want, calls):
        fn = call[0]
        gv, gm = _one(col)
        assert np.array_equal(gm, w["valid"]), fn
        if w["exact"] is not None and (fn == "avg" or gv.dtype.kind == "f"):
            exact, mag, k = w["exact"]
            nan = np.isnan(exact)
            assert np.array_equal(np.isnan(gv) & gm, nan & gm), fn
            ok = gm & ~nan
            bar = 16 * np.log2(np.maximum(k, 2)) * 2.0 ** -53 * mag + 1e-300
            if fn == "avg":   # the sum's bar over the count, plus the division's rounding
                cnt = np.maximum(w["count"], 1)
                want_avg = exact / cnt
                assert np.all(np.abs(gv[ok] - want_avg[ok]) <= bar[ok] / cnt[ok] + np.abs(want_avg[ok]) * 2.0 ** -52), fn
            else:
                extra = np.abs(exact) * 2.0 ** -24 if gv.dtype == np.float32 else 0   # one more rounding, to f32
                assert np.all(np.abs(gv[ok].astype(np.longdouble) - exact[ok]) <= (bar + extra)[ok]), fn
        else:
            g, x = gv[gm], np.asarray(w["values"])[gm]
            if g.dtype.kind == "f":
                nan = np.isnan(g)
                assert np.array_equal(nan, np.isnan(x)), fn
                g, x = g[~nan], x[~nan]
            u = np.dtype(f"u{g.dtype.itemsize}")
            bad = np.nonzero(g.view(u) != np.ascontiguousarray(x, dtype=g.dtype).view(u))[0]
            assert bad.size == 0, (fn, bad[:5], g[bad[:5]], x[bad[:5]])


def _run(rdf, ctx, part, order, calls, lens):
    """part: [(values, mask)]; order: [((values, mask), descending)]; calls: [(fn, (values, mask) or None, arg)].  Uploads chunked by
    lens, runs the GPU and the oracle, compares, and returns the GPU columns."""
    up = {}

    def chunks(vm):
        if id(vm) not in up:
            ch = _chunks(rdf, vm[0], vm[1], lens)
            up[id(vm)] = (ch, rdf.Column.upload(ch, ctx=ctx))
        return up[id(vm)]

    pc = [chunks(p) for p in part]
    oc = [(chunks(o), d) for o, d in order]
    gpu_calls, ora_calls = [], []
    for fn, x, arg in calls:
        if x is None:
            gpu_calls.append((fn,))
            ora_calls.append((fn, None, None))
        elif fn in ("lag", "lead"):
            gpu_calls.append((fn, chunks(x)[1], arg[0], arg[1]))
            ora_calls.append((fn, chunks(x)[0], arg))
        else:
            gpu_calls.append((fn, chunks(x)[1], arg))
            ora_calls.append((fn, chunks(x)[0], arg))
    got = rdf.window([c[1] for c in pc], [(c[1], d) for c, d in oc], gpu_calls)
    want = W.window([c[0] for c in pc], [(c[0], d) for c, d in oc], ora_calls, n=sum(lens))
    _check(got, want, ora_calls)
    return got, (pc, oc, gpu_calls)


def _all_calls(x, dt, frame="range", default=None):
    out = []
    for fn in ALL:
        if fn in ("row_number", "rank", "dense_rank", "percent_rank", "cume_dist"):
            out.append((fn, None, None))
        elif fn in ("lag", "lead"):
            out.append((fn, x, (1, default)))
        elif not (fn == "avg" and np.dtype(dt).itemsize == 8 and np.dtype(dt).kind != "f"):
            out.append((fn, x, frame))
    return out


DTYPES = ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "float32", "float64"]


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
def test_every_value_dtype(rdf, ctx, dt):
    rng = np.random.default_rng(DTYPES.index(dt) + 1)
    lens = [3000, 1, 0, 4097, 64]
    n = sum(lens)
    k, km = _values(rng, n, "int32", 0.05, card=20)
    o, om = _values(rng, n, "float64", 0.05, card=30)
    x = _values(rng, n, dt, 0.15)
    default = np.array(7, dtype=dt).item()
    for frame in ("rows", "range", "partition"):
        _run(rdf, ctx, [(k, km)], [((o, om), True)], _all_calls(x, dt, frame, default), lens)


@pytest.mark.gpu
@pytest.mark.parametrize("n_part,n_order", [(0, 1), (1, 0), (2, 2), (16, 16), (0, 16), (16, 0)])
def test_key_counts_and_directions(rdf, ctx, n_part, n_order):
    rng = np.random.default_rng(10 * n_part + n_order)
    lens = [2500, 3333, 17]
    n = sum(lens)
    kinds = ["int8", "float32", "uint16", "int64", "float64", "uint8", "int16", "uint32"]
    card = 2 if n_part + n_order > 8 else 6
    part = [_values(rng, n, kinds[i % 8], 0.05, card=card) for i in range(n_part)]
    order = [(_values(rng, n, kinds[(i + 3) % 8], 0.05, card=card), i % 2 == 1) for i in range(n_order)]
    x = _values(rng, n, "float64", 0.1)
    xi = _values(rng, n, "int32", 0.1)
    calls = _all_calls(x, "float64", "range") + [("sum", xi, "rows"), ("max", xi, "partition"), ("lead", xi, (3, None)), ("count", x, "rows")]
    _run(rdf, ctx, part, order, calls, lens)


@pytest.mark.gpu
def test_no_keys_reads_sliced_chunks_in_place(rdf, ctx):
    """No partition and no order: row-order running aggregates over sliced chunks whose validity starts at a bit offset."""
    rng = np.random.default_rng(5)
    P = rdf.PrimitiveArray
    base = rng.uniform(-1e3, 1e3, 20_000)
    bm = rng.random(20_000) > 0.2
    base_i = rng.integers(-2 ** 31, 2 ** 31, 20_000).astype(np.int32)
    xch = [P.from_numpy(base, bm).slice(3, 7000), P.from_numpy(base, bm).slice(7100, 1), P.from_numpy(base, bm).slice(9005, 9000)]
    ich = [P.from_numpy(base_i, bm).slice(5, 7000), P.from_numpy(base_i, bm).slice(7101, 1), P.from_numpy(base_i, bm).slice(9001, 9000)]
    cx, ci = rdf.Column.upload(xch, ctx=ctx), rdf.Column.upload(ich, ctx=ctx)
    calls = [("sum", "rows"), ("avg", "rows"), ("min", "range"), ("max", "partition"), ("count", "rows")]
    got = rdf.window([], [], [(fn, cx, fr) for fn, fr in calls] + [(fn, ci, fr) for fn, fr in calls] +
                     [("lag", cx, 2), ("lead", ci, 1, -1), ("row_number",), ("rank",), ("cume_dist",)])
    ora = [(fn, xch, fr) for fn, fr in calls] + [(fn, ich, fr) for fn, fr in calls] + \
          [("lag", xch, (2, None)), ("lead", ich, (1, -1)), ("row_number", None, None), ("rank", None, None), ("cume_dist", None, None)]
    _check(got, W.window([], [], ora), ora)


@pytest.mark.gpu
def test_edge_shapes(rdf, ctx):
    P = rdf.PrimitiveArray
    empty = rdf.Column.upload([P.from_numpy(np.zeros(0, np.int32))], ctx=ctx)
    res = rdf.window([empty], [(empty, False)], [("rank",), ("lag", empty, 1), ("sum", empty, "rows"), ("avg", empty, "range")])
    assert [len(r) for r in res] == [0, 0, 0, 0]
    rng = np.random.default_rng(4)
    for n in (1, 2047, 2049, 70_001):
        x = _values(rng, n, "float64", 0.1)
        uniq = (rng.permutation(n).astype(np.int64), None)              # every row its own partition
        _run(rdf, ctx, [uniq], [], _all_calls(x, "float64", "rows"), [n])
        _run(rdf, ctx, [], [], _all_calls(x, "float64", "range", 1.5), [n])


@pytest.mark.gpu
def test_one_partition_over_many_tiles(rdf, ctx):
    """1.5e6 rows in one partition: the segmented scan carries across ~730 tiles; the same bits on a second run."""
    rng = np.random.default_rng(9)
    n = 1_500_003
    o = _values(rng, n, "int64", 0.01, card=50_000)
    x = _values(rng, n, "float64", 0.05)
    xi = _values(rng, n, "int16", 0.05)
    calls = [("rank", None, None), ("cume_dist", None, None), ("sum", x, "rows"), ("sum", x, "range"), ("avg", x, "rows"),
             ("min", x, "rows"), ("max", xi, "range"), ("sum", xi, "rows"), ("count", xi, "partition")]
    got, (pc, oc, gcalls) = _run(rdf, ctx, [], [(o, False)], calls, [700_000, 800_003])
    again = rdf.window([c[1] for c in pc], [(c[1], d) for c, d in oc], gcalls)
    for a, b in zip(got, again):
        (p, pm), (q, qm) = _one(a), _one(b)
        u = np.dtype(f"u{p.dtype.itemsize}")
        assert np.array_equal(pm, qm) and np.array_equal(p.view(u), q.view(u))


@pytest.mark.gpu
def test_shared_spec_and_repeated_calls(rdf, ctx):
    rng = np.random.default_rng(12)
    n = 30_000
    k = _values(rng, n, "uint8", 0.0, card=40)
    o = _values(rng, n, "float32", 0.1, card=100)
    x = _values(rng, n, "float32", 0.1)
    calls = [("rank", None, None), ("rank", None, None), ("sum", x, "range"), ("sum", x, "range"), ("lag", x, (2, None)),
             ("lag", x, (2, None)), ("row_number", None, None), ("percent_rank", None, None)]
    got, _ = _run(rdf, ctx, [k], [(o, True)], calls, [n])
    for a, b in ((0, 1), (2, 3), (4, 5)):
        (p, pm), (q, qm) = _one(got[a]), _one(got[b])
        u = np.dtype(f"u{p.dtype.itemsize}")
        assert np.array_equal(pm, qm) and np.array_equal(p.view(u), q.view(u))


@pytest.mark.gpu
def test_device_generated_2_pow_24_rows(rdf, ctx):
    n = 2 ** 24 + 5
    lens = [2 ** 23, 2 ** 23 + 5]
    k = rdf.Column.generate(rdf.I8, lens, kind=2, col_id=1, ctx=ctx)
    o = rdf.Column.generate(rdf.I16, lens, kind=2, col_id=2, null_mod=97, ctx=ctx)
    x = rdf.Column.generate(rdf.F64, lens, kind=0, lo=-1.0, hi=1.0, col_id=3, null_mod=13, ctx=ctx)
    got = rdf.window([k], [(o, True)], [("row_number",), ("rank",), ("lag", x, 1), ("sum", x, "rows"), ("max", x, "range")])
    kch, och, xch = k.download(), o.download(), x.download()
    ora = [("row_number", None, None), ("rank", None, None), ("lag", xch, (1, None)), ("sum", xch, "rows"), ("max", xch, "range")]
    _check(got, W.window([kch], [(och, True)], ora, n=n), ora)


@pytest.mark.gpu
def test_pool_and_errors(rdf, ctx):
    N = rdf.native
    P = rdf.PrimitiveArray
    a = rdf.Column.upload([P.from_numpy(np.arange(100, dtype=np.int32))], ctx=ctx)
    a99 = rdf.Column.upload([P.from_numpy(np.arange(99, dtype=np.int32))], ctx=ctx)
    i64 = rdf.Column.upload([P.from_numpy(np.arange(100, dtype=np.int64))], ctx=ctx)
    flag = a.compare(N.GT, 50.0)
    ctx.synchronize()
    before = pool_used(ctx)
    res = rdf.window([a], [(a, True)], [("rank",), ("lag", a, 1), ("sum", a, "range"), ("min", a, "rows")])
    for r in res:
        r.free()
    ctx.synchronize()
    assert pool_used(ctx) == before

    def call(n_part, part, n_order, order, calls):
        pk = (C.c_void_p * max(len(part), 1))(*[c.handle for c in part])
        ok = (N.SortKeyC * max(len(order), 1))()
        for i, (c, d) in enumerate(order):
            ok[i].column, ok[i].descending = c.handle.value, d
        arr = (N.WindowCall * max(len(calls), 1))()
        for j, (fn, col, frame, off) in enumerate(calls):
            arr[j].function, arr[j].frame, arr[j].offset = fn, frame, off
            arr[j].column = col.handle.value if col is not None else None
        out = (C.c_void_p * max(len(calls), 1))()
        st = N.lib().bdf_window_dev(ctx.handle, n_part, pk if part else None, n_order, ok if order else None, len(calls), arr, out)
        assert all(out[j] is None for j in range(len(calls)))
        return st

    rank = (N.WIN_RANK, None, 0, 0)
    assert call(17, [a] * 17, 0, [], [rank]) == N.INVALID
    assert call(0, [], 17, [(a, 0)] * 17, [rank]) == N.INVALID
    assert call(1, [a], 0, [], [rank] * 65) == N.INVALID
    assert call(1, [], 0, [], [rank]) == N.INVALID                                    # null pointer
    assert call(1, [a], 0, [], [(N.WIN_LAG, a, 0, -1)]) == N.INVALID                  # negative offset
    assert call(1, [a], 0, [], [(N.WIN_RANK, a, 0, 0)]) == N.INVALID                  # a ranking call with a column
    assert call(1, [a], 0, [], [(N.WIN_SUM, None, 0, 0)]) == N.INVALID                # an aggregate without one
    assert call(0, [], 0, [], [rank]) == N.INVALID                                    # nothing to count rows by
    assert call(1, [a], 0, [], [(99, a, 0, 0)]) == N.UNSUPPORTED
    assert call(1, [a], 0, [], [(N.WIN_SUM, a, 7, 0)]) == N.UNSUPPORTED
    assert call(1, [flag], 0, [], [rank]) == N.UNSUPPORTED
    assert call(1, [a], 0, [], [(N.WIN_AVG, i64, 0, 0)]) == N.UNSUPPORTED
    assert call(1, [a], 1, [(a99, 0)], [rank]) == N.LENGTH_MISMATCH
    huge = rdf.Column.generate(rdf.I8, [2 ** 31, 2 ** 31], kind=2, ctx=ctx)              # 2^32 rows: one too many for UInt32 positions
    assert call(1, [huge], 0, [], [rank]) == N.UNSUPPORTED
    huge.free()
    with pytest.raises(rdf.UnsupportedType):
        rdf.window([a], [], [("ntile", a)])
    with pytest.raises(rdf.UnsupportedType):
        rdf.window([a], [], [("sum", a, "groups")])
    ctx.synchronize()
    assert pool_used(ctx) == before


@pytest.mark.gpu
def test_multi_gpu_context_is_refused(rdf):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU: no multi-GPU context")
    fleet = rdf.Context.multi(0)
    try:
        fk = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.arange(10, dtype=np.int64))], ctx=fleet)
        with pytest.raises(rdf.UnsupportedType):
            rdf.window([fk], [], [("row_number",)])
    finally:
        fleet.close()


@pytest.mark.gpu
def test_device_frame_window_and_evaluate(rdf, ctx):
    from rust_dataframe_b200.frame import select, window

    path = os.path.join(ROOT, "tests", "golden", "uk_cities_with_headers.csv")
    frame = rdf.DeviceFrame.from_csv(path, ctx=ctx)
    host = {n: c.download() for n, c in frame.columns.items()}
    out = frame.window([], [("lng", True)], [("r", "rank"), ("lat", "lag", "lat", 1)])
    assert list(out.schema) == ["lng", "r", "lat"]   # lat replaced, as with_column does
    lat, lng = [np.concatenate([a.value_slice() for a in host[c]]) for c in ("lat", "lng")]
    ora = W.window([], [(host["lng"], True)], [("rank", None, None), ("lag", host["lat"], (1, None))])
    _check([out.column("r"), out.column("lat")], ora, [("rank",), ("lag",)])
    ev = frame.evaluate([window([], [], [("running", "sum", "lat", "rows")]), select(["running"])])
    got, gm = _one(ev.column("running"))
    assert gm.all() and np.allclose(got, np.cumsum(lat), rtol=1e-13, atol=0)
    order = np.argsort(-lng, kind="stable")
    assert _one(out.column("r"))[0][order[0]] == 1
