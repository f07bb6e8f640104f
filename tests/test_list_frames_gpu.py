"""List columns in device frames on the GPU: take and filter of whole lists, collect_list / collect_set per group, frames that carry
list columns, and lists written to Arrow IPC -- each against tests/list_frame_oracle.py or pyarrow, bit for bit."""
import math
import os

import numpy as np
import pyarrow as pa
import pytest

import list_frame_oracle as lfo
from helpers import pool_used

pytestmark = pytest.mark.gpu

NP = [np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64, np.float32, np.float64]
PA = [pa.int8(), pa.int16(), pa.int32(), pa.int64(), pa.uint8(), pa.uint16(), pa.uint32(), pa.uint64(), pa.float32(), pa.float64()]


def bits(x, dt):
    if x is None:
        return None
    a = np.array([x], dtype=NP[dt])
    return int(a.view(f"u{a.itemsize}")[0])


def lists_bits(lists, dt):
    return [None if l is None else [bits(x, dt) for x in l] for l in lists]


def make_chunk(rng, dt, n, sliced=False):
    """A ListArray of n lists: null lists spanning elements, empty lists, null elements, NaN / +-0.0; sliced: list offset != 0 and
    child offset != 0."""
    lens = rng.integers(0, 9, n)
    total = int(lens.sum())
    if dt >= 8:
        pool = np.array([0.0, -0.0, np.nan, 1.5, -2.0, 3.0, 2.0], dtype=NP[dt])
        vals = pool[rng.integers(0, len(pool), total)]
    else:
        vals = rng.integers(0, 100, total).astype(NP[dt])
    emask = rng.random(total) < 0.15
    child = pa.array(vals, type=PA[dt], mask=emask)
    if sliced:
        pad = np.zeros(2, dtype=NP[dt])
        child = pa.array(np.concatenate([pad, vals, pad]), type=PA[dt], mask=np.concatenate([[True, False], emask, [False, True]])).slice(2, total)
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    lvalid = rng.random(n) >= 0.1
    arr = pa.Array.from_buffers(pa.list_(PA[dt]), n, [pa.py_buffer(np.packbits(lvalid, bitorder="little")), pa.py_buffer(offsets)],
                                null_count=int((~lvalid).sum()), children=[child])
    if sliced and n >= 10:
        arr = arr.slice(3, n - 5)
    return arr


def to_lists(arr):
    return [None if x is None else list(x) for x in arr.to_pylist()]


def upload(rdf, ctx, arrays):
    return rdf.ListColumn.upload([rdf.ListArray.from_arrow(a) for a in arrays], ctx)


def down_chunks(lc):
    return [ch.to_pylist() for ch in lc.download()]


def u32_col(rdf, ctx, idx):
    mask = np.array([i is not None for i in idx], dtype=bool)
    vals = np.array([0 if i is None else i for i in idx], dtype=np.uint32)
    return rdf.Column.upload([rdf.PrimitiveArray.from_numpy(vals, mask if not mask.all() else None)], ctx)


def bool_col(rdf, ctx, chunks):
    arrays = [rdf.BooleanArray.from_numpy(np.array([bool(b) for b in c], dtype=bool), np.array([b is not None for b in c], dtype=bool))
              for c in chunks]
    return rdf.Column.upload(arrays, ctx)


def exact_null_counts(lc, chunks):
    for i, ch in enumerate(chunks):
        assert lc.chunk_info(i)["null_count"] == sum(l is None for l in ch)


@pytest.mark.parametrize("dt", range(10))
def test_take_against_the_oracle(rdf, ctx, dt):
    rng = np.random.default_rng(dt)
    arrays = [make_chunk(rng, dt, n, sliced=k % 2 == 1) for k, n in enumerate((40, 0, 300, 1, 57, 123))]
    lists = sum((to_lists(a) for a in arrays), [])
    lc = upload(rdf, ctx, arrays)
    n = len(lists)
    cases = [list(rng.permutation(n)), [int(i) for i in rng.integers(0, n, 3 * n)], [None if rng.random() < 0.2 else int(i) for i in rng.integers(0, n, n)],
             [n - 1] * 50, []]
    for idx in cases:
        got = lc.take(u32_col(rdf, ctx, idx))
        assert got.n_chunks == 1
        want = lfo.take(lists, idx)
        chunks = down_chunks(got)
        assert lists_bits(chunks[0], dt) == lists_bits(want, dt)
        exact_null_counts(got, [want])
        assert got.chunk_info(0)["n_elements"] == sum(len(l) for l in want if l is not None)   # only valid lists' elements
        if dt < 8:   # pyarrow's take of the same chunks (NaN != NaN: the float types are checked by bits above)
            assert to_lists(pa.chunked_array(arrays, pa.list_(PA[dt])).take(pa.array(idx, pa.uint32()))) == chunks[0]


@pytest.mark.parametrize("dt", range(10))
def test_filter_keeps_the_chunks(rdf, ctx, dt):
    rng = np.random.default_rng(100 + dt)
    arrays = [make_chunk(rng, dt, n, sliced=k % 2 == 0) for k, n in enumerate((40, 0, 300, 1, 77))]
    lc = upload(rdf, ctx, arrays)
    per = [to_lists(a) for a in arrays]
    masks = [[None if rng.random() < 0.1 else bool(b) for b in rng.random(len(p)) < 0.5] for p in per]
    got = lc.filter(bool_col(rdf, ctx, masks))
    assert got.n_chunks == len(arrays)
    chunks = down_chunks(got)
    want = [lfo.filter_(p, m) for p, m in zip(per, masks)]
    assert [len(c) for c in chunks] == [len(w) for w in want]
    for c, w in zip(chunks, want):
        assert lists_bits(c, dt) == lists_bits(w, dt)
    exact_null_counts(got, want)
    with pytest.raises(rdf.ComputeError):   # mask chunks of other lengths
        lc.filter(bool_col(rdf, ctx, [[True] * len(p) for p in reversed(per)]))


def test_hot_list_take(rdf, ctx):
    """One list of 1e7 elements among 1e7 one-element lists, taken in reverse: the element gather spreads the hot list over the GPU."""
    hot, n_small = 10_000_000, 10_000_000
    rng = np.random.default_rng(3)
    vals = rng.integers(-1000, 1000, hot + n_small).astype(np.int64)
    offsets = np.concatenate([[0], [hot], hot + np.arange(1, n_small + 1)]).astype(np.int32)
    lc = rdf.ListColumn.upload([rdf.ListArray(rdf.I64, offsets, None, 0, n_small + 1, 0, rdf.PrimitiveArray.from_numpy(vals))], ctx)
    idx = np.arange(n_small, -1, -1, dtype=np.uint32)
    got = lc.take(rdf.Column.upload([rdf.PrimitiveArray.from_numpy(idx)], ctx)).download()[0]
    assert np.array_equal(got.offsets[-2:], [n_small, n_small + hot])
    v = got.values.value_slice()
    assert np.array_equal(v[:n_small], vals[hot:][::-1]) and np.array_equal(v[n_small:], vals[:hot])


def test_errors_leak_nothing(rdf, ctx):
    lc = rdf.ListColumn.upload([rdf.ListArray.from_pylist(rdf.I32, [[1, 2], [], None]), rdf.ListArray.from_pylist(rdf.I32, [[3]])], ctx)
    idx = u32_col(rdf, ctx, [0, 4])
    mask = bool_col(rdf, ctx, [[True, False, True]])
    ctx.synchronize()
    before = pool_used(ctx)
    with pytest.raises(rdf.ComputeError):   # BDF_INVALID: index past the end
        lc.take(idx)
    with pytest.raises(rdf.ComputeError):   # BDF_LENGTH_MISMATCH: one mask chunk for two list chunks
        lc.filter(mask)
    r = lc.take(u32_col(rdf, ctx, [3, None, 2]))
    assert r.download()[0].to_pylist() == [[3], None, None]
    r.free()
    ctx.synchronize()
    assert pool_used(ctx) == before
    fleet = rdf.Context.multi(1)
    lib = rdf.native.lib()
    import ctypes as C
    h = C.c_void_p()
    assert lib.bdf_list_take_dev(fleet.handle, lc.handle, idx.handle, C.byref(h)) == rdf.native.UNSUPPORTED


def _key_col(rng, dt, n, n_distinct, null_frac=0.05):
    vals = rng.integers(0, n_distinct, n).astype(NP[dt])
    return vals, rng.random(n) < null_frac


def _pylist(vals, mask):
    return [None if m else v for v, m in zip(vals.tolist() if vals.dtype.kind != "f" else list(vals), mask)]


def _check_collect(rdf, ctx, keys_np, x_np, dt, chunks=(0.3, 0.0, 0.7)):
    n = len(x_np[0])
    cuts = [0] + [int(round(n * sum(chunks[:i + 1]))) for i in range(len(chunks))]
    up = lambda v, m: rdf.Column.upload([rdf.PrimitiveArray.from_numpy(v[a:b], ~m[a:b]) for a, b in zip(cuts, cuts[1:])], ctx)
    kcols = [up(v, m) for v, m in keys_np]
    xc = up(*x_np)
    keys_py = [_pylist(v, m) for v, m in keys_np]
    x_py = _pylist(*x_np)
    gk, res = rdf.group_by(kcols, [(xc, "collect_list"), (xc, "collect_set"), (xc, "count")])
    want_l, want_s = lfo.collect_list(keys_py, x_py), lfo.collect_set(keys_py, x_py)
    assert isinstance(res[0], rdf.ListColumn) and isinstance(res[1], rdf.ListColumn) and isinstance(res[2], rdf.Column)
    got_l, got_s = res[0].download(), res[1].download()
    assert len(got_l) == 1 and len(got_s) == 1
    assert lists_bits(got_l[0].to_pylist(), dt) == lists_bits([l for _, l in want_l], dt)
    assert lists_bits(got_s[0].to_pylist(), dt) == lists_bits([l for _, l in want_s], dt)
    assert res[0].chunk_info(0)["null_count"] == 0 and res[1].chunk_info(0)["null_count"] == 0
    for k, col in enumerate(gk):
        assert col.download()[0].to_pylist() == [key[k] for key, _ in want_l]


@pytest.mark.parametrize("dt", range(10))
def test_collect_against_the_oracle(rdf, ctx, dt):
    rng = np.random.default_rng(200 + dt)
    n = 5000
    if dt >= 8:
        pool = np.array([0.0, -0.0, np.nan, 1.5, -2.0, 3.0, np.inf], dtype=NP[dt])
        xv = pool[rng.integers(0, len(pool), n)]
    else:
        xv = rng.integers(0, 40, n).astype(NP[dt])
    xm = rng.random(n) < 0.2
    kv, km = _key_col(rng, 2, n, 300)
    xm[kv == 7] = True   # an all-null group
    kv[:3] = 1000        # one-row groups
    kv[:3] += np.arange(3, dtype=kv.dtype)
    _check_collect(rdf, ctx, [(kv, km)], (xv, xm), dt)


@pytest.mark.parametrize("n_keys", [2, 16])
def test_collect_with_many_keys(rdf, ctx, n_keys):
    rng = np.random.default_rng(n_keys)
    n = 4000
    keys = [_key_col(rng, 2 if k % 2 == 0 else 9, n, 3 if n_keys == 16 else 20) for k in range(n_keys)]
    xv, xm = rng.integers(-50, 50, n).astype(np.int64), rng.random(n) < 0.1
    _check_collect(rdf, ctx, keys, (xv, xm), 3)


def test_collect_mixed_with_other_aggregates_sorts_once_per_collect_set_column(rdf, ctx):
    N = rdf.native
    rng = np.random.default_rng(5)
    n = 10000
    k = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(rng.integers(0, 100, n).astype(np.int32))], ctx)
    x = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(rng.normal(size=n), rng.random(n) > 0.1)], ctx)
    y = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(rng.integers(0, 9, n).astype(np.int16))], ctx)
    ctx.synchronize()
    ctx.profile_enable(True)
    _, res = rdf.group_by([k], [(x, "sum"), (x, "collect_list"), (y, "collect_set"), (x, "count"), (y, "first"), (y, "collect_set"),
                                (x, "collect_set")])
    recs = ctx.profile_read()
    ctx.profile_enable(False)
    sorts = [r for r in recs if r["kernel"] == N.KERNEL_NAMES[N.K_SORT]]
    assert len(sorts) == 1 + 2   # the key sort, then one second sort for y and one for x
    kinds = [type(r).__name__ for r in res]
    assert kinds == ["Column", "ListColumn", "ListColumn", "Column", "Column", "ListColumn", "ListColumn"]
    assert down_chunks(res[2]) == down_chunks(res[5])
    with pytest.raises(rdf.UnsupportedType):   # the entry without list outputs does not know the ids
        import ctypes as C
        aggs = (N.GroupAggC * 1)()
        aggs[0].column, aggs[0].function = x.handle.value if isinstance(x.handle, C.c_void_p) else x.handle, N.GROUP_COLLECT_LIST
        hk, out, ng = (C.c_void_p * 1)(), (C.c_void_p * 1)(), C.c_int64()
        N.raise_for_status(N.lib().bdf_group_by_dev(ctx.handle, 1, (C.c_void_p * 1)(k.handle), 1, aggs, hk, out, C.byref(ng)))
    t = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.arange(n, dtype=np.int32))], ctx).with_temporal(rdf.TemporalType.date32())
    with pytest.raises(rdf.UnsupportedType):
        rdf.group_by([k], [(t, "collect_list")])


def _frame(rdf, ctx, rng, lens):
    """Two list columns and two numeric columns with the same chunks, and the pyarrow table of the same data."""
    la = [make_chunk(rng, 3, n, sliced=True) for n in lens]
    lens = [len(a) for a in la]   # a slice is shorter than n
    lb = [make_chunk(rng, 9, n) for n in lens]
    k = [pa.array(rng.integers(0, 20, n).astype(np.int32), mask=rng.random(n) < 0.05) for n in lens]
    x = [pa.array(rng.normal(size=n)) for n in lens]
    frame = rdf.DeviceFrame.from_host({"k": [rdf.PrimitiveArray.from_arrow(a) for a in k], "x": [rdf.PrimitiveArray.from_arrow(a) for a in x]}, ctx=ctx)
    frame = frame.with_column("tags", upload(rdf, ctx, la)).with_column("w", upload(rdf, ctx, lb))
    table = pa.Table.from_batches([pa.record_batch([a, b, c, d], names=["k", "x", "tags", "w"]) for a, b, c, d in zip(k, x, la, lb)])
    return frame, table


def _as_table(frame):
    base = frame.columns and __import__("rust_dataframe_b200").native.LIST_BASE
    cols = {}
    for (name, chunks), dt in zip(frame.to_host().items(), frame.schema.values()):
        typ = pa.list_(PA[dt - base]) if dt >= base else PA[dt]
        cols[name] = pa.array(sum((c.to_pylist() for c in chunks), []), typ)
    return pa.table(cols)


def _same(got, want):
    assert got.column_names == want.column_names
    for name in want.column_names:
        g, w = got[name].to_pylist(), want[name].to_pylist()
        if pa.types.is_list(want.schema.field(name).type) and pa.types.is_floating(want.schema.field(name).type.value_type):
            dt = 9
            assert lists_bits(g, dt) == lists_bits(w, dt), name
        else:
            assert [None if v is None or (isinstance(v, float) and math.isnan(v)) else v for v in g] == \
                   [None if v is None or (isinstance(v, float) and math.isnan(v)) else v for v in w], name


def test_frames_carry_list_columns(rdf, ctx):
    import pyarrow.compute as pc
    from rust_dataframe_b200 import frame as F

    rng = np.random.default_rng(9)
    frame, table = _frame(rdf, ctx, rng, (100, 0, 333, 7))
    assert frame.schema["tags"] == rdf.native.LIST_BASE + rdf.I64 and frame.schema["w"] == rdf.native.LIST_BASE + rdf.F64
    # filter keeps the chunks, on a comparison of a numeric column
    got = frame.filter(("gt", F.col("x"), F.lit(0.0)))
    assert [got.columns["tags"].chunk_info(i)["len"] for i in range(4)] == [got.columns["k"].chunk_info(i)["len"] for i in range(4)]
    _same(_as_table(got), table.filter(pc.greater(table["x"], 0.0)))
    # sort (stable, nulls last) = take by the sort's permutation
    got = frame.sort([("k", False)])
    order = pc.sort_indices(table, [("k", "ascending")], null_placement="at_end")
    _same(_as_table(got), table.take(order))
    _same(_as_table(frame.limit(50)), table.slice(0, 50))
    _same(_as_table(frame.select(["tags", "x"])), table.select(["x", "tags"]))
    # a LEFT join: a right row without a partner gives NULL lists
    right = rdf.DeviceFrame.from_host({"k2": [rdf.PrimitiveArray.from_numpy(np.arange(0, 10, dtype=np.int32))]}, ctx=ctx)
    right = right.with_column("r", rdf.ListColumn.upload([rdf.ListArray.from_pylist(rdf.I32, [[i] * (i % 3) for i in range(10)])], ctx))
    got = frame.join(right, [("k", "k2")], "left")
    host = _as_table(got)
    kk = host["k"].to_pylist()
    assert host["r"].to_pylist() == [[k] * (k % 3) if k is not None and k < 10 else None for k in kk]
    # window leaves the list columns untouched
    w = frame.window(["k"], [("x", False)], [("rn", "row_number")])
    _same(_as_table(w).select(["tags", "w"]), table.select(["tags", "w"]))
    # refusals before any device work
    for bad in (lambda: frame.sort([("tags", False)]), lambda: frame.filter(("gt", F.col("tags"), F.lit(1.0))),
                lambda: frame.evaluate([F.calculate("add", ["tags", "x"], "y")]), lambda: frame.aggregate(["tags"], [("sum", ["x"])]),
                lambda: frame.aggregate(["k"], [("sum", ["tags"])]), lambda: frame.join(frame, [("tags", "tags")], "inner"),
                lambda: frame.window(["tags"], [], [("r", "row_number")])):
        with pytest.raises(rdf.UnsupportedType):
            bad()


def test_to_arrow_writes_lists(rdf, ctx, tmp_path):
    rng = np.random.default_rng(13)
    frame, table = _frame(rdf, ctx, rng, (64, 0, 1000, 3))
    rows = [frame.columns["k"].chunk_info(i)["len"] for i in range(4)]
    path = str(tmp_path / "lists.arrow")
    frame.to_arrow(path)
    back = pa.ipc.open_file(path).read_all()
    back.validate(full=True)
    assert back.schema.field("tags").type == pa.list_(pa.field("item", pa.int64()))
    _same(back, table)
    reader = pa.ipc.open_file(path)
    assert [reader.get_batch(i).num_rows for i in range(reader.num_record_batches)] == rows   # list chunk b = batch b
    with rdf.IpcFile(path) as f:
        cols = f.read(["tags", "w"], ctx=ctx)
        for name, dt in (("tags", 3), ("w", 9)):
            got = sum((ch.to_pylist() for ch in cols[name].download()), [])
            assert lists_bits(got, dt) == lists_bits(table[name].to_pylist(), dt)
    # a group-by result written straight away
    k = frame.columns["k"]
    gk, res = rdf.group_by([k], [(frame.columns["x"], "collect_list")])
    out = rdf.DeviceFrame({"k": gk[0], "xs": res[0]})
    out.to_arrow(str(tmp_path / "g.arrow"))
    pa.ipc.open_file(str(tmp_path / "g.arrow")).read_all().validate(full=True)


def test_csv_and_parquet_refuse_lists(rdf, ctx, tmp_path):
    rng = np.random.default_rng(17)
    frame, _ = _frame(rdf, ctx, rng, (10,))
    for write, name in ((frame.to_csv, "f.csv"), (frame.to_parquet, "f.parquet")):
        p = str(tmp_path / name)
        with pytest.raises(rdf.UnsupportedType):
            write(p)
        assert not os.path.exists(p)
