"""DataFrame::to_parquet on the device: files written by bdf_parquet_write read back by pyarrow.parquet and by this library's own reader,
bit for bit (floats as bits: -0.0 and NaN payloads), over every numeric, Boolean and temporal type, null fractions, writer options and
chunk layouts (odd chunk lengths, Arrow arrays with an offset, filter and take outputs); the metadata the rules promise (row groups,
codec, dictionary pages, encodings, statistics); dictionary edge cases; the reference's to_parquet data; read/write loops; a
multi-block frame; a fixed launch count; zero rows; and the refusals, which leave an existing file untouched."""
import base64
import os

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pyarrow.csv as pacsv
import pyarrow.parquet as pq
import pytest

import parquet_helpers as H
from helpers import pool_used

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "uk_cities_with_headers.csv")

N_ROWS = 5000
NUMERIC = [pa.int8(), pa.int16(), pa.int32(), pa.int64(), pa.uint8(), pa.uint16(), pa.uint32(), pa.uint64(), pa.float32(), pa.float64()]
TEMPORAL = ([pa.date32(), pa.date64(), pa.time32("s"), pa.time32("ms"), pa.time64("us"), pa.time64("ns")] +
            [pa.timestamp(u, tz=tz) for u in ("s", "ms", "us", "ns") for tz in (None, "UTC", "+01:00")])
TYPES = NUMERIC + [pa.bool_()] + TEMPORAL
OPTIONS = {"defaults": {}, "snappy": {"compression": "snappy"}, "plain": {"dictionary": False}, "rg1000": {"row_group_rows": 1000}}
LAYOUTS = ["one", "1024", "odd", "offset", "filter", "take"]


def _values(t: pa.DataType, n: int, rng) -> pa.Array:
    """Values with repeats (so dictionaries form), extremes, and for floats -0.0, NaN payloads and infinities."""
    if pa.types.is_boolean(t):
        return pa.array(rng.integers(0, 2, n).astype(bool))
    if pa.types.is_floating(t):
        np_t = np.float32 if t == pa.float32() else np.float64
        v = np.round(rng.normal(size=n) * 10).astype(np_t)
        special = np.array([0.0, -0.0, np.inf, -np.inf, np.nan], dtype=np_t)
        v[rng.integers(0, n, n // 20)] = special[rng.integers(0, 5, n // 20)]
        bits = v.view(np.uint32 if np_t == np.float32 else np.uint64)
        bits[:3] = [0x7FC00001, 0xFFC00002, 0x7FF00000 + 5] if np_t == np.float32 else [0x7FF8000000000001, 0xFFF8000000000002, 0x7FF0000000000005]
        return pa.array(v)
    if pa.types.is_integer(t):
        info = np.iinfo(t.to_pandas_dtype())
        v = rng.integers(info.min, info.max, n, dtype=t.to_pandas_dtype(), endpoint=True)
        v[: n // 2] = v[: n // 2] % 97   # half of them from a small set
        v[2], v[3] = info.min, info.max
        return pa.array(v, type=t)
    phys = pa.int32() if t.bit_width == 32 else pa.int64()
    if pa.types.is_date64(t):   # whole days, as Arrow's Date64 holds them (a day's remainder would not survive DATE)
        v = rng.integers(-10 ** 7, 10 ** 7, n) * 86400000
    elif pa.types.is_time32(t):
        v = rng.integers(0, 86400 * (1 if t.unit == "s" else 1000), n)
    elif pa.types.is_time64(t):
        v = rng.integers(0, 86400 * (10 ** 6 if t.unit == "us" else 10 ** 9), n)
    elif pa.types.is_timestamp(t):
        lim = {"s": 10 ** 10, "ms": 10 ** 13, "us": 10 ** 16, "ns": 10 ** 18}[t.unit]
        v = rng.integers(-lim, lim, n)
    else:
        v = rng.integers(-10 ** 6, 10 ** 6, n)
    v[: n // 3] = v[: n // 3] % 50
    return pa.array(v.astype(phys.to_pandas_dtype()), type=phys).cast(t)


def _with_nulls(arr: pa.Array, frac: float, rng) -> pa.Array:
    if frac == 0:
        return arr
    mask = rng.random(len(arr)) < frac
    return pc.if_else(pa.array(mask), pa.nulls(len(arr), arr.type), arr)


def _chunks(arr: pa.Array, layout: str):
    n = len(arr)
    if layout == "one":
        return [arr]
    if layout == "1024":
        return [arr.slice(s, 1024) for s in range(0, n, 1024)]
    if layout in ("odd", "filter", "take"):
        cuts, s, k = [], 0, 0
        while s < n:
            ln = [7, 0, 1999, 1, 3333][k % 5]
            cuts.append(arr.slice(s, min(ln, n - s)))
            s += ln
            k += 1
        return cuts
    assert layout == "offset"   # arrays that start mid-byte: sliced from a longer array
    pad = pa.concat_arrays([_values(arr.type, 13, np.random.default_rng(0)), arr])
    return [pad.slice(13 + s, 1500) for s in range(0, n, 1500)]


def _to_host(a: pa.Array, rdf):
    if pa.types.is_boolean(a.type):
        vbuf, dbuf = a.buffers()
        bits = np.frombuffer(dbuf, dtype=np.uint8)
        valid = np.frombuffer(vbuf, dtype=np.uint8) if vbuf is not None else None
        return rdf.BooleanArray(bits, valid, a.offset, len(a), a.null_count if vbuf is not None else 0, keepalive=a)
    return rdf.PrimitiveArray.from_arrow(a)


def _device_column(rdf, ctx, arr: pa.Array, layout: str, rng):
    """(device Column, the Arrow array it holds)."""
    col = rdf.Column.upload([_to_host(c, rdf) for c in _chunks(arr, layout)], ctx=ctx,
                            dtype=10 if pa.types.is_boolean(arr.type) else None)
    col.temporal = rdf.TemporalType.from_arrow(arr.type)
    if layout == "filter":
        keep = rng.random(len(arr)) < 0.6
        mask = rdf.Column.upload([_to_host(c, rdf) for c in _chunks(pa.array(keep), "odd")], ctx=ctx, dtype=10)
        out = col.filter(mask)
        out.temporal = col.temporal
        return out, arr.filter(pa.array(keep))
    if layout == "take":
        idx = rng.integers(0, len(arr), 3000).astype(np.uint32)
        out = col.take(rdf.Column.upload([rdf.PrimitiveArray.from_numpy(idx)], ctx=ctx))
        out.temporal = col.temporal
        return out, arr.take(pa.array(idx))
    return col, arr


def _bits(a) -> tuple:
    """(values as unsigned bits with nulls zeroed, validity) of an Arrow array; temporal values as their integers."""
    a = a.combine_chunks() if isinstance(a, pa.ChunkedArray) else a
    valid = np.asarray(a.is_valid())
    if pa.types.is_boolean(a.type):
        return np.where(valid, np.asarray(pc.fill_null(a, False)), False).astype(np.uint64), valid
    if pa.types.is_temporal(a.type):
        a = a.cast(pa.int32() if a.type.bit_width == 32 else pa.int64())
    v = np.asarray(pc.fill_null(a, pa.scalar(0).cast(a.type)) if a.null_count else a)
    v = v.view(f"u{v.dtype.itemsize}").astype(np.uint64)
    return np.where(valid, v, 0), valid


def _stored(t: pa.DataType, a: pa.Array) -> pa.Array:
    """What this library's reader gives for a column of type t: Date64 as Date32 days, Time32(s) and Timestamp(s) as milliseconds."""
    if pa.types.is_date64(t):
        return pa.array(np.floor_divide(np.asarray(a.cast(pa.int64()).fill_null(0)), 86400000).astype(np.int32), mask=~np.asarray(a.is_valid()))
    if (pa.types.is_time32(t) or pa.types.is_timestamp(t)) and t.unit == "s":
        phys = pa.int32() if pa.types.is_time32(t) else pa.int64()
        v = np.asarray(a.cast(phys).fill_null(0)).astype(phys.to_pandas_dtype()) * 1000
        return pa.array(v, type=phys, mask=~np.asarray(a.is_valid()))
    return a


def _frame(rdf, ctx, layout, null_frac, seed=0, types=TYPES, n=N_ROWS):
    rng = np.random.default_rng(seed)
    cols, want = {}, {}
    for k, t in enumerate(types):
        if layout == "filter" and pa.types.is_boolean(t):
            continue   # the filter kernel takes no Boolean values (the take layout covers a gathered Boolean column)
        arr = _with_nulls(_values(t, n, rng), null_frac, rng)
        col, exp = _device_column(rdf, ctx, arr, layout, np.random.default_rng(seed + 1))   # the same rows kept in every column
        cols[f"c{k}"] = col
        want[f"c{k}"] = exp
    return cols, want


def _check_file(rdf, ctx, path, want):
    """pyarrow reads the file as it reads its own file of the same table, bit for bit; the ARROW:schema entry holds the Arrow types;
    this library's reader gives the stored values."""
    ref = str(path) + ".pyarrow.parquet"
    pq.write_table(pa.table(want), ref)
    expect = pq.read_table(ref)
    got = pq.read_table(path)
    assert got.column_names == list(want)
    for name in want:
        g, e = got.column(name), expect.column(name)
        assert g.type == e.type, name
        gv, gm = _bits(g)
        ev, em = _bits(e)
        assert np.array_equal(gm, em) and np.array_equal(gv, ev), name
    entry = pq.ParquetFile(path).metadata.metadata[b"ARROW:schema"]
    schema = pa.ipc.read_schema(pa.py_buffer(base64.b64decode(entry)))
    assert schema.names == list(want) and [f.type for f in schema] == [a.type for a in want.values()]
    if got.num_rows == 0:
        return
    with rdf.ParquetFile(path, batch_size=1 << 20) as f:
        cols = f.read(list(want), ctx=ctx)
        for name, exp in want.items():
            chunks = cols[name].download()
            gv = np.concatenate([np.asarray(c.value_bits() if hasattr(c, "value_bits") else c.value_slice().view(f"u{c.value_slice().dtype.itemsize}")).astype(np.uint64)
                                 for c in chunks])
            gm = np.concatenate([np.asarray(c.valid_mask(), dtype=bool) for c in chunks])
            ev, em = _bits(_stored(exp.type, exp))
            assert np.array_equal(gm, em) and np.array_equal(np.where(gm, gv, 0), ev), name


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("opt", list(OPTIONS))
@pytest.mark.parametrize("null_frac", [0.0, 0.1, 1.0])
def test_round_trip_matrix(rdf, ctx, tmp_path, layout, opt, null_frac):
    cols, want = _frame(rdf, ctx, layout, null_frac, seed=LAYOUTS.index(layout))
    p = str(tmp_path / "t.parquet")
    rdf.write_parquet(p, cols, **OPTIONS[opt])
    _check_file(rdf, ctx, p, want)
    md = pq.ParquetFile(p).metadata
    n = len(next(iter(want.values())))
    if opt == "rg1000":
        assert [md.row_group(g).num_rows for g in range(md.num_row_groups)] == [min(1000, n - s) for s in range(0, n, 1000)]
    else:
        lens = [len(c) for c in _chunks(pa.array(np.zeros(N_ROWS)), layout)] if layout not in ("filter", "take") else None
        if lens is not None:
            assert [md.row_group(g).num_rows for g in range(md.num_row_groups)] == [x for x in lens if x]
    for g in range(md.num_row_groups):
        for i, t in enumerate(want[k].type for k in want):
            cm = md.row_group(g).column(i)
            assert cm.compression == ("SNAPPY" if opt == "snappy" else "UNCOMPRESSED")
            st = cm.statistics
            assert st is not None and st.has_null_count
            if st.null_count == cm.num_values:   # no valid value: no dictionary and no min / max
                assert not cm.has_dictionary_page and not st.has_min_max and st.null_count == cm.num_values
            elif opt == "plain" or pa.types.is_boolean(t):
                assert not cm.has_dictionary_page and "PLAIN_DICTIONARY" not in cm.encodings
            else:
                assert cm.has_dictionary_page and "PLAIN_DICTIONARY" in cm.encodings


@pytest.mark.parametrize("null_frac", [0.0, 0.3])
def test_statistics_equal_numpy(rdf, ctx, tmp_path, null_frac):
    rng = np.random.default_rng(3)
    cols, want = {}, {}
    for k, t in enumerate(NUMERIC):
        arr = _with_nulls(_values(t, 4000, rng), null_frac, rng)
        if t in (pa.uint32(), pa.uint64()):   # values above 2^31 / 2^63 must order as unsigned
            v = np.asarray(arr.fill_null(0)).copy()
            v[5] = np.iinfo(v.dtype).max - 3
            arr = pa.array(v, type=t, mask=~np.asarray(arr.is_valid()))
        cols[f"c{k}"], want[f"c{k}"] = _device_column(rdf, ctx, arr, "1024", rng)
    p = str(tmp_path / "s.parquet")
    rdf.write_parquet(p, cols, row_group_rows=1500)
    md = pq.ParquetFile(p).metadata
    for i, (name, arr) in enumerate(want.items()):
        for g in range(md.num_row_groups):
            part = arr.slice(g * 1500, 1500)
            v = np.asarray(part.drop_null())
            if v.dtype.kind == "f":
                v = v[~np.isnan(v)]
            st = md.row_group(g).column(i).statistics
            assert st.null_count == part.null_count
            assert st.min == v.min() and st.max == v.max(), name


def test_float_dictionary_keeps_bits(rdf, ctx, tmp_path):
    nan1, nan2 = np.array([0x7FF8000000000001, 0xFFF8000000000007], dtype=np.uint64).view(np.float64)
    v = np.array([0.0, -0.0, nan1, nan2, 0.0, -0.0, nan2, nan1] * 100)
    col = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(v)], ctx=ctx)
    p = str(tmp_path / "d.parquet")
    rdf.write_parquet(p, {"x": col})
    pages = H.chunk_pages(p, 0)
    assert pages[0][0][1] == 2 and pages[0][0][7][1] == 4   # a dictionary page of 4 entries
    got = np.asarray(pq.read_table(p).column("x").combine_chunks()).view(np.uint64)
    assert np.array_equal(got, v.view(np.uint64))
    st = pq.ParquetFile(p).metadata.row_group(0).column(0).statistics
    assert np.signbit(st.min) and not np.signbit(st.max) and st.min == 0 and st.max == 0


def test_dictionary_fallback_and_size(rdf, ctx, tmp_path):
    big = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.arange(1 << 18, dtype=np.float64) * 1.5)], ctx=ctx)
    p = str(tmp_path / "big.parquet")
    rdf.write_parquet(p, {"x": big})
    cm = pq.ParquetFile(p).metadata.row_group(0).column(0)
    assert not cm.has_dictionary_page and "PLAIN_DICTIONARY" not in cm.encodings
    assert np.array_equal(pq.read_table(p).column("x").to_numpy(), np.arange(1 << 18) * 1.5)
    v = np.random.default_rng(1).integers(0, 50, 200_000).astype(np.int64)
    small = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(v)], ctx=ctx)
    pd_, pp = str(tmp_path / "dict.parquet"), str(tmp_path / "plain.parquet")
    rdf.write_parquet(pd_, {"x": small})
    rdf.write_parquet(pp, {"x": small}, dictionary=False)
    dsz = pq.ParquetFile(pd_).metadata.row_group(0).column(0).total_compressed_size
    psz = pq.ParquetFile(pp).metadata.row_group(0).column(0).total_compressed_size
    assert dsz < psz / 4
    assert np.array_equal(pq.read_table(pd_).column("x").to_numpy(), v)


def test_reference_to_parquet(rdf, ctx, tmp_path):
    """The reference's test_parquet_io: uk_cities CSV, lat + lng as lat_lng_sum, to_parquet; the Utf8 city is left out by from_csv."""
    fr = rdf.DeviceFrame.from_csv(GOLDEN, ctx=ctx)
    fr = fr.with_column("lat_lng_sum", fr.column("lat").add(fr.column("lng")))
    p = str(tmp_path / "uk.parquet")
    fr.to_parquet(p)
    got = pq.read_table(p)
    t = pacsv.read_csv(GOLDEN)
    for n in ("lat", "lng"):
        assert np.array_equal(got.column(n).to_numpy(), t.column(n).to_numpy()), n
    assert np.array_equal(got.column("lat_lng_sum").to_numpy(), t.column("lat").to_numpy() + t.column("lng").to_numpy())


def test_loops_and_determinism(rdf, ctx, tmp_path):
    src = str(tmp_path / "src.parquet")
    t = H.table(7000, seed=9, null_frac=0.1)
    pq.write_table(t, src, row_group_size=3000)
    fr = rdf.DeviceFrame.from_parquet(src, batch_size=2048, ctx=ctx)
    a, b = str(tmp_path / "a.parquet"), str(tmp_path / "b.parquet")
    fr.to_parquet(a, compression="snappy")
    fr.to_parquet(b, compression="snappy")
    assert open(a, "rb").read() == open(b, "rb").read()
    got = pq.read_table(a)
    for n in fr.columns:
        want = t.column(n)
        if pa.types.is_date64(want.type) or (pa.types.is_temporal(want.type) and getattr(want.type, "unit", "") == "s"):
            continue   # the reader's documented unit departures
        gv, gm = _bits(got.column(n))
        ev, em = _bits(want)
        assert np.array_equal(gm, em) and np.array_equal(gv, ev), n


def test_three_blocks(rdf, ctx, tmp_path):
    n = 30_000_000
    rng = np.random.default_rng(5)
    a = np.arange(n, dtype=np.int64)
    b = np.round(rng.normal(size=n), 2)
    c = rng.integers(0, 1000, n).astype(np.int32)
    chunk = 1 << 22
    cols = {k: rdf.Column.upload([rdf.PrimitiveArray.from_numpy(v[s:s + chunk]) for s in range(0, n, chunk)], ctx=ctx)
            for k, v in (("a", a), ("b", b), ("c", c))}
    p = str(tmp_path / "big.parquet")
    rdf.write_parquet(p, cols, compression="snappy")
    got = pq.read_table(p)
    assert np.array_equal(got.column("a").to_numpy(), a)
    assert np.array_equal(got.column("b").to_numpy().view(np.uint64), b.view(np.uint64))
    assert np.array_equal(got.column("c").to_numpy(), c)


def test_launch_count_is_fixed(rdf, ctx, tmp_path):
    cols, _ = _frame(rdf, ctx, "one", 0.1, types=[pa.int64(), pa.float64(), pa.bool_()], n=250_000)
    counts = []
    for rg in (0, 1000, 100_000):
        before = ctx.launch_count()
        rdf.write_parquet(str(tmp_path / f"r{rg}.parquet"), cols, row_group_rows=rg)
        counts.append(ctx.launch_count() - before)
    assert counts[0] == counts[1] == counts[2], counts


def test_zero_rows(rdf, ctx, tmp_path):
    col = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.zeros(0, dtype=np.int32))], ctx=ctx)
    ts = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.zeros(0, dtype=np.int64))], ctx=ctx)
    ts.temporal = rdf.TemporalType.timestamp("us", "UTC")
    p = str(tmp_path / "empty.parquet")
    rdf.write_parquet(p, {"x": col, "t": ts})
    assert pq.ParquetFile(p).metadata.num_row_groups == 0
    t = pq.read_table(p)
    assert t.num_rows == 0 and t.schema.field("x").type == pa.int32() and t.schema.field("t").type == pa.timestamp("us", tz="UTC")
    with pytest.raises(rdf.ReferencePanic):
        rdf.ParquetFile(p)


def test_refusals_leave_the_file(rdf, ctx, tmp_path):
    p = tmp_path / "keep.parquet"
    p.write_bytes(b"existing contents")
    a = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.arange(10, dtype=np.int64))], ctx=ctx)
    b = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.arange(4, dtype=np.int64)),
                           rdf.PrimitiveArray.from_numpy(np.arange(6, dtype=np.int64))], ctx=ctx)
    bad = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.arange(10, dtype=np.int32))], ctx=ctx)
    lst = rdf.ListColumn.upload([rdf.ListArray.from_arrow(pa.array([[1, 2], [3]], type=pa.list_(pa.int64())))], ctx=ctx)
    flag = rdf.Column.upload([rdf.BooleanArray.from_numpy(np.arange(10) % 2 == 0)], ctx=ctx, dtype=10)
    many = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.zeros((1 << 20) + 1, dtype=np.int8))], ctx=ctx)
    ctx.synchronize()
    used = pool_used(ctx)
    with pytest.raises(rdf.ComputeError, match="different length"):   # BDF_LENGTH_MISMATCH
        rdf.write_parquet(str(p), {"a": a, "b": b})
    for kw in ({"compression": "gzip"},):
        with pytest.raises(ValueError):
            rdf.write_parquet(str(p), {"a": a}, **kw)
    with pytest.raises(rdf.ComputeError, match="row_group_rows"):
        rdf.write_parquet(str(p), {"a": a}, row_group_rows=-1)
    bad.temporal = rdf.TemporalType.timestamp("us")   # an Int32 column cannot hold a Timestamp
    with pytest.raises(rdf.ComputeError, match="temporal"):
        rdf.write_parquet(str(p), {"a": bad})
    bad.temporal = rdf.TemporalType(4, 3)             # Time32(ns) does not exist
    with pytest.raises(rdf.ComputeError, match="does not take time unit"):
        rdf.write_parquet(str(p), {"a": bad})
    flag.temporal = rdf.TemporalType.date32()         # a Boolean column cannot hold a Date
    with pytest.raises(rdf.ComputeError, match="does not hold temporal kind"):
        rdf.write_parquet(str(p), {"a": flag})
    with pytest.raises(rdf.ComputeError, match="column chunks"):   # 2^20 + 1 row groups of one row
        rdf.write_parquet(str(p), {"a": many}, row_group_rows=1)
    with pytest.raises(rdf.UnsupportedType):
        rdf.write_parquet(str(p), {"a": lst})
    assert p.read_bytes() == b"existing contents"
    with pytest.raises(rdf.ComputeError, match="cannot create"):
        rdf.write_parquet(str(tmp_path / "no" / "such" / "dir.parquet"), {"a": a})
    ctx.synchronize()
    assert pool_used(ctx) == used
    m = rdf.Context.multi(0)
    try:
        col = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.arange(10, dtype=np.int64))], ctx=m)
        with pytest.raises(rdf.UnsupportedType, match="one GPU"):
            rdf.write_parquet(str(p), {"a": col})
    finally:
        m.close()
    assert p.read_bytes() == b"existing contents"


def _serial_snappy(tmp_path):
    """The host build of parquet_encode.cuh's serial snappy_fragment (test_parquet_write.py's driver), or None without g++."""
    import shutil
    import subprocess

    from test_parquet_write import CSRC, DRIVER

    gxx = shutil.which("g++")
    if gxx is None:
        return None
    (tmp_path / "drv.cpp").write_text(DRIVER)
    exe = str(tmp_path / "pqenc")
    subprocess.check_call([gxx, "-std=c++17", "-O2", "-I", CSRC, str(tmp_path / "drv.cpp"), "-o", exe])

    def run(body: bytes) -> bytes:
        (tmp_path / "in").write_bytes(body)
        subprocess.check_call([exe, "z", str(tmp_path / "in"), str(tmp_path / "out")], stdout=subprocess.DEVNULL)
        return (tmp_path / "out").read_bytes()
    return run


def test_multi_page_dictionary_chunks_with_nulls(rdf, ctx, tmp_path):
    """Chunks of two data pages (2^17 rows, then the rest) with nulls and dictionaries (ids across the tiles of later pages, mixed level pages); row groups
    that keep a dictionary between row groups that fall back to PLAIN (the kept ids and entries are compacted); statistics of the
    converted temporal values; and every snappy page body equal to the serial snappy_fragment's stream of the uncompressed body."""
    n, rg = 330_000, 165_000
    rng = np.random.default_rng(21)
    valid = rng.random(n) > 0.1
    low = rng.integers(0, 300, n)
    # row group 0: low cardinality (a dictionary); row group 1: 165 000 distinct Float64 values (1.3 MB of entries: PLAIN)
    f = np.where(np.arange(n) < rg, low / 8.0, np.arange(n) * 1.25)
    arrays = {
        "i64": pa.array(low * 1_000_003, mask=~valid),
        "f64": pa.array(f, mask=~valid),
        "d64": pa.array((low - 150) * 86400000, mask=~valid).cast(pa.date64()),
        "t32s": pa.array((low * 97).astype(np.int32), mask=~valid).cast(pa.time32("s")),
        "tss": pa.array(low * 1_000_000_007 - 10 ** 11, mask=~valid).cast(pa.timestamp("s", tz="UTC")),
    }
    cols = {k: _device_column(rdf, ctx, a, "odd", rng)[0] for k, a in arrays.items()}
    pn, ps = str(tmp_path / "n.parquet"), str(tmp_path / "s.parquet")
    rdf.write_parquet(pn, cols, row_group_rows=rg)
    rdf.write_parquet(ps, cols, row_group_rows=rg, compression="snappy")
    for p in (pn, ps):
        _check_file(rdf, ctx, p, arrays)
    md = pq.ParquetFile(pn).metadata
    assert md.num_row_groups == 2
    for i, name in enumerate(arrays):
        for g in range(2):
            cm = md.row_group(g).column(i)
            assert cm.has_dictionary_page == (name != "f64" or g == 0), (name, g)
            part = _stored(arrays[name].type, arrays[name].slice(g * rg, rg))
            m = np.asarray(part.is_valid())
            vals = np.asarray(part.drop_null())   # the stored physical values: days, milliseconds
            st = cm.statistics
            assert st.null_count == int((~m).sum())
            assert st.min_raw == vals.min() and st.max_raw == vals.max(), (name, g)
    # a chunk of the snappy file has the same pages as the uncompressed one, each body the serial compressor's stream of it
    serial = _serial_snappy(tmp_path)
    if serial is None:
        pytest.skip("g++ is not installed")
    for i in range(len(arrays)):
        plain, comp = H.chunk_pages(pn, i), H.chunk_pages(ps, i)
        assert len(plain) == len(comp) >= 3
        for (hp, bp), (hs, bs) in zip(plain, comp):
            assert hs[2] == hp[2] == len(bp)   # the uncompressed size
            assert bs == serial(bp)
