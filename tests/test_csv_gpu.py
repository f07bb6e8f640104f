"""DataFrame::from_csv on the device against tests/csv_oracle.py: every value bit for bit, and the same null slots."""
import json
import os
import struct

import numpy as np
import pytest

import csv_oracle as co
from helpers import pool_used

HERE = os.path.dirname(os.path.abspath(__file__))
UK = os.path.join(HERE, "golden", "uk_cities_with_headers.csv")


def _host(col):
    """(values as bit patterns, valid mask, [chunk lengths], [has_validity]) of a device column."""
    chunks = col.download()
    vals, valid, lens, hv = [], [], [], []
    for a in chunks:
        m = a.valid_mask()
        if hasattr(a, "value_bits"):
            v = np.asarray(a.value_bits(), dtype=bool)
        else:
            v = np.asarray(a.value_slice())
            if v.dtype == np.float64:
                v = v.view(np.uint64)
            elif v.dtype == np.float32:
                v = v.view(np.uint32)
        vals.append(v); valid.append(np.asarray(m, dtype=bool)); lens.append(a.length); hv.append(a.validity is not None)
    return np.concatenate(vals) if vals else np.zeros(0), np.concatenate(valid) if valid else np.zeros(0, bool), lens, hv


def _check(rdf, ctx, tmp_path, data: bytes, batch_size=1024, columns=None, **kw):
    p = tmp_path / "t.csv"
    p.write_bytes(data)
    ref = co.read(data, batch_size=batch_size, **kw)
    with rdf.CsvFile(str(p), batch_size=batch_size, ctx=ctx, **kw) as f:
        assert [n for n, _, _ in f.schema] == ref.names
        assert [dt if dt >= 0 else co.UTF8 for _, dt, _ in f.schema] == ref.dtypes
        if kw.get("schema") is None:
            assert [nl for _, _, nl in f.schema] == ref.nullable
        assert f.num_rows == ref.num_rows
        idx = [i for i, dt in enumerate(ref.dtypes) if dt != co.UTF8] if columns is None else columns
        cols = f.read(idx)
        stats = f.stats()
        for i in idx:
            v, m, lens, hv = _host(cols[ref.names[i]])
            rv, rm = ref.column(i)
            assert np.array_equal(m, rm)
            assert np.array_equal(v[m], rv[rm].astype(v.dtype) if v.size else rv[rm])
            n = ref.num_rows
            assert lens == [min(batch_size, n - s) for s in range(0, n, batch_size)]
            nulls = [int((~rm[s:s + batch_size]).sum()) for s in range(0, n, batch_size)]
            assert hv == [k > 0 for k in nulls]
    return ref, stats


@pytest.mark.gpu
def test_uk_cities_reference_asserts(rdf, ctx):
    gold = json.load(open(os.path.join(HERE, "golden", "uk_cities.json")))
    df = rdf.DeviceFrame.from_csv(UK, ctx=ctx)
    assert list(df.schema) == ["lat", "lng"]                        # test_read_csv_to_dataframe: city (Utf8) is skipped
    assert all(dt == rdf.F64 for dt in df.schema.values())
    assert len(df.column("lat")) == 37 and df.column("lat").n_chunks == 1
    lat = np.concatenate([a.value_slice() for a in df.column("lat").download()])
    lng = np.concatenate([a.value_slice() for a in df.column("lng").download()])
    assert lat.view(np.uint64).tolist() == np.array(gold["lat"], np.float64).view(np.uint64).tolist()
    assert lng.view(np.uint64).tolist() == np.array(gold["lng"], np.float64).view(np.uint64).tolist()
    s = df.column("lat").add(df.column("lng"))                     # test_dataframe_ops
    assert s.download()[0].value_slice()[0] == 57.653484 - 3.335724
    assert df.column("lng").unary(rdf.native.ABS).download()[0].value_slice()[0] == 3.335724
    with_cols = df.with_column("lat_lng", s)                        # test_with_columns
    assert list(with_cols.schema) == ["lat", "lng", "lat_lng"]
    total = df.column("lat").sum()
    assert abs(total - 1948.1160980000002) <= 1e-9 * 1948.1160980000002
    with rdf.CsvFile(UK, ctx=ctx) as f:
        assert f.schema == [("city", -1, False), ("lat", rdf.F64, False), ("lng", rdf.F64, False)]
        with pytest.raises(rdf.UnsupportedType):
            f.read(["city"])


def _mixed_file(rng, n, with_nulls=True):
    lines = ["i8,i16,i32,i64,u8,u16,u32,u64,f32,f64,b,s"]
    for r in range(n):
        row = [str(rng.integers(-128, 128)), str(rng.integers(-2 ** 15, 2 ** 15)), str(rng.integers(-2 ** 31, 2 ** 31)),
               str(int(rng.integers(-2 ** 63, 2 ** 63 - 1))), str(rng.integers(0, 256)), str(rng.integers(0, 2 ** 16)),
               str(rng.integers(0, 2 ** 32)), str(int(rng.integers(0, 2 ** 63)) * 2 + 1), repr(float(np.float32(rng.normal() * 10.0 ** rng.integers(-40, 37)))),
               repr(float(rng.normal() * 10.0 ** rng.integers(-300, 300))), ["true", "False", "TRUE"][r % 3], f'"a, ""{r}"""']
        if with_nulls:
            row = [("" if rng.random() < 0.1 and k < 11 else v) for k, v in enumerate(row)]
        lines.append(",".join(row))
    return ("\n".join(lines) + "\n").encode()


@pytest.mark.gpu
def test_every_dtype_explicit_schema(rdf, ctx, tmp_path):
    rng = np.random.default_rng(1)
    data = _mixed_file(rng, 3000)
    schema = list(range(10)) + [co.BOOL, co.UTF8]
    _check(rdf, ctx, tmp_path, data, schema=schema, batch_size=1000)
    _check(rdf, ctx, tmp_path, data, schema=schema[:-1] + [-1], batch_size=7)


@pytest.mark.gpu
@pytest.mark.parametrize("batch", [1, 7, 1000, 1024, 100000])
def test_batch_sizes(rdf, ctx, tmp_path, batch):
    rng = np.random.default_rng(batch)
    lines = ["a,b,c"] + [f"{rng.integers(-9, 9)},{'' if r % 5 == 0 else rng.random()},{'true' if r % 3 else 'false'}" for r in range(2500)]
    _check(rdf, ctx, tmp_path, "\n".join(lines).encode(), batch_size=batch)


@pytest.mark.gpu
def test_edge_bytes(rdf, ctx, tmp_path):
    _check(rdf, ctx, tmp_path, b"a,b\r1,2.5\r\r3,4\r")                                  # \r only, blank lines
    _check(rdf, ctx, tmp_path, b"a,b\r\n1,2.5\r\n\r\n3,4")                              # CRLF, no final newline
    _check(rdf, ctx, tmp_path, b"\xef\xbb\xbfa,b\n1,2\n")                               # BOM: skipped, the name is "a"
    ref, _ = _check(rdf, ctx, tmp_path, b'a,s,b\n1,"multi\nline, field",2\n3,"x""y",4\n')
    assert ref.names == ["a", "s", "b"]
    _check(rdf, ctx, tmp_path, b'a,b\n"1"2,"3"\n4,5\n')                                 # "1"2 -> 12
    _check(rdf, ctx, tmp_path, b'a,b\n1,2\n3,"4')                                       # unterminated quote at end of file
    _check(rdf, ctx, tmp_path, b'a,b\n1,ab"c\n2,x\n')                                   # a quote inside an unquoted field
    _check(rdf, ctx, tmp_path, b"a,b\n1,\n,2.0\n")                                      # a trailing empty field, nulls
    _check(rdf, ctx, tmp_path, b"\n\n\na,b\n1,2\n\n")                                   # leading blank lines
    # without a header the device itself reads field 0, which must skip the leading terminators too
    _check(rdf, ctx, tmp_path, b"\r\n\n1,2\n3,4\n", has_header=False)
    _check(rdf, ctx, tmp_path, b"\r\n1,2\r\n3,4\r\n", has_header=False, schema=[co.I64, co.I64])
    _check(rdf, ctx, tmp_path, b"\r\r\n\ntrue,2.5\n", has_header=False)


@pytest.mark.gpu
def test_long_fields_and_wide_files(rdf, ctx, tmp_path):
    long = "x" * 9000                                                                   # longer than one CTA's 4096 bytes
    _check(rdf, ctx, tmp_path, ("a,s,b\n" + "".join(f'{i},"{long},{i}",{i * 0.5}\n' for i in range(50))).encode())
    mb = '"' + "y\n," * 350_000 + '"'                                                   # a 1 MB quoted field
    _check(rdf, ctx, tmp_path, f"a,s\n1,{mb}\n2,z\n".encode())
    rng = np.random.default_rng(3)
    head = ",".join(f"c{k}" for k in range(300))
    rows = [",".join(str(v) for v in rng.integers(-1000, 1000, 300)) for _ in range(200)]
    _check(rdf, ctx, tmp_path, (head + "\n" + "\n".join(rows)).encode(), batch_size=64)


@pytest.mark.gpu
@pytest.mark.parametrize("delim", [";", "\t", "|"])
def test_delimiters_and_projection(rdf, ctx, tmp_path, delim):
    data = delim.join(["a", "b", "c"]) + "\n" + "\n".join(delim.join([str(i), f"{i}.25", "true"]) for i in range(100))
    _check(rdf, ctx, tmp_path, data.encode(), delimiter=delim, columns=[2, 0])
    _check(rdf, ctx, tmp_path, data.encode(), delimiter=delim, has_header=False)


@pytest.mark.gpu
def test_max_records_then_parse_error(rdf, ctx, tmp_path):
    data = b"a,b\n1,2\n3,4\n5,6.5\n"
    p = tmp_path / "m.csv"
    p.write_bytes(data)
    with rdf.CsvFile(str(p), max_records=2, ctx=ctx) as f:
        assert f.schema == [("a", rdf.I64, False), ("b", rdf.I64, False)]
        with pytest.raises(rdf.ParseError, match=r"^Error while parsing value 6.5 for column 1 at line 3$"):
            f.read()
        assert len(f.read(["a"])["a"]) == 3
    p.write_bytes(data[4:])
    with rdf.CsvFile(str(p), has_header=False, max_records=2, ctx=ctx) as f:   # without a header the line is the record index
        assert f.schema == [("column_1", rdf.I64, False), ("column_2", rdf.I64, False)]
        with pytest.raises(rdf.ParseError, match=r"^Error while parsing value 6.5 for column 1 at line 2$"):
            f.read([1])


FLOAT_HARD = ["2.2250738585072011e-308", "2.2250738585072014e-308", "4.9e-324", "2.4703282292062327e-324", "2.4703282292062328e-324",
              "1.7976931348623157e308", "1.7976931348623158e308", "1e309", "1e-400", "-1e-400", "9007199254740993", "9007199254740992.5",
              "1.00000000000000011102230246251565404236316680908203125", "1.00000000000000011102230246251565404236316680908203124",
              "3.4028235e38", "3.4028236e38", "1.4e-45", "7.0064923216240862e-46", "7.006492321624087e-46", "0.1", "1e23",
              "123456789012345678901234567890", "0.000000000000000000000000000000001", "-0", "+.5", "1.", "INF", "-Infinity", "nan", "-NaN",
              "8.589973e9", "16777217", "16777216.999999999999999999999", "1e-45", "0e999999999999"] + [
              "1" + "0" * 24 + str(k) + "e-" + str(k) for k in range(1, 40)] + ["0." + "9" * 30 + str(k) for k in range(10)]


@pytest.mark.gpu
def test_float_hard_cases_and_exact_fallback(rdf, ctx, tmp_path):
    data = ("a,b\n" + "\n".join(f"{s},{s}" for s in FLOAT_HARD) + "\n").encode()
    _, stats = _check(rdf, ctx, tmp_path, data, schema=[co.F32, co.F64])
    assert stats["exact_fields"] > 0


@pytest.mark.gpu
def test_integer_overflow_and_unsigned_minus_zero(rdf, ctx, tmp_path):
    cases = [(co.I64, "9223372036854775807", True), (co.I64, "-9223372036854775808", True), (co.I64, "9223372036854775808", False),
             (co.U8, "255", True), (co.U8, "256", False), (co.U8, "-0", False), (co.I8, "-0", True), (co.U64, "18446744073709551615", True),
             (co.U64, "18446744073709551616", False), (co.I32, "+7", True), (co.I16, "1.0", False), (co.I16, " 1", False)]
    for dt, s, ok in cases:
        data = f"x\n1\n{s}\n".encode()
        p = tmp_path / "i.csv"
        p.write_bytes(data)
        with rdf.CsvFile(str(p), schema=[dt], ctx=ctx) as f:
            if ok:
                v, m, _, _ = _host(f.read()["x"])
                assert int(v[1]) == int(s)
            else:
                with pytest.raises(rdf.ParseError, match=f"^Error while parsing value {s} for column 0 at line 2$"):
                    f.read()


@pytest.mark.gpu
def test_ten_million_rows_and_repeatability(rdf, ctx, tmp_path):
    rng = np.random.default_rng(7)
    n = 10_000_000
    ids = rng.integers(-2 ** 62, 2 ** 62, n)
    lat = np.round(rng.uniform(-90, 90, n), 6)
    flag = rng.random(n) < 0.5
    lat_s = np.char.mod("%.6f", lat)
    null = rng.random(n) < 0.01
    lat_s[null] = ""
    body = np.char.add(np.char.add(np.char.add(ids.astype(str), ","), lat_s), np.where(flag, ",true", ",false"))
    p = tmp_path / "big.csv"
    with open(p, "wb") as fh:
        fh.write(b"id,lat,flag\n")
        fh.write("\n".join(body.tolist()).encode())
    with rdf.CsvFile(str(p), ctx=ctx) as f:
        assert f.schema == [("id", rdf.I64, False), ("lat", rdf.F64, True), ("flag", rdf.native.BOOL, False)]
        first = f.read()
        again = f.read()
    want_lat = np.array([float(s) if s else 0.0 for s in lat_s.tolist()]).view(np.uint64)
    for name, want, mask in [("id", ids, np.ones(n, bool)), ("lat", want_lat, ~null), ("flag", flag, np.ones(n, bool))]:
        v, m, lens, _ = _host(first[name])
        assert np.array_equal(m, mask)
        assert np.array_equal(v[m], want[mask].astype(v.dtype))
        v2, m2, _, _ = _host(again[name])
        assert np.array_equal(v, v2) and np.array_equal(m, m2)
        assert len(lens) == (n + 1023) // 1024


@pytest.mark.gpu
def test_errors_leak_nothing(rdf, ctx, tmp_path):
    N = rdf.native

    def write(name, data):
        p = tmp_path / name
        p.write_bytes(data)
        return str(p)

    ctx.synchronize()
    before = pool_used(ctx)
    with pytest.raises(rdf.ComputeError, match=r"CSV error: record 2 \(line: 3, byte: 8\): found record with 3 fields, but the previous record has 2 fields"):
        rdf.CsvFile(write("u.csv", b"a,b\n1,2\n3,4,5\n6,7\n"), ctx=ctx)
    with pytest.raises(rdf.ComputeError, match="found record with 1 fields, but the previous record has 2 fields"):
        rdf.CsvFile(write("v.csv", b"a,b\n1,2\n" * 2000 + b"3\n"), max_records=5, ctx=ctx)
    with pytest.raises(rdf.ReferencePanic):
        rdf.CsvFile(write("h.csv", b"a,b\n"), ctx=ctx)
    with pytest.raises(rdf.ReferencePanic):
        rdf.CsvFile(write("e.csv", b""), ctx=ctx)
    with pytest.raises(rdf.UnsupportedType):
        rdf.CsvFile(write("s.csv", b"a\n1\n"), schema=[12], ctx=ctx)
    with pytest.raises(rdf.ComputeError):
        rdf.CsvFile(write("n.csv", b"a\n1\n"), schema=[co.I64, co.I64], ctx=ctx)
    with pytest.raises(rdf.ComputeError):
        rdf.CsvFile(str(tmp_path / "missing.csv"), ctx=ctx)
    with rdf.CsvFile(write("p.csv", b"a,b\n1,x\n2,3\n"), schema=[co.I64, co.I64], ctx=ctx) as f:
        with pytest.raises(rdf.ParseError, match=r"^Error while parsing value x for column 1 at line 1$"):
            f.read()
        with pytest.raises(rdf.ComputeError):
            f.read([5])
    ctx.synchronize()
    assert pool_used(ctx) == before
    fleet = rdf.Context.multi(0)
    try:
        with pytest.raises(rdf.UnsupportedType):
            rdf.CsvFile(UK, ctx=fleet)
    finally:
        fleet.close()
