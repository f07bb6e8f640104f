"""The CSV reader's restated rules (tests/csv_oracle.py) against the golden data and independent parsers; no GPU."""
import csv
import io
import json
import os
import struct

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import csv_oracle as co

HERE = os.path.dirname(os.path.abspath(__file__))
UK = os.path.join(HERE, "golden", "uk_cities_with_headers.csv")


def test_uk_cities_through_the_oracle():
    t = co.read(open(UK, "rb").read())
    assert t.names == ["city", "lat", "lng"]
    assert t.dtypes == [co.UTF8, co.F64, co.F64] and t.nullable == [False, False, False]
    assert t.num_rows == 37
    gold = json.load(open(os.path.join(HERE, "golden", "uk_cities.json")))
    for i, name in [(1, "lat"), (2, "lng")]:
        v, m = t.column(i)
        assert m.all()
        assert v.tolist() == np.array(gold[name], np.float64).view(np.uint64).tolist()
    lat0 = struct.unpack("<d", struct.pack("<Q", int(t.column(1)[0][0])))[0]
    lng0 = struct.unpack("<d", struct.pack("<Q", int(t.column(2)[0][0])))[0]
    assert (lat0, lng0) == (57.653484, -3.335724)


_field = st.text(alphabet='ab,"\r\n x', max_size=6)


@settings(max_examples=400, deadline=None)
@given(st.lists(st.lists(_field, min_size=1, max_size=4), min_size=1, max_size=6), st.sampled_from(["\n", "\r\n", "\r"]), st.booleans())
def test_dfa_matches_python_csv(rows, term, final_newline):
    buf = io.StringIO(newline="")
    w = csv.writer(buf, lineterminator=term, quoting=csv.QUOTE_MINIMAL)
    for r in rows:
        w.writerow(r)
    text = buf.getvalue()
    if not final_newline and text.endswith(term):
        text = text[: -len(term)]
    want = [r for r in csv.reader(io.StringIO(text, newline="")) if r]   # Python yields blank rows; csv-core skips them
    got = [[v.decode() for v in rec] for rec in co.records(text.encode())]
    assert got == want


@pytest.mark.parametrize("text,want", [
    (b'ab"c,d\n', [[b'ab"c', b"d"]]),          # a quote inside an unquoted field is literal
    (b'"ab"cd,e\n', [[b"abcd", b"e"]]),         # bytes after the closing quote are appended
    (b'"a""b"\n', [[b'a"b']]),
    (b'"a,\nb",c', [[b"a,\nb", b"c"]]),
    (b'a,"unterminated\n', [[b"a", b"unterminated\n"]]),   # end of file ends the field
    (b"\xef\xbb\xbfa,b\n", [[b"a", b"b"]]),     # BOM skipped
    (b"\r\n\r\na\r\r\nb", [[b"a"], [b"b"]]),
    (b"a,\n", [[b"a", b""]]),
    (b"\r\n\n1,2\n", [[b"1", b"2"]]),        # leading terminators make no record
])
def test_dfa_cases(text, want):
    assert co.records(text) == want


def test_inference_classes_and_merge():
    cls = {b"": None, b'""x': co.UTF8, b"TrUe": co.BOOL, b"false": co.BOOL, b"-1.5": co.F64, b"12": co.I64, b"-0": co.I64, b"1e5": co.UTF8,
           b".5": co.UTF8, b"+1": co.UTF8, b"inf": co.UTF8, b"1.": co.UTF8, b"truex": co.UTF8, b"\xd9\xa1": co.UTF8}
    for v, c in cls.items():
        assert co.classify(v) == c, v
    assert co.merge({co.I64}) == co.I64 and co.merge({co.F64, co.I64}) == co.F64
    assert co.merge({co.BOOL, co.I64}) == co.UTF8 and co.merge({co.F64, co.UTF8}) == co.UTF8
    t = co.read(b'a,b,c,d\n1,,true,"""q"""\n2.5,,false,x\n')
    assert t.dtypes == [co.F64, co.UTF8, co.BOOL, co.UTF8] and t.nullable == [False, True, False, False]
    t = co.read(b"a\n1\n2\nx\n", max_records=2)
    assert t.dtypes == [co.I64]


def test_line_numbers_and_error_texts():
    t = co.read(b"a,b\n1,2\n3,x\n", schema=[co.I64, co.I64])
    with pytest.raises(co.ParseError, match="^Error while parsing value x for column 1 at line 2$"):
        t.column(1)
    t = co.read(b"1,2\n3,x\n", has_header=False, schema=[co.I64, co.I64])
    with pytest.raises(co.ParseError, match="at line 1$"):
        t.column(1)
    t = co.read(b'a\n"multi\nline"\n7\nbad\n', schema=[co.I64])   # records, not physical lines
    with pytest.raises(co.ParseError, match="value multi\nline for column 0 at line 1$"):
        t.column(0)
    with pytest.raises(co.CsvError, match="found record with 3 fields, but the previous record has 2 fields"):
        co.read(b"a,b\n1,2,3\n")
    with pytest.raises(co.Panic):
        co.read(b"a,b\n")


def test_numbers_against_pyarrow():
    pa = pytest.importorskip("pyarrow")
    pacsv = pytest.importorskip("pyarrow.csv")
    rng = np.random.default_rng(5)
    floats = [repr(float(x)) for x in rng.normal(size=300) * 10.0 ** rng.integers(-300, 300, 300)]
    floats += [f"{rng.integers(0, 10 ** 9)}.{rng.integers(0, 10 ** 9):09d}e{rng.integers(-320, 300)}" for _ in range(300)]
    floats += ["2.2250738585072011e-308", "4.9e-324", "1e-400", "1.7976931348623159e308", "0.1", "1.", ".5", "-0"]
    ints = [str(int(x)) for x in rng.integers(-2 ** 63, 2 ** 63 - 1, 300)] + ["-0", "9223372036854775807"]
    for vals, dt, pt in [(floats, co.F64, pa.float64()), (floats, co.F32, pa.float32()), (ints, co.I64, pa.int64())]:
        data = ("x\n" + "\n".join(vals) + "\n").encode()
        got, valid = co.read(data, schema=[dt]).column(0)
        tbl = pacsv.read_csv(io.BytesIO(data), convert_options=pacsv.ConvertOptions(column_types={"x": pt}))
        want = tbl.column("x").to_numpy()
        if dt == co.F64:
            want = want.astype(np.float64).view(np.uint64)
        elif dt == co.F32:
            want = want.astype(np.float32).view(np.uint32)
        assert valid.all()
        assert got.tolist() == want.tolist()


def test_value_grammars():
    F64 = co.F64
    assert co.parse_float_bits(b"1_0", F64) is None and co.parse_float_bits(b" 1", F64) is None
    assert co.parse_float_bits(b".", F64) is None and co.parse_float_bits(b"1e", F64) is None
    assert co.parse_float_bits(b"-NaN", F64) == 0xFFF8000000000000 and co.parse_float_bits(b"Infinity", co.F32) == 0x7F800000
    assert co.parse_float_bits(b"3.4028236e38", co.F32) == 0x7F800000 and co.parse_float_bits(b"1.4e-45", co.F32) == 1
    # the exponent and the digits together decide the magnitude
    assert co.parse_float_bits(b"0." + b"0" * 500 + b"1e450", co.F32) == 0
    assert co.parse_float_bits(b"0." + b"0" * 500 + b"1e501", co.F32) == struct.unpack("<I", struct.pack("<f", 1.0))[0]
    assert co.parse_float_bits(b"1" + b"0" * 400 + b"e-400", co.F32) == struct.unpack("<I", struct.pack("<f", 1.0))[0]
    assert co.parse_float_bits(b"0.00001e-40", co.F32) == 1 and co.parse_float_bits(b"123e99999999999", co.F32) == 0x7F800000
    assert co.parse_float_bits(b"0e99999999999", co.F32) == 0
    assert co.parse_int(b"-0", co.U8) is None and co.parse_int(b"-0", co.I8) == 0 and co.parse_int(b"256", co.U8) is None
    assert co.parse_int(b"-128", co.I8) == -128 and co.parse_int(b"128", co.I8) is None and co.parse_int(b"+", co.I8) is None
    assert co.parse_bool(b"TRUE") is True and co.parse_bool(b"no") is None


def test_csv_abi_constants(rdf):
    N = rdf.native
    assert N.PARSE == 9 and N.KERNEL_NAMES[N.K_CSV] == "csv" and N.UTF8 == 11
    assert issubclass(rdf.ParseError, rdf.ArrowError)
    assert [f for f, _ in N.CsvOptions._fields_] == ["has_header", "delimiter", "max_records", "batch_size"]
