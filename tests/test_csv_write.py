"""The CSV writer's rules without a GPU: tests/csv_write_oracle.py against Python's own float printing, pinned strings, read-back by
pyarrow and Python's csv module, and the generated power tables."""
import csv
import io
import os
import subprocess
import sys

import numpy as np
import pytest

import csv_write_oracle as wo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "rust-dataframe_b200", "csrc")


def test_float_oracle_matches_python_repr_digit_for_digit():
    """np.format_float_positional(unique=True) gives the same shortest digits as repr (which prints with an exponent)."""
    rng = np.random.default_rng(7)
    bits = rng.integers(0, 2 ** 64, 100_000, dtype=np.uint64)
    for v in bits.view(np.float64):
        if not np.isfinite(v) or v == 0:
            continue
        got = wo.format_float(v)
        assert float(got) == v
        r = repr(float(v)).lstrip("-").split("e")[0].replace(".", "").lstrip("0").rstrip("0")
        assert got.lstrip("-").replace(".", "").lstrip("0").rstrip("0") == r, (v, got)


@pytest.mark.parametrize("value,dtype,want", [
    (1.0, np.float64, "1"), (0.1, np.float64, "0.1"), (1e20, np.float64, "100000000000000000000"), (1e-7, np.float64, "0.0000001"),
    (0.1, np.float32, "0.1"), (16777216.0, np.float32, "16777216"),
    (np.finfo(np.float32).max, np.float32, "340282350000000000000000000000000000000"),
    (np.nan, np.float64, "NaN"), (-np.nan, np.float32, "NaN"), (np.inf, np.float64, "inf"), (-np.inf, np.float32, "-inf"),
    (-0.0, np.float64, "-0"), (0.0, np.float32, "0"),
])
def test_pinned_float_strings(value, dtype, want):
    assert wo.format_float(dtype(value)) == want


def test_pinned_longest_float_field():
    tiny = np.array([1], np.uint64).view(np.float64)[0]
    s = wo.format_float(-tiny)
    assert len(s) == 327 and s.startswith("-0.000") and s.endswith("5")
    s32 = wo.format_float(-np.array([1], np.uint32).view(np.float32)[0])
    assert len(s32) <= 48


def test_pinned_integers_booleans_and_the_empty_record():
    assert wo.format_values(3, np.array([np.iinfo(np.int64).min], np.int64)) == ["-9223372036854775808"]
    assert wo.format_values(7, np.array([np.iinfo(np.uint64).max], np.uint64)) == ["18446744073709551615"]
    assert wo.format_values(wo.BOOL, np.array([True, False])) == ["true", "false"]
    text = wo.write([("x", 2, np.array([1, 2], np.int32), np.array([True, False]))])
    assert text == b'x\n1\n""\n'
    assert wo.write([("a", 2, np.array([1], np.int32), None), ("b", 2, np.array([2], np.int32), np.array([False]))]) == b"a,b\n1,\n"
    assert wo.write([("a", 2, np.zeros(0, np.int32), None)]) == b"a\n"
    assert wo.write([("a", 2, np.zeros(0, np.int32), None)], has_header=False) == b""


def test_header_quoting():
    assert wo.header(["a", "b,c", 'd"e', "f\ng", "h\ri"]) == 'a,"b,c","d""e","f\ng","h\ri"\n'
    assert wo.header(["a;b", "c,d"], ";") == '"a;b";c,d\n'
    assert wo.header([""]) == '""\n' and wo.header(["", "x"]) == ",x\n"


def _frame(rng, n):
    f64 = rng.integers(0, 2 ** 64, n, dtype=np.uint64).view(np.float64)
    f32 = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32).view(np.float32)
    i64 = rng.integers(np.iinfo(np.int64).min, np.iinfo(np.int64).max, n, dtype=np.int64, endpoint=True)
    b = rng.random(n) < 0.5
    valid = rng.random(n) >= 0.1
    return [("f64", wo.F64, f64, valid), ("f32", wo.F32, f32, None), ("i64", 3, i64, valid), ("b", wo.BOOL, b, valid)]


def test_python_csv_reads_the_oracle_text_back():
    rng = np.random.default_rng(3)
    cols = _frame(rng, 5000)
    text = wo.write(cols, delim=";").decode()
    recs = list(csv.reader(io.StringIO(text), delimiter=";"))
    assert recs[0] == ["f64", "f32", "i64", "b"] and len(recs) == 5001
    for j, (_, dt, vals, valid) in enumerate(cols):
        for r in range(5000):
            s = recs[r + 1][j]
            if valid is not None and not valid[r]:
                assert s == ""
                continue
            if dt == wo.F64:
                got = np.float64(float(s))
                assert (np.isnan(got) and np.isnan(vals[r])) or got.view(np.uint64) == vals[r].view(np.uint64)
            elif dt == wo.F32:
                got = np.float32(s)   # numpy rounds the decimal straight to f32
                assert (np.isnan(got) and np.isnan(vals[r])) or got.view(np.uint32) == vals[r].view(np.uint32)
            elif dt == wo.BOOL:
                assert s == ("true" if vals[r] else "false")
            else:
                assert int(s) == int(vals[r])


def test_pyarrow_reads_the_oracle_text_back():
    pa = pytest.importorskip("pyarrow")
    pcsv = pytest.importorskip("pyarrow.csv")
    rng = np.random.default_rng(5)
    cols = _frame(rng, 3000)
    text = wo.write(cols)
    types = {"f64": pa.float64(), "f32": pa.float32(), "i64": pa.int64(), "b": pa.bool_()}
    # pyarrow's default null spellings include NaN: only the empty field is a NULL here
    t = pcsv.read_csv(io.BytesIO(text), convert_options=pcsv.ConvertOptions(column_types=types, null_values=[""], strings_can_be_null=True))
    for name, dt, vals, valid in cols:
        col = t.column(name).combine_chunks()
        m = np.ones(len(vals), bool) if valid is None else valid
        assert np.array_equal(~np.asarray(col.is_null()), m), name
        want = vals[m]
        if dt in (wo.F32, wo.F64):
            got = col.to_numpy(zero_copy_only=False)[m].astype(want.dtype)
            same = (got.view(f"u{want.itemsize}") == want.view(f"u{want.itemsize}")) | (np.isnan(got) & np.isnan(want))
            assert same.all(), name
        else:
            assert [x for x, ok in zip(col.to_pylist(), m) if ok] == want.tolist(), name


def test_one_generator_reproduces_the_power_tables():
    out = subprocess.run([sys.executable, os.path.join(CSRC, "gen_csv_pow5.py")], capture_output=True, text=True, check=True).stdout
    assert out == open(os.path.join(CSRC, "csv_pow5.cuh")).read()


def test_csv_write_abi_entries(rdf):
    N = rdf.native
    assert N.KERNEL_NAMES[N.K_CSV_WRITE] == "csv_write" and N.K_CSV_WRITE == 16 and N.K_MOMENTS == 15
    assert "bdf_csv_write" in N.EXPORTED_SYMBOLS
    assert callable(rdf.write_csv) and callable(rdf.DeviceFrame.to_csv)


def test_header_layout_of_the_options_struct(tmp_path):
    src = tmp_path / "o.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200df.h"\n'
                   'int main(void){printf("%zu %zu %d\\n", sizeof(bdf_csv_write_options), offsetof(bdf_csv_write_options, delimiter), '
                   '(int)BDF_K_CSV_WRITE);return 0;}\n')
    exe = tmp_path / "o"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    assert subprocess.check_output([str(exe)]).split() == [b"8", b"4", b"16"]
