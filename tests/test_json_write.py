"""The JSON writer's rules without a GPU: tests/json_write_oracle.py against Python's json module, pyarrow and datetime, pinned strings,
the device formatter (json_format.cuh) compiled for the host against the oracle over millions of float patterns and every Date32 day
of chrono's range, and the ABI."""
import ctypes as C
import datetime
import io
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

import json_write_oracle as wo

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "rust-dataframe_b200", "csrc")


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    cxx = shutil.which("g++")
    if cxx is None:
        pytest.skip("g++ is not installed: json_format.cuh cannot be compiled for the host")
    so = str(tmp_path_factory.mktemp("json_harness") / "json_format_harness.so")
    subprocess.run([cxx, "-O2", "-std=c++17", "-D__device__=", "-I", CSRC, "-shared", "-fPIC", os.path.join(HERE, "json_format_harness.cpp"),
                    "-o", so], check=True)
    lib = C.CDLL(so)
    lib.jh_format_floats.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_char_p, C.c_int64]
    lib.jh_format_floats.restype = C.c_int64
    lib.jh_format_dates.argtypes = [C.c_int32, C.c_int64, C.c_void_p]
    lib.jh_format_temporal.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_int, C.c_char_p, C.c_char_p, C.c_int64]
    lib.jh_format_temporal.restype = C.c_int64
    return lib


def _floats(lib, bits, width):
    bits = np.ascontiguousarray(bits, dtype=np.uint64)
    cap = 64 * len(bits) + 64
    buf = C.create_string_buffer(cap)
    n = lib.jh_format_floats(bits.ctypes.data, len(bits), width, buf, cap)
    assert n >= 0
    return buf.raw[:n].decode().split("\n")[:-1]


def _temporal(lib, vals, temporal):
    kind, unit, tz = temporal
    ups = 1 if kind == wo.DATE32 else 1000 if kind == wo.DATE64 else wo.PER_SEC[unit]
    upd = 1 if kind == wo.DATE32 else 86400 * ups
    jt = {wo.DATE32: 1, wo.DATE64: 1, wo.TIMESTAMP: 2, wo.TIME32: 3, wo.TIME64: 3}[kind]
    off, sfx = wo.tz_suffix(tz) if kind == wo.TIMESTAMP else (0, "")
    frac = 0 if kind in (wo.DATE32, wo.DATE64) else 3 * unit
    v = np.ascontiguousarray(vals, dtype=np.int64)
    cap = 64 * len(v) + 64
    buf = C.create_string_buffer(cap)
    n = lib.jh_format_temporal(v.ctypes.data, len(v), jt, upd, ups, off * ups, frac, sfx.encode(), buf, cap)
    assert n >= 0
    return buf.raw[:n].decode().split("\n")[:-1]


# ---- pinned strings -------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("value,f32,want", [
    (1.0, False, "1.0"), (-0.0, False, "-0.0"), (0.0, True, "0.0"), (1e16, False, "1e16"), (1e15, False, "1000000000000000.0"),
    (1e-7, False, "1e-7"), (1e-5, False, "0.00001"), (5e-324, False, "5e-324"), (0.1, False, "0.1"), (123.456, False, "123.456"),
    (1e13, True, "1e13"), (1e12, True, "1000000000000.0"), (1e-6, True, "0.000001"), (1e-7, True, "1e-7"),
    (float(np.finfo(np.float32).max), True, "3.4028235e38"), (1.5e-7, False, "1.5e-7"), (-2.5e300, False, "-2.5e300"),
    (float("nan"), False, None), (float("inf"), True, None), (float("-inf"), False, None),
])
def test_pinned_float_strings(harness, value, f32, want):
    assert wo.format_float(value, f32) == want
    bits = np.array([value], np.float32).view(np.uint32).astype(np.uint64) if f32 else np.array([value], np.float64).view(np.uint64)
    assert _floats(harness, bits, 32 if f32 else 64) == [want or "null"]


def test_pinned_integers_and_booleans():
    assert wo.format_scalar(3, np.iinfo(np.int64).min) == "-9223372036854775808"
    assert wo.format_scalar(7, np.iinfo(np.uint64).max) == "18446744073709551615"
    assert wo.format_scalar(wo.BOOL, True) == "true" and wo.format_scalar(wo.BOOL, False) == "false"


@pytest.mark.parametrize("temporal,value,want", [
    ((wo.DATE32, 0, None), -719162, '"0001-01-01"'),
    ((wo.DATE32, 0, None), 2932897, '"+10000-01-01"'),
    ((wo.DATE32, 0, None), -719834, '"-0001-03-01"'),
    ((wo.DATE32, 0, None), wo.MIN_DAY, '"-262144-01-01"'),
    ((wo.DATE32, 0, None), wo.MAX_DAY, '"+262143-12-31"'),
    ((wo.DATE64, wo.MILLISECOND, None), -1, '"1969-12-31"'),
    ((wo.TIMESTAMP, wo.MICROSECOND, None), -1, '"1969-12-31T23:59:59.999999"'),
    ((wo.TIMESTAMP, wo.SECOND, "UTC"), 0, '"1970-01-01T00:00:00Z"'),
    ((wo.TIMESTAMP, wo.MILLISECOND, "+00:00"), 1, '"1970-01-01T00:00:00.001Z"'),
    ((wo.TIMESTAMP, wo.MILLISECOND, "+05:30"), 1700000000123, '"2023-11-15T03:43:20.123+05:30"'),
    ((wo.TIMESTAMP, wo.NANOSECOND, "-08:00"), 0, '"1969-12-31T16:00:00.000000000-08:00"'),
    ((wo.TIME32, wo.SECOND, None), 86399, '"23:59:59"'),
    ((wo.TIME32, wo.MILLISECOND, None), 0, '"00:00:00.000"'),
    ((wo.TIME64, wo.NANOSECOND, None), 86399999999999, '"23:59:59.999999999"'),
])
def test_pinned_temporal_strings(harness, temporal, value, want):
    assert wo.format_temporal(temporal, value) == want
    assert _temporal(harness, [value], temporal) == [want]


def test_temporal_range_and_named_zones_are_refused_by_the_oracle():
    with pytest.raises(ValueError):
        wo.format_temporal((wo.DATE32, 0, None), wo.MIN_DAY - 1)
    with pytest.raises(ValueError):
        wo.format_temporal((wo.TIME64, wo.MICROSECOND, None), 86400 * 10 ** 6)
    with pytest.raises(ValueError):
        wo.format_temporal((wo.TIMESTAMP, wo.SECOND, "Europe/Paris"), 0)


def test_name_escapes():
    assert wo.escape_name('a"b\\c') == '"a\\"b\\\\c"'
    assert wo.escape_name("\b\f\n\r\t") == '"\\b\\f\\n\\r\\t"'
    assert wo.escape_name("\x00\x1f\x7f") == '"\\u0000\\u001f\x7f"'
    assert wo.escape_name("é ü") == '"é ü"'
    for name in ['a"b\\c', "\x01x\ty", "é", "", " "]:
        assert json.loads(wo.escape_name(name)) == name


def test_empty_frame_and_null_members():
    cols = [{"name": "a", "dtype": 2, "values": np.array([1, 2], np.int32), "valid": np.array([True, False])},
            {"name": "b", "dtype": wo.F64, "values": np.array([np.nan, 1.0])}]
    assert wo.write(cols) == b'{"a":1}\n{"b":1.0}\n'
    assert wo.write(cols, explicit_nulls=True) == b'{"a":1,"b":null}\n{"a":null,"b":1.0}\n'
    assert wo.write([{"name": "a", "dtype": 2, "values": np.array([1], np.int32), "valid": np.array([False])}]) == b"{}\n"
    assert wo.write([{"name": "a", "dtype": 2, "values": np.zeros(0, np.int32)}]) == b""
    lists = [{"name": "l", "dtype": 3, "lists": [[1, None, 3], [], None]}]
    assert wo.write(lists) == b'{"l":[1,null,3]}\n{"l":[]}\n{}\n'
    assert wo.write(lists, explicit_nulls=True) == b'{"l":[1,null,3]}\n{"l":[]}\n{"l":null}\n'


# ---- the oracle against independent readers --------------------------------------------------------------------------------------

def _frame(rng, n):
    f64 = rng.integers(0, 2 ** 64, n, dtype=np.uint64).view(np.float64)
    f32 = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32).view(np.float32)
    i64 = rng.integers(np.iinfo(np.int64).min, np.iinfo(np.int64).max, n, dtype=np.int64, endpoint=True)
    u64 = rng.integers(0, np.iinfo(np.uint64).max, n, dtype=np.uint64, endpoint=True)
    b = rng.random(n) < 0.5
    valid = rng.random(n) >= 0.1
    lists = [None if rng.random() < 0.1 else [None if rng.random() < 0.1 else float(x) for x in rng.normal(size=rng.integers(0, 5))]
             for _ in range(n)]
    return [{"name": "f64", "dtype": wo.F64, "values": f64, "valid": valid}, {"name": "f32", "dtype": wo.F32, "values": f32},
            {"name": "i64", "dtype": 3, "values": i64, "valid": valid}, {"name": "u64", "dtype": 7, "values": u64},
            {"name": "b", "dtype": wo.BOOL, "values": b, "valid": valid}, {"name": "l", "dtype": wo.F64, "lists": lists}]


def test_python_json_reads_the_oracle_text_back():
    rng = np.random.default_rng(3)
    cols = _frame(rng, 3000)
    for explicit in (False, True):
        lines = wo.write(cols, explicit_nulls=explicit).decode().split("\n")
        assert lines[-1] == "" and len(lines) == 3001
        for r, line in enumerate(lines[:-1]):
            obj = json.loads(line)
            assert list(obj) == [c["name"] for c in cols if explicit or wo._value(c, r) is not None]
            for c in cols:
                got = obj.get(c["name"])
                if c.get("lists") is not None:
                    assert got == c["lists"][r]
                    continue
                v = c["values"][r]
                if (c.get("valid") is not None and not c["valid"][r]) or (c["dtype"] in (wo.F32, wo.F64) and not np.isfinite(v)):
                    assert got is None
                elif c["dtype"] == wo.F64:
                    assert np.float64(got).view(np.uint64) == v.view(np.uint64)
                elif c["dtype"] == wo.F32:
                    s = line.split(f'"{c["name"]}":')[1].split(",")[0].split("}")[0]
                    assert np.float32(s).view(np.uint32) == v.view(np.uint32)   # numpy rounds the decimal straight to f32
                elif c["dtype"] == wo.BOOL:
                    assert got is bool(v)
                else:
                    assert got == int(v)


def test_integral_floats_stay_floats_under_inference():
    text = wo.write([{"name": "x", "dtype": wo.F64, "values": np.array([1.0, 2.0, -0.0])}])
    assert text == b'{"x":1.0}\n{"x":2.0}\n{"x":-0.0}\n'
    assert all(isinstance(json.loads(l)["x"], float) for l in text.decode().splitlines())


def test_pyarrow_reads_the_oracle_text_back():
    pa = pytest.importorskip("pyarrow")
    pj = pytest.importorskip("pyarrow.json")
    rng = np.random.default_rng(5)
    cols = _frame(rng, 2000)
    text = wo.write(cols)
    schema = pa.schema([("f64", pa.float64()), ("f32", pa.float64()), ("i64", pa.int64()), ("u64", pa.uint64()), ("b", pa.bool_()),
                        ("l", pa.list_(pa.float64()))])
    t = pj.read_json(io.BytesIO(text), parse_options=pj.ParseOptions(explicit_schema=schema))
    for c in cols:
        got = t.column(c["name"]).to_pylist()
        if c.get("lists") is not None:
            assert got == c["lists"]
            continue
        for r, g in enumerate(got):
            v = c["values"][r]
            if (c.get("valid") is not None and not c["valid"][r]) or (c["dtype"] in (wo.F32, wo.F64) and not np.isfinite(v)):
                assert g is None
            elif c["dtype"] == wo.F64:
                assert np.float64(g).view(np.uint64) == v.view(np.uint64)
            elif c["dtype"] == wo.F32:
                assert np.float32(np.float64(g)) == v or np.float32(g) == v   # pyarrow reads f64 and narrows
            elif c["dtype"] == wo.BOOL:
                assert g is bool(v)
            else:
                assert g == int(v)


def test_oracle_dates_match_datetime():
    rng = np.random.default_rng(11)
    days = np.concatenate([rng.integers(-719162, 2932896, 20000), [-719162, 2932896, 0, -1]])
    slots = wo.date_slots(days)
    for i, d in enumerate(days):
        want = '"' + (datetime.date(1970, 1, 1) + datetime.timedelta(days=int(d))).isoformat() + '"'
        assert wo.format_temporal((wo.DATE32, 0, None), int(d)) == want
        assert bytes(slots[i]).rstrip(b"\0").decode() == want
    for d in rng.integers(wo.MIN_DAY, wo.MAX_DAY, 20000).tolist() + [wo.MIN_DAY, wo.MAX_DAY, -719528, -719529, 2932897]:
        assert bytes(wo.date_slots(np.array([d]))[0]).rstrip(b"\0").decode() == wo.format_temporal((wo.DATE32, 0, None), d)


def test_oracle_timestamps_match_datetime():
    rng = np.random.default_rng(12)
    for unit in range(4):
        ups = wo.PER_SEC[unit]
        for v in rng.integers(-2 ** 62 // max(1, 10 ** 9 // ups) // 4, 2 ** 62 // max(1, 10 ** 9 // ups) // 4, 300).tolist():
            for tz, off in ((None, 0), ("+05:30", 19800), ("-11:15", -40500)):
                s, sub = divmod(v + off * ups, ups)
                want_dt = datetime.datetime(1970, 1, 1) + datetime.timedelta(seconds=s)
                frac = f".{sub:0{3 * unit}d}" if unit else ""
                want = '"' + want_dt.strftime("%Y-%m-%dT%H:%M:%S").rjust(19, "0") + frac + (tz or "") + '"'
                if 1 <= want_dt.year <= 9999:
                    assert wo.format_temporal((wo.TIMESTAMP, unit, tz), v) == want


# ---- the device formatter, compiled for the host, against the oracle ----------------------------------------------------------

@pytest.mark.parametrize("width", [32, 64])
def test_format_millions_of_patterns_match_the_oracle(harness, width):
    rng = np.random.default_rng(40 + width)
    n = 4_200_000
    if width == 32:
        bits = rng.integers(0, 2 ** 32, n, dtype=np.uint64)
        # every biased exponent's edges and the decimal layout thresholds
        edges = np.array([np.float32(10.0) ** k for k in range(-45, 39)] + [np.nextafter(np.float32(10.0) ** k, np.float32(0)) for k in range(-44, 39)],
                         np.float32).view(np.uint32).astype(np.uint64)
    else:
        bits = rng.integers(0, 2 ** 64, n, dtype=np.uint64)
        edges = np.array([10.0 ** k for k in range(-323, 309)] + [np.nextafter(10.0 ** k, 0) for k in range(-322, 309)], np.float64).view(np.uint64)
    bits = np.concatenate([bits, edges, edges | np.uint64(1 << (width - 1)), np.arange(64, dtype=np.uint64)])
    got = _floats(harness, bits, width)
    vals = bits.astype(np.uint32).view(np.float32) if width == 32 else bits.view(np.float64)
    if width == 64:   # repr gives the same shortest, closest digits, much faster than numpy's per-value formatting
        want = [wo.format_f64_repr(v) for v in vals.tolist()]
    else:
        want = [wo.format_float(v, True) or "null" for v in vals]
    bad = [(hex(int(b)), g, w) for b, g, w in zip(bits, got, want) if g != w]
    assert not bad, bad[:10]


def test_fast_float64_layout_agrees_with_the_oracle():
    rng = np.random.default_rng(9)
    for v in rng.integers(0, 2 ** 64, 20000, dtype=np.uint64).view(np.float64).tolist() + [1e16, 1e15, 1e-5, 1e-6, 5e-324, 0.5, 123.0]:
        assert wo.format_f64_repr(v) == (wo.format_float(v, False) or "null"), v


def test_every_date32_day_of_chronos_range_matches_the_oracle(harness):
    step = 1 << 22
    buf = np.zeros((step, 16), np.uint8)
    for first in range(wo.MIN_DAY, wo.MAX_DAY + 1, step):
        n = min(step, wo.MAX_DAY + 1 - first)
        harness.jh_format_dates(first, n, buf.ctypes.data)
        want = wo.date_slots(np.arange(first, first + n, dtype=np.int64))
        if not np.array_equal(buf[:n], want):
            i = int(np.nonzero((buf[:n] != want).any(axis=1))[0][0])
            raise AssertionError((first + i, bytes(buf[i]), bytes(want[i])))


def test_temporal_text_of_every_kind_matches_the_oracle(harness):
    rng = np.random.default_rng(13)
    for kind, unit in [(wo.DATE32, 0), (wo.DATE64, 1), (wo.TIME32, 0), (wo.TIME32, 1), (wo.TIME64, 2), (wo.TIME64, 3)] + \
                      [(wo.TIMESTAMP, u) for u in range(4)]:
        for tz in ([None, "UTC", "Z", "+00:00", "+05:30", "-23:59", "-00:00"] if kind == wo.TIMESTAMP else [None]):
            ups = 1000 if kind == wo.DATE64 else wo.PER_SEC[unit]
            if kind in (wo.TIME32, wo.TIME64):
                vals = np.concatenate([rng.integers(0, 86400 * ups, 3000), [0, 86400 * ups - 1]])
            elif kind == wo.DATE32:
                vals = np.concatenate([rng.integers(wo.MIN_DAY, wo.MAX_DAY + 1, 3000), [wo.MIN_DAY, wo.MAX_DAY]])
            else:
                lo = max(wo.MIN_DAY * 86400 * ups + 86400 * ups, -2 ** 63)
                hi = min(wo.MAX_DAY * 86400 * ups - 86400 * ups, 2 ** 63 - 1)
                vals = np.concatenate([rng.integers(lo, hi, 3000, dtype=np.int64), [lo, hi, -1, 0, 1]])
            got = _temporal(harness, vals, (kind, unit, tz))
            want = [wo.format_temporal((kind, unit, tz), int(v)) for v in vals]
            assert got == want, [(v, g, w) for v, g, w in zip(vals, got, want) if g != w][:5]


# ---- ABI ------------------------------------------------------------------------------------------------------------------------

def test_json_write_abi_entries(rdf):
    N = rdf.native
    assert N.LAUNCH_KERNEL_NAMES[N.K_JSON_WRITE] == "json_write" and N.K_JSON_WRITE == 24 and N.K_HIST == 23
    assert N.LAUNCH_KERNEL_NAMES[:len(N.KERNEL_NAMES)] == N.KERNEL_NAMES
    assert "bdf_json_write" in N.EXPORTED_SYMBOLS
    assert callable(rdf.write_json) and callable(rdf.DeviceFrame.to_json)


def test_header_layout_of_the_options_struct(tmp_path):
    src = tmp_path / "o.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200df.h"\n'
                   'int main(void){printf("%zu %zu %d %d\\n", sizeof(bdf_json_write_options), offsetof(bdf_json_write_options, explicit_nulls), '
                   '(int)BDF_K_JSON_WRITE, (int)BDF_K_HIST);return 0;}\n')
    exe = tmp_path / "o"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    assert subprocess.check_output([str(exe)]).split() == [b"4", b"0", b"24", b"23"]
