"""DataFrame::from_json on the device against tests/json_oracle.py: every value bit for bit, the same null slots, chunk lengths and
bitmaps, lists included."""
import struct

import numpy as np
import pytest

import json_oracle as jo
from csv_oracle import BOOL, F32, F64, I8, I16, I32, I64, U8, U16, U32, U64
from helpers import pool_used

pytestmark = pytest.mark.gpu


def _host(col):
    vals, valid, lens, hv = [], [], [], []
    for a in col.download():
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
    return np.concatenate(vals), np.concatenate(valid), lens, hv


def _list_host(lc):
    rows, lens, hv = [], [], []
    for ch in lc.download():
        lens.append(ch.length)
        hv.append(ch.validity is not None)
        vals = np.asarray(ch.values.value_slice())
        if vals.dtype.kind == "f":
            vals = vals.view(f"u{vals.dtype.itemsize}")
        vm = ch.values.valid_mask()
        lm = [True] * ch.length if ch.validity is None else [bool((ch.validity[k >> 3] >> (k & 7)) & 1) for k in range(ch.length)]
        assert ch.offsets[0] == 0
        for k in range(ch.length):
            s, e = int(ch.offsets[k]), int(ch.offsets[k + 1])
            rows.append(None if not lm[k] else [int(vals[j]) if vm[j] else None for j in range(s, e)])
    return rows, lens, hv


def check(rdf, ctx, tmp_path, data: bytes, batch_size=1024, schema=None, max_records=None):
    p = tmp_path / "t.json"
    p.write_bytes(data)
    ref = jo.read(data, schema=schema, max_records=max_records, batch_size=batch_size)
    with rdf.JsonFile(str(p), schema=schema, max_records=max_records, batch_size=batch_size, ctx=ctx) as f:
        assert [n for n, _, _ in f.schema] == ref.names
        assert [dt for _, dt, _ in f.schema] == ref.dtypes
        assert [nl for _, _, nl in f.schema] == ref.nullable
        assert f.num_rows == ref.num_rows
        n = ref.num_rows
        want_lens = [min(batch_size, n - s) for s in range(0, n, batch_size)]
        idx = [i for i, dt in enumerate(ref.dtypes) if 0 <= dt <= BOOL]
        cols = f.read(idx)
        exact = f.stats()["exact_fields"]
        for i in idx:
            v, m, lens, hv = _host(cols[ref.names[i]])
            rv, rm = ref.column(i)
            assert np.array_equal(m, rm), ref.names[i]
            assert np.array_equal(v, rv.astype(v.dtype)), ref.names[i]   # NULL slots are zero on both sides
            assert lens == want_lens
            assert hv == [bool((~rm[s:s + batch_size]).any()) for s in range(0, n, batch_size)]
        for i in [i for i, dt in enumerate(ref.dtypes) if dt >= jo.LIST_BASE]:
            rows, lens, hv = _list_host(f.read_list(i))
            want = ref.list_column(i)
            assert rows == want, ref.names[i]
            assert lens == want_lens
            assert hv == [any(x is None for x in want[s:s + batch_size]) for s in range(0, n, batch_size)]
    return ref, exact


def test_escapes_and_brackets_in_strings(rdf, ctx, tmp_path):
    data = (b'{"s": "a\\"b", "x": 1, "t": "\\\\", "u": "\\u00e9\\ud83d\\ude00"}\n'
            b'{"s": "[{:,}]", "x": 2, "t": "\\\\\\\\", "q\\"k": 3}\n'
            b'{"s": "\\\\\\"}", "x": 3, "t": "} ] , :", "\\u0078": 4}\n')
    ref, _ = check(rdf, ctx, tmp_path, data)
    assert ref.names == ["s", "x", "t", "u", 'q"k'] and ref.column(1)[0].tolist() == [1, 2, 4]


def test_key_order_duplicates_missing_nulls(rdf, ctx, tmp_path):
    lines = ['{"a": 1, "b": 2.5, "c": true}', '{"c": false, "a": 2}', '{"b": null, "b": 7, "a": 3, "a": 4}', '{}', '{"d": 1, "a": null}']
    check(rdf, ctx, tmp_path, ("\n".join(lines) + "\n").encode())


def test_line_ends_bom_blank_lines(rdf, ctx, tmp_path):
    check(rdf, ctx, tmp_path, b'\xef\xbb\xbf\n  \r\n{"a": 1}\r\n\t\n{"a": 2, "b": [1, 2]}\r\n\n{"a": 3}')


def test_inference(rdf, ctx, tmp_path):
    data = (b'{"i": 1, "m": 1, "ls": 3, "e": [], "o": {"x": [1, 2]}, "s": "str", "n": null, "bl": [true]}\n'
            b'{"i": -9223372036854775808, "m": 2.5, "ls": [1, 2], "e": [null, 4], "o": {}, "s": "t", "n": null}\n'
            b'{"m": 1e3, "ls": [1.5], "e": []}\n')
    ref, _ = check(rdf, ctx, tmp_path, data)
    assert ref.dtypes == [I64, F64, jo.LIST_BASE + F64, jo.LIST_BASE + I64, -1, -1, -1, -1]
    check(rdf, ctx, tmp_path, data, max_records=1)


def test_explicit_schema_every_type(rdf, ctx, tmp_path):
    rng = np.random.default_rng(5)
    lines = []
    for r in range(300):
        lines.append('{"i8": %d, "i16": %d, "i32": %d, "i64": %d, "u8": %d, "u16": %d, "u32": %d, "u64": %d, "f32": %r, "f64": %r, '
                     '"b": %s, "l8": [%d, null, %d], "lf": [%r], "l64": %d, "skip": "x"}' % (
                         rng.integers(-130, 130), rng.integers(-40000, 40000), rng.integers(-2**31, 2**31), rng.integers(-2**63, 2**63),
                         rng.integers(-5, 260), rng.integers(0, 70000), rng.integers(0, 2**32 + 5), int(rng.integers(0, 2**63)) * 2 + 1,
                         float(rng.normal()), float(rng.normal() * 1e100), "true" if r % 3 else "false", rng.integers(-130, 130),
                         rng.integers(0, 5), float(rng.random()), rng.integers(0, 10)))
    schema = [("i8", I8), ("i16", I16), ("i32", I32), ("i64", I64), ("u8", U8), ("u16", U16), ("u32", U32), ("u64", U64), ("f32", F32),
              ("f64", F64), ("b", BOOL), ("l8", jo.LIST_BASE + I8), ("lf", jo.LIST_BASE + F32), ("l64", jo.LIST_BASE + U64),
              ("skip", -1), ("absent", I32)]
    for bs in (1, 7, 1024):
        check(rdf, ctx, tmp_path, ("\n".join(lines) + "\n").encode(), batch_size=bs, schema=schema)


def test_float_edges(rdf, ctx, tmp_path):
    vals = ["1e308", "1e-400", "-0.0", "0.0", "5e-324", "2.2250738585072011e-308", "4.9406564584124654e-324", "1.7976931348623157e308",
            "1.401298464324817e-45", "3.4028235677973366e38", "0.1000000000000000055511151231257827021181583404541015625",
            "9007199254740993.0000000000000000001", "1.00000005960464477539062500000000000001", "123456789012345678901234567890"]
    data = "".join('{"f": %s, "g": %s}\n' % (v, v) for v in vals).encode()
    ref, exact = check(rdf, ctx, tmp_path, data, schema=[("f", F64), ("g", F32)])
    assert exact > 0   # more than 19 significant digits at a rounding boundary reach the host's exact path


def test_integer_range_edges(rdf, ctx, tmp_path):
    lines = []
    for lo, hi in [(-128, 127), (-32768, 32767), (-2**31, 2**31 - 1), (-2**63, 2**63 - 1)]:
        lines += [str(lo - 1), str(lo), str(hi), str(hi + 1)]
    lines += ["0", "-0", "255", "256", "65535", "65536", str(2**32 - 1), str(2**32), str(2**64 - 1), str(2**64), "1.0", "1e2", "true", '"1"']
    data = "".join('{"v": %s}\n' % v for v in lines).encode()
    for t in range(8):
        check(rdf, ctx, tmp_path, data, schema=[("v", t)])


@pytest.mark.parametrize("bad,line", [(b'{"a": 1}\n[1]', 2), (b'{"a": NaN}', 1), (b'{"a": Infinity}', 1), (b'{"a": +1}', 1),
                                      (b'{"a": 01}', 1), (b'{"a": 1.}', 1), (b'{"a": .5}', 1), (b'\n{"a": "x', 2), (b'{"a": "\\q"}', 1),
                                      (b'{"a": [1}', 1), (b'{"a": 1}}', 1), (b'{"a": 1,}', 1), (b'{"a" 1}', 1), (b'{"a": 1}\n\n\n1', 4)])
def test_malformed(rdf, ctx, tmp_path, bad, line):
    with pytest.raises(jo.JsonError) as ei:
        jo.read(bad)
    assert ei.value.line == line
    p = tmp_path / "bad.json"
    p.write_bytes(bad)
    before = pool_used(ctx)
    with pytest.raises(rdf.ArrowError) as ei:
        rdf.JsonFile(str(p), ctx=ctx)
    assert f"JSON error at line {line}, byte " in str(ei.value)
    assert pool_used(ctx) == before


def test_empty_file_and_refusals(rdf, ctx, tmp_path):
    before = pool_used(ctx)
    for data in (b"", b"\n \r\n\n"):
        p = tmp_path / "e.json"
        p.write_bytes(data)
        with pytest.raises(rdf.ReferencePanic):
            rdf.JsonFile(str(p), ctx=ctx)
    p = tmp_path / "s.json"
    p.write_bytes(b'{"a": "x", "l": [1], "n": 2}\n')
    with rdf.JsonFile(str(p), ctx=ctx) as f:
        with pytest.raises(rdf.UnsupportedType):
            f.read(["a"])
        with pytest.raises(rdf.UnsupportedType):
            f.read(["l"])
        with pytest.raises(rdf.UnsupportedType):
            f.read_list("n")
    with pytest.raises(rdf.UnsupportedType):
        rdf.JsonFile(str(p), schema=[("a", jo.LIST_BASE + BOOL)], ctx=ctx)
    assert pool_used(ctx) == before


def test_large_file(rdf, ctx, tmp_path):
    """1e6 records whose boundaries straddle many tiles of the newline pass; keys in varying order."""
    rng = np.random.default_rng(11)
    n = 1_000_000
    ids = rng.integers(-2**40, 2**40, n)
    xs = rng.normal(size=n)
    lens = rng.integers(0, 5, n)
    parts = []
    for r in range(n):
        tags = ",".join(str(int(t)) for t in range(lens[r]))
        if r % 2:
            parts.append('{"id":%d,"x":%r,"tags":[%s],"ok":%s}' % (ids[r], float(xs[r]), tags, "true" if r % 3 else "false"))
        else:
            parts.append('{"tags":[%s], "x":%r ,"id":%d, "s":"r%d"}' % (tags, float(xs[r]), ids[r], r))
    data = ("\n".join(parts) + "\n").encode()
    check(rdf, ctx, tmp_path, data)


def test_frame_pipeline_against_pandas(rdf, ctx, tmp_path):
    pd = pytest.importorskip("pandas")
    rng = np.random.default_rng(3)
    n = 5000
    k, v = rng.integers(0, 20, n), rng.integers(-1000, 1000, n)
    data = "".join('{"k": %d, "v": %d, "w": %r, "s": "x"}\n' % (k[i], v[i], float(v[i]) / 8) for i in range(n)).encode()
    p = tmp_path / "f.json"
    p.write_bytes(data)
    df = rdf.DeviceFrame.from_json(str(p), ctx=ctx)
    assert list(df.schema) == ["k", "v", "w"]
    pdf = pd.DataFrame({"k": k, "v": v, "w": v / 8})
    host = df.filter(("gt", ("col", "v"), ("scalar", 0))).sort([("v", False)]).to_host()
    want = pdf[pdf.v > 0].sort_values("v", kind="stable")
    assert np.concatenate([c.value_slice() for c in host["v"]]).tolist() == want.v.tolist()
    assert np.concatenate([c.value_slice() for c in host["w"]]).tolist() == want.w.tolist()
    keys, res = rdf.group_by([df.column("k")], [(df.column("v"), "sum")])
    want_g = pdf.groupby("k").v.sum()
    assert keys[0].download()[0].value_slice().tolist() == want_g.index.tolist()
    assert res[0].download()[0].value_slice().tolist() == want_g.tolist()


def test_list_functions(rdf, ctx, tmp_path):
    data = b'{"t": [1, 2, 3]}\n{"t": []}\n{"t": null}\n{"t": [2, null]}\n{"t": 2}\n{}\n{"t": [4]}\n'
    p = tmp_path / "l.json"
    p.write_bytes(data)
    ref = jo.read(data, schema=[("t", jo.LIST_BASE + I32)])
    lists = ref.list_column(0)
    with rdf.JsonFile(str(p), schema=[("t", jo.LIST_BASE + I32)], batch_size=3, ctx=ctx) as f:
        lc = f.read_list("t")
        has2 = []
        for a in lc.array_contains(2).download():
            m = a.valid_mask()
            b = a.value_bits()
            has2 += [bool(b[i]) if m[i] else None for i in range(a.length)]
        assert has2 == [None if l is None else 2 in l for l in lists]
        rows, vals = lc.explode()
        want = [(r, x) for r, l in enumerate(lists) if l for x in l]
        got_rows = rows.download()[0].value_slice().tolist()
        va = vals.download()[0]
        vm = va.valid_mask()
        got = [(r, int(x) if vm[i] else None) for i, (r, x) in enumerate(zip(got_rows, va.value_slice().tolist()))]
        assert got == want
