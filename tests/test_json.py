"""The line-delimited JSON oracle (tests/json_oracle.py) against pyarrow's JSON reader where the two agree, and on hand-written cases
for every rule of include/b200df.h, the departures included.  No GPU needed."""
import io
import struct

import numpy as np
import pytest

import json_oracle as jo
from csv_oracle import BOOL, F32, F64, I8, I64, U8, U64

pa = pytest.importorskip("pyarrow")
pajson = pytest.importorskip("pyarrow.json")


def gen_file(rng, n):
    """Seeded records with int / float / bool / null / numeric-list keys, missing keys and keys in varying order."""
    lines = []
    for _ in range(n):
        items = []
        if rng.random() < 0.9:
            items.append(("id", str(int(rng.integers(-2**62, 2**62)))))
        if rng.random() < 0.8:
            items.append(("x", "null" if rng.random() < 0.1 else repr(float(rng.normal() * 10 ** int(rng.integers(-5, 6))))))
        if rng.random() < 0.8:
            items.append(("mix", str(int(rng.integers(-99, 99))) if rng.random() < 0.5 else repr(float(rng.random()))))
        if rng.random() < 0.8:
            items.append(("ok", "true" if rng.random() < 0.5 else "false"))
        if rng.random() < 0.8:
            k = int(rng.integers(0, 4))
            items.append(("tags", "[" + ", ".join(str(int(t)) for t in rng.integers(0, 100, k)) + "]"))
        rng.shuffle(items)
        lines.append("{" + ", ".join(f'"{k}": {v}' for k, v in items) + "}")
    return ("\n".join(lines) + "\n").encode()


@pytest.mark.parametrize("seed,batch", [(1, 1024), (2, 7), (3, 100)])
def test_oracle_matches_pyarrow(seed, batch):
    rng = np.random.default_rng(seed)
    data = gen_file(rng, 500)
    ref = jo.read(data, batch_size=batch)
    t = pajson.read_json(io.BytesIO(data), read_options=pajson.ReadOptions(block_size=1 << 20))
    assert set(ref.names) == set(t.column_names)
    for i, name in enumerate(ref.names):
        col = t.column(name).to_pylist()
        typ = t.schema.field(name).type
        if ref.dtypes[i] >= jo.LIST_BASE:
            assert pa.types.is_list(typ)
            got = ref.list_column(i)
            want = [None if v is None else [None if x is None else int(x) for x in v] for v in col]
            assert got == want
            continue
        assert ref.dtypes[i] == {pa.int64(): I64, pa.float64(): F64, pa.bool_(): BOOL}[typ]
        vals, valid = ref.column(i)
        assert valid.tolist() == [v is not None for v in col]
        for v, m, w in zip(vals.tolist(), valid.tolist(), col):
            if not m:
                continue
            if typ == pa.float64():
                assert v == struct.unpack("<Q", struct.pack("<d", w))[0]
            else:
                assert v == w


def test_records_and_errors():
    assert jo.read(b'\xef\xbb\xbf{"a": 1}\r\n\n  \t\r\n{"a": 2}').column(0)[0].tolist() == [1, 2]   # BOM, CRLF, blank lines, no final \n
    for bad, line in [(b'{"a": 1}\n[1]', 2), (b'{"a": NaN}', 1), (b'{"a": Infinity}', 1), (b'{"a": +1}', 1), (b'{"a": 01}', 1),
                      (b'{"a": 1.}', 1), (b'{"a": .5}', 1), (b'\n{"a": "x', 2), (b'{"a": "\\q"}', 1), (b'{"a": [1}', 1), (b'{"a": 1}}', 1),
                      (b'{"a": 1,}', 1), (b'{"a" 1}', 1), (b'1', 1)]:
        with pytest.raises(jo.JsonError) as ei:
            jo.read(bad)
        assert ei.value.line == line, bad
    with pytest.raises(jo.Panic):
        jo.read(b"")
    with pytest.raises(jo.Panic):
        jo.read(b"\n \n\r\n")


def test_keys_order_and_last_wins():
    t = jo.read(b'{"b": 1, "a": 2, "b": 3}\n{"c": true, "\\u0061": 5}')
    assert t.names == ["b", "a", "c"]
    assert t.column(0)[0].tolist() == [3, 0] and t.column(0)[1].tolist() == [True, False]
    assert t.column(1)[0].tolist() == [2, 5]
    assert t.nullable == [True, False, True]


def test_inference_table():
    cases = [
        (b'{"a": 1}\n{"a": 2.5}', F64), (b'{"a": 1}\n{"a": 9223372036854775808}', F64), (b'{"a": -9223372036854775808}', I64),
        (b'{"a": true}\n{"a": null}', BOOL), (b'{"a": [1, 2]}\n{"a": [1.5]}', jo.LIST_BASE + F64), (b'{"a": 3}\n{"a": [1]}', jo.LIST_BASE + I64),
        (b'{"a": [null]}\n{"a": []}\n{"a": [1]}', jo.LIST_BASE + I64), (b'{"a": []}', -1), (b'{"a": "x"}', -1), (b'{"a": {"b": 1}}', -1),
        (b'{"a": true}\n{"a": 1}', -1), (b'{"a": [[1]]}', -1), (b'{"a": [true]}', -1), (b'{"a": null}', -1), (b'{"a": [1, "x"]}', -1),
    ]
    for data, want in cases:
        assert jo.read(data).dtypes == [want], data


def test_max_records_and_schema():
    data = b'{"a": 1}\n{"a": 1.5, "b": true}'
    t = jo.read(data, max_records=1)
    assert t.names == ["a"] and t.dtypes == [I64]
    assert t.column(0)[1].tolist() == [True, False]   # 1.5 does not convert to Int64: NULL
    t = jo.read(data, schema=[("b", BOOL), ("z", F32), ("a", U8)])
    assert t.column(0)[1].tolist() == [False, True]
    assert t.column(1)[1].tolist() == [False, False]
    assert t.column(2)[0].tolist() == [1, 0] and t.column(2)[1].tolist() == [True, False]


def test_values():
    data = b'{"i": -0, "u": -0, "f": 1e-400, "g": 1e400, "s": "1", "l": 5, "b": 1}\n{"i": 128, "u": 255, "f": -0.0, "g": 0.1, "s": 2, "l": [1, null, 1.5, 300], "b": false}'
    t = jo.read(data, schema=[("i", I8), ("u", U8), ("f", F64), ("g", F32), ("s", U64), ("l", jo.LIST_BASE + U8), ("b", BOOL)])
    assert t.column(0)[1].tolist() == [True, False]
    assert t.column(1)[1].tolist() == [False, True]
    assert t.column(2)[0].tolist() == [0, 1 << 63]
    assert t.column(3)[0].tolist() == [0x7F800000, struct.unpack("<I", struct.pack("<f", 0.1))[0]]
    assert t.column(4)[1].tolist() == [False, True]
    assert t.list_column(5) == [[5], [1, None, None, None]]
    assert t.column(6)[1].tolist() == [False, True]


def test_pyarrow_departure_on_nonconforming_values():
    """Departure 4: a value that does not convert is NULL here; pyarrow refuses the file."""
    data = b'{"a": 1}\n{"a": "x"}'
    assert jo.read(data, schema=[("a", I64)]).column(0)[1].tolist() == [True, False]
    with pytest.raises(pa.ArrowInvalid):
        pajson.read_json(io.BytesIO(data), parse_options=pajson.ParseOptions(explicit_schema=pa.schema([("a", pa.int64())])))
