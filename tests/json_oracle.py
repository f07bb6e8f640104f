"""The line-delimited JSON reader's rules (include/b200df.h) restated in plain Python: json.loads with hooks that keep the key order
and the number literals, then the inference table and the conversions.  Float64 values come from float(), Float32 values from
csv_oracle's exact rounding (f32_from_fraction through parse_float_bits)."""
from __future__ import annotations

import json
from typing import List, Optional, Sequence, Tuple

import numpy as np

import csv_oracle as co
from csv_oracle import BOOL, BOM, F32, F64, I64, UTF8

LIST_BASE = 32
NP = [np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64, np.uint32, np.uint64]   # floats as bits

# value classes (json_parse.cuh)
NULL, BOOLC, INT, FLOAT, STR, OBJ, LIST_INT, LIST_FLOAT, LIST_OTHER, LIST_EMPTY, MISSING = (1 << i for i in range(11))


class JsonError(Exception):
    def __init__(self, line: int, what: str):
        super().__init__(f"JSON error at line {line}: {what}")
        self.line = line


class Panic(Exception):
    pass


class Int(str):
    """An integer literal, its text kept."""


class Flt(str):
    """A number literal with a fraction or an exponent, its text kept."""


class Obj(list):
    """An object: its (key, value) pairs in order, repeats included."""


def _constant(s):
    raise ValueError(f"{s} is not JSON")


def records(data: bytes) -> List[Obj]:
    """The records of a file; JsonError(line) for a malformed one."""
    if data.startswith(BOM):
        data = data[3:]
    out = []
    for i, line in enumerate(data.split(b"\n")):
        if not line.strip(b" \t\r\n"):
            continue
        try:
            obj = json.loads(line.decode("utf-8"), object_pairs_hook=Obj, parse_int=Int, parse_float=Flt, parse_constant=_constant)
        except ValueError as e:
            raise JsonError(i + 1, str(e)) from None
        if not isinstance(obj, Obj):
            raise JsonError(i + 1, "the record is not an object")
        out.append(obj)
    return out


def classify(v) -> int:
    if v is None:
        return NULL
    if isinstance(v, bool):
        return BOOLC
    if isinstance(v, Int):
        return INT if -(1 << 63) <= int(v) < (1 << 63) else FLOAT
    if isinstance(v, Flt):
        return FLOAT
    if isinstance(v, str):
        return STR
    if isinstance(v, Obj):
        return OBJ
    el = 0
    for x in v:
        c = classify(x)
        el |= OBJ if c & (LIST_INT | LIST_FLOAT | LIST_OTHER | LIST_EMPTY) else c
    if el & (BOOLC | STR | OBJ):
        return LIST_OTHER
    return LIST_FLOAT if el & FLOAT else LIST_INT if el & INT else LIST_EMPTY


def coerce(bits: int) -> int:
    t = bits & ~(NULL | MISSING)
    if t & (STR | OBJ | LIST_OTHER):
        return -1
    if t & BOOLC:
        return BOOL if t == BOOLC else -1
    lst = t & (LIST_INT | LIST_FLOAT | LIST_EMPTY)
    fl, it = t & (FLOAT | LIST_FLOAT), t & (INT | LIST_INT)
    if not fl and not it:
        return -1
    scalar = F64 if fl else I64
    return LIST_BASE + scalar if lst else scalar


def convert(v, dtype: int) -> Optional[int]:
    """The scalar's value (floats as bits), or None when it does not convert."""
    if dtype == BOOL:
        return int(v) if isinstance(v, bool) else None
    if not isinstance(v, (Int, Flt)):
        return None
    if dtype in (F32, F64):
        return co.parse_float_bits(v.encode(), dtype)
    return co.parse_int(v.encode(), dtype)


class Table:
    def __init__(self, names, dtypes, nullable, rows, batch_size):
        self.names, self.dtypes, self.nullable, self.rows, self.batch_size = names, dtypes, nullable, rows, batch_size

    @property
    def num_rows(self) -> int:
        return len(self.rows)

    def cells(self, i: int) -> list:
        name = self.names[i]
        return [r.get(name) if name in r else None for r in self.rows]

    def column(self, i: int) -> Tuple[np.ndarray, np.ndarray]:
        """(values, valid): the value bits in the column's numpy type (floats as unsigned bits, Boolean as bool), NULL slots 0."""
        dt = self.dtypes[i]
        vals, valid = [], []
        for v in self.cells(i):
            x = convert(v, dt) if v is not None else None
            vals.append(0 if x is None else x)
            valid.append(x is not None)
        np_dt = np.bool_ if dt == BOOL else NP[dt]
        return np.array(vals, dtype=object).astype(np_dt) if vals else np.zeros(0, np_dt), np.array(valid, dtype=bool)

    def list_column(self, i: int) -> list:
        """Per row: None (a NULL list) or the element bits, None for a null element."""
        t = self.dtypes[i] - LIST_BASE
        out = []
        for v in self.cells(i):
            if isinstance(v, list) and not isinstance(v, Obj):
                out.append([None if x is None else convert(x, t) for x in v])
            elif isinstance(v, (Int, Flt)):
                out.append([convert(v, t)])
            else:
                out.append(None)
        return out


def read(data: bytes, schema: Optional[Sequence[Tuple[str, int]]] = None, max_records: Optional[int] = None, batch_size: int = 1024) -> Table:
    recs = records(data)
    if not recs:
        raise Panic("no records")
    rows = []
    order = {}   # keys in the order first seen
    for r in recs:
        d = {}
        for k, v in r:
            d[k] = v   # the last value wins
            order.setdefault(k)
        rows.append(d)
    if schema is not None:
        names = [n for n, _ in schema]
        dtypes = [-1 if t in (UTF8, -1) else t for _, t in schema]
        nullable = [True] * len(names)
    else:
        look = rows if max_records is None or max_records < 0 else rows[:max_records]
        names = [k for k in order if any(k in r for r in look)]
        dtypes, nullable = [], []
        for k in names:
            bits = 0
            for r in look:
                bits |= classify(r[k]) if k in r else MISSING
            dtypes.append(coerce(bits))
            nullable.append(bool(bits & (NULL | MISSING)))
    return Table(names, dtypes, nullable, rows, batch_size)
