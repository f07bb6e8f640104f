"""The CSV reader's rules (include/b200df.h "CSV files straight to the device") restated in Python: a byte-level csv-core DFA,
the inference regexes and merge table, and the value grammars with exact conversions.  The checker, never the thing under test.

Floats are converted only after the exact grammar matched (Python's float() also accepts '1_0' and whitespace); float64 comes from
float() (correctly rounded), float32 is rounded from the exact Fraction, ties to even."""
from __future__ import annotations

import math
import re
import struct
from fractions import Fraction
from typing import List, Optional, Sequence

import numpy as np

SR, SF, IF, IQ, QQ = range(5)
I8, I16, I32, I64, U8, U16, U32, U64, F32, F64, BOOL, UTF8 = range(12)
BOM = b"\xef\xbb\xbf"


class CsvError(Exception):
    pass


class ParseError(Exception):
    pass


class Panic(Exception):
    pass


def records(data: bytes, delim: int = ord(",")) -> List[List[bytes]]:
    """csv-core's record DFA: the unquoted fields of every record (a leading UTF-8 BOM is skipped)."""
    if data.startswith(BOM):
        data = data[3:]
    out, rec, cur, st = [], [], bytearray(), SR
    for b in data:
        t = b in (13, 10)
        if st == IQ:
            if b == 34:
                st = QQ
            else:
                cur.append(b)
            continue
        if st == QQ and b == 34:
            cur.append(34)
            st = IQ
            continue
        if st == SR and t:
            continue
        if b == delim:
            rec.append(bytes(cur)); cur = bytearray(); st = SF
        elif t:
            rec.append(bytes(cur)); cur = bytearray(); out.append(rec); rec = []; st = SR
        elif b == 34 and st in (SR, SF):
            st = IQ
        else:
            cur.append(b); st = IF
    if st != SR:
        rec.append(bytes(cur)); out.append(rec)
    return out


def states(data: bytes, delim: int = ord(","), start: int = SR) -> List[int]:
    """The DFA state before every byte of data (records()' transitions, from `start`), and after the last one: len(data) + 1 entries."""
    out, st = [start], start
    for b in data:
        t = b in (13, 10)
        if st == IQ:
            st = QQ if b == 34 else IQ
        elif st == QQ and b == 34:
            st = IQ
        elif b == delim:
            st = SF
        elif t:
            st = SR
        elif b == 34 and st in (SR, SF):
            st = IQ
        else:
            st = IF
        out.append(st)
    return out


_BOOL = re.compile(rb"(?i)^(true)$|^(false)$")
_DEC = re.compile(rb"^-?(\d+\.\d+)$", re.ASCII)
_INT = re.compile(rb"^-?(\d+)$", re.ASCII)


def classify(v: bytes) -> Optional[int]:
    """None for an empty field (a null), else the inferred type of one value."""
    if v == b"":
        return None
    if v.startswith(b'"'):
        return UTF8
    if _BOOL.fullmatch(v) and not v.endswith(b"\n"):
        return BOOL
    if _DEC.fullmatch(v):
        return F64
    if _INT.fullmatch(v):
        return I64
    return UTF8


def merge(types: set) -> int:
    if len(types) == 1:
        return next(iter(types))
    if types == {I64, F64}:
        return F64
    return UTF8


_INT_RE = re.compile(rb"[+-]?[0-9]+")
_FLOAT_RE = re.compile(rb"[+-]?([0-9]+\.?[0-9]*|\.[0-9]+)([eE][+-]?[0-9]+)?")
_SPECIAL_RE = re.compile(rb"([+-]?)(inf|infinity|nan)", re.IGNORECASE)
_BITS = {I8: 8, I16: 16, I32: 32, I64: 64, U8: 8, U16: 16, U32: 32, U64: 64}


def parse_int(v: bytes, dtype: int) -> Optional[int]:
    if not _INT_RE.fullmatch(v):
        return None
    x = int(v)
    bits = _BITS[dtype]
    if dtype >= U8:
        return x if (not v.startswith(b"-") and x < 1 << bits) else None
    return x if -(1 << (bits - 1)) <= x < 1 << (bits - 1) else None


def f32_from_fraction(x: Fraction) -> float:
    """x rounded to the nearest float32, ties to even (overflow to inf)."""
    if x == 0:
        return 0.0
    neg, a = x < 0, abs(x)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    e = max(e, -126)
    q = Fraction(2) ** (e - 23)
    m = a / q
    n = math.floor(m)
    r = m - n
    if r > Fraction(1, 2) or (r == Fraction(1, 2) and n % 2 == 1):
        n += 1
    v = n * q
    if v >= Fraction(2) ** 128:
        return -math.inf if neg else math.inf
    return -float(v) if neg else float(v)


def parse_float_bits(v: bytes, dtype: int) -> Optional[int]:
    """The bit pattern of Rust's FromStr for f32 / f64, or None."""
    m = _SPECIAL_RE.fullmatch(v)
    if m:
        neg = m.group(1) == b"-"
        if m.group(2).lower() == b"nan":
            bits = 0x7FF8000000000000 if dtype == F64 else 0x7FC00000
        else:
            bits = 0x7FF0000000000000 if dtype == F64 else 0x7F800000
        return bits | ((1 << 63 if dtype == F64 else 1 << 31) if neg else 0)
    if not _FLOAT_RE.fullmatch(v):
        return None
    s = v.decode()
    if dtype == F64:
        return struct.unpack("<Q", struct.pack("<d", float(s)))[0]
    mant, _, exp = s.lower().partition("e")
    sign = -1 if mant.startswith("-") else 1
    mant = mant.lstrip("+-")
    ip, _, fp = mant.partition(".")
    digits = int(ip + fp or "0")
    scale = (int(exp) if exp else 0) - len(fp)   # value = digits * 10^scale, exactly
    mag = scale + len(str(digits))                # digits * 10^scale < 10^mag
    if digits == 0 or mag < -60:                  # below half the smallest subnormal (1.4e-45): zero
        x = Fraction(0)
    elif mag > 60:                                # at least 10^59: above the largest float32, infinity
        x = Fraction(10) ** 60
    else:
        x = Fraction(digits) * Fraction(10) ** scale
    f = f32_from_fraction(x)
    bits = struct.unpack("<I", struct.pack("<f", f))[0]
    return bits | (1 << 31 if sign < 0 else 0)


def parse_bool(v: bytes) -> Optional[bool]:
    s = v.decode("utf-8", "replace").lower()
    return True if s == "true" else False if s == "false" else None


class Table:
    def __init__(self, names, dtypes, nullable, rows, has_header, batch_size):
        self.names, self.dtypes, self.nullable = names, dtypes, nullable
        self.rows, self.has_header, self.batch_size = rows, has_header, batch_size

    @property
    def num_rows(self) -> int:
        return len(self.rows)

    def column(self, i: int):
        """(values, valid) as numpy: values are the bit patterns' dtype (float columns as uint bits)."""
        dt = self.dtypes[i]
        vals, valid = [], []
        for r, rec in enumerate(self.rows):
            v = rec[i]
            if v == b"":
                vals.append(0); valid.append(False); continue
            if dt == BOOL:
                x = parse_bool(v)
            elif dt in (F32, F64):
                x = parse_float_bits(v, dt)
            else:
                x = parse_int(v, dt)
            if x is None:
                raise ParseError(f"Error while parsing value {v.decode('utf-8', 'replace')} for column {i} at line {r + self.has_header}")
            vals.append(int(x)); valid.append(True)
        np_dt = {F32: np.uint32, F64: np.uint64, BOOL: np.bool_}.get(dt)
        if np_dt is None:
            np_dt = {I8: np.int8, I16: np.int16, I32: np.int32, I64: np.int64, U8: np.uint8, U16: np.uint16, U32: np.uint32, U64: np.uint64}[dt]
        return np.array(vals, dtype=object).astype(np_dt) if vals else np.zeros(0, np_dt), np.array(valid, dtype=bool)


def read(data: bytes, has_header: bool = True, delimiter: str = ",", max_records: Optional[int] = None, batch_size: int = 1024,
         schema: Optional[Sequence[int]] = None) -> Table:
    recs = records(data, ord(delimiter))
    if not recs:
        raise Panic("no records")
    k = len(recs[0])
    for r, rec in enumerate(recs):
        if len(rec) != k:
            raise CsvError(f"found record with {len(rec)} fields, but the previous record has {k} fields (record {r})")
    names = [v.decode("utf-8", "replace") for v in recs[0]] if has_header else [f"column_{i + 1}" for i in range(k)]
    rows = recs[1:] if has_header else recs
    if not rows:
        raise Panic("no data records")
    if schema is not None:
        dtypes = [UTF8 if t in (UTF8, -1) else t for t in schema]
        nullable = [True] * k
    else:
        look = rows if max_records is None else rows[:max_records]
        dtypes, nullable = [], []
        for i in range(k):
            cls = [classify(rec[i]) for rec in look]
            dtypes.append(merge({c for c in cls if c is not None}) if any(c is not None for c in cls) else UTF8)
            nullable.append(any(c is None for c in cls))
    return Table(names, dtypes, nullable, rows, 1 if has_header else 0, batch_size)
