"""A restatement of the CSV writer's rules (include/b200df.h, "CSV files straight from the device") in numpy and Python.

Columns are (name, dtype, values, valid) with dtype 0..9 or 10 (Boolean), values a numpy array of the native type (bool for Boolean)
and valid a bool mask or None.  Floats: numpy's shortest round-trip digits in the value's own type (format_float_positional with
unique=True), with Rust's spellings of the special values.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np

BOOL = 10
F32, F64 = 8, 9
REFUSED_DELIMITERS = b"0123456789-.\"\r\nNaintruefls\x00"

Column = Tuple[str, int, np.ndarray, Optional[np.ndarray]]


def format_float(v) -> str:
    """Rust's Display of an f32 / f64 (the numpy scalar's own type decides which)."""
    if np.isnan(v):
        return "NaN"
    if np.isinf(v):
        return "inf" if v > 0 else "-inf"
    if v == 0:
        return "-0" if np.signbit(v) else "0"
    return np.format_float_positional(v, unique=True, trim="-")


def format_values(dtype: int, values: np.ndarray) -> List[str]:
    if dtype == BOOL:
        return ["true" if b else "false" for b in values.tolist()]
    if dtype in (F32, F64):
        return [format_float(v) for v in values]
    return [str(int(v)) for v in values.tolist()]


def quote_name(name: str, delim: str, only: bool) -> str:
    if (only and name == "") or any(ch in name for ch in ('"', "\r", "\n", delim)):
        return '"' + name.replace('"', '""') + '"'
    return name


def header(names: Sequence[str], delim: str = ",") -> str:
    return delim.join(quote_name(n, delim, len(names) == 1) for n in names) + "\n"


def write(columns: Sequence[Column], has_header: bool = True, delim: str = ",") -> bytes:
    assert delim.encode() not in REFUSED_DELIMITERS
    rows = len(columns[0][2]) if columns else 0
    fields = []
    for _, dt, vals, valid in columns:
        text = format_values(dt, vals)
        if valid is not None:
            text = [t if ok else "" for t, ok in zip(text, valid.tolist())]
        fields.append(text)
    out = [header([c[0] for c in columns], delim)] if has_header else []
    one = len(columns) == 1
    for r in range(rows):
        rec = delim.join(f[r] for f in fields)
        out.append(('""' if one and rec == "" else rec) + "\n")
    return "".join(out).encode()
