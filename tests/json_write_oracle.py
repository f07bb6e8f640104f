"""The JSON writer's rules (include/b200df.h "line-delimited JSON files straight from the device") restated in Python from the header
alone: ryu's float layout over numpy's shortest digits, chrono's years, RFC 3339 suffixes and serde_json's name escapes.

A column is a dict: name, dtype (0..9, BOOL), values (numpy array), valid (bool array or None), and optionally temporal = (kind, unit,
tz) or lists = a Python list of rows, each None (a null list) or a list of element values (None for a null element)."""
from __future__ import annotations

import math

import numpy as np

BOOL = 10
F32, F64 = 8, 9
DATE32, DATE64, TIMESTAMP, TIME32, TIME64 = 1, 2, 3, 4, 5
SECOND, MILLISECOND, MICROSECOND, NANOSECOND = 0, 1, 2, 3
PER_SEC = [1, 1000, 1000000, 1000000000]
MIN_DAY, MAX_DAY = -96465658, 95026601   # chrono's NaiveDate range


def format_float(v, f32: bool):
    """The text of a float, or None for NaN / inf (written as null)."""
    v = np.float32(v) if f32 else np.float64(v)
    if not np.isfinite(v):
        return None
    neg = bool(np.signbit(v))
    if v == 0:
        return "-0.0" if neg else "0.0"
    sci = np.format_float_scientific(abs(v), unique=True, trim="-")   # shortest digits in the value's own type
    mant, exp = sci.split("e")
    digits = mant.replace(".", "").rstrip("0") or "0"
    kk = int(exp) + 1
    n = len(digits)
    top, low = (13, -6) if f32 else (16, -5)
    if n <= kk <= top:
        s = digits + "0" * (kk - n) + ".0"
    elif 0 < kk <= top:
        s = digits[:kk] + "." + digits[kk:]
    elif low < kk <= 0:
        s = "0." + "0" * (-kk) + digits
    else:
        s = digits[0] + ("." + digits[1:] if n > 1 else "") + "e" + str(kk - 1)
    return ("-" if neg else "") + s


def format_f64_repr(v: float) -> str:
    """format_float(v, False) (with "null" for NaN / inf) from repr's shortest, closest digits: much faster for millions of values."""
    if math.isnan(v) or math.isinf(v):
        return "null"
    if v == 0:
        return "-0.0" if math.copysign(1.0, v) < 0 else "0.0"
    r = repr(abs(v))
    mant, _, exp = r.partition("e")
    ip, _, fp = mant.partition(".")
    digits = (ip + fp).lstrip("0")
    kk = len(ip.lstrip("0")) + int(exp or 0) if ip.strip("0") else int(exp or 0) - (len(fp) - len(fp.lstrip("0")))
    digits = digits.rstrip("0")
    n = len(digits)
    if n <= kk <= 16:
        s = digits + "0" * (kk - n) + ".0"
    elif 0 < kk <= 16:
        s = digits[:kk] + "." + digits[kk:]
    elif -5 < kk <= 0:
        s = "0." + "0" * (-kk) + digits
    else:
        s = digits[0] + ("." + digits[1:] if n > 1 else "") + "e" + str(kk - 1)
    return ("-" if v < 0 else "") + s


def format_scalar(dtype: int, v):
    if dtype == BOOL:
        return "true" if v else "false"
    if dtype in (F32, F64):
        return format_float(v, dtype == F32)
    return str(int(v))


def civil_from_days(z: int):
    """Hinnant's civil_from_days in Python's unbounded integers (// is floor division already)."""
    z += 719468
    era = z // 146097
    doe = z - era * 146097
    yoe = (doe - doe // 1460 + doe // 36524 - doe // 146096) // 365
    y = yoe + era * 400
    doy = doe - (365 * yoe + yoe // 4 - yoe // 100)
    mp = (5 * doy + 2) // 153
    d = doy - (153 * mp + 2) // 5 + 1
    m = mp + 3 if mp < 10 else mp - 9
    return y + (m <= 2), m, d


def chrono_year(y: int) -> str:
    """chrono's %Y: 4 digits for 0..9999, '+' and the digits above, '-' and at least 4 digits below 0."""
    if 0 <= y <= 9999:
        return f"{y:04d}"
    if y > 9999:
        return f"+{y}"
    return f"-{-y:04d}"


def tz_suffix(tz):
    """(offset in seconds, suffix) of a Timestamp tz; raises ValueError for a named zone."""
    if tz is None:
        return 0, ""
    if tz in ("UTC", "Z", "+00:00"):
        return 0, "Z"
    if len(tz) == 6 and tz[0] in "+-" and tz[1:3].isdigit() and tz[3] == ":" and tz[4:].isdigit() and int(tz[1:3]) <= 23 and int(tz[4:]) <= 59:
        sec = (int(tz[1:3]) * 3600 + int(tz[4:]) * 60) * (-1 if tz[0] == "-" else 1)
        return sec, tz
    raise ValueError(f"named zone {tz!r}")


def format_temporal(temporal, v: int) -> str:
    kind, unit, tz = temporal
    v = int(v)
    if kind == DATE32:
        if not MIN_DAY <= v <= MAX_DAY:
            raise ValueError(f"date {v} out of range")
        y, m, d = civil_from_days(v)
        return f'"{chrono_year(y)}-{m:02d}-{d:02d}"'
    ups = 1000 if kind == DATE64 else PER_SEC[unit]
    upd = 86400 * ups
    if kind in (TIME32, TIME64):
        if not 0 <= v < upd:
            raise ValueError(f"time of day {v} out of range")
        days, tod = 0, v
    else:
        off = tz_suffix(tz)[0] * ups if kind == TIMESTAMP else 0
        days, tod = divmod(v + off, upd)   # floor division
        if not MIN_DAY <= days <= MAX_DAY:
            raise ValueError(f"date {v} out of range")
    frac_digits = 0 if kind == DATE64 else 3 * unit
    secs, sub = divmod(tod, ups)
    clock = f"{secs // 3600:02d}:{secs // 60 % 60:02d}:{secs % 60:02d}" + (f".{sub:0{frac_digits}d}" if frac_digits else "")
    if kind in (TIME32, TIME64):
        return f'"{clock}"'
    y, m, d = civil_from_days(days)
    date = f"{chrono_year(y)}-{m:02d}-{d:02d}"
    if kind == DATE64:
        return f'"{date}"'
    return f'"{date}T{clock}{tz_suffix(tz)[1]}"'


def escape_name(name: str) -> str:
    """serde_json's string escapes over the name's UTF-8 bytes, in quotes."""
    out = bytearray(b'"')
    short = {0x22: b'\\"', 0x5C: b"\\\\", 0x08: b"\\b", 0x0C: b"\\f", 0x0A: b"\\n", 0x0D: b"\\r", 0x09: b"\\t"}
    for ch in name.encode():
        if ch in short:
            out += short[ch]
        elif ch < 0x20:
            out += b"\\u%04x" % ch
        else:
            out.append(ch)
    out += b'"'
    return out.decode()


def date_slots(days: np.ndarray, width: int = 16) -> np.ndarray:
    """The Date32 text of each day (quotes included), left-aligned in `width` zero-padded bytes: the vectorised form of
    format_temporal for (DATE32, 0, None), for checking millions of days at once."""
    z = days.astype(np.int64) + 719468
    era = z // 146097   # numpy's // floors
    doe = z - era * 146097
    yoe = (doe - doe // 1460 + doe // 36524 - doe // 146096) // 365
    doy = doe - (365 * yoe + yoe // 4 - yoe // 100)
    mp = (5 * doy + 2) // 153
    d = doy - (153 * mp + 2) // 5 + 1
    m = np.where(mp < 10, mp + 3, mp - 9)
    y = yoe + era * 400 + (m <= 2)
    mag = np.abs(y)
    ndig = np.maximum(4, np.floor(np.log10(np.maximum(mag, 1))).astype(np.int64) + 1)
    ndig = ndig + (mag >= 10 ** ndig) - (mag < 10 ** (ndig - 1)) * (ndig > 4)   # exact at powers of ten
    sign = (y < 0) | (y > 9999)
    ylen = ndig + sign
    out = np.zeros((len(days), width), np.uint8)
    rows = np.arange(len(days))
    out[:, 0] = ord('"')
    out[sign, 1] = np.where(y[sign] < 0, ord("-"), ord("+"))
    for k in range(int(ndig.max()) if len(days) else 0):   # digit k from the right of the year
        has = k < ndig
        col = sign + ndig - k   # 1-based position after the quote
        out[rows[has], col[has]] = ord("0") + (mag[has] // 10 ** k) % 10
    tail = np.stack([np.full_like(m, ord("-")), ord("0") + m // 10, ord("0") + m % 10, np.full_like(m, ord("-")),
                     ord("0") + d // 10, ord("0") + d % 10, np.full_like(m, ord('"'))], axis=1)
    for k in range(7):
        out[rows, 1 + ylen + k] = tail[:, k]
    return out


def _value(col, r):
    """The text of row r's member, or None for a NULL member."""
    if col.get("lists") is not None:
        row = col["lists"][r]
        if row is None:
            return None
        parts = []
        for x in row:
            t = None if x is None else format_scalar(col["dtype"], x)
            parts.append("null" if t is None else t)
        return "[" + ",".join(parts) + "]"
    if col.get("valid") is not None and not col["valid"][r]:
        return None
    v = col["values"][r]
    if col.get("temporal") is not None:
        return format_temporal(col["temporal"], v)
    return format_scalar(col["dtype"], v)


def n_rows(col) -> int:
    return len(col["lists"]) if col.get("lists") is not None else len(col["values"])


def write(cols, explicit_nulls: bool = False) -> bytes:
    n = n_rows(cols[0]) if cols else 0
    names = [escape_name(c["name"]) + ":" for c in cols]
    lines = []
    for r in range(n):
        members = []
        for c, nm in zip(cols, names):
            t = _value(c, r)
            if t is None:
                if explicit_nulls:
                    members.append(nm + "null")
                continue
            members.append(nm + t)
        lines.append("{" + ",".join(members) + "}\n")
    return "".join(lines).encode()
