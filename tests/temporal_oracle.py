"""The rules of include/b200df.h "dates and timestamps", restated in vectorised numpy int64 (no datetime, no pyarrow): floor division
into (days, time of day), Hinnant's civil_from_days / days_from_civil, chrono's date range, the Spark 2.4 rules and the fixed
MONTHS_BETWEEN double sequence.  Every function returns (values, valid) with values 0 under NULL, as the device writes them."""
import numpy as np

MIN_DAY, MAX_DAY = -96465658, 95026601          # -262144-01-01 ..= 262143-12-31
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
DATE32, DATE64, TIMESTAMP, TIME32, TIME64 = range(1, 6)
PER_SEC = [1, 1000, 1000000, 1000000000]

FNS = ["year", "quarter", "month", "day_of_month", "day_of_year", "day_of_week", "hour", "minute", "second", "to_date", "date_add",
       "date_sub", "add_months", "last_day", "next_day", "date_trunc", "unix_timestamp", "to_timestamp"]
TRUNC = ["year", "quarter", "month", "week", "day", "hour", "minute", "second"]


def per_day(kind, unit):
    """Units per day of the stored value (1 for Date32) and units per second."""
    if kind == DATE32:
        return 1, 1
    if kind == DATE64:
        return 86400000, 1000
    return 86400 * PER_SEC[unit], PER_SEC[unit]


def tz_offset_seconds(tz):
    """Fixed offset of a tz string, or None for a named zone (the device refuses those for civil functions)."""
    if tz is None or tz in ("UTC", "Z"):
        return 0
    if len(tz) == 6 and tz[0] in "+-" and tz[1:3].isdigit() and tz[3] == ":" and tz[4:6].isdigit():
        hh, mm = int(tz[1:3]), int(tz[4:6])
        if hh <= 23 and mm <= 59:
            return (-1 if tz[0] == "-" else 1) * (hh * 3600 + mm * 60)
    return None


def civil_from_days(z):
    z = np.asarray(z, dtype=np.int64) + 719468
    era = z // 146097
    doe = z - era * 146097
    yoe = (doe - doe // 1460 + doe // 36524 - doe // 146096) // 365
    doy = doe - (365 * yoe + yoe // 4 - yoe // 100)
    mp = (5 * doy + 2) // 153
    d = doy - (153 * mp + 2) // 5 + 1
    m = np.where(mp < 10, mp + 3, mp - 9)
    y = yoe + era * 400 + (m <= 2)
    return y, m, d


def days_from_civil(y, m, d):
    y = np.asarray(y, dtype=np.int64) - (np.asarray(m) <= 2)
    m = np.asarray(m, dtype=np.int64)
    era = y // 400
    yoe = y - era * 400
    doy = (153 * np.where(m > 2, m - 3, m + 9) + 2) // 5 + np.asarray(d, dtype=np.int64) - 1
    doe = yoe * 365 + yoe // 4 - yoe // 100 + doy
    return era * 146097 + doe - 719468


def days_in_month(y, m):
    y = np.asarray(y, dtype=np.int64)
    m = np.asarray(m, dtype=np.int64)
    leap = (y % 4 == 0) & ((y % 100 != 0) | (y % 400 == 0))
    return np.where(m == 2, np.where(leap, 29, 28), np.where((m == 4) | (m == 6) | (m == 9) | (m == 11), 30, 31))


def split(v, kind, unit, off_sec=0):
    """(days, time of day) by floor division, then a fixed offset in seconds applied (local time)."""
    v = np.asarray(v, dtype=np.int64)
    upd, ups = per_day(kind, unit)
    if upd == 1:
        return v.copy(), np.zeros_like(v)
    days = v // upd
    tod = v - days * upd + off_sec * ups
    days = days + (tod >= upd) - (tod < 0)
    tod = np.where(tod >= upd, tod - upd, np.where(tod < 0, tod + upd, tod))
    return days, tod


def in_range(days):
    return (days >= MIN_DAY) & (days <= MAX_DAY)


def result_dtype(fn, kind):
    if fn in ("to_date", "date_add", "date_sub", "add_months", "last_day", "next_day"):
        return np.int32
    if fn == "date_trunc":
        return np.int32 if kind in (DATE32, TIME32) else np.int64
    if fn in ("unix_timestamp", "to_timestamp"):
        return np.int64
    return np.int32


def unary(fn, kind, unit, tz, values, valid, arg=0):
    """One temporal function over a column of stored values; valid is the input validity.  Returns (values, valid)."""
    v = np.asarray(values, dtype=np.int64)
    valid = np.asarray(valid, dtype=bool).copy()
    upd, ups = per_day(kind, unit)
    odt = result_dtype(fn, kind)
    if kind in (TIME32, TIME64):
        ok = valid & (v >= 0) & (v < upd)
        t = np.where(ok, v, 0)
        r = {"hour": t // (3600 * ups), "minute": (t // (60 * ups)) % 60, "second": (t // ups) % 60}[fn]
        return np.where(ok, r, 0).astype(odt), ok
    if fn in ("unix_timestamp", "to_timestamp"):
        days, tod = split(v, kind, unit, 0)
        ok = valid & in_range(days)
        if fn == "unix_timestamp":
            r = np.where(ok, days, 0) * 86400 + np.where(ok, tod, 0) // ups
            return np.where(ok, r, 0).astype(np.int64), ok
        dst = PER_SEC[arg]
        if kind == DATE32:
            mul, div = 86400 * dst, 1
        else:
            mul, div = (dst // ups, 1) if dst >= ups else (1, ups // dst)
        if div > 1:
            r = v // div
        else:
            fits = (v <= I64_MAX // mul) & (v >= -((1 << 63) // mul))
            ok &= fits
            r = np.where(fits, v, 0) * mul
        return np.where(ok, r, 0).astype(np.int64), ok
    off = tz_offset_seconds(tz) if kind == TIMESTAMP else 0
    assert off is not None, "a named zone is refused"
    days, tod = split(v, kind, unit, off)
    ok = valid & in_range(days)
    d = np.where(ok, days, 0)
    tod = np.where(ok, tod, 0)
    y, m, dd = civil_from_days(d)
    if fn == "year":
        r = y
    elif fn == "quarter":
        r = (m - 1) // 3 + 1
    elif fn == "month":
        r = m
    elif fn == "day_of_month":
        r = dd
    elif fn == "day_of_year":
        r = d - days_from_civil(y, 1, 1) + 1
    elif fn == "day_of_week":
        r = (d + 4) % 7 + 1
    elif fn in ("hour", "minute", "second"):
        if upd == 1:
            r = np.zeros_like(d)
        else:
            r = {"hour": tod // (3600 * ups), "minute": (tod // (60 * ups)) % 60, "second": (tod // ups) % 60}[fn]
    elif fn == "to_date":
        r = d
    elif fn in ("date_add", "date_sub"):
        r = d + arg if fn == "date_add" else d - arg
        ok &= in_range(r)
    elif fn == "last_day":
        r = days_from_civil(y, m, days_in_month(y, m))
    elif fn == "next_day":
        delta = (arg - ((d + 4) % 7 + 1)) % 7
        r = d + np.where(delta == 0, 7, delta)
        ok &= in_range(r)
    elif fn == "add_months":
        total = y * 12 + (m - 1) + arg
        ny = total // 12
        nm = total - ny * 12 + 1
        yok = (ny >= -262144) & (ny <= 262143)
        ok &= yok
        ny = np.where(yok, ny, 1970)
        last = days_in_month(ny, nm)
        nd = np.where((dd == days_in_month(y, m)) | (dd > last), last, dd)
        r = days_from_civil(ny, nm, nd)
    elif fn == "date_trunc":
        unit_t = TRUNC[arg]
        ntod = np.zeros_like(tod)
        if unit_t == "year":
            nd = days_from_civil(y, 1, 1)
        elif unit_t == "quarter":
            nd = days_from_civil(y, (m - 1) // 3 * 3 + 1, 1)
        elif unit_t == "month":
            nd = days_from_civil(y, m, 1)
        elif unit_t == "week":
            nd = d - (d + 3) % 7
        else:
            nd = d
            if unit_t != "day":
                q = {"hour": 3600, "minute": 60, "second": 1}[unit_t] * ups
                ntod = tod - tod % q
        ok &= nd >= MIN_DAY
        if upd == 1:
            r = nd
        else:   # the instant may leave i64: exact Python integers
            big = nd.astype(object) * upd + ntod.astype(object) - off * ups
            fits = np.array([I64_MIN <= x <= I64_MAX for x in big], dtype=bool)
            ok &= fits
            r = np.array([x if f else 0 for x, f in zip(big, fits)], dtype=np.int64)
    else:
        raise ValueError(fn)
    return np.where(ok, r, 0).astype(odt), ok


def side(kind, unit, tz, values):
    off = tz_offset_seconds(tz) if kind == TIMESTAMP else 0
    days, tod = split(values, kind, unit, off)
    _, ups = per_day(kind, unit)
    return days, tod // ups


def binary(fn, ta, a, va, tb, b, vb):
    """DATE_DIFF(a, b) -> Int32 or MONTHS_BETWEEN(a, b) -> Float64.  ta / tb are (kind, unit, tz)."""
    da, sa = side(*ta, a)
    db, sb = side(*tb, b)
    ok = np.asarray(va, bool) & np.asarray(vb, bool) & in_range(da) & in_range(db)
    da, db = np.where(ok, da, 0), np.where(ok, db, 0)
    if fn == "date_diff":
        return np.where(ok, da - db, 0).astype(np.int32), ok
    y1, m1, d1 = civil_from_days(da)
    y2, m2, d2 = civil_from_days(db)
    month_diff = ((y1 * 12 + m1) - (y2 * 12 + m2)).astype(np.float64)
    same = (d1 == d2) | ((d1 == days_in_month(y1, m1)) & (d2 == days_in_month(y2, m2)))
    sec_diff = ((d1 - d2) * 86400 + (np.where(ok, sa, 0) - np.where(ok, sb, 0))).astype(np.float64)
    diff = month_diff + sec_diff / 2678400.0
    t = diff * 1e8
    k = np.floor(t)
    k = np.where(t - k >= 0.5, k + 1.0, k)
    r = np.where(same, month_diff, k / 1e8)
    return np.where(ok, r, 0.0), ok
