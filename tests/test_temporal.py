"""CPU checks of the date and timestamp functions (include/b200df.h "dates and timestamps"): the numpy oracle against Python's datetime,
numpy datetime64 and pyarrow.compute, the recalled Spark documentation examples, bdf_temporal_result over every (fn, type, arg), and
the IPC description of temporal columns.  No GPU."""
import datetime as dt
import os
import re

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pyarrow.ipc as pai
import pytest

import temporal_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPOCH = dt.date(1970, 1, 1)
UNITS = ["s", "ms", "us", "ns"]


def days_of(d: dt.date) -> int:
    return (d - EPOCH).days


def one(fn, kind, unit, tz, value, arg=0):
    v, ok = O.unary(fn, kind, unit, tz, np.array([value], np.int64), np.array([True]), arg)
    return v[0].item() if ok[0] else None


# ---- the oracle against independent calendars ----------------------------------------------------------------------------------

def test_oracle_against_python_datetime_every_day_sample():
    rng = np.random.default_rng(1)
    lo, hi = days_of(dt.date(1, 1, 1)), days_of(dt.date(9999, 12, 31))
    days = np.unique(np.concatenate([rng.integers(lo, hi + 1, 200000), np.arange(lo, lo + 800), np.arange(hi - 800, hi + 1),
                                     np.arange(-1000, 1000)]))
    y, m, d = O.civil_from_days(days)
    dates = [EPOCH + dt.timedelta(days=int(x)) for x in days]
    assert (y == [t.year for t in dates]).all() and (m == [t.month for t in dates]).all() and (d == [t.day for t in dates]).all()
    assert (O.days_from_civil(y, m, d) == days).all()
    valid = np.ones(days.shape, bool)
    doy, _ = O.unary("day_of_year", O.DATE32, 0, None, days, valid)
    assert (doy == [t.timetuple().tm_yday for t in dates]).all()
    dow, _ = O.unary("day_of_week", O.DATE32, 0, None, days, valid)
    assert (dow == [t.isoweekday() % 7 + 1 for t in dates]).all()   # Spark: Sunday = 1
    last, _ = O.unary("last_day", O.DATE32, 0, None, days, valid)
    assert (O.civil_from_days(last + 1)[2] == 1).all()


def test_oracle_times_of_day_against_datetime():
    rng = np.random.default_rng(2)
    base = dt.datetime(1970, 1, 1)
    for unit, ups in zip(UNITS, O.PER_SEC):
        v = rng.integers(-(2 ** 62) // max(1, 1000000000 // ups) // 1000, (2 ** 62) // max(1, 1000000000 // ups) // 1000, 20000)
        v = np.concatenate([v, [-1, 0, 1, 86400 * ups - 1, 86400 * ups, -86400 * ups]])
        valid = np.ones(v.shape, bool)
        us = (v.astype(object) * 1000000) // ups
        ok = [dt.datetime.min <= base + dt.timedelta(microseconds=int(x)) <= dt.datetime.max if abs(int(x)) < 2 ** 62 else False for x in us]
        for fn, get in [("hour", lambda t: t.hour), ("minute", lambda t: t.minute), ("second", lambda t: t.second), ("year", lambda t: t.year)]:
            got, gok = O.unary(fn, O.TIMESTAMP, O.PER_SEC.index(ups), None, v, valid)
            for i in np.nonzero(ok)[0][:3000]:
                t = base + dt.timedelta(microseconds=int(us[i]))
                assert gok[i] and got[i] == get(t), (unit, fn, int(v[i]))
    assert one("hour", O.TIMESTAMP, 2, None, -1) == 23 and one("second", O.TIMESTAMP, 2, None, -1) == 59   # floor, not truncation


def test_oracle_against_numpy_datetime64_whole_chrono_range():
    days = np.unique(np.concatenate([np.linspace(O.MIN_DAY, O.MAX_DAY, 300001).astype(np.int64), [O.MIN_DAY, O.MAX_DAY, 0, -1]]))
    d64 = days.astype("datetime64[D]")
    y = d64.astype("datetime64[Y]").astype(np.int64) + 1970
    m = d64.astype("datetime64[M]").astype(np.int64) % 12 + 1
    d = (d64 - d64.astype("datetime64[M]")).astype(np.int64) + 1
    oy, om, od = O.civil_from_days(days)
    assert (oy == y).all() and (om == m).all() and (od == d).all()
    _, ok = O.unary("year", O.DATE32, 0, None, np.array([O.MIN_DAY - 1, O.MIN_DAY, O.MAX_DAY, O.MAX_DAY + 1]), np.ones(4, bool))
    assert ok.tolist() == [False, True, True, False]
    y2, m2, d2 = O.civil_from_days(np.array([O.MIN_DAY, O.MAX_DAY]))
    assert y2.tolist() == [-262144, 262143] and m2.tolist() == [1, 12] and d2.tolist() == [1, 31]


TYPES = ([(pa.date32(), O.DATE32, 0, None), (pa.date64(), O.DATE64, 1, None)] +
         [(pa.timestamp(u, tz=tz), O.TIMESTAMP, i, tz) for i, u in enumerate(UNITS) for tz in (None, "+05:30", "-08:00")])


@pytest.mark.parametrize("typ,kind,unit,tz", TYPES, ids=[str(t[0]) for t in TYPES])
def test_oracle_against_pyarrow_compute(typ, kind, unit, tz):
    rng = np.random.default_rng(3)
    upd, ups = O.per_day(kind, unit)
    lo, hi = days_of(dt.date(1700, 1, 1)), days_of(dt.date(2250, 12, 31))
    v = rng.integers(lo, hi, 5000) * upd + (rng.integers(0, upd, 5000) if upd > 1 else 0)
    if kind == O.DATE64:
        v = v - v % 86400000 + rng.integers(0, 86400000, 5000)
    v = np.concatenate([v, np.array([0, -1, upd - 1, -upd, upd]) if upd > 1 else np.array([0, -1, 1])]).astype(np.int64)
    arr = pa.array(v.astype(np.int32 if kind == O.DATE32 else np.int64)).view(typ)   # tz-aware: pyarrow's fields are local, the same rule
    valid = np.ones(v.shape, bool)
    checks = [("year", pc.year), ("month", pc.month), ("day_of_month", pc.day), ("day_of_year", pc.day_of_year), ("quarter", pc.quarter),
              ("day_of_week", lambda a: pc.add(pc.day_of_week(a, count_from_zero=True, week_start=7), 1))]
    if kind == O.TIMESTAMP:   # pyarrow has no hour kernel for dates
        checks += [("hour", pc.hour), ("minute", pc.minute), ("second", pc.second)]
    for fn, f in checks:
        want = np.asarray(f(arr).to_numpy(zero_copy_only=False), dtype=np.int64)
        got, ok = O.unary(fn, kind, unit, tz, v, valid)
        assert ok.all() and (got.astype(np.int64) == want).all(), fn
    for name, arg in [("day", 4), ("week", 3), ("month", 2), ("year", 0), ("hour", 5)]:
        if kind != O.TIMESTAMP and name == "hour":
            continue
        want = pc.floor_temporal(arr, unit=name, week_starts_monday=True)
        want = np.asarray(want.cast(pa.int32() if kind == O.DATE32 else pa.int64()).to_numpy(zero_copy_only=False), np.int64)
        got, ok = O.unary("date_trunc", kind, unit, tz, v, valid, arg)
        assert ok.all() and (got.astype(np.int64) == want).all(), name


def test_spark_documentation_examples():
    D = lambda s: days_of(dt.date.fromisoformat(s))
    assert one("day_of_week", O.DATE32, 0, None, D("2009-07-30")) == 5
    assert one("day_of_year", O.DATE32, 0, None, D("2016-04-09")) == 100
    assert one("quarter", O.DATE32, 0, None, D("2016-08-31")) == 3
    assert one("add_months", O.DATE32, 0, None, D("2016-08-31"), 1) == D("2016-09-30")
    assert one("add_months", O.DATE32, 0, None, D("2019-02-28"), 1) == D("2019-03-31")   # Spark 2.4's last-day rule
    assert one("last_day", O.DATE32, 0, None, D("2009-01-12")) == D("2009-01-31")
    assert one("next_day", O.DATE32, 0, None, D("2015-01-14"), 3) == D("2015-01-20")   # Tuesday
    assert one("date_add", O.DATE32, 0, None, D("2016-07-30"), 1) == D("2016-07-31")
    assert one("date_trunc", O.DATE32, 0, None, D("2009-02-12"), 2) == D("2009-02-01")
    ts = int(dt.datetime(2015, 3, 5, 9, 32, 5, 359000).replace(tzinfo=dt.timezone.utc).timestamp() * 1000) * 1000
    assert one("date_trunc", O.TIMESTAMP, 2, None, ts, 5) == int(dt.datetime(2015, 3, 5, 9, tzinfo=dt.timezone.utc).timestamp()) * 1000000
    dd, _ = O.binary("date_diff", (O.DATE32, 0, None), np.array([D("2009-07-31")]), [True], (O.DATE32, 0, None), np.array([D("2009-07-30")]), [True])
    assert dd[0] == 1
    t1 = int(dt.datetime(1997, 2, 28, 10, 30, tzinfo=dt.timezone.utc).timestamp())
    mb, _ = O.binary("months_between", (O.TIMESTAMP, 0, None), np.array([t1]), [True], (O.DATE32, 0, None), np.array([D("1996-10-30")]), [True])
    assert mb[0] == 3.94959677


# ---- bdf_temporal_result: every (fn, type, arg) ----------------------------------------------------------------------------------

def _expect(fn, kind, unit, tz, arg):
    """(status name, dtype) the header's rules predict."""
    valid_type = ((kind == O.DATE32) or (kind == O.DATE64 and unit == 1) or (kind == O.TIMESTAMP and 0 <= unit <= 3) or
                  (kind == O.TIME32 and unit in (0, 1)) or (kind == O.TIME64 and unit in (2, 3)))
    if not valid_type:
        return "ComputeError", None
    name = O.FNS[fn]
    if kind in (O.TIME32, O.TIME64) and name not in ("hour", "minute", "second"):
        return "UnsupportedType", None
    if name in ("date_add", "date_sub", "add_months") and not (-(2 ** 31) <= arg < 2 ** 31):
        return "ComputeError", None
    if name == "next_day" and not 1 <= arg <= 7:
        return "ComputeError", None
    if name == "date_trunc" and not 0 <= arg <= 7:
        return "ComputeError", None
    if name == "to_timestamp" and not 0 <= arg <= 3:
        return "ComputeError", None
    if kind == O.TIMESTAMP and name not in ("unix_timestamp", "to_timestamp") and O.tz_offset_seconds(tz) is None:
        return "UnsupportedType", None
    return "ok", {np.int32: 2, np.int64: 3}[O.result_dtype(name, kind)]


def test_temporal_result_every_combination(rdf):
    T = rdf.TemporalType
    args = [-(2 ** 31) - 1, -(2 ** 31), -1, 0, 1, 3, 4, 7, 8, 2 ** 31 - 1, 2 ** 31]
    n = 0
    for kind in range(0, 7):
        for unit in range(-1, 5):
            for tz in ([None, "UTC", "Z", "+00:00", "+05:30", "-23:59", "+24:00", "Europe/Paris", "05:30"] if kind == O.TIMESTAMP else [None]):
                for fn in range(len(O.FNS)):
                    for arg in args:
                        status, dtype = _expect(fn, kind, unit, tz, arg)
                        if kind in (0, 6):
                            status = "ComputeError"
                        try:
                            got_dt, got_t = rdf.temporal_result(fn, T(kind, unit, tz), arg)
                            got = "ok"
                        except rdf.ArrowError as e:
                            got = type(e).__name__
                        assert got == status, (kind, unit, tz, O.FNS[fn], arg, got)
                        n += 1
                        if got != "ok":
                            continue
                        assert got_dt == dtype
                        name = O.FNS[fn]
                        if name == "date_trunc":
                            assert got_t == T(kind, unit, tz)
                        elif name == "to_timestamp":
                            assert got_t == T(O.TIMESTAMP, arg, tz if kind == O.TIMESTAMP else None)
                        elif O.result_dtype(name, kind) == np.int32 and name in ("to_date", "date_add", "date_sub", "add_months", "last_day", "next_day"):
                            assert got_t == T.date32()
                        else:
                            assert got_t is None
    assert n > 10000
    with pytest.raises(rdf.ComputeError):
        rdf.temporal_result(18, T.date32())
    with pytest.raises(rdf.ComputeError):
        rdf.temporal_result(-1, T.date32())


# ---- IPC description --------------------------------------------------------------------------------------------------------------

def test_ipc_describes_temporal_columns(rdf, tmp_path):
    cols = {"d32": pa.array([1, None], pa.date32()), "d64": pa.array([86400000, None], pa.date64()), "x": pa.array([1, 2], pa.int64()),
            "t32s": pa.array([1, 2], pa.time32("s")), "t32ms": pa.array([1, 2], pa.time32("ms")), "t64us": pa.array([1, 2], pa.time64("us")),
            "t64ns": pa.array([1, 2], pa.time64("ns")), "dur": pa.array([1, 2], pa.duration("s"))}
    for u in UNITS:
        for tz in (None, "UTC", "+05:30", "America/New_York"):
            cols[f"ts_{u}_{tz}"] = pa.array([1, None], pa.timestamp(u, tz=tz))
    tb = pa.table(cols)
    path = str(tmp_path / "t.arrow")
    with pai.new_file(path, tb.schema) as w:
        w.write_table(tb)
    f = rdf.IpcFile(path)
    dtypes = {name: d for name, d, _ in f.schema}
    assert dtypes["x"] == rdf.I64 and all(d == -1 for n, d in dtypes.items() if n != "x")   # schema is unchanged
    T = rdf.TemporalType
    want = {"d32": T.date32(), "d64": T.date64(), "t32s": T.time32("s"), "t32ms": T.time32("ms"), "t64us": T.time64("us"), "t64ns": T.time64("ns")}
    for u in UNITS:
        for tz in (None, "UTC", "+05:30", "America/New_York"):
            want[f"ts_{u}_{tz}"] = T.timestamp(u, tz)
    assert f.temporal_columns == want
    for name, field in zip(tb.schema.names, tb.schema):
        if name in want:
            assert want[name].to_arrow() == field.type
    f.close()


def test_ipc_malformed_timezone_still_opens(rdf, tmp_path):
    """A Timestamp field whose timezone string does not decode is stepped over, as before temporal columns were read: the file opens."""
    tb = pa.table({"ts": pa.array([1, 2], pa.timestamp("us", tz="+05:30")), "x": pa.array([3, 4], pa.int64())})
    path = str(tmp_path / "bad_tz.arrow")
    with pai.new_file(path, tb.schema) as w:
        w.write_table(tb)
    raw = bytearray(open(path, "rb").read())
    n = 0
    at = raw.find(b"+05:30")
    while at >= 0:   # every copy of the schema: the string's length prefix now points past the end of the file
        raw[at - 4:at] = (0x7FFFFFF0).to_bytes(4, "little")
        n += 1
        at = raw.find(b"+05:30", at + 1)
    assert n >= 1
    open(path, "wb").write(bytes(raw))
    f = rdf.IpcFile(path)
    assert [(name, d) for name, d, _ in f.schema] == [("ts", -1), ("x", rdf.I64)]
    assert f.temporal_columns == {}
    f.close()


def test_header_declares_the_temporal_abi():
    text = open(os.path.join(ROOT, "include", "b200df.h")).read()
    for sym in ["bdf_temporal", "bdf_temporal_dev", "bdf_temporal_binary_dev", "bdf_temporal_result", "bdf_ipc_temporal_column",
                "bdf_ipc_read_temporal", "bdf_ipc_write_typed"]:
        assert re.search(r"\b" + sym + r"\s*\(", text), sym
    for name in ["bdf_temporal_kind", "bdf_time_unit", "bdf_temporal_type", "bdf_temporal_fn", "bdf_temporal_binary_fn", "bdf_trunc_unit",
                 "BDF_K_TEMPORAL", "Spark 3 dropped", "parity unpinned", "FLOOR division"]:
        assert name.lower() in text.lower(), name
    assert "#define BDF_ABI_VERSION 3" in text


def test_python_mirror_names(rdf):
    for name in list(rdf.native.TEMPORAL_FNS) + ["date_diff", "months_between"]:
        assert callable(getattr(rdf.ScalarFunctions, name)), name
        assert callable(getattr(rdf.Column, name)), name
    assert rdf.native.KERNEL_NAMES[rdf.native.K_TEMPORAL] == "temporal"
