"""Bounded window frames and value functions without a GPU: the numpy oracle (tests/window_frame_oracle.py) against SQLite's ROWS /
RANGE BETWEEN frames and against written-out expectations for what SQLite cannot show, the planner, and the C header's new enum
values and struct layout against the ctypes binding."""
import ctypes as C
import datetime
import math
import os
import sqlite3
import subprocess
from collections import OrderedDict

import numpy as np
import pytest

import window_frame_oracle as F
from test_window import _load, _sql_column, arr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SQLITE_FRAMES = sqlite3.sqlite_version_info >= (3, 30, 0)
BOUNDS = [None, -3, -1, 0, 2]   # UNBOUNDED, n PRECEDING, CURRENT ROW, m FOLLOWING


def _sql_bound(v, upper):
    if v is None:
        return "UNBOUNDED FOLLOWING" if upper else "UNBOUNDED PRECEDING"
    if v == 0:
        return "CURRENT ROW"
    return f"{abs(v)} {'PRECEDING' if v < 0 else 'FOLLOWING'}"


def _table(rng, n):
    p = rng.integers(0, 3, n)
    o = rng.integers(0, 12, n)
    om = rng.random(n) > 0.15
    of = rng.choice([-2.5, -1.0, 0.0, 0.5, 1.5, 4.0, 9.0], n)
    ofm = rng.random(n) > 0.15
    xf = rng.uniform(-100, 100, n)
    xi = rng.integers(-1000, 1000, n)
    xm = rng.random(n) > 0.25
    return dict(p=(p, np.ones(n, bool)), o=(o, om), of=(of, ofm), xf=(xf, xm), xi=(xi, xm))


def _compare(got, want, fn, expr):
    for i, w in enumerate(want):
        if fn == "sum" and w is None:
            w = 0   # an empty frame sums to 0 here; SQLite gives NULL
        if w is None:
            assert not got["valid"][i], (expr, i)
            continue
        assert got["valid"][i], (expr, i, w)
        v = got["values"][i]
        if isinstance(w, float) or got["values"].dtype.kind == "f":
            assert math.isclose(float(v), float(w), rel_tol=1e-12, abs_tol=1e-9), (expr, i, v, w)
        else:
            assert int(v) == int(w), (expr, i, v, w)


@pytest.mark.skipif(not SQLITE_FRAMES, reason="SQLite before 3.30 has no NULLS LAST")
@pytest.mark.parametrize("seed", [1, 2])
def test_rows_between_matches_sqlite(rdf, seed):
    rng = np.random.default_rng(seed)
    n = 120
    tab = _table(rng, n)
    db = _load(tab)
    ch = {c: arr(rdf, rdf.F64 if tab[c][0].dtype.kind == "f" else rdf.I64, tab[c][0], tab[c][1]) for c in tab}
    spec = "PARTITION BY p ORDER BY o ASC NULLS LAST, rowid"
    for s in BOUNDS:
        for e in BOUNDS:
            if s is not None and e is not None and s > e:
                continue
            frame = ("rows", s, e)
            sql = f"{spec} ROWS BETWEEN {_sql_bound(s, False)} AND {_sql_bound(e, True)}"
            calls = [(fn, ch[x], frame) for fn in ("sum", "count", "min", "max", "avg") for x in ("xf", "xi")]
            calls += [("first_value", ch["xi"], (frame, None, False)), ("last_value", ch["xf"], (frame, None, False)),
                      ("nth_value", ch["xi"], (frame, 2, False))]
            exprs = [f"{fn}({x})" for fn in ("sum", "count", "min", "max", "avg") for x in ("xf", "xi")]
            exprs += ["first_value(xi)", "last_value(xf)", "nth_value(xi, 2)"]
            got = F.window([ch["p"]], [(ch["o"], False)], calls)
            for g, (fn, _, _), expr in zip(got, calls, exprs):
                _compare(g, _sql_column(db, expr, sql), fn, f"{expr} {sql}")


@pytest.mark.skipif(not SQLITE_FRAMES, reason="SQLite before 3.30 has no NULLS LAST")
@pytest.mark.parametrize("key", ["o", "of"])
@pytest.mark.parametrize("desc", [False, True])
def test_range_between_matches_sqlite(rdf, key, desc):
    rng = np.random.default_rng(3 + desc)
    n = 150
    tab = _table(rng, n)
    db = _load(tab)
    ch = {c: arr(rdf, rdf.F64 if tab[c][0].dtype.kind == "f" else rdf.I64, tab[c][0], tab[c][1]) for c in tab}
    offs = [None, -3, 0, 2] if key == "o" else [None, -1.5, 0.0, 2.5]
    direction = "DESC" if desc else "ASC"
    for s in offs:
        for e in offs:
            if s is not None and e is not None and s > e:
                continue
            frame = ("range", s, e)
            sql = f"PARTITION BY p ORDER BY {key} {direction} NULLS LAST RANGE BETWEEN {_sql_bound(s, False)} AND {_sql_bound(e, True)}"
            calls = [(fn, ch["xf"], frame) for fn in ("sum", "count", "min", "max", "avg")] + [("count", ch["xi"], frame)]
            calls += [("first_value", ch["xi"], (frame, None, False)), ("last_value", ch["xi"], (frame, None, False))]
            exprs = [f"{fn}(xf)" for fn in ("sum", "count", "min", "max", "avg")] + ["count(xi)", "first_value(xi)", "last_value(xi)"]
            got = F.window([ch["p"]], [(ch[key], desc)], calls)
            for g, (fn, _, _), expr in zip(got, calls, exprs):
                want = _sql_column(db, expr, sql)
                if fn in ("first_value", "last_value"):   # peers tie in SQLite's unspecified order: compare the frame's bounds instead
                    continue
                _compare(g, want, fn, f"{expr} {sql}")
            # first_value / last_value over peers: any value of the bounding peer group is right; check the bounds hold one
            s_pos, e_pos = got[6]["bounds"]
            cnt = np.array([0 if w is None else w for w in _sql_column(db, "count(*)", sql)])
            assert np.array_equal(np.maximum(e_pos - s_pos + 1, 0), cnt), sql


def test_value_functions_written_out(rdf):
    x = arr(rdf, rdf.I32, [10, 20, 30, 40, 50, 60], [1, 0, 0, 1, 0, 1])
    k = arr(rdf, rdf.I32, [1, 1, 1, 1, 2, 2])
    r = F.window([k], [], [("first_value", x, (("rows", -1, 1), None, False)), ("first_value", x, (("rows", -1, 1), None, True)),
                           ("last_value", x, (("rows", None, 0), None, True)), ("nth_value", x, (("rows", None, None), 2, True)),
                           ("nth_value", x, ("partition", 3, False)), ("last_value", x, (("rows", 1, 2), None, False))])
    assert r[0]["valid"].tolist() == [True, True, False, False, False, False] and r[0]["values"][:2].tolist() == [10, 10]
    assert r[1]["values"].tolist() == [10, 10, 40, 40, 60, 60] and r[1]["valid"].tolist() == [True, True, True, True, True, True]
    assert r[2]["values"].tolist() == [10, 10, 10, 40, 0, 60] and r[2]["valid"].tolist() == [True, True, True, True, False, True]   # forward fill
    assert r[3]["values"].tolist() == [40, 40, 40, 40, 0, 0] and r[3]["valid"].tolist() == [True] * 4 + [False] * 2
    assert r[4]["valid"].tolist() == [False] * 6                       # the third row of partition 1 is null; partition 2 has two
    assert r[5]["valid"].tolist() == [False, True, True, False, True, False]     # 1..2 rows ahead, clipped to the partition
    assert r[5]["values"][[1, 2, 4]].tolist() == [40, 40, 60]


def test_nan_inf_and_null_keys_written_out(rdf):
    nan, inf = float("nan"), float("inf")
    o = arr(rdf, rdf.F64, [-inf, 1.0, 2.0, inf, nan, nan, 3.0, -0.0], [1, 1, 1, 1, 1, 1, 0, 1])
    x = arr(rdf, rdf.I64, [1, 2, 4, 8, 16, 32, 64, 128])
    # ascending: -inf, -0.0, 1, 2, inf, NaN, NaN, null
    r = F.window([], [(o, False)], [("sum", x, ("range", -1.0, 0.0)), ("sum", x, ("range", 0.0, None)), ("sum", x, ("range", None, 1.0))])
    assert r[0]["values"].tolist() == [1, 2 + 128, 4 + 2, 8, 16 + 32, 16 + 32, 64, 128 + 2 - 2 + 0]
    assert r[1]["values"].tolist() == [255, 255 - 1 - 128, 255 - 1 - 128 - 2, 8 + 16 + 32 + 64, 16 + 32 + 64, 16 + 32 + 64, 64, 255 - 1]
    assert r[2]["values"].tolist() == [1, 1 + 128 + 2 + 4, 1 + 128 + 2 + 4, 1 + 128 + 2 + 4 + 8, 1 + 2 + 4 + 8 + 16 + 32 + 128,
                                       1 + 2 + 4 + 8 + 16 + 32 + 128, 255, 1 + 128 + 2]
    # descending: NaN, NaN, inf, 2, 1, -0.0, -inf, null; PRECEDING points to larger keys
    r = F.window([], [(o, True)], [("sum", x, ("range", -1.0, 0.0)), ("count", x, ("range", None, 0.0))])
    assert r[0]["values"].tolist() == [1, 2 + 4, 4, 8, 16 + 32, 16 + 32, 64, 128 + 2]
    assert r[1]["values"].tolist() == [7, 4 + 1, 4, 3, 2, 2, 8, 6]


def test_integer_key_edges_written_out(rdf):
    o = arr(rdf, rdf.I8, [-128, -127, 0, 126, 127], [1, 1, 1, 1, 1])
    x = arr(rdf, rdf.I32, [1, 2, 4, 8, 16])
    r = F.window([], [(o, False)], [("sum", x, ("range", -300, -1)), ("sum", x, ("range", 1, 300)), ("sum", x, ("range", -1, 1)),
                                    ("sum", x, ("range", -(2 ** 63) + 1, 2 ** 63 - 2))])
    assert r[0]["values"].tolist() == [0, 1, 3, 7, 15]
    assert r[1]["values"].tolist() == [30, 28, 24, 16, 0]
    assert r[2]["values"].tolist() == [3, 3, 4, 24, 24]
    assert r[3]["values"].tolist() == [31] * 5
    u = arr(rdf, rdf.U8, [0, 1, 5, 255])
    r = F.window([], [(u, True)], [("sum", arr(rdf, rdf.I32, [1, 2, 4, 8]), ("range", -1, 3))])
    # descending: 255, 5, 1, 0; a row's frame is v - 3 <= k <= v + 1 (a negative start over an unsigned key)
    assert r[0]["values"].tolist() == [1 + 2, 1 + 2, 4, 8]   # 0 - 3 < 0 takes in every key below


def test_timestamp_key_with_timedelta(rdf):
    from rust_dataframe_b200.functions import _frame_offset

    ts = (rdf.I64, rdf.TemporalType(rdf.arrays.TIMESTAMP, "ms"))
    assert _frame_offset(datetime.timedelta(days=-7), ts, False) == -7 * 86_400_000
    assert _frame_offset(datetime.timedelta(seconds=3), (rdf.I64, rdf.TemporalType(rdf.arrays.TIMESTAMP, "ns")), True) == 3 * 10 ** 9
    assert _frame_offset(datetime.timedelta(days=2), (rdf.I32, rdf.TemporalType(rdf.arrays.DATE32)), True) == 2
    assert _frame_offset(None, ts, False) == -(2 ** 63)
    with pytest.raises(rdf.ComputeError):
        _frame_offset(datetime.timedelta(hours=1), (rdf.I32, rdf.TemporalType(rdf.arrays.DATE32)), True)
    day = 86_400_000
    o = arr(rdf, rdf.I64, [0, 3 * day, 7 * day, 8 * day, 20 * day])
    x = arr(rdf, rdf.F64, [1.0, 2.0, 4.0, 8.0, 16.0])
    r = F.window([], [(o, False)], [("sum", x, ("range", -7 * day, 0))])
    assert r[0]["values"].tolist() == [1.0, 3.0, 7.0, 14.0, 16.0]


def _schema(rdf):
    return OrderedDict([("k", rdf.I32), ("x", rdf.F64), ("i", rdf.I16), ("b", rdf.native.BOOL)])


def test_plan_window_value_functions_and_errors(rdf):
    plan = rdf.plan_window(_schema(rdf), ["k"], [("x", False)], [("f", "first_value", "i"), ("l", "last_value", "x", ("rows", -2, 2), True),
                                                                 ("n", "nth_value", "i", 3), ("m", "avg", "i", ("range", -1.5, 0.0))])
    assert plan[-4:] == [("f", rdf.I16), ("l", rdf.F64), ("n", rdf.I16), ("m", rdf.F64)]
    with pytest.raises(rdf.UnsupportedType):
        rdf.plan_window(_schema(rdf), [], [], [("r", "ntile", "x")])
    with pytest.raises(rdf.ComputeError):
        rdf.plan_window(_schema(rdf), [], [], [("r", "first_value")])
    from rust_dataframe_b200.functions import _window_call

    class Col:   # what _window_call reads of a column
        handle, dtype = None, rdf.F64

    with pytest.raises(rdf.UnsupportedType):
        _window_call(("sum", Col(), "groups"), True)
    with pytest.raises(rdf.UnsupportedType):
        _window_call(("sum", Col(), ("groups", -1, 1)), True)
    k = _window_call(("nth_value", Col(), 4, ("range", None, 2.5), True), True, (rdf.F64, None))
    assert (k.function, k.offset, k.frame, k.start_f, k.end_f, k.ignore_nulls) == (rdf.native.WIN_NTH_VALUE, 4, rdf.native.FRAME_RANGE_BETWEEN,
                                                                                  -math.inf, 2.5, 1)
    k = _window_call(("sum", Col(), ("rows", -99, None)), True)
    assert (k.frame, k.start, k.end) == (rdf.native.FRAME_ROWS_BETWEEN, -99, 2 ** 63 - 1)


def test_frame_types_match_the_header(tmp_path, rdf):
    N = rdf.native
    src = tmp_path / "ft.c"
    fields = ["function", "frame", "column", "offset", "default_bits", "has_default", "ignore_nulls", "start", "end", "start_f", "end_f"]
    src.write_text("#include <stdio.h>\n#include <stddef.h>\n#include \"b200df.h\"\n"
                   "int main(void){printf(\"%d %d %d %d %d %zu" + " %zu" * len(fields) + "\\n\","
                   " (int)BDF_WIN_FIRST_VALUE, (int)BDF_WIN_LAST_VALUE, (int)BDF_WIN_NTH_VALUE, (int)BDF_FRAME_ROWS_BETWEEN,"
                   " (int)BDF_FRAME_RANGE_BETWEEN, sizeof(bdf_window_call)" +
                   "".join(f", offsetof(bdf_window_call, {f})" for f in fields) + ");return 0;}\n")
    exe = tmp_path / "ft"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got[:3] == [N.WINDOW_FNS[k] for k in ("first_value", "last_value", "nth_value")] == [12, 13, 14]
    assert got[3:5] == [N.FRAME_ROWS_BETWEEN, N.FRAME_RANGE_BETWEEN] == [3, 4]
    W = N.WindowCall
    assert got[5:] == [C.sizeof(W)] + [getattr(W, f).offset for f in fields]
