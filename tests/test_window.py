"""Window functions without a GPU: the numpy oracle (tests/window_oracle.py) against SQLite's window functions and against written-out
expectations, the planner's schemas and errors, and the C header's window types against the ctypes binding."""
import ctypes as C
import math
import os
import sqlite3
import subprocess
from collections import OrderedDict

import numpy as np
import pytest

import window_oracle as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SQLITE_WINDOWS = sqlite3.sqlite_version_info >= (3, 30, 0)   # window functions and NULLS LAST


def arr(rdf, dtype, values, valid=None):
    """One chunk, as the list of chunks the oracle takes."""
    v = np.asarray(values, dtype=rdf.NP_DTYPES[dtype])
    return [rdf.PrimitiveArray.from_numpy(v, None if valid is None else np.asarray(valid, bool))]


def _sqlite_table(rng, n):
    """Partition keys with nulls, order keys with ties and nulls, value columns without NaN (SQLite has no NaN)."""
    p1 = rng.integers(0, 4, n)
    p1m = rng.random(n) > 0.1
    p2 = rng.choice([-1.5, 0.5, 2.0], n)
    o1 = rng.integers(0, 6, n)
    o1m = rng.random(n) > 0.15
    o2 = rng.choice([-2.0, 1.0, 3.5, 7.25], n)
    o2m = rng.random(n) > 0.1
    xf = rng.uniform(-100, 100, n)
    xi = rng.integers(-1000, 1000, n)
    xm = rng.random(n) > 0.2
    return dict(p1=(p1, p1m), p2=(p2, np.ones(n, bool)), o1=(o1, o1m), o2=(o2, o2m), xf=(xf, xm), xi=(xi, xm))


def _load(tab):
    db = sqlite3.connect(":memory:")
    names = list(tab)
    db.execute(f"CREATE TABLE t ({', '.join(names)})")
    n = len(tab[names[0]][0])
    rows = [tuple((tab[c][0][i].item() if tab[c][1][i] else None) for c in names) for i in range(n)]
    db.executemany(f"INSERT INTO t VALUES ({', '.join('?' * len(names))})", rows)
    return db


def _sql_column(db, expr, window):
    return [r[0] for r in db.execute(f"SELECT {expr} OVER ({window}) FROM t ORDER BY rowid")]


@pytest.mark.skipif(not SQLITE_WINDOWS, reason="SQLite before 3.30 has no window functions / NULLS LAST")
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_oracle_matches_sqlite(rdf, seed):
    rng = np.random.default_rng(seed)
    n = 300
    tab = _sqlite_table(rng, n)
    db = _load(tab)
    ch = {c: arr(rdf, rdf.F64 if tab[c][0].dtype.kind == "f" else rdf.I64, tab[c][0], tab[c][1]) for c in tab}
    part = [ch["p1"], ch["p2"]]
    order = [(ch["o1"], False), (ch["o2"], True)]
    spec = "PARTITION BY p1, p2 ORDER BY o1 ASC NULLS LAST, o2 DESC NULLS LAST"
    spec_rowid = spec + ", rowid"

    def check(calls, sql, window):
        got = W.window(part, order, calls)
        for g, (fn, _, _), expr in zip(got, calls, sql):
            want = _sql_column(db, expr, window)
            for i in range(n):
                w = want[i]
                if fn == "sum" and w is None:
                    w = 0   # AggregateFunctions::sum: an empty frame sums to 0
                if w is None:
                    assert not g["valid"][i], (expr, i)
                    continue
                assert g["valid"][i], (expr, i, w)
                v = g["values"][i]
                if isinstance(w, float) or g["values"].dtype.kind == "f":
                    assert math.isclose(float(v), float(w), rel_tol=1e-12, abs_tol=1e-9), (expr, i, v, w)
                else:
                    assert int(v) == int(w), (expr, i, v, w)

    check([("rank", None, None), ("dense_rank", None, None), ("percent_rank", None, None), ("cume_dist", None, None)],
          ["rank()", "dense_rank()", "percent_rank()", "cume_dist()"], spec)
    check([("row_number", None, None), ("lag", ch["xf"], (1, None)), ("lead", ch["xi"], (2, -7)), ("lag", ch["xi"], (0, None))],
          ["row_number()", "lag(xf, 1)", "lead(xi, 2, -7)", "lag(xi, 0)"], spec_rowid)
    for frame, window, sql_frame in (("rows", spec_rowid, "ROWS BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW"),
                                     ("range", spec, "RANGE BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW"),
                                     ("partition", spec_rowid, "ROWS BETWEEN UNBOUNDED PRECEDING AND UNBOUNDED FOLLOWING")):
        calls = [(fn, ch[x], frame) for fn in ("sum", "count", "min", "max", "avg") for x in ("xf", "xi")]
        check(calls, [f"{fn}({x})" for fn in ("sum", "count", "min", "max", "avg") for x in ("xf", "xi")], f"{window} {sql_frame}")


def test_oracle_written_out_keys(rdf):
    """NaN, -0.0 and nulls in partition and order keys: one partition per value class, nulls last in both directions."""
    nan = float("nan")
    p = arr(rdf, rdf.F64, [nan, 0.0, -0.0, nan, 1.0, 0.0], [1, 1, 1, 1, 1, 0])
    o = arr(rdf, rdf.F32, [2.0, nan, 1.0, -0.0, 5.0, 3.0], [1, 1, 0, 1, 1, 1])
    r = W.window([p], [(o, False)], [("row_number", None, None), ("rank", None, None)])
    # partitions: {NaN: rows 0, 3}, {0.0 / -0.0: rows 1, 2}, {1.0: row 4}, {null: row 5}
    assert r[0]["values"].tolist() == [2, 1, 2, 1, 1, 1]
    r = W.window([p], [(o, True)], [("row_number", None, None)])
    assert r[0]["values"].tolist() == [1, 1, 2, 2, 1, 1]   # descending: NaN first, the null row last
    o2 = arr(rdf, rdf.F64, [0.0, -0.0, nan, nan, 1.0, 1.0], [1, 1, 1, 1, 0, 0])
    r = W.window([], [(o2, False)], [("rank", None, None), ("dense_rank", None, None), ("cume_dist", None, None)])
    assert r[0]["values"].tolist() == [1, 1, 3, 3, 5, 5]
    assert r[1]["values"].tolist() == [1, 1, 2, 2, 3, 3]
    assert r[2]["values"].tolist() == [2 / 6, 2 / 6, 4 / 6, 4 / 6, 1.0, 1.0]


def test_oracle_written_out_values(rdf):
    nan = float("nan")
    x8 = arr(rdf, rdf.I8, [100, 100, -128, 5], [1, 1, 1, 0])
    r = W.window([], [], [("sum", x8, "rows"), ("count", x8, "rows"), ("min", x8, "partition"), ("max", x8, "rows")])
    assert r[0]["values"].tolist() == [100, -56, 72, 72]        # wraps in Int8
    assert r[1]["values"].tolist() == [1, 2, 3, 3]
    assert r[2]["values"].tolist() == [-128] * 4
    assert r[3]["values"].tolist() == [100, 100, 100, 100]
    xf = arr(rdf, rdf.F64, [1.0, nan, -0.0, 0.0, 2.0], [1, 1, 1, 1, 0])
    k = arr(rdf, rdf.I32, [0, 0, 1, 1, 1])
    r = W.window([k], [], [("min", xf, "rows"), ("max", xf, "rows"), ("avg", xf, "partition")])
    got_min = r[0]["values"]
    assert got_min[0] == 1.0 and got_min[1] == 1.0 and np.signbit(got_min[2]) and np.signbit(got_min[3]) and np.signbit(got_min[4])
    assert r[1]["values"][0] == 1.0 and np.isnan(r[1]["values"][1]) and np.signbit(r[1]["values"][2]) and not np.signbit(r[1]["values"][3])
    assert r[2]["valid"].tolist() == [True] * 5
    allnull = arr(rdf, rdf.I32, [1, 2], [0, 0])
    r = W.window([], [], [("sum", allnull, "rows"), ("min", allnull, "rows"), ("avg", allnull, "rows")])
    assert r[0]["values"].tolist() == [0, 0] and r[0]["valid"].all()
    assert not r[1]["valid"].any() and not r[2]["valid"].any()


def test_oracle_written_out_shifts(rdf):
    k = arr(rdf, rdf.I32, [1, 1, 2, 1, 2])
    x = arr(rdf, rdf.U64, [10, 20, 30, 40, 50], [1, 0, 1, 1, 1])
    big = np.iinfo(np.uint64).max
    r = W.window([k], [], [("lag", x, (1, big)), ("lead", x, (1, None)), ("lag", x, (0, None)), ("lead", x, (5, 7))])
    assert r[0]["values"].tolist() == [big, 10, big, 0, 30] and r[0]["valid"].tolist() == [True, True, True, False, True]
    assert r[1]["values"].tolist() == [0, 40, 50, 0, 0] and r[1]["valid"].tolist() == [False, True, True, False, False]
    assert r[2]["valid"].tolist() == [True, False, True, True, True]
    assert r[3]["values"].tolist() == [7] * 5


def _schema(rdf):
    return OrderedDict([("k", rdf.I32), ("x", rdf.F64), ("i", rdf.I64), ("b", rdf.native.BOOL)])


def test_plan_window_schema(rdf):
    plan = rdf.plan_window(_schema(rdf), ["k"], [("x", True)],
                           [("rn", "row_number"), ("pr", "percent_rank"), ("s", "sum", "i", "range"), ("c", "count", "x"), ("a", "avg", "x"),
                            ("x", "lag", "x", 1, 0.0)])
    assert plan == [("k", rdf.I32), ("i", rdf.I64), ("b", rdf.native.BOOL), ("rn", rdf.U32), ("pr", rdf.F64), ("s", rdf.I64), ("c", rdf.I64),
                    ("a", rdf.F64), ("x", rdf.F64)]


def test_plan_window_errors(rdf):
    s = _schema(rdf)
    with pytest.raises(rdf.ComputeError):
        rdf.plan_window(s, ["nope"], [], [("r", "row_number")])
    with pytest.raises(rdf.ComputeError):
        rdf.plan_window(s, [], [("nope", False)], [("r", "row_number")])
    with pytest.raises(rdf.ComputeError):
        rdf.plan_window(s, [], [], [("r", "sum", "nope")])
    with pytest.raises(rdf.UnsupportedType):
        rdf.plan_window(s, ["b"], [], [("r", "row_number")])
    with pytest.raises(rdf.UnsupportedType):
        rdf.plan_window(s, [], [], [("r", "avg", "i")])
    with pytest.raises(rdf.UnsupportedType):
        rdf.plan_window(s, [], [], [("r", "ntile", "x")])


def test_plan_fusion_keeps_every_column_a_window_reads():
    """A run of Calculations before a window is not fused when the window reads an intermediate; its outputs are new columns."""
    from rust_dataframe_b200 import F64, I32
    from rust_dataframe_b200.frame import calculate, plan_fusion, select, window

    schema = OrderedDict([("k", I32), ("x", F64), ("y", F64)])
    steps = [calculate("add", ["x", "y"], "t"), calculate("multiply", ["t", "y"], "u"), window(["k"], [("t", False)], [("s", "sum", "u")]),
             select(["k", "s"])]
    assert [k for k, _ in plan_fusion(schema, steps)] == ["calculate", "calculate", "window", "select"]
    steps2 = [calculate("add", ["x", "y"], "t"), calculate("multiply", ["t", "y"], "u"), window(["k"], [("x", False)], [("s", "sum", "u")]),
              select(["k", "s"])]
    assert [k for k, _ in plan_fusion(schema, steps2)] == ["fused", "window", "select"]


def test_window_types_match_the_header(tmp_path, rdf):
    N = rdf.native
    src = tmp_path / "wt.c"
    src.write_text("#include <stdio.h>\n#include <stddef.h>\n#include \"b200df.h\"\n"
                   "int main(void){printf(\"%d %d %d %d %d %d %d %d %d %d %d %d  %d %d %d  %d  %zu %zu %zu %zu %zu %zu %zu\\n\","
                   " (int)BDF_WIN_ROW_NUMBER, (int)BDF_WIN_RANK, (int)BDF_WIN_DENSE_RANK, (int)BDF_WIN_PERCENT_RANK, (int)BDF_WIN_CUME_DIST,"
                   " (int)BDF_WIN_LAG, (int)BDF_WIN_LEAD, (int)BDF_WIN_SUM, (int)BDF_WIN_COUNT, (int)BDF_WIN_MIN, (int)BDF_WIN_MAX, (int)BDF_WIN_AVG,"
                   " (int)BDF_FRAME_ROWS, (int)BDF_FRAME_RANGE, (int)BDF_FRAME_PARTITION, (int)BDF_K_WINDOW, sizeof(bdf_window_call),"
                   " offsetof(bdf_window_call, function), offsetof(bdf_window_call, frame), offsetof(bdf_window_call, column),"
                   " offsetof(bdf_window_call, offset), offsetof(bdf_window_call, default_bits), offsetof(bdf_window_call, has_default));"
                   "return 0;}\n")
    exe = tmp_path / "wt"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    names = ["row_number", "rank", "dense_rank", "percent_rank", "cume_dist", "lag", "lead", "sum", "count", "min", "max", "avg"]
    assert got[:12] == [N.WINDOW_FNS[k] for k in names]
    assert got[12:15] == [N.WINDOW_FRAMES[k] for k in ("rows", "range", "partition")]
    assert got[15] == N.K_WINDOW and N.KERNEL_NAMES[N.K_WINDOW] == "window"
    W_ = N.WindowCall
    assert got[16:] == [C.sizeof(W_), W_.function.offset, W_.frame.offset, W_.column.offset, W_.offset.offset, W_.default_bits.offset,
                        W_.has_default.offset]
