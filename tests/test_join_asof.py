"""CPU checks of the as-of and existence joins: the numpy restatement in tests/asof_oracle.py against pandas.merge_asof and against
an inner join, the planned schemas of the frame steps, the Python argument errors and the layout of bdf_asof_spec.  No GPU needed."""
import ctypes as C
import datetime
import os
import subprocess
import types
import zlib
from collections import OrderedDict

import numpy as np
import pandas as pd
import pytest

import asof_oracle as ao
import join_oracle as jo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _pandas_asof(lv, rv, lb, rb, direction, exact, tolerance):
    """Right row numbers (-1 = none) that pandas.merge_asof picks; both sides sorted by `on`, no nulls."""
    left = pd.DataFrame({"on": lv, **{f"k{j}": b for j, b in enumerate(lb)}})
    right = pd.DataFrame({"on": rv, "ri": np.arange(len(rv), dtype=np.int64), **{f"k{j}": b for j, b in enumerate(rb)}})
    by = [f"k{j}" for j in range(len(lb))] or None
    m = pd.merge_asof(left, right, on="on", by=by, direction=direction, allow_exact_matches=exact, tolerance=tolerance)
    return m["ri"].fillna(-1).astype(np.int64).to_numpy()


@pytest.mark.parametrize("dtype", ["int64", "float64"])
@pytest.mark.parametrize("n_by", [0, 1, 2])
@pytest.mark.parametrize("direction", ao.DIRECTIONS)
@pytest.mark.parametrize("exact", [True, False])
@pytest.mark.parametrize("tolerance", [None, 0, 3])
def test_oracle_matches_pandas_merge_asof(dtype, n_by, direction, exact, tolerance):
    rng = np.random.default_rng(zlib.crc32(repr((dtype, n_by, direction, exact, tolerance)).encode()))
    nl, nr = 700, 400
    lv = np.sort(rng.integers(-60, 60, nl)).astype(dtype)
    rv = np.sort(rng.integers(-60, 60, nr), kind="stable").astype(dtype)   # many ties: last / first by right row order
    lb = [rng.integers(0, 4, nl).astype(np.int32) for _ in range(n_by)]
    rb = [rng.integers(0, 4, nr).astype(np.int32) for _ in range(n_by)]
    tol = None if tolerance is None else (float(tolerance) if dtype == "float64" else int(tolerance))
    want = _pandas_asof(lv, rv, lb, rb, direction, exact, tol)
    ones = lambda n: np.ones(n, bool)
    got = ao.join_asof((lv, ones(nl)), (rv, ones(nr)), [(b, ones(nl)) for b in lb], [(b, ones(nr)) for b in rb], direction, exact, tol)
    assert np.array_equal(got, want)


def test_oracle_pandas_ties_from_the_issue():
    """r = [1, 2, 2, 2, 5]: l = 2 takes the last 2 backward and the first 2 forward; a nearest tie at l = 4 over [3, 3, 5, 5] takes the
    last 3."""
    r = np.array([1, 2, 2, 2, 5], np.int64)
    one = lambda v: (v, np.ones(len(v), bool))
    assert ao.join_asof(one(np.array([2])), one(r), direction="backward").tolist() == [3]
    assert ao.join_asof(one(np.array([2])), one(r), direction="forward").tolist() == [1]
    assert ao.join_asof(one(np.array([4])), one(np.array([3, 3, 5, 5])), direction="nearest").tolist() == [1]
    assert _pandas_asof(np.array([2]), r, [], [], "backward", True, None).tolist() == [3]
    assert _pandas_asof(np.array([4]), np.array([3, 3, 5, 5]), [], [], "nearest", True, None).tolist() == [1]


def test_oracle_nulls_nan_and_wide_distances():
    v = lambda *x, dt=np.int64: np.array(x, dt)
    lo, hi = np.iinfo(np.int64).min, np.iinfo(np.int64).max
    l, r = (v(hi, 0), np.ones(2, bool)), (v(lo), np.ones(1, bool))
    assert ao.join_asof(l, r, tolerance=2 ** 64 - 2).tolist() == [-1, 0]         # INT64_MAX - INT64_MIN = 2^64 - 1: no wrap
    assert ao.join_asof(l, r, tolerance=2 ** 63 - 1).tolist() == [-1, -1]
    u = np.iinfo(np.uint64).max
    assert ao.join_asof((v(u, dt=np.uint64), np.ones(1, bool)), (v(0, dt=np.uint64), np.ones(1, bool)), tolerance=u).tolist() == [0]
    f = (v(np.nan, 1.0, np.inf, -0.0, 2.0, dt=np.float64), np.array([True, True, True, True, False]))
    rf = (v(0.0, np.inf, np.nan, 1.0, dt=np.float64), np.array([True, True, True, False]))
    assert ao.join_asof(f, rf).tolist() == [-1, 0, 1, 0, -1]                      # NaN and null keys match nothing; inf == inf
    assert ao.join_asof(f, rf, tolerance=0.5).tolist() == [-1, -1, 1, 0, -1]      # inf - inf is distance 0
    assert ao.join_asof(f, rf, direction="forward", allow_exact_matches=False).tolist() == [-1, 1, -1, 1, -1]


@pytest.mark.parametrize("seed", range(4))
def test_semi_and_anti_are_the_deduplicated_inner_join(seed):
    rng = np.random.default_rng(seed)
    nl, nr = 3000, 1200
    left = [(rng.integers(0, 40, nl).astype(np.int32), rng.random(nl) > 0.1), (rng.integers(0, 3, nl).astype(np.float64), rng.random(nl) > 0.05)]
    right = [(rng.integers(0, 40, nr).astype(np.int32), rng.random(nr) > 0.1), (rng.integers(0, 3, nr).astype(np.float64), np.ones(nr, bool))]
    li, _ = jo.join_indices(left, right, "inner")
    semi, anti = ao.join_exists(left, right, False), ao.join_exists(left, right, True)
    assert np.array_equal(semi, np.unique(li))
    assert np.array_equal(np.sort(np.concatenate([semi, anti])), np.arange(nl))


# ---- the frame layer: schemas, lazy steps, argument errors -------------------------------------------------------------------

def test_plan_join_existence_and_asof_schemas(rdf):
    from rust_dataframe_b200 import frame as F

    a = OrderedDict([("t", rdf.I64), ("x", rdf.F64), ("k", rdf.I32)])
    b = OrderedDict([("t", rdf.I64), ("y", rdf.F32), ("k", rdf.I32)])
    for how in ("left_semi", "left_anti"):
        assert rdf.plan_join(a, b, [("k", "k")], how) == list(a.items())
        with pytest.raises(rdf.ComputeError, match="Join column does not exist in table B"):
            rdf.plan_join(a, b, [("k", "zz")], how)
        with pytest.raises(rdf.ComputeError, match="Join columns must have compatible types"):
            rdf.plan_join(a, b, [("x", "y")], how)
    assert rdf.plan_join(a, b, [("k", "k")]) == rdf.plan_join(a, b, [("k", "k")], "inner")
    other = types.SimpleNamespace(schema=b)
    steps = [F.join(other, [("k", "k")], "left_semi"), F.join_asof(other, "t", by=[("k", "k")]), F.select(["a.t", "y"])]
    walk = F._schema_walk(a, steps)
    assert list(walk[1].items()) == list(a.items())
    assert list(walk[2]) == ["a.t", "x", "a.k", "b.t", "y", "b.k"]
    assert list(walk[3]) == ["a.t", "y"]
    assert F._columns_read(steps[1]) == {"t", "k"}
    assert F._columns_read(F.join_asof(other, "t", "u", [("k", "j")])) == {"t", "k"}
    bad = F._schema_walk(a, [F.join_asof(other, "x", "t")])   # Float64 against Int64: refused when evaluated
    assert bad[-1] == OrderedDict()


def test_join_asof_argument_errors(rdf):
    from rust_dataframe_b200.functions import _asof_tolerance

    TT = rdf.TemporalType
    col = lambda dtype, t=None: types.SimpleNamespace(dtype=dtype, temporal=t, ctx=None, handle=None)
    assert _asof_tolerance(None, col(rdf.I64)) == (0, 0, 0.0)
    assert _asof_tolerance(5, col(rdf.I32)) == (1, 5, 0.0)
    assert _asof_tolerance(float("inf"), col(rdf.F32)) == (1, 0, float("inf"))
    ms = datetime.timedelta(milliseconds=1)
    assert _asof_tolerance(ms, col(rdf.I64, TT.timestamp("ns"))) == (1, 1_000_000, 0.0)
    assert _asof_tolerance(datetime.timedelta(days=2), col(rdf.I32, TT.date32())) == (1, 2, 0.0)
    assert _asof_tolerance(datetime.timedelta(seconds=3), col(rdf.I64, TT.date64())) == (1, 3000, 0.0)
    with pytest.raises(rdf.ComputeError, match="whole number"):
        _asof_tolerance(datetime.timedelta(microseconds=1500), col(rdf.I64, TT.timestamp("ms")))
    with pytest.raises(rdf.ComputeError, match="timedelta"):
        _asof_tolerance(ms, col(rdf.I64))
    for bad, c in ((-1, col(rdf.I64)), (float("nan"), col(rdf.F64)), (-0.5, col(rdf.F32)), (2 ** 63, col(rdf.U64)), (1.5, col(rdf.I64))):
        with pytest.raises(rdf.ComputeError):
            _asof_tolerance(bad, c)
    with pytest.raises(rdf.UnsupportedType, match="direction"):
        rdf.join_asof_indices(col(rdf.I64), col(rdf.I64), direction="closest")
    with pytest.raises(rdf.ComputeError, match="left and a right"):
        rdf.join_asof_indices(col(rdf.I64), col(rdf.I64), [col(rdf.I32)], [])
    with pytest.raises(rdf.UnsupportedType, match="temporal"):
        rdf.join_asof_indices(col(rdf.I64, TT.timestamp("ms")), col(rdf.I64, TT.timestamp("us")))


def test_asof_spec_layout_and_enums(tmp_path, rdf):
    N = rdf.native
    src = tmp_path / "asof.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200df.h"\n'
                   "int main(void){printf(\"%zu %zu %zu %zu %zu %zu %d %d %d %d\\n\", sizeof(bdf_asof_spec), offsetof(bdf_asof_spec, allow_exact_matches),"
                   " offsetof(bdf_asof_spec, has_tolerance), offsetof(bdf_asof_spec, tolerance), offsetof(bdf_asof_spec, tolerance_f),"
                   " offsetof(bdf_asof_spec, direction), BDF_JOIN_LEFT_SEMI, BDF_JOIN_LEFT_ANTI, BDF_ASOF_FORWARD, BDF_ASOF_NEAREST);return 0;}\n")
    exe = tmp_path / "asof"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    S = N.AsofSpec
    assert got == [C.sizeof(S), S.allow_exact_matches.offset, S.has_tolerance.offset, S.tolerance.offset, S.tolerance_f.offset,
                   S.direction.offset, N.JOIN_LEFT_SEMI, N.JOIN_LEFT_ANTI, N.ASOF_FORWARD, N.ASOF_NEAREST]
    assert N.JOIN_TYPES["left_semi"] == 4 and N.JOIN_TYPES["left_anti"] == 5
    assert "bdf_join_asof_dev" in N.EXPORTED_SYMBOLS
