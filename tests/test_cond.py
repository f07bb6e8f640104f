"""CPU checks of null handling and conditional selection: the numpy restatement in cond_oracle.py against pyarrow, SQLite and
hand-written Spark cases; the bdf_arg layout against gcc; fill_null's column eligibility; and the planner keeping a column
that only a null-test filter reads.  No GPU is needed."""
import ctypes as C
import math
import os
import sqlite3
import struct
import subprocess
from collections import OrderedDict

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import cond_oracle as co

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RNG_SEED = 20261017


def _arg(rng, n, dtype, null_frac, lo=-50, hi=50):
    v = rng.integers(lo, hi, n).astype(dtype)
    return v, rng.random(n) >= null_frac


def _to_pa(a):
    v, m = a
    return pa.array(v, mask=~m)


def _from_pa(arr, dtype):
    m = np.asarray(arr.is_valid())
    v = np.asarray(arr.fill_null(0) if arr.type != pa.bool_() else arr.fill_null(False)).astype(dtype)
    return v, m


@pytest.mark.parametrize("dtype", [np.int32, np.float64, np.uint8])
@pytest.mark.parametrize("k", [1, 2, 3, 7])
def test_coalesce_matches_pyarrow(dtype, k):
    rng = np.random.default_rng(RNG_SEED + k)
    args = [_arg(rng, 500, dtype, f) for f in np.linspace(0.0, 0.9, k)]
    want = _from_pa(pc.coalesce(*[_to_pa(a) for a in args]), dtype)
    assert co.same(co.coalesce(args), want)


@pytest.mark.parametrize("dtype", [np.int16, np.float32, np.uint64])
@pytest.mark.parametrize("k", [2, 3, 5])
def test_greatest_least_match_pyarrow_without_nan(dtype, k):
    rng = np.random.default_rng(RNG_SEED + 10 + k)
    args = [_arg(rng, 400, dtype, f, 0, 30) for f in np.linspace(0.1, 0.8, k)]
    pas = [_to_pa(a) for a in args]
    assert co.same(co.greatest(args), _from_pa(pc.max_element_wise(*pas, skip_nulls=True), dtype))
    assert co.same(co.least(args), _from_pa(pc.min_element_wise(*pas, skip_nulls=True), dtype))


@pytest.mark.parametrize("branches", [1, 2, 4])
def test_case_when_matches_pyarrow(branches):
    """Arrow's case_when with every NULL condition first replaced by false (fill_null) is the SQL rule the oracle states: a NULL
    condition counts as false."""
    rng = np.random.default_rng(RNG_SEED + 20 + branches)
    n = 600
    conds = [(rng.random(n) < 0.3, rng.random(n) >= 0.2) for _ in range(branches)]
    values = [_arg(rng, n, np.int64, 0.15) for _ in range(branches)] + [_arg(rng, n, np.int64, 0.3)]
    cond_pa = [pa.array(c, mask=~m) for c, m in conds]
    struct_ = pa.StructArray.from_arrays([pc.fill_null(c, False) for c in cond_pa], [f"c{i}" for i in range(branches)])
    want = _from_pa(pc.case_when(struct_, *[_to_pa(v) for v in values]), np.int64)
    assert co.same(co.case_when(conds, values), want)
    # the missing ELSE is NULL
    no_else = values[:-1] + [co.scalar(None, n, np.int64)]
    want2 = _from_pa(pc.case_when(struct_, *[_to_pa(v) for v in values[:-1]]), np.int64)
    assert co.same(co.case_when(conds, no_else), want2)
    if branches == 1:   # if_else is the one-branch form
        want3 = _from_pa(pc.if_else(pc.fill_null(cond_pa[0], False), _to_pa(values[0]), _to_pa(values[1])), np.int64)
        assert co.same(co.case_when(conds, values), want3)


def _sqlite_rows(cols):
    n = len(cols[0][0])
    return [tuple(int(v[i]) if m[i] else None for v, m in cols) for i in range(n)]


def _unpack(rows, dtype):
    v = np.array([0 if r is None else r for r in rows], dtype=dtype)
    return v, np.array([r is not None for r in rows])


def test_coalesce_case_when_ifnull_match_sqlite():
    rng = np.random.default_rng(RNG_SEED + 30)
    n = 300
    a, b, c = (_arg(rng, n, np.int64, f) for f in (0.3, 0.5, 0.2))
    c1, c2 = (rng.random(n) < 0.4, rng.random(n) >= 0.3), (rng.random(n) < 0.5, rng.random(n) >= 0.3)
    db = sqlite3.connect(":memory:")
    db.execute("CREATE TABLE t (i INTEGER, a INTEGER, b INTEGER, c INTEGER, c1 INTEGER, c2 INTEGER)")
    rows = _sqlite_rows([a, b, c, c1, c2])
    db.executemany("INSERT INTO t VALUES (?, ?, ?, ?, ?, ?)", [(i,) + r for i, r in enumerate(rows)])

    def q(sql):
        return [r[0] for r in db.execute(f"SELECT {sql} FROM t ORDER BY i")]

    assert co.same(co.coalesce([a, b, c]), _unpack(q("COALESCE(a, b, c)"), np.int64))
    assert co.same(co.coalesce([a, co.scalar(7, n, np.int64)]), _unpack(q("IFNULL(a, 7)"), np.int64))
    conds = [(c1[0], c1[1]), (c2[0], c2[1])]
    assert co.same(co.case_when(conds, [a, b, c]), _unpack(q("CASE WHEN c1 THEN a WHEN c2 THEN b ELSE c END"), np.int64))
    assert co.same(co.case_when(conds, [a, b, co.scalar(None, n, np.int64)]), _unpack(q("CASE WHEN c1 THEN a WHEN c2 THEN b END"), np.int64))


def _one(x, valid=True):
    return np.array([0.0 if x is None else x], dtype=np.float64), np.array([valid and x is not None])


def test_spark_cases():
    nan, inf = float("nan"), float("inf")
    v, m = co.greatest([_one(nan), _one(inf)])
    assert m[0] and math.isnan(v[0])                                  # greatest(NaN, inf) = NaN
    v, m = co.greatest([_one(-0.0), _one(0.0)])
    assert m[0] and struct.pack("<d", v[0]) == struct.pack("<d", -0.0)  # the earliest of equal values keeps its bits
    v, m = co.least([_one(0.0), _one(-0.0)])
    assert m[0] and struct.pack("<d", v[0]) == struct.pack("<d", 0.0)
    v, m = co.least([_one(None), _one(1.0)])
    assert m[0] and v[0] == 1.0                                       # least(NULL, 1) = 1
    v, m = co.nanvl(_one(None), _one(1.0))
    assert not m[0]                                                   # nanvl(NULL, 1) = NULL
    v, m = co.nanvl(_one(nan), _one(None))
    assert not m[0]                                                   # nanvl(NaN, NULL) = NULL
    v, m = co.nanvl(_one(nan), _one(2.0))
    assert m[0] and v[0] == 2.0
    v, m = co.is_nan(_one(None))
    assert m[0] and not v[0]                                          # isnan(NULL) = false
    v, m = co.case_when([(np.array([False]), np.array([False]))], [_one(1.0), _one(2.0)])
    assert m[0] and v[0] == 2.0                                       # CASE WHEN NULL THEN 1 ELSE 2 = 2
    v, m = co.coalesce([_one(nan), _one(1.0)])
    assert m[0] and math.isnan(v[0])                                  # NaN is a value, not a null
    payload = np.array([0x7FF8000000000123], dtype=np.uint64).view(np.float64)
    v, m = co.coalesce([(payload, np.array([True]))])
    assert v.view(np.uint64)[0] == 0x7FF8000000000123                 # NaN payloads survive


def test_null_tests():
    a = (np.array([1.0, float("nan"), 3.0, float("nan")]), np.array([True, True, False, False]))
    assert list(co.is_null(a)[0]) == [False, False, True, True]
    assert list(co.is_not_null(a)[0]) == [True, True, False, False]
    assert list(co.is_nan(a)[0]) == [False, True, False, False]
    assert not co.is_nan((np.arange(4, dtype=np.int32), np.ones(4, bool)))[0].any()


def test_bdf_arg_layout_and_enums(tmp_path, rdf):
    src = tmp_path / "arg.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200df.h"\n'
                   'int main(void){printf("%zu %zu %zu %zu %d %d %d %d %d\\n", sizeof(bdf_arg), offsetof(bdf_arg, column), offsetof(bdf_arg, bits),'
                   ' offsetof(bdf_arg, valid), BDF_ROW_COALESCE, BDF_ROW_GREATEST, BDF_ROW_LEAST, BDF_ROW_NANVL, BDF_IS_NAN);return 0;}\n')
    exe = tmp_path / "arg"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    N = rdf.native
    assert got[:4] == [C.sizeof(N.Arg), N.Arg.column.offset, N.Arg.bits.offset, N.Arg.valid.offset]
    assert got[4:] == [N.ROW_COALESCE, N.ROW_GREATEST, N.ROW_LEAST, N.ROW_NANVL, N.IS_NAN]
    for name in ("bdf_rowwise_dev", "bdf_case_when_dev", "bdf_null_test_dev"):
        assert name in N.EXPORTED_SYMBOLS


def test_fill_null_eligibility(rdf):
    from rust_dataframe_b200.frame import fill_value_fits as fits

    I8, I32, U8, U64, F32, F64, BOOL = rdf.I8, rdf.I32, rdf.U8, rdf.U64, rdf.F32, rdf.F64, rdf.native.BOOL
    assert fits(I8, 127) and not fits(I8, 128) and not fits(U8, -1) and fits(U64, 2 ** 64 - 1)
    assert fits(F32, 2 ** 24) and not fits(F32, 2 ** 24 + 1) and fits(F64, 2 ** 53) and not fits(F64, 2 ** 53 + 1)
    assert fits(F64, 0.1) and not fits(F32, 0.1) and fits(F32, 0.5) and fits(F32, float("nan")) and fits(F32, float("inf"))
    assert not fits(I32, 1.0) and not fits(I32, True) and fits(BOOL, True) and not fits(BOOL, 1)


def test_scalar_bits(rdf):
    from rust_dataframe_b200.functions import _scalar_bits

    assert _scalar_bits(rdf.I8, -1) == 0xFF and _scalar_bits(rdf.F64, -0.0) == 1 << 63
    assert _scalar_bits(rdf.F32, 1.0) == 0x3F800000 and _scalar_bits(rdf.native.BOOL, True) == 1
    for dtype, v in ((rdf.I8, 300), (rdf.F32, 0.1), (rdf.I32, 1.5), (rdf.native.BOOL, 1)):
        with pytest.raises(rdf.UnsupportedType):
            _scalar_bits(dtype, v)


def test_planner_keeps_a_column_only_a_null_test_reads(rdf):
    """A Calculation whose output only an is_null filter reads, and that a later select drops, must not be fused away."""
    from rust_dataframe_b200.frame import Calculation, filter_, is_nan, is_not_null, is_null, plan_fusion, select

    schema = OrderedDict([("a", rdf.F64), ("b", rdf.F64)])
    for test in (is_null, is_not_null, is_nan):
        steps = [("calculate", Calculation("add", ["a", "b"], "c")), ("calculate", Calculation("multiply", ["c", "a"], "d")),
                 filter_(test("c")), select(["d"])]
        planned = plan_fusion(schema, steps)
        outputs = {arg.output for kind, arg in planned if kind in ("calculate", "fused")}
        assert "c" in outputs, planned
        assert planned[-2][0] == "filter" and planned[-2][1] == (test.__name__, ("col", "c"))
