"""Distinct rows and set operations without a GPU: the numpy oracle (tests/setops_oracle.py) against pandas' duplicated, SQLite's
INTERSECT / EXCEPT and collections.Counter arithmetic; the C header's new section; and the frame layer's refusals, which must come
before any device call."""
import os
import sqlite3
import subprocess
from collections import Counter, OrderedDict

import numpy as np
import pandas as pd
import pytest

import setops_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _canon_row(row):
    """A row of Python values under the library's equality: one NaN, -0.0 == 0.0, None for NULL."""
    out = []
    for x in row:
        if x is None:
            out.append(None)
        elif isinstance(x, float) and x != x:
            out.append("nan")
        else:
            out.append(x + 0.0 if isinstance(x, float) else x)
    return tuple(out)


def _rows(keys):
    cols = [[(None if not m else (float(v) if np.asarray(v).dtype.kind == "f" else int(v))) for v, m in zip(vals, mask)] for vals, mask in keys]
    return list(zip(*cols))


def _random_keys(rng, n, card, nulls=True, nans=True):
    f = (rng.integers(0, card, n) - card // 2).astype(np.float64) * 0.5
    if nans:
        f[rng.random(n) < 0.1] = np.nan
    f[rng.random(n) < 0.1] = -0.0
    i = rng.integers(0, card, n).astype(np.int32)
    fm = np.ones(n, bool) if not nulls else rng.random(n) >= 0.1
    im = np.ones(n, bool) if not nulls else rng.random(n) >= 0.1
    return [(f, fm), (i, im)]


@pytest.mark.parametrize("keep", so.KEEPS)
@pytest.mark.parametrize("seed", range(4))
def test_duplicated_matches_pandas(keep, seed):
    rng = np.random.default_rng(seed)
    n = 3000
    f = (rng.integers(0, 6, n) - 3).astype(np.float64)
    f[rng.random(n) < 0.15] = np.nan
    f[rng.random(n) < 0.15] = -0.0
    i = rng.integers(0, 5, n)
    im = rng.random(n) >= 0.2
    df = pd.DataFrame({"f": f, "i": pd.array(np.where(im, i, 0), dtype="Int64")})
    df.loc[~im, "i"] = pd.NA
    want = df.duplicated(keep=keep).to_numpy()
    got = so.duplicated([(f, np.ones(n, bool)), (i, im)], keep)
    assert np.array_equal(got, want)


def test_duplicated_zero_signs_and_nan_payloads_are_one_value():
    v = np.array([0.0, -0.0, np.nan, -np.nan, 1.0, 0.0], np.float64)
    v[3] = np.frombuffer(np.uint64(0xfff0000000000123).tobytes(), np.float64)[0]   # another NaN payload
    assert so.duplicated([(v, np.ones(6, bool))], "first").tolist() == [False, True, False, True, False, True]
    assert so.duplicated([(v, np.array([1, 1, 1, 1, 0, 0], bool))], False).tolist() == [True] * 6


def _sqlite(left_rows, right_rows, op, n_keys):
    con = sqlite3.connect(":memory:")
    names = ", ".join(f"k{j}" for j in range(n_keys))
    for t, rows in (("l", left_rows), ("r", right_rows)):
        con.execute(f"CREATE TABLE {t} ({names})")
        con.executemany(f"INSERT INTO {t} VALUES ({', '.join('?' * n_keys)})", rows)
    sql = {"intersect": "INTERSECT", "except": "EXCEPT"}[op]
    out = con.execute(f"SELECT {names} FROM l {sql} SELECT {names} FROM r").fetchall()
    con.close()
    return out


@pytest.mark.parametrize("op", ["intersect", "except"])
@pytest.mark.parametrize("seed", range(4))
def test_distinct_set_ops_match_sqlite(op, seed):
    rng = np.random.default_rng(100 + seed)
    left, right = _random_keys(rng, 2000, 8, nans=False), _random_keys(rng, 1500, 8, nans=False)
    mask = so.set_op(left, right, op)
    lrows = _rows(left)
    got = [_canon_row(r) for r, k in zip(lrows, mask) if k]
    want = [_canon_row(r) for r in _sqlite(lrows, _rows(right), op, 2)]
    assert len(got) == len(set(got))                 # distinct: one copy of every kept row
    assert set(got) == set(want)
    first = {}
    for j, r in enumerate(lrows):                    # the kept copy is the first one
        first.setdefault(_canon_row(r), j)
    assert all(first[_canon_row(lrows[j])] == j for j in np.flatnonzero(mask))


@pytest.mark.parametrize("op", ["intersect_all", "except_all"])
@pytest.mark.parametrize("seed", range(4))
def test_all_forms_match_counter_arithmetic(op, seed):
    rng = np.random.default_rng(200 + seed)
    left, right = _random_keys(rng, 2500, 6), _random_keys(rng, 2000, 6)
    mask = so.set_op(left, right, op)
    lc = Counter(_canon_row(r) for r in _rows(left))
    rc = Counter(_canon_row(r) for r in _rows(right))
    want = lc & rc if op == "intersect_all" else lc - rc
    lrows = [_canon_row(r) for r in _rows(left)]
    assert Counter(r for r, k in zip(lrows, mask) if k) == want
    seen = Counter()                                 # the kept copies are the earliest ones
    for r, k in zip(lrows, mask):
        assert k == (seen[r] < want[r])
        seen[r] += 1


@pytest.mark.parametrize("op", so.OPS)
def test_every_run_shape(op):
    """Every (cl, cr) in 0..5 x 0..5 as its own run: the run keeps exactly its first q(cl, cr) left rows."""
    lv, rv = [], []
    for cl in range(6):
        for cr in range(6):
            key = cl * 6 + cr
            lv += [key] * cl
            rv += [key] * cr
    lv, rv = np.array(lv, np.int16), np.array(rv, np.int16)
    mask = so.set_op([(lv, np.ones(lv.size, bool))], [(rv, np.ones(rv.size, bool))], op)
    for key in np.unique(lv):
        rows = mask[lv == key]
        q = int(so.q_of(op, int((lv == key).sum()), int((rv == key).sum())))
        assert rows.tolist() == [True] * q + [False] * (rows.size - q)


def test_header_section_compiles_and_enums(tmp_path):
    src = tmp_path / "setops.c"
    src.write_text(
        '#include <stdio.h>\n#include "b200df.h"\n'
        "typedef char enum_values[(BDF_KEEP_FIRST == 0 && BDF_KEEP_LAST == 1 && BDF_KEEP_NONE == 2 && BDF_SETOP_INTERSECT == 0 &&"
        " BDF_SETOP_INTERSECT_ALL == 1 && BDF_SETOP_EXCEPT == 2 && BDF_SETOP_EXCEPT_ALL == 3 && BDF_K_GROUP == 11 && BDF_K_SELECT == 22 &&"
        " BDF_K_HIST == 23 && BDF_ABI_VERSION == 3) ? 1 : -1];\n"
        "int main(void){enum_values ok = {0}; (void)ok;"
        "int (*a)(bdf_ctx*, int32_t, const bdf_col* const*, int32_t, bdf_col**) = bdf_duplicated_dev;"
        "int (*b)(bdf_ctx*, int32_t, int32_t, const bdf_col* const*, const bdf_col* const*, bdf_col**) = bdf_set_op_dev;"
        "int (*c)(bdf_ctx*, int32_t, const bdf_col* const*, bdf_col**) = bdf_concat_dev;"
        "int (*d)(bdf_ctx*, int32_t, const bdf_list* const*, bdf_list**) = bdf_list_concat_dev;"
        "return (a && b && c && d) ? 0 : 1;}\n")
    obj = tmp_path / "setops.o"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", str(src), "-o", str(obj)])


def test_enum_values_and_bindings(rdf):
    N = rdf.native
    assert (N.KEEP_FIRST, N.KEEP_LAST, N.KEEP_NONE) == (0, 1, 2)
    assert [N.SET_OPS[k] for k in so.OPS] == [0, 1, 2, 3]
    for name in ("bdf_duplicated_dev", "bdf_set_op_dev", "bdf_concat_dev", "bdf_list_concat_dev", "bdf_bool_widen_dev"):
        assert name in N.EXPORTED_SYMBOLS
    text = open(os.path.join(ROOT, "include", "b200df.h")).read()
    assert "typedef enum { BDF_KEEP_FIRST = 0, BDF_KEEP_LAST, BDF_KEEP_NONE } bdf_keep;" in text
    assert "typedef enum { BDF_SETOP_INTERSECT = 0, BDF_SETOP_INTERSECT_ALL, BDF_SETOP_EXCEPT, BDF_SETOP_EXCEPT_ALL } bdf_setop;" in text
    assert "BDF_K_SELECT, BDF_K_HIST } bdf_kernel_id;" in text and "#define BDF_ABI_VERSION 3" in text


# ---- the frame layer refuses before any device work -------------------------------------------------------------------------

class _FakeColumn:
    def __init__(self, dtype, temporal=None):
        self.dtype, self.temporal = dtype, temporal


def _fake_list(rdf, dtype):
    class FakeList(rdf.ListColumn):
        def __init__(self):
            self.handle = None

        @property
        def dtype(self):
            return dtype

        def free(self):
            pass
    return FakeList()


@pytest.fixture
def no_device(rdf, monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("a device call was made")
    monkeypatch.setattr(rdf.native, "lib", refuse)
    monkeypatch.setattr(rdf.functions.N, "lib", refuse)
    return rdf


def _frame(rdf, cols):
    return rdf.DeviceFrame(OrderedDict(cols))


@pytest.mark.parametrize("op", ["union", "union_by_name", "intersect", "intersect_all", "subtract", "except_all"])
def test_frames_refuse_mismatched_schemas(no_device, op):
    rdf = no_device
    a = _frame(rdf, [("x", _FakeColumn(rdf.I32)), ("y", _FakeColumn(rdf.F64))])
    for b in (_frame(rdf, [("x", _FakeColumn(rdf.I32))]),
              _frame(rdf, [("x", _FakeColumn(rdf.I64)), ("y", _FakeColumn(rdf.F64))]),
              _frame(rdf, [("x", _FakeColumn(rdf.I32)), ("y", _FakeColumn(rdf.F32))])):
        with pytest.raises(rdf.UnsupportedType, match="Union can only be performed on tables with compatible column types"):
            getattr(a, op)(b)
    c = _frame(rdf, [("x", _FakeColumn(rdf.I32, "date32")), ("y", _FakeColumn(rdf.F64))])   # a Date32 column against an Int32 one
    with pytest.raises(rdf.UnsupportedType, match="compatible column types"):
        getattr(a, op)(c)


def test_frames_refuse_different_temporal_types(no_device):
    rdf = no_device
    a = _frame(rdf, [("x", _FakeColumn(rdf.I64, "timestamp[us]"))])
    b = _frame(rdf, [("x", _FakeColumn(rdf.I64, "timestamp[ms]"))])
    for op in ("union", "intersect", "except_all"):
        with pytest.raises(rdf.UnsupportedType, match="compatible column types"):
            getattr(a, op)(b)


def test_frames_refuse_list_keys_and_17_columns(no_device):
    rdf = no_device
    lst = _frame(rdf, [("x", _FakeColumn(rdf.I32)), ("l", _fake_list(rdf, rdf.I32))])
    for call in (lambda: lst.distinct(), lambda: lst.duplicated(), lambda: lst.drop_duplicates(["l"]), lambda: lst.intersect(lst),
                 lambda: lst.except_all(lst), lambda: lst.subtract(lst)):
        with pytest.raises(rdf.UnsupportedType, match="list column"):
            call()
    wide = _frame(rdf, [(f"c{j}", _FakeColumn(rdf.I8)) for j in range(17)])
    for call in (lambda: wide.distinct(), lambda: wide.duplicated(), lambda: wide.intersect_all(wide), lambda: wide.subtract(wide)):
        with pytest.raises(rdf.UnsupportedType, match="1..16"):
            call()
    with pytest.raises(rdf.UnsupportedType, match="keep"):
        rdf.duplicated([_FakeColumn(rdf.I8)], keep=True)


def test_lazy_steps_schema_and_columns_read(rdf):
    F = rdf.frame
    other = _frame(rdf, [("p", _FakeColumn(rdf.I32)), ("q", _FakeColumn(rdf.F64))])
    schema = OrderedDict([("a", rdf.I32), ("b", rdf.F64)])
    steps = [F.distinct(["b"]), F.set_op(other, "intersect_all"), F.distinct()]
    walk = F._schema_walk(schema, steps)
    assert [list(s.items()) for s in walk] == [list(schema.items())] * 4
    assert F._columns_read(steps[0]) == {"b"}
    assert F._columns_read(steps[1], schema) == {"a", "b"}
    assert F._columns_read(steps[2], schema) == {"a", "b"}
    bad = F._schema_walk(schema, [F.set_op(_frame(rdf, [("p", _FakeColumn(rdf.I32))]), "union")])
    assert list(bad[-1].items()) == []
    # a column that only the comparison reads is still observable before the step
    calc = F.calculate("add", ["b", "b"], "c")
    needed = F._needed_after([calc, F.distinct()], ["a", "b", "c"], F._schema_walk(schema, [calc, F.distinct()]))
    assert "c" in needed[0]


def test_a_failed_filter_frees_the_columns_already_filtered(rdf, monkeypatch):
    freed = []

    class Fake:
        def __init__(self, name):
            self.name = name

        def free(self):
            freed.append(self.name)

        def logical_not(self):
            return Fake("not-mask")

    def filter_any(c, m):
        if c.name == "c":
            raise rdf.ComputeError("the filter failed")
        return Fake(c.name + "-kept")

    monkeypatch.setattr(rdf.functions, "filter_any", filter_any)
    f = rdf.DeviceFrame(OrderedDict((n, Fake(n)) for n in "abc"))
    with pytest.raises(rdf.ComputeError):
        f._keep(Fake("mask"), invert=True)
    assert sorted(freed) == ["a-kept", "b-kept", "mask", "not-mask"]
