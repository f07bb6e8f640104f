"""The equi-join without a GPU: the numpy restatement (tests/join_oracle.py) on the data of the reference's three join tests,
against pyarrow's hash join and pandas' merge on many small shapes, DeviceFrame's plan (plan_join) and the join type enum."""
import json
import os
import subprocess

import numpy as np
import pytest

import join_oracle as jo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NULL = -1


def _fixture():
    with open(os.path.join(ROOT, "tests", "golden", "join_tables.json")) as fh:
        d = json.load(fh)

    def col(values):
        if any(isinstance(x, str) for x in values):   # float.hex() strings
            v = np.array([0.0 if x is None else float.fromhex(x) for x in values])
        else:
            v = np.array([0 if x is None else x for x in values], np.int32)
        return v, np.array([x is not None for x in values])

    j1, j2 = d["join_test_j1"], d["join_test_j2"]
    return {k: col(j1[k]) for k in ("a", "b")}, {k: col(j2[k]) for k in ("d", "f")}, j1["c"], j2["e"]


def _pairs(how, left, right):
    li, ri = jo.join_indices(left, right, how)
    return [(None if a == NULL else a, None if b == NULL else b) for a, b in zip(li.tolist(), ri.tolist())]


def test_reference_left_join_on_b_eq_d():
    """src/dataframe.rs test_left_join: 9 rows."""
    j1, j2, c, e = _fixture()
    got = _pairs("left", [j1["b"]], [j2["d"]])
    assert got == [(0, 0), (1, 1), (2, 2), (3, 3), (3, 4), (3, 5), (4, 6), (5, 7), (6, None)]
    assert [(c[a], e[b] if b is not None else None) for a, b in got][3:6] == [("delta", "iota"), ("delta", "kappa"), ("delta", "mu")]


def test_reference_right_join_on_a_eq_d():
    """src/dataframe.rs test_right_join: 10 rows; the null `a` rows of j1 match nothing."""
    j1, j2, _, _ = _fixture()
    assert _pairs("right", [j1["a"]], [j2["d"]]) == [(None, 0), (1, 1), (2, 2), (None, 3), (None, 4), (None, 5), (None, 6), (5, 7), (6, 7),
                                                     (None, 8)]


def test_reference_inner_join_on_a_eq_d():
    """src/dataframe.rs test_inner_join: 4 rows."""
    j1, j2, _, _ = _fixture()
    assert _pairs("inner", [j1["a"]], [j2["d"]]) == [(1, 1), (2, 2), (5, 7), (6, 7)]


def test_full_join_on_a_eq_d_is_the_sql_full_outer_join():
    """13 rows: the 7 LEFT rows, then the 6 right rows nobody matched.  The reference's FullJoin arm (join.rs:109-133) would give
    7: the 4 matched pairs and the 3 null-key rows of j1, dropping every unmatched row whose key is valid."""
    j1, j2, _, _ = _fixture()
    got = _pairs("full", [j1["a"]], [j2["d"]])
    assert got == [(0, None), (1, 1), (2, 2), (3, None), (4, None), (5, 7), (6, 7),
                   (None, 0), (None, 3), (None, 4), (None, 5), (None, 6), (None, 8)]
    assert len(got) == 13


def test_float_keys_of_the_fixture():
    """j2.f joined with itself: NaN matches NaN, inf matches inf, the null row matches nothing."""
    _, j2, _, _ = _fixture()
    got = _pairs("left", [j2["f"]], [j2["f"]])
    assert got == [(i, i if i != 4 else None) for i in range(9)]


DTYPES = ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "float32", "float64"]


def _side(rng, n, dtypes, card, null_frac):
    cols = []
    for dt in dtypes:
        dt = np.dtype(dt)
        if dt.kind == "f":
            v = (rng.integers(0, card, n) - card // 2).astype(dt) * dt.type(0.5)
            v[rng.random(n) < 0.15] = np.nan
            v[rng.random(n) < 0.15] = -0.0
        else:
            v = rng.integers(0, card, n).astype(dt)
        cols.append((v, rng.random(n) >= null_frac))
    return cols


def _multiset(li, ri):
    return sorted(zip(li.tolist(), ri.tolist()))


def test_oracle_against_pyarrow_join():
    import pyarrow as pa
    from hypothesis import given, settings, strategies as st

    kinds = {"left": "left outer", "right": "right outer", "inner": "inner", "full": "full outer"}

    @settings(max_examples=150, deadline=None)
    @given(st.integers(0, 14), st.integers(0, 14), st.lists(st.sampled_from(DTYPES), min_size=1, max_size=3), st.integers(1, 4),
           st.floats(0, 0.4), st.integers(0, 2 ** 31))
    def run(nl, nr, dtypes, card, null_frac, seed):
        rng = np.random.default_rng(seed)
        left, right = _side(rng, nl, dtypes, card, null_frac), _side(rng, nr, dtypes, card, null_frac)

        def table(cols, prefix, n):   # pyarrow compares float keys bitwise: -0.0 is handed over as 0.0
            t = {f"{prefix}{k}": pa.array(np.where(v == 0, 0, v).astype(v.dtype), mask=~m) for k, (v, m) in enumerate(cols)}
            t[f"{prefix}row"] = pa.array(np.arange(n, dtype=np.int64))
            return pa.table(t)

        lt, rt = table(left, "l", nl), table(right, "r", nr)
        lk, rk = [f"l{k}" for k in range(len(dtypes))], [f"r{k}" for k in range(len(dtypes))]
        for how in jo.HOWS:
            li, ri = jo.join_indices(left, right, how)
            j = lt.join(rt, lk, rk, join_type=kinds[how], use_threads=False)
            want = sorted((NULL if a is None else a, NULL if b is None else b)
                          for a, b in zip(j.column("lrow").to_pylist(), j.column("rrow").to_pylist()))
            assert _multiset(li, ri) == want, how

    run()


def test_oracle_against_pandas_merge_without_null_keys():
    import pandas as pd
    from hypothesis import given, settings, strategies as st

    kinds = {"left": "left", "right": "right", "inner": "inner", "full": "outer"}

    @settings(max_examples=150, deadline=None)
    @given(st.integers(0, 14), st.integers(0, 14), st.lists(st.sampled_from(DTYPES), min_size=1, max_size=3), st.integers(1, 4),
           st.integers(0, 2 ** 31))
    def run(nl, nr, dtypes, card, seed):
        rng = np.random.default_rng(seed)
        left, right = _side(rng, nl, dtypes, card, 0.0), _side(rng, nr, dtypes, card, 0.0)
        names = [f"k{k}" for k in range(len(dtypes))]
        ldf = pd.DataFrame({**{n: v for n, (v, _) in zip(names, left)}, "lrow": np.arange(nl)})
        rdf = pd.DataFrame({**{n: v for n, (v, _) in zip(names, right)}, "rrow": np.arange(nr)})
        for how in jo.HOWS:
            li, ri = jo.join_indices(left, right, how)
            m = ldf.merge(rdf, on=names, how=kinds[how])
            want = sorted((NULL if pd.isna(a) else int(a), NULL if pd.isna(b) else int(b)) for a, b in zip(m["lrow"], m["rrow"]))
            assert _multiset(li, ri) == want, how

    run()


def test_oracle_order():
    """The whole output, not just the set of pairs: left rows in row order, partners in right row order, FULL's tail in right row
    order, RIGHT = LEFT with the sides swapped."""
    rng = np.random.default_rng(5)
    left, right = _side(rng, 300, ["int16", "float64"], 4, 0.1), _side(rng, 200, ["int16", "float64"], 4, 0.1)
    for how in jo.HOWS:
        li, ri = jo.join_indices(left, right, how)
        if how == "right":
            assert np.array_equal(ri, np.sort(ri)) and set(ri.tolist()) == set(range(200))
            r2, l2 = jo.join_indices(right, left, "left")
            assert np.array_equal(li, l2) and np.array_equal(ri, r2)
            continue
        head = li if how != "full" else li[li >= 0]
        assert np.array_equal(head, np.sort(head))
        for i in np.unique(head):
            part = ri[:len(head)][head == i]
            assert np.array_equal(part, np.sort(part))
        if how == "full":
            assert (li[len(head):] == NULL).all() and np.array_equal(ri[len(head):], np.sort(ri[len(head):]))


def test_plan_join():
    from rust_dataframe_b200 import F64, I32, I64, ComputeError, UnsupportedType, plan_join
    from rust_dataframe_b200 import native

    BOOL = native.BOOL

    a = {"a": I32, "b": I32, "x": F64}
    b = {"d": I32, "x": F64, "f": F64}
    assert plan_join(a, b, [("b", "d")]) == [("a", I32), ("b", I32), ("a.x", F64), ("d", I32), ("b.x", F64), ("f", F64)]
    assert plan_join(a, b, [("a", "d"), ("x", "f")]) == plan_join(a, b, [("b", "d")])
    with pytest.raises(ComputeError, match="Join columns do not exist in tables"):
        plan_join(a, b, [("nope", "nope")])
    with pytest.raises(ComputeError, match="Join column does not exist in table A"):
        plan_join(a, b, [("nope", "d")])
    with pytest.raises(ComputeError, match="Join column does not exist in table B"):
        plan_join(a, b, [("a", "nope")])
    with pytest.raises(ComputeError, match="Join columns must have compatible types"):
        plan_join(a, b, [("a", "f")])
    with pytest.raises(ComputeError, match="Join column does not exist in table B"):   # try_join's order: criterion by criterion
        plan_join(a, b, [("a", "nope"), ("a", "f")])
    with pytest.raises(UnsupportedType):
        plan_join({"p": BOOL}, {"q": BOOL}, [("p", "q")])
    with pytest.raises(ComputeError, match="Join criteria cannot be empty"):
        plan_join(a, b, [])
    with pytest.raises(ComputeError):
        plan_join({"a": I64}, {"a": I32}, [("a", "a")])


def test_plan_fusion_keeps_every_column_a_join_passes_on():
    """A run of Calculations before a join is not fused when the join would carry an intermediate into its output."""
    from collections import OrderedDict

    from rust_dataframe_b200 import F64, I32
    from rust_dataframe_b200.frame import calculate, join, plan_fusion, select

    class Other:
        schema = OrderedDict([("k", I32), ("z", F64)])

    schema = OrderedDict([("k", I32), ("x", F64), ("y", F64)])
    steps = [calculate("add", ["x", "y"], "t"), calculate("multiply", ["t", "y"], "u"), join(Other(), [("k", "k")], "inner"),
             select(["a.k", "t", "u"])]
    assert [k for k, _ in plan_fusion(schema, steps)] == ["calculate", "calculate", "join", "select"]
    steps2 = [calculate("add", ["x", "y"], "t"), calculate("multiply", ["t", "y"], "u"), select(["k", "u"]),
              join(Other(), [("k", "k")], "inner")]
    assert [k for k, _ in plan_fusion(schema, steps2)] == ["fused", "select", "join"]


def test_join_types_match_the_header(tmp_path):
    import rust_dataframe_b200 as rdf

    src = tmp_path / "jt.c"
    src.write_text("#include <stdio.h>\n#include \"b200df.h\"\n"
                   "int main(void){printf(\"%d %d %d %d %d\\n\", (int)BDF_JOIN_LEFT, (int)BDF_JOIN_RIGHT, (int)BDF_JOIN_INNER,"
                   " (int)BDF_JOIN_FULL, (int)BDF_K_JOIN);return 0;}\n")
    exe = tmp_path / "jt"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    N = rdf.native
    assert got == [N.JOIN_TYPES["left"], N.JOIN_TYPES["right"], N.JOIN_TYPES["inner"], N.JOIN_TYPES["full"], N.K_JOIN]
    assert N.KERNEL_NAMES[N.K_JOIN] == "join"
