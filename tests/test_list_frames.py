"""List columns in frames without a GPU: the oracle of tests/list_frame_oracle.py against pyarrow, the planners' refusals of a list
column, and the header's new ABI."""
import os
import subprocess

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import list_frame_oracle as lfo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lists(rng, n):
    out = []
    for _ in range(n):
        if rng.random() < 0.1:
            out.append(None)
        else:
            out.append([None if rng.random() < 0.15 else int(v) for v in rng.integers(-5, 5, rng.integers(0, 6))])
    return out


def test_take_and_filter_oracle_against_pyarrow():
    rng = np.random.default_rng(1)
    lists = _lists(rng, 300)
    arr = pa.array(lists, pa.list_(pa.int64()))
    idx = [None if rng.random() < 0.1 else int(i) for i in rng.integers(0, len(lists), 500)]
    assert lfo.take(lists, idx) == pc.take(arr, pa.array(idx, pa.uint32())).to_pylist()
    mask = [None if rng.random() < 0.1 else bool(b) for b in rng.random(len(lists)) < 0.5]
    assert lfo.filter_(lists, mask) == pc.filter(arr, pa.array(mask, pa.bool_())).to_pylist()
    with pytest.raises(IndexError):
        lfo.take(lists, [len(lists)])


@pytest.mark.parametrize("n_keys", [1, 2])
def test_collect_oracle_against_pyarrow(n_keys):
    rng = np.random.default_rng(n_keys)
    n = 2000
    keys = [[None if rng.random() < 0.05 else int(v) for v in rng.integers(0, 30, n)] for _ in range(n_keys)]
    x = [None if rng.random() < 0.2 else float(v) for v in rng.integers(-4, 4, n)]
    names = [f"k{i}" for i in range(n_keys)]
    t = pa.table({**{nm: pa.array(k, pa.int32()) for nm, k in zip(names, keys)}, "x": pa.array(x, pa.float64())})
    # pyarrow's "list" keeps nulls and drops nothing: compare on the rows with a valid x, groups without one are the oracle's []
    valid = t.filter(pc.is_valid(t["x"]))
    g = valid.group_by(names, use_threads=False).aggregate([("x", "list"), ("x", "distinct", pc.CountOptions(mode="only_valid"))])
    want_list = {tuple(r[nm] for nm in names): r["x_list"] for r in g.to_pylist()}
    want_set = {tuple(r[nm] for nm in names): sorted(r["x_distinct"]) for r in g.to_pylist()}
    got_list, got_set = lfo.collect_list(keys, x), lfo.collect_set(keys, x)
    assert [k for k, _ in got_list] == [k for k, _ in got_set]
    assert [k for k, _ in got_list] == sorted({tuple(c[r] for c in keys) for r in range(n)}, key=lambda k: tuple(lfo._order(v) for v in k))
    for (k, l), (_, s) in zip(got_list, got_set):
        assert l == want_list.get(k, [])
        assert s == want_set.get(k, [])


def test_collect_set_float_rules():
    nan = float("nan")
    keys = [[1, 1, 1, 1, 1, 2, 2, None]]
    x = [-0.0, 0.0, nan, 1.0, nan, None, None, 3.0]
    got = lfo.collect_set(keys, x)
    assert [k for k, _ in got] == [(1,), (2,), (None,)]
    s = got[0][1]
    assert len(s) == 3 and str(s[0]) == "-0.0" and s[1] == 1.0 and np.isnan(s[2])   # the first occurrence's bits
    assert got[1][1] == [] and got[2][1] == [3.0]
    assert lfo.collect_list(keys, x)[1][1] == []


def test_planners_refuse_a_list_column(rdf):
    from rust_dataframe_b200 import frame as F

    N = rdf.native
    schema = {"k": rdf.I32, "x": rdf.F64, "tags": N.LIST_BASE + rdf.I64}
    with pytest.raises(rdf.UnsupportedType):
        F.plan_aggregate(schema, ["tags"], [("sum", ["x"])])
    with pytest.raises(rdf.UnsupportedType):
        F.plan_aggregate(schema, ["k"], [("count", ["tags"])])
    with pytest.raises(rdf.UnsupportedType):
        F.plan_join(schema, {"tags": N.LIST_BASE + rdf.I64}, [("tags", "tags")])
    with pytest.raises(rdf.UnsupportedType):
        F.plan_window(schema, ["tags"], [], [("r", "row_number")])
    with pytest.raises(rdf.UnsupportedType):
        F.plan_window(schema, ["k"], [], [("s", "sum", "tags")])
    # the list column is carried by the plans that do not name it
    assert ("tags", N.LIST_BASE + rdf.I64) in F.plan_window(schema, ["k"], [], [("s", "sum", "x")])
    assert ("a.tags", N.LIST_BASE + rdf.I64) in F.plan_join(schema, {"k": rdf.I32, "tags": N.LIST_BASE + rdf.F32}, [("k", "k")])


def test_header_declares_the_list_frame_abi(tmp_path, rdf):
    src = tmp_path / "abi.c"
    src.write_text("""
#include <stdio.h>
#include "b200df.h"
typedef char check_collect_list[BDF_GROUP_COLLECT_LIST == 48 ? 1 : -1];
typedef char check_collect_set[BDF_GROUP_COLLECT_SET == 49 ? 1 : -1];
typedef char check_mode[BDF_GROUP_MODE == 33 ? 1 : -1];
int main(void) {
    int (*take)(bdf_ctx*, const bdf_list*, const bdf_col*, bdf_list**) = bdf_list_take_dev;
    int (*filt)(bdf_ctx*, const bdf_list*, const bdf_col*, bdf_list**) = bdf_list_filter_dev;
    int (*grp)(bdf_ctx*, int32_t, const bdf_col* const*, int32_t, const bdf_group_agg*, bdf_col**, bdf_col**, bdf_list**, int64_t*) =
        bdf_group_by_lists_dev;
    int (*wr)(bdf_ctx*, const char*, int32_t, const char* const*, const bdf_col* const*, const bdf_temporal_type*, const bdf_list* const*) =
        bdf_ipc_write_lists;
    printf("%d %d %d\\n", BDF_GROUP_COLLECT_LIST, BDF_GROUP_COLLECT_SET, take != 0 && filt != 0 && grp != 0 && wr != 0);
    return 0;
}
""")
    exe = tmp_path / "abi"
    lib_dir = os.path.join(ROOT, "rust-dataframe_b200")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe),
                           "-L", lib_dir, "-lb200df", "-Wl,-rpath," + lib_dir])
    for name in ("bdf_list_take_dev", "bdf_list_filter_dev", "bdf_group_by_lists_dev", "bdf_ipc_write_lists"):
        assert name in rdf.native.EXPORTED_SYMBOLS
    assert rdf.native.COLLECT_FNS == {"collect_list": 48, "collect_set": 49}
