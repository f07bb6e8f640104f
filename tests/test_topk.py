"""Top-k without a GPU: the rounds restated in numpy (topk_oracle.py) against the C oracle's stable lexsort, the planner's rewrite of
sort -> limit into one top_k step, and the header's new section."""
import os
import subprocess
from collections import OrderedDict

import numpy as np
import pytest

import topk_oracle as to

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TYPES = ["I8", "I16", "I32", "I64", "U8", "U16", "U32", "U64", "F32", "F64"]


def _values(rng, npdt, n, card):
    if npdt.kind == "f":
        pool = np.array([np.nan, -0.0, 0.0, np.inf, -np.inf, 1.5, -1.5, 2.0, -7.25, 1e300 if npdt.itemsize == 8 else 3e38], npdt)
        return pool[rng.integers(0, min(card, pool.size), n)]
    info = np.iinfo(npdt)
    pool = np.array(sorted({info.min, info.max, 0, 1, info.max - 1, info.min + 1, 5, 17}), npdt)
    return pool[rng.integers(0, min(card, pool.size), n)] if card <= pool.size else rng.integers(info.min, info.max, n, dtype=npdt, endpoint=True)


def _chunks(rdf, v, m, rng):
    cuts = np.sort(rng.integers(0, len(v) + 1, rng.integers(0, 3)))
    bounds = [0, *cuts.tolist(), len(v)]
    return [rdf.PrimitiveArray.from_numpy(v[a:b].copy(), m[a:b].copy()) for a, b in zip(bounds[:-1], bounds[1:])]


def _boundaries(want, keys):
    """Positions in sort order where the tuple of the first j criteria changes, for every j, and one either side."""
    out = set()
    for j in range(1, len(keys) + 1):
        prev = None
        for i, r in enumerate(want):
            cur = tuple((bool(m[r]), int(k[r]) if m[r] else 0) for k, m in keys[:j])
            if cur != prev:
                out |= {i - 1, i, i + 1}
            prev = cur
    return out


def test_rounds_equal_the_oracles_sort_prefix(rdf, oracle):
    rng = np.random.default_rng(2024)
    cases = 0
    for case in range(2000):
        n = int(rng.integers(0, 40))
        n_keys = int(rng.integers(1, 5))
        crit, host, keys = [], [], []
        for _ in range(n_keys):
            dtype = getattr(rdf, TYPES[int(rng.integers(0, len(TYPES)))])
            npdt = np.dtype(rdf.NP_DTYPES[dtype])
            card = int(rng.choice([1, 2, 3, 5, 10, 1000]))
            v = _values(rng, npdt, n, card)
            m = rng.random(n) >= rng.choice([0.0, 0.1, 0.5, 1.0])
            desc = bool(rng.integers(0, 2))
            crit.append((v, m, desc))
            host.append((_chunks(rdf, v, m, rng) or [rdf.PrimitiveArray.from_numpy(v, m)], desc))
            keys.append((to.sort_key(v), m))
        st, want = oracle.lexsort_indices(host)
        assert st == oracle.OK
        ks = {0, 1, n - 1, n, n + 5} | _boundaries(want, keys)
        for k in sorted(x for x in ks if x >= 0):
            got = to.top_k(crit, k)
            assert np.array_equal(got, want[:k]), (case, k, got, want[:k])
            cases += 1
    assert cases > 15_000


def test_the_rounds_choose_without_sorting_every_row():
    v = np.array([5, 1, 4, 1, 3, 1, 2], np.int32)
    ok = np.ones(7, bool)
    assert to.chosen_rows([(v, ok, False)], 3).tolist() == [1, 3, 5]           # three ties at the threshold, all needed
    assert to.chosen_rows([(v, ok, False)], 2).tolist() == [1, 3]              # the first two ties in row order
    assert to.chosen_rows([(v, ok, True)], 2).tolist() == [0, 2]
    nulls = np.array([True, False, True, False, True, True, False])
    assert to.chosen_rows([(v, nulls, True)], 5).tolist() == [0, 1, 2, 4, 5]   # every valid row, then the first null
    assert to.top_k([(v, nulls, True)], 5).tolist() == [0, 2, 4, 5, 1]
    f = np.array([np.nan, -0.0, 0.0, -np.nan, np.inf], np.float64)
    assert to.top_k([(f, np.ones(5, bool), False)], 5).tolist() == [1, 2, 4, 0, 3]


# ---- the planner --------------------------------------------------------------------------------------------------------------

SCHEMA = OrderedDict([("a", 5), ("b", 9), ("c", 2)])


def _plan(rdf, steps, **kw):
    return rdf.plan_fusion(SCHEMA, steps, **kw)


def test_rewrite_of_adjacent_and_separated_steps(rdf):
    F = rdf.frame
    crit = [("a", True), ("b", False)]
    assert _plan(rdf, [F.sort(crit), F.limit(7)]) == [("top_k", (crit, 7))]
    assert _plan(rdf, [F.sort(crit), F.select(["a", "c"]), F.drop(["c"]), F.limit(3)]) == \
        [("top_k", (crit, 3)), ("select", ["a", "c"]), ("drop", ["c"])]
    assert _plan(rdf, [F.limit(9), F.sort(crit), F.limit(-2), F.limit(1)]) == [("limit", 9), ("top_k", (crit, -2)), ("limit", 1)]
    assert _plan(rdf, [F.sort(crit), F.limit(4), F.sort([("c", False)]), F.drop(["b"]), F.limit(2)]) == \
        [("top_k", (crit, 4)), ("top_k", ([("c", False)], 2)), ("drop", ["b"])]


def test_no_rewrite_across_row_changing_steps(rdf):
    F = rdf.frame
    crit = [("a", False)]
    other = rdf.DeviceFrame(OrderedDict())
    between = [F.filter_(("gt", ("col", "a"), ("scalar", 0))), F.calculate("sin", ["b"], "s"), F.join(other, [("a", "a")], "inner"),
               F.window([], [("a", False)], [("r", "row_number")]), F.distinct(["a"])]
    for step in between:
        plan = _plan(rdf, [F.sort(crit), step, F.limit(5)])
        assert plan[0] == ("sort", crit) and plan[-1] == ("limit", 5), step
    assert _plan(rdf, [F.limit(5)]) == [("limit", 5)]
    assert _plan(rdf, [F.select(["a"]), F.limit(5)]) == [("select", ["a"]), ("limit", 5)]
    assert _plan(rdf, [F.sort(crit)]) == [("sort", crit)]


def test_unfused_evaluation_runs_the_steps_as_written(rdf):
    calls = []

    class Recorder:
        def __getattr__(self, name):
            def step(*args):
                calls.append(name)
                return self
            return step

    F = rdf.frame
    steps = [F.sort([("a", False)]), F.select(["a"]), F.limit(3)]
    rdf.DeviceFrame.evaluate(Recorder(), steps, fuse=False)
    assert calls == ["sort", "select", "limit"]
    calls.clear()
    rec = Recorder()
    rec.schema = SCHEMA
    rdf.DeviceFrame.evaluate(rec, steps)
    assert calls == ["top_k", "select"]


# ---- the header ---------------------------------------------------------------------------------------------------------------

def test_header_declares_and_exports_the_entry(rdf, tmp_path):
    src = tmp_path / "topk.c"
    src.write_text(
        '#include <stdio.h>\n#include "b200df.h"\n'
        "typedef char ids[(BDF_K_SELECT == 22 && BDF_K_HIST == 23 && BDF_ABI_VERSION == 3) ? 1 : -1];\n"
        "int main(void){ids ok = {0}; (void)ok;"
        "int (*f)(bdf_ctx*, int32_t, const bdf_sort_key*, int64_t, bdf_col**) = bdf_top_k_indices_dev;"
        "return f ? 0 : 1;}\n")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", str(src), "-o",
                           str(tmp_path / "topk.o")])
    assert "bdf_top_k_indices_dev" in rdf.native.EXPORTED_SYMBOLS
