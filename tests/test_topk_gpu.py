"""Top-k on the device (bdf_top_k_indices_dev, DeviceFrame.top_k and the lazy sort -> limit rewrite).  The first k rows of a
stable sort have exactly one right answer, so indices are compared for EQUALITY with the C oracle's lexsort and with the
device sort's first k entries, and frames bit for bit with sort(...).limit(...)."""
import ctypes as C
from collections import OrderedDict

import numpy as np
import pytest

from helpers import pool_used

pytestmark = pytest.mark.gpu

DTYPES = ["I8", "I16", "I32", "I64", "U8", "U16", "U32", "U64", "F32", "F64"]
LENS = [0, 1, 31, 2049, 0, 10_007, 70_001]


def _key(rdf, rng, dtype, lens, null_frac=0.1, card=None, sliced=True, specials=True):
    """Host chunks of one key column: sliced chunks (validity at a bit offset), planted -0.0 / NaN / inf for floats."""
    npdt = np.dtype(rdf.NP_DTYPES[dtype])
    out = []
    for j, n in enumerate(lens):
        pad = (3 + 5 * j) % 23 if sliced else 0
        m = n + pad + 2
        if card is not None:
            v = rng.integers(0, card, m).astype(npdt)
        elif npdt.kind == "f":
            v = np.round(rng.normal(0, 50, m)).astype(npdt)
            if specials and m > 16:
                at = rng.choice(m, 8, replace=False)
                v[at] = np.array([np.nan, -0.0, 0.0, np.inf, -np.inf, -np.nan, 1.5, -1.5], npdt)
        else:
            info = np.iinfo(npdt)
            v = rng.integers(max(info.min, -300), min(info.max, 300), m, dtype=npdt, endpoint=True)
        valid = rng.random(m) >= null_frac if null_frac else None
        a = rdf.PrimitiveArray.from_numpy(v, valid)
        a.null_count = -1 if a.validity is not None else 0
        out.append(a.slice(pad, n))
    return out


def _indices(col):
    got = col.download()
    assert len(got) == 1 and got[0].validity is None
    return got[0].value_slice().copy()


def _check(rdf, oracle, crit_host, ks):
    """crit_host: [(chunks, descending)].  For every k: top_k == oracle lexsort[:k] == device sort[:k]."""
    cols = [(rdf.Column.upload(ch), d) for ch, d in crit_host]
    st, want = oracle.lexsort_indices(crit_host)
    assert st == oracle.OK
    full = _indices(rdf.sort_indices(cols))
    assert np.array_equal(full, want)
    for k in ks:
        got = _indices(rdf.top_k_indices(cols, k))
        assert got.dtype == np.uint32 and len(got) == min(k, len(want)), k
        bad = np.flatnonzero(got != want[:k])
        assert bad.size == 0, f"k={k}: differ at {bad[:5]}: got {got[bad[:5]]}, want {want[bad[:5]]}"


def _ks(n, extra=()):
    return sorted({0, 1, 2, 7, n // 100, n // 10, n // 2, 5 * n // 8, 5 * n // 8 + 1, n - 1, n, n + 5, *[e for e in extra if e >= 0]})


@pytest.mark.parametrize("tname", DTYPES)
def test_every_type_both_directions(rdf, ctx, oracle, tname):
    dtype = getattr(rdf, tname)
    rng = np.random.default_rng(300 + dtype)
    n = sum(LENS)
    for desc in (False, True):
        key = _key(rdf, rng, dtype, LENS)
        valid = sum(int(a.valid_mask().sum()) for a in key)
        _check(rdf, oracle, [(key, desc)], _ks(n, (valid - 1, valid, valid + 1)))   # k on the valid / null boundary


def test_ties_through_three_criteria(rdf, ctx, oracle):
    rng = np.random.default_rng(11)
    lens = [5000, 0, 33, 40_000, 7]
    n = sum(lens)
    for desc in ((False, True, False), (True, False, True)):
        k1 = _key(rdf, rng, rdf.I8, lens, 0.05, card=3)
        k2 = _key(rdf, rng, rdf.F64, lens, 0.1, card=4)
        k3 = _key(rdf, rng, rdf.U16, lens, 0.1, card=5)
        _check(rdf, oracle, list(zip([k1, k2, k3], desc)), _ks(n, (3, 100, 1000, 5000)))


def test_all_null_all_equal_and_all_tied_keys(rdf, ctx, oracle):
    rng = np.random.default_rng(12)
    lens = [3000, 0, 4097, 61]
    n = sum(lens)
    all_null = _key(rdf, rng, rdf.I32, lens, null_frac=1.0)
    equal = _key(rdf, rng, rdf.F64, lens, null_frac=0, card=1)
    second = _key(rdf, rng, rdf.I64, lens, 0.2)
    ks = _ks(n, (5, 300))
    _check(rdf, oracle, [(all_null, False), (second, True)], ks)
    _check(rdf, oracle, [(equal, True), (second, False)], ks)
    _check(rdf, oracle, [(equal, False)], ks)                                   # every criterion equal: the earliest rows win
    _check(rdf, oracle, [(equal, False), (_key(rdf, rng, rdf.U8, lens, 0, card=1), True)], ks)
    _check(rdf, oracle, [(all_null, True)], ks)


def test_unsliced_word_aligned_chunks(rdf, ctx, oracle):
    rng = np.random.default_rng(13)
    lens = [4096, 2048, 32, 1000]   # chunks that own their bitmap words, then one that does not end on a word
    for tname in ("I8", "F32", "U64"):
        key = _key(rdf, rng, getattr(rdf, tname), lens, 0.1, sliced=False)
        _check(rdf, oracle, [(key, True), (_key(rdf, rng, rdf.I16, lens, 0.1, sliced=False), False)], _ks(sum(lens), (100,)))


def test_crossover_both_sides_and_launch_records(rdf, ctx):
    rng = np.random.default_rng(14)
    n = 1 << 20
    key = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(rng.normal(0, 1, n))], ctx=ctx)
    full = _indices(rdf.sort_indices([(key, False)]))
    for k, sorts_all in ((5 * n // 8, False), (5 * n // 8 + 1, True)):   # the crossover: k > 5n / 8 sorts every row
        ctx.profile_enable(True)
        got = _indices(rdf.top_k_indices([(key, False)], k))
        recs = ctx.profile_read()
        ctx.profile_enable(False)
        assert np.array_equal(got, full[:k])
        assert any(r["kernel"] == "sort" and r["rows"] == n for r in recs) == sorts_all, k
        assert sorts_all or any(r["kernel"] == "select" for r in recs)


# ---- frames ---------------------------------------------------------------------------------------------------------------------

def _frame(rdf, ctx, rng, lens):
    n = sum(lens)
    ts = rdf.TemporalType.timestamp("us")

    def up(v, m):
        chunks, at = [], 0
        for ln in lens:
            chunks.append(rdf.PrimitiveArray.from_numpy(v[at:at + ln].copy(), m[at:at + ln].copy()))
            at += ln
        return rdf.Column.upload(chunks, ctx=ctx)

    cols = OrderedDict()
    cols["k"] = up(rng.integers(0, 20, n).astype(np.int32), rng.random(n) >= 0.1)
    cols["x"] = up(np.round(rng.normal(0, 5, n)), rng.random(n) >= 0.05)
    cols["t"] = up(rng.integers(0, 30, n).astype(np.int64) * 3_600_000_000, rng.random(n) >= 0.05).with_temporal(ts)
    cols["flag"] = rdf.Column.upload([rdf.BooleanArray.from_numpy(rng.random(ln) < 0.5, rng.random(ln) >= 0.1) for ln in lens], ctx=ctx)
    arrays = [rdf.ListArray.from_pylist(rdf.I32, [None if rng.random() < 0.1 else [int(x) for x in rng.integers(0, 9, rng.integers(0, 4))]
                                                  for _ in range(ln)]) for ln in lens]
    cols["lst"] = rdf.ListColumn.upload(arrays, ctx)
    return rdf.DeviceFrame(cols)


def _values(col):
    if type(col).__name__ == "ListColumn":
        return [r for a in col.download() for r in a.to_pylist()]
    out = []
    for a in col.download():
        if hasattr(a, "value_bits"):
            out += [bool(b) if ok else None for b, ok in zip(a.value_bits(), a.valid_mask())]
        else:
            vals = a.value_slice()
            out += [vals[j].tobytes() if ok else None for j, ok in enumerate(a.valid_mask())]
    return out


def _same_frames(a, b, what):
    assert list(a.columns) == list(b.columns), what
    for name in a.columns:
        assert a.columns[name].n_chunks == b.columns[name].n_chunks, (what, name)
        assert _values(a.columns[name]) == _values(b.columns[name]), (what, name)
        assert getattr(a.columns[name], "temporal", None) == getattr(b.columns[name], "temporal", None), (what, name)


def test_frame_top_k_equals_sort_then_limit(rdf, ctx):
    rng = np.random.default_rng(21)
    f = _frame(rdf, ctx, rng, [700, 0, 1300, 500])
    n = 2500
    for crit in ([("k", False)], [("k", True), ("x", False)], [("t", True), ("k", False), ("x", True)]):
        for k in (-3, 0, 1, 10, 300, n // 2, 5 * n // 8, 5 * n // 8 + 1, n - 1, n, n + 7):
            _same_frames(f.top_k(crit, k), f.sort(crit).limit(k), (crit, k))


def test_lazy_sort_limit_runs_as_one_step(rdf, ctx):
    rng = np.random.default_rng(22)
    f = _frame(rdf, ctx, rng, [1000, 1500])
    F = rdf.frame
    plans = [
        [F.sort([("k", False), ("x", True)]), F.limit(40)],
        [F.sort([("x", True)]), F.select(["x", "k", "lst"]), F.drop(["k"]), F.limit(100)],
        [F.sort([("k", True)]), F.limit(-1)],
        [F.sort([("k", False)]), F.limit(5000), F.sort([("x", False)]), F.limit(3)],
        [F.select(["k", "x", "t"]), F.sort([("k", False)]), F.filter_(("gt", ("col", "x"), ("scalar", 0.0))), F.limit(30)],
    ]
    for steps in plans:
        planned = rdf.plan_fusion(f.schema, steps)
        n_sort = sum(1 for s in steps if s[0] == "sort")
        fused = sum(1 for s in planned if s[0] == "top_k")
        assert fused == (0 if any(s[0] == "filter" for s in steps) else n_sort), planned
        _same_frames(f.evaluate(steps), f.evaluate(steps, fuse=False), steps)


# ---- errors ---------------------------------------------------------------------------------------------------------------------

def test_errors_match_the_sort_and_leak_nothing(rdf, ctx):
    N = rdf.native
    P = rdf.PrimitiveArray
    a = rdf.Column.upload([P.from_numpy(np.arange(10, dtype=np.int32))], ctx=ctx)
    s = rdf.Column.upload([P.from_numpy(np.arange(7, dtype=np.int32))], ctx=ctx)
    b = rdf.Column.upload([rdf.BooleanArray.from_numpy(np.arange(10) % 2 == 0)], ctx=ctx)
    ctx.synchronize()
    before = pool_used(ctx)
    h = C.c_void_p()
    lib = N.lib()

    def keys(*cols):
        arr = (N.SortKeyC * max(len(cols), 1))()
        for i, c in enumerate(cols):
            arr[i].column, arr[i].descending = c.handle, 0
        return arr

    cases = [(0, keys(a), C.byref(h)), (1, None, C.byref(h)), (1, keys(a), None), (1, keys(b), C.byref(h)), (2, keys(a, s), C.byref(h)),
             (2, keys(b, s), C.byref(h))]
    for j, (nk, ks, out) in enumerate(cases):   # the sort's status for every refused call, each leaving the pool as it was
        want = lib.bdf_sort_indices_dev(ctx.handle, nk, ks, out)
        assert want != N.OK
        assert lib.bdf_top_k_indices_dev(ctx.handle, nk, ks, 3, out) == want, j
        ctx.synchronize()
        assert pool_used(ctx) == before, j
    assert lib.bdf_top_k_indices_dev(ctx.handle, 1, keys(a), -1, C.byref(h)) == N.INVALID
    assert lib.bdf_top_k_indices_dev(ctx.handle, 2, keys(a, s), -1, C.byref(h)) == N.LENGTH_MISMATCH   # the sort's checks first
    ctx.synchronize()
    assert pool_used(ctx) == before
    for k in (0, 3, 6, 10):   # success frees every temporary
        idx = rdf.top_k_indices([(a, True)], k)
        assert _indices(idx).tolist() == list(range(9, 9 - k, -1))
        idx.free()
        ctx.synchronize()
        assert pool_used(ctx) == before, k
    with pytest.raises(rdf.ComputeError):
        rdf.top_k_indices([], 3)
    rng = np.random.default_rng(23)
    f = _frame(rdf, ctx, rng, [40])
    for crit in ([], [("lst", False)], [("flag", False)], [("nope", False)]):
        with pytest.raises(Exception) as refused:
            f.sort(crit)
        want = type(refused.value)
        with pytest.raises(want):
            f.top_k(crit, 5)
        with pytest.raises(want):
            f.evaluate([rdf.frame.sort(crit), rdf.frame.limit(5)])
    fleet = rdf.Context.multi(0)
    try:
        fk = rdf.Column.upload([P.from_numpy(np.arange(10, dtype=np.int64))], ctx=fleet)
        with pytest.raises(rdf.UnsupportedType):
            rdf.top_k_indices([(fk, False)], 3)
    finally:
        fleet.close()


# ---- scale ----------------------------------------------------------------------------------------------------------------------

def test_hundred_million_rows_take_the_fast_path(rdf, ctx):
    rng = np.random.default_rng(10 ** 8)
    n, k, chunk = 100_000_000, 1000, 4_000_000
    chunks = [rdf.PrimitiveArray.from_numpy(rng.normal(0, 1, chunk), rng.random(chunk) >= 0.1) for _ in range(n // chunk)]
    key = rdf.Column.upload(chunks, ctx=ctx)
    del chunks
    ctx.profile_enable(True)
    got = _indices(rdf.top_k_indices([(key, True)], k))
    recs = ctx.profile_read()
    ctx.profile_enable(False)
    assert not any(r["kernel"] == "sort" and r["rows"] == n for r in recs)
    full = rdf.sort_indices([(key, True)])
    assert np.array_equal(got, _indices(full)[:k])
    full.free()
    key.free()
