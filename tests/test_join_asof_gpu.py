"""The as-of join (bdf_join_asof_dev) on the GPU, element for element against the numpy restatement in tests/asof_oracle.py (itself
checked against pandas.merge_asof in tests/test_join_asof.py)."""
import ctypes as C
import datetime
import itertools

import numpy as np
import pytest

import asof_oracle as ao
from helpers import pool_used

DTYPES = ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "float32", "float64"]


def _upload(rdf, ctx, values, mask, lens, sliced=False):
    """Chunks of the given lengths; `sliced`: every chunk is a slice at an odd offset of a larger array (validity bit offsets)."""
    P = rdf.PrimitiveArray
    out, row = [], 0
    for k, n in enumerate(lens):
        v, m = values[row:row + n], mask[row:row + n]
        if sliced:
            off = 3 + k
            pad_v = np.concatenate([np.zeros(off, v.dtype), v, np.zeros(5, v.dtype)])
            pad_m = np.concatenate([np.zeros(off, bool), m, np.ones(5, bool)])
            out.append(P.from_numpy(pad_v, pad_m).slice(off, n))
        else:
            out.append(P.from_numpy(v, m))
        row += n
    assert row == len(values)
    return rdf.Column.upload(out, ctx=ctx)


def _indices(col):
    arrs = col.download()
    assert len(arrs) == 1
    v, m = arrs[0].value_slice(), arrs[0].valid_mask()
    return np.where(m, v.astype(np.int64), -1)


def _run(rdf, ctx, lon, ron, lby, rby, llens, rlens, sliced=False, **kw):
    lo = _upload(rdf, ctx, *lon, llens, sliced)
    ro = _upload(rdf, ctx, *ron, rlens, sliced)
    lb = [_upload(rdf, ctx, *k, llens, sliced) for k in lby]
    rb = [_upload(rdf, ctx, *k, rlens, sliced) for k in rby]
    idx = rdf.join_asof_indices(lo, ro, lb, rb, **kw)
    assert idx.dtype == rdf.U32 and idx.n_chunks == 1
    return _indices(idx)


def _check(rdf, ctx, lon, ron, lby, rby, llens, rlens, sliced=False, combos=None, tolerances=(None,)):
    combos = combos or list(itertools.product(ao.DIRECTIONS, (True, False)))
    for (direction, exact), tol in itertools.product(combos, tolerances):
        got = _run(rdf, ctx, lon, ron, lby, rby, llens, rlens, sliced, direction=direction, allow_exact_matches=exact, tolerance=tol)
        want = ao.join_asof(lon, ron, lby, rby, direction, exact, tol)
        assert len(got) == len(lon[0])
        assert np.array_equal(got, want), (direction, exact, tol, np.nonzero(got != want)[0][:10])


def _key(rng, n, dt, card, null_frac):
    dt = np.dtype(dt)
    if dt.kind == "f":
        v = (rng.integers(0, card, n) - card // 2).astype(dt) * dt.type(0.5)
    elif dt.kind == "i":
        v = (rng.integers(0, card, n) - card // 2).astype(dt)
    else:
        v = rng.integers(0, card, n).astype(dt)
    return v, rng.random(n) >= null_frac


# every numeric `on` dtype, with 0, 1 or 3 `by` keys; duplicate keys and nulls on both sides; ragged chunks
@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
def test_asof_matches_the_oracle(rdf, ctx, dt):
    rng = np.random.default_rng(DTYPES.index(dt) + 11)
    nl, nr = 9000, 5000
    card = 100 if np.dtype(dt).itemsize > 1 else 60
    n_by = DTYPES.index(dt) % 4 if DTYPES.index(dt) % 4 != 2 else 3
    lon, ron = _key(rng, nl, dt, card, 0.05), _key(rng, nr, dt, card, 0.05)
    by_types = ["int32", "float64", "uint8"][:n_by]
    lby = [_key(rng, nl, t, 5, 0.03) for t in by_types]
    rby = [_key(rng, nr, t, 5, 0.03) for t in by_types]
    tols = (None, 0, 3) if np.dtype(dt).kind != "f" else (None, 0.0, 1.5, np.inf)
    _check(rdf, ctx, lon, ron, lby, rby, [4000, 0, 1, 4999], [2500, 2500], tolerances=tols)


@pytest.mark.gpu
@pytest.mark.parametrize("sliced", [False, True])
def test_asof_many_ragged_and_sliced_chunks(rdf, ctx, sliced):
    rng = np.random.default_rng(5)
    llens = [int(x) for x in rng.integers(0, 70, 120)]
    rlens = [1, 33, 2047, 2049, 0, 31, 95]
    nl, nr = sum(llens), sum(rlens)
    lon, ron = _key(rng, nl, "int64", 400, 0.1), _key(rng, nr, "int64", 400, 0.1)
    lby, rby = [_key(rng, nl, "int16", 7, 0.1)], [_key(rng, nr, "int16", 7, 0.1)]
    _check(rdf, ctx, lon, ron, lby, rby, llens, rlens, sliced, tolerances=(None, 2))


@pytest.mark.gpu
def test_asof_sixteen_by_keys(rdf, ctx):
    rng = np.random.default_rng(16)
    nl, nr = 6000, 4000
    types = ["int8", "uint16", "int32", "float32"] * 4
    lby = [_key(rng, nl, t, 2, 0.01) for t in types]
    rby = [_key(rng, nr, t, 2, 0.01) for t in types]
    lby[15], rby[15] = _key(rng, nl, "int64", 3, 0.0), _key(rng, nr, "int64", 3, 0.0)
    lon, ron = _key(rng, nl, "float64", 300, 0.02), _key(rng, nr, "float64", 300, 0.02)
    _check(rdf, ctx, lon, ron, lby, rby, [nl], [1000, 3000], tolerances=(None, 4.0))


@pytest.mark.gpu
def test_asof_ties_take_last_backward_and_first_forward(rdf, ctx):
    ones = lambda n: np.ones(n, bool)
    r = np.array([1, 2, 2, 2, 5], np.int64)
    l = np.array([2, 4, 0, 5, 9], np.int64)
    got = {d: _run(rdf, ctx, (l, ones(5)), (r, ones(5)), [], [], [5], [2, 3], direction=d).tolist() for d in ao.DIRECTIONS}
    assert got == {"backward": [3, 3, -1, 4, 4], "forward": [1, 4, 0, 4, -1], "nearest": [3, 4, 0, 4, 4]}
    tie = _run(rdf, ctx, (np.array([4], np.int64), ones(1)), (np.array([3, 3, 5, 5], np.int64), ones(4)), [], [], [1], [4], direction="nearest")
    assert tie.tolist() == [1]
    # equal right keys spread over rows out of order: last / first by RIGHT ROW ORDER, not by position in the sort
    rng = np.random.default_rng(8)
    rv = rng.integers(0, 20, 20_000).astype(np.int32)
    lv = rng.integers(-2, 22, 30_000).astype(np.int32)
    _check(rdf, ctx, (lv, ones(30_000)), (rv, ones(20_000)), [], [], [30_000], [7000, 13_000])


@pytest.mark.gpu
def test_asof_integer_extremes_and_wrap_free_tolerance(rdf, ctx):
    ones = lambda n: np.ones(n, bool)
    i64 = np.iinfo(np.int64)
    lv = np.array([i64.max, i64.min, 0, i64.max, -1, 1], np.int64)
    rv = np.array([i64.min, i64.max, 0, i64.min + 1, i64.max - 1], np.int64)
    for tol in (None, 0, 1, 2 ** 63 - 1, 2 ** 63 - 2):
        _check(rdf, ctx, (lv, ones(6)), (rv, ones(5)), [], [], [6], [5], tolerances=(tol,))
    u = np.iinfo(np.uint64).max
    lu = np.array([u, 0, u - 1, 2 ** 63, 2 ** 63 - 1], np.uint64)
    ru = np.array([0, u, 2 ** 63, 1], np.uint64)
    for tol in (None, 0, 1, 2 ** 63 - 1):
        _check(rdf, ctx, (lu, ones(5)), (ru, ones(4)), [], [], [5], [4], tolerances=(tol,))
    for dt in ("int8", "int16", "int32", "uint8", "uint16", "uint32"):
        info = np.iinfo(dt)
        lv = np.array([info.max, info.min, 0, info.max - 1], dt)
        rv = np.array([info.min, info.max, 1], dt)
        _check(rdf, ctx, (lv, ones(4)), (rv, ones(3)), [], [], [4], [3], tolerances=(None, 0, int(info.max) - int(info.min) - 1, int(info.max) - int(info.min)))


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["float32", "float64"])
def test_asof_float_edges(rdf, ctx, dt):
    tiny = np.finfo(dt).smallest_subnormal
    vals = np.array([np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, tiny, -tiny, 2 * tiny, 1.0, -1.0, np.finfo(dt).max, -np.finfo(dt).max], dt)
    rng = np.random.default_rng(3)
    lv, rv = rng.choice(vals, 3000), rng.choice(vals, 800)
    lm, rm = rng.random(3000) > 0.05, rng.random(800) > 0.05
    _check(rdf, ctx, (lv, lm), (rv, rm), [], [], [1000, 2000], [800], tolerances=(None, 0.0, float(tiny), 1.0, float(np.finfo(dt).max), np.inf))
    lb, rb = [_key(rng, 3000, "int8", 3, 0.05)], [_key(rng, 800, "int8", 3, 0.05)]
    _check(rdf, ctx, (lv, lm), (rv, rm), lb, rb, [3000], [400, 400], tolerances=(None, 0.0, 1.0))


@pytest.mark.gpu
def test_asof_edge_shapes(rdf, ctx):
    rng = np.random.default_rng(4)
    some, few = _key(rng, 5000, "int64", 50, 0.1), _key(rng, 300, "int64", 50, 0.1)
    empty = (np.zeros(0, np.int64), np.ones(0, bool))
    by_s, by_f, by_e = _key(rng, 5000, "int32", 4, 0.1), _key(rng, 300, "int32", 4, 0.1), (np.zeros(0, np.int32), np.ones(0, bool))
    _check(rdf, ctx, some, empty, [], [], [5000], [0])                   # an empty right side
    _check(rdf, ctx, empty, some, [], [], [0], [5000])                   # an empty left side
    _check(rdf, ctx, some, empty, [by_s], [by_e], [5000], [0])
    _check(rdf, ctx, empty, empty, [], [], [0], [0])
    all_null = (few[0], np.zeros(300, bool))
    _check(rdf, ctx, some, all_null, [], [], [5000], [300])               # an all-null right side
    _check(rdf, ctx, some, few, [by_s], [(by_f[0], np.zeros(300, bool))], [5000], [300])   # every right by key null


@pytest.mark.gpu
def test_asof_one_hot_group_beside_a_million_singletons(rdf, ctx):
    rng = np.random.default_rng(6)
    n_single = 1_000_000
    hot = 200_000
    rby = np.concatenate([np.arange(n_single, dtype=np.int64) + 1, np.zeros(hot, np.int64)])
    ron = rng.integers(0, 10 ** 9, rby.size).astype(np.int64)
    perm = rng.permutation(rby.size)
    rby, ron = rby[perm], ron[perm]
    nl = 1_500_000
    lby = np.where(rng.random(nl) < 0.5, 0, rng.integers(1, n_single + 1, nl)).astype(np.int64)
    lon = rng.integers(0, 10 ** 9, nl).astype(np.int64)
    ones = lambda n: np.ones(n, bool)
    _check(rdf, ctx, (lon, ones(nl)), (ron, ones(rby.size)), [(lby, ones(nl))], [(rby, ones(rby.size))], [nl], [rby.size],
           combos=[("backward", True), ("nearest", False)], tolerances=(None, 10 ** 6))


@pytest.mark.gpu
def test_asof_ten_million_left_by_a_million_right(rdf, ctx):
    rng = np.random.default_rng(10)
    nl, nr = 10_000_000, 1_000_000
    lon, ron = (rng.integers(0, 10 ** 12, nl).astype(np.int64), rng.random(nl) > 0.01), (rng.integers(0, 10 ** 12, nr).astype(np.int64), rng.random(nr) > 0.01)
    lby, rby = [_key(rng, nl, "int32", 1000, 0.01)], [_key(rng, nr, "int32", 1000, 0.01)]
    _check(rdf, ctx, lon, ron, lby, rby, [nl], [nr], combos=[("backward", True), ("forward", False), ("nearest", True)], tolerances=(None, 10 ** 9))


@pytest.mark.gpu
def test_asof_same_bits_on_a_second_run(rdf, ctx):
    rng = np.random.default_rng(21)
    lon, ron = _key(rng, 300_000, "float64", 5000, 0.05), _key(rng, 200_000, "float64", 5000, 0.05)
    lby, rby = [_key(rng, 300_000, "int32", 50, 0.05)], [_key(rng, 200_000, "int32", 50, 0.05)]
    for d in ao.DIRECTIONS:
        a = _run(rdf, ctx, lon, ron, lby, rby, [300_000], [200_000], direction=d, tolerance=20.0)
        b = _run(rdf, ctx, lon, ron, lby, rby, [300_000], [200_000], direction=d, tolerance=20.0)
        assert np.array_equal(a, b)


@pytest.mark.gpu
def test_asof_timestamps_through_device_frame(rdf, ctx):
    """Trades against the last quote of the same symbol at or before them, within 2 ms, with a list column riding along."""
    P = rdf.PrimitiveArray
    TT = rdf.TemporalType
    rng = np.random.default_rng(12)
    nt, nq = 5000, 3000
    t_trade = rng.integers(0, 10 ** 7, nt).astype(np.int64)          # microseconds
    t_quote = rng.integers(0, 10 ** 7, nq).astype(np.int64)
    s_trade, s_quote = rng.integers(0, 5, nt).astype(np.int32), rng.integers(0, 5, nq).astype(np.int32)
    bid = rng.random(nq)
    trades = rdf.DeviceFrame.from_host({"time": [P.from_numpy(t_trade[:2000]), P.from_numpy(t_trade[2000:])],
                                        "sym": [P.from_numpy(s_trade[:2000]), P.from_numpy(s_trade[2000:])]}, ctx=ctx)
    trades.columns["time"].with_temporal(TT.timestamp("us"))
    quotes = rdf.DeviceFrame.from_host({"time": [P.from_numpy(t_quote)], "sym": [P.from_numpy(s_quote)], "bid": [P.from_numpy(bid)]}, ctx=ctx)
    quotes.columns["time"].with_temporal(TT.timestamp("us"))
    lists = rdf.ListColumn.upload([rdf.ListArray.from_pylist(rdf.I32, [[i, i + 1] if i % 7 else None for i in range(nq)])], ctx)
    quotes = quotes.with_column("tags", lists)
    tol = datetime.timedelta(milliseconds=2)
    g = trades.join_asof(quotes, "time", by=[("sym", "sym")], tolerance=tol)
    assert list(g.schema) == ["a.time", "a.sym", "b.time", "b.sym", "bid", "tags"]
    assert g.columns["a.time"].temporal == TT.timestamp("us") and g.columns["b.time"].temporal == TT.timestamp("us")
    ones = lambda n: np.ones(n, bool)
    want = ao.join_asof((t_trade, ones(nt)), (t_quote, ones(nq)), [(s_trade, ones(nt))], [(s_quote, ones(nq))], tolerance=2000)
    h = g.to_host()
    got_bid = h["bid"][0]
    assert np.array_equal(got_bid.valid_mask(), want >= 0)
    assert np.array_equal(got_bid.value_slice()[want >= 0], bid[want[want >= 0]])
    assert np.array_equal(np.concatenate([a.value_slice() for a in h["a.time"]]), t_trade)
    assert h["tags"][0].to_pylist() == [[int(w), int(w) + 1] if w >= 0 and w % 7 else None for w in want]
    from rust_dataframe_b200.frame import join_asof

    lazy = trades.evaluate([join_asof(quotes, "time", by=[("sym", "sym")], tolerance=tol)])
    assert np.array_equal(lazy.to_host()["bid"][0].valid_mask(), want >= 0)
    with pytest.raises(rdf.ComputeError, match="timedelta"):
        trades.join_asof(quotes, "sym", tolerance=tol)
    quotes.columns["time"].with_temporal(TT.timestamp("ms"))
    with pytest.raises(rdf.UnsupportedType):
        trades.join_asof(quotes, "time")


@pytest.mark.gpu
def test_asof_errors_leak_nothing(rdf, ctx):
    P, N = rdf.PrimitiveArray, rdf.native
    a = rdf.Column.upload([P.from_numpy(np.arange(10, dtype=np.int64))], ctx=ctx)
    a11 = rdf.Column.upload([P.from_numpy(np.arange(11, dtype=np.int64))], ctx=ctx)
    f = rdf.Column.upload([P.from_numpy(np.arange(10, dtype=np.float64))], ctx=ctx)
    flag = rdf.Column.upload([rdf.BooleanArray.from_numpy(np.arange(10) % 2 == 0)], ctx=ctx)
    huge = rdf.Column.generate(rdf.I8, [2 ** 31, 2 ** 31], kind=2, ctx=ctx)   # 2^32 rows: one too many for UInt32 indices
    one8 = rdf.Column.upload([P.from_numpy(np.zeros(1, np.int8))], ctx=ctx)

    def call(lon, ron, lby=(), rby=(), direction=0, exact=1, has_tol=0, tol=0, tol_f=0.0, n_by=None, spec=True):
        n = len(lby) if n_by is None else n_by
        lb = (C.c_void_p * max(len(lby), 1))(*[k.handle for k in lby])
        rb = (C.c_void_p * max(len(rby), 1))(*[k.handle for k in rby])
        s = N.AsofSpec(direction, exact, has_tol, tol, tol_f)
        h = C.c_void_p()
        st = N.lib().bdf_join_asof_dev(ctx.handle, lon.handle if lon else None, ron.handle if ron else None, n, lb, rb,
                                       C.byref(s) if spec else None, C.byref(h))
        assert h.value is None
        return st, (N.lib().bdf_last_error() or b"").decode()

    ctx.synchronize()
    before = pool_used(ctx)
    assert call(a, a, [a] * 17, [a] * 17)[0] == N.INVALID
    assert call(a, a, n_by=-1)[0] == N.INVALID
    assert call(None, a)[0] == N.INVALID
    assert call(a, a, spec=False)[0] == N.INVALID
    assert call(a, a, has_tol=1, tol=-1)[0] == N.INVALID
    assert call(f, f, has_tol=1, tol_f=float("nan"))[0] == N.INVALID
    assert call(f, f, has_tol=1, tol_f=-1e-300)[0] == N.INVALID
    assert call(a, a, direction=3)[0] == N.UNSUPPORTED
    assert call(flag, flag)[0] == N.UNSUPPORTED
    assert call(a, a, [flag], [flag])[0] == N.UNSUPPORTED
    assert call(a, f) == (N.UNSUPPORTED, "Join columns must have compatible types")
    assert call(a, a, [a], [f]) == (N.UNSUPPORTED, "Join columns must have compatible types")
    assert call(a, a, [a11], [a])[0] == N.LENGTH_MISMATCH
    assert call(a, a, [a], [a11])[0] == N.LENGTH_MISMATCH
    assert call(one8, huge)[0] == N.UNSUPPORTED
    with pytest.raises(rdf.UnsupportedType):
        rdf.join_asof_indices(a, a, direction="closest")
    ctx.synchronize()
    assert pool_used(ctx) == before
    fleet = rdf.Context.multi(0)
    try:
        fk = rdf.Column.upload([P.from_numpy(np.arange(10, dtype=np.int64))], ctx=fleet)
        with pytest.raises(rdf.UnsupportedType):
            rdf.join_asof_indices(fk, fk)
    finally:
        fleet.close()
