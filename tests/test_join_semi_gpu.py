"""LEFT SEMI and LEFT ANTI joins (bdf_join_indices_dev) on the GPU, element for element against tests/asof_oracle.join_exists (itself
checked against a de-duplicated inner join in tests/test_join_asof.py)."""
import ctypes as C

import numpy as np
import pytest

import asof_oracle as ao
from helpers import pool_used

DTYPES = ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "float32", "float64"]


def _upload(rdf, ctx, values, mask, lens, sliced=False):
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
    return rdf.Column.upload(out, ctx=ctx)


def _keys(rng, n, dtypes, card, null_frac):
    cols = []
    for dt in dtypes:
        dt = np.dtype(dt)
        if dt.kind == "f":
            v = (rng.integers(0, card, n) - card // 2).astype(dt) * dt.type(0.5)
            v[rng.random(n) < 0.05] = np.nan
            v[rng.random(n) < 0.05] = -0.0
        elif dt.kind == "i":
            v = (rng.integers(0, card, n) - card // 2).astype(dt)
        else:
            v = rng.integers(0, card, n).astype(dt)
        cols.append((v, rng.random(n) >= null_frac))
    return cols


def _run(rdf, ctx, left, right, how, llens, rlens, sliced=(False, False)):
    lk = [_upload(rdf, ctx, v, m, llens, sliced[0]) for v, m in left]
    rk = [_upload(rdf, ctx, v, m, rlens, sliced[1]) for v, m in right]
    li, ri = rdf.join_indices(lk, rk, how)
    assert ri is None and li.dtype == rdf.U32 and li.n_chunks == 1
    arr = li.download()[0]
    assert arr.null_count == 0 and bool(arr.valid_mask().all())
    return arr.value_slice().astype(np.int64)


def _check(rdf, ctx, left, right, llens, rlens, sliced=(False, False)):
    semi = _run(rdf, ctx, left, right, "left_semi", llens, rlens, sliced)
    anti = _run(rdf, ctx, left, right, "left_anti", llens, rlens, sliced)
    assert np.array_equal(semi, ao.join_exists(left, right, False))
    assert np.array_equal(anti, ao.join_exists(left, right, True))
    assert np.array_equal(np.sort(np.concatenate([semi, anti])), np.arange(len(left[0][0])))   # disjoint, and every left row


@pytest.mark.gpu
@pytest.mark.parametrize("i,dt", list(enumerate(DTYPES)))
def test_semi_anti_match_the_oracle(rdf, ctx, i, dt):
    rng = np.random.default_rng(40 + i)
    dtypes = [dt, "int16", "float64"][: 1 + i % 3]
    card = 40 if np.dtype(dt).itemsize > 1 else 12
    left, right = _keys(rng, 23_000, dtypes, card, 0.05), _keys(rng, 7_000, dtypes, card, 0.05)
    _check(rdf, ctx, left, right, [10_000, 0, 1, 12_999], [4000, 3000])


@pytest.mark.gpu
@pytest.mark.parametrize("sliced", [(True, False), (False, True), (True, True)])
def test_semi_anti_sliced_and_ragged_chunks(rdf, ctx, sliced):
    rng = np.random.default_rng(7)
    llens = [int(x) for x in rng.integers(0, 90, 150)]
    left, right = _keys(rng, sum(llens), ["int32", "float32"], 30, 0.1), _keys(rng, 6_500, ["int32", "float32"], 30, 0.1)
    _check(rdf, ctx, left, right, llens, [5000, 1, 0, 1499], sliced)


@pytest.mark.gpu
def test_semi_anti_sixteen_keys_and_edge_shapes(rdf, ctx):
    rng = np.random.default_rng(16)
    types = ["int8", "uint16", "int32", "float32"] * 4
    left, right = _keys(rng, 8000, types, 2, 0.01), _keys(rng, 5000, types, 2, 0.01)
    _check(rdf, ctx, left, right, [8000], [5000])
    some = _keys(rng, 5000, ["int64"], 50, 0.1)
    empty = [(np.zeros(0, np.int64), np.ones(0, bool))]
    _check(rdf, ctx, some, empty, [5000], [0])
    _check(rdf, ctx, empty, some, [0], [5000])
    _check(rdf, ctx, empty, empty, [0], [0])
    nulls = [(np.zeros(100, np.int8), np.zeros(100, bool))]
    _check(rdf, ctx, nulls, nulls, [100], [100])           # null keys never match: every row is ANTI
    lv = np.array([0.0, -0.0, np.nan, -np.nan, 1.0, np.inf, -np.inf, 2.0])
    rv = np.array([np.nan, -0.0, np.inf, 1.0, 3.0])
    for dt in (np.float32, np.float64):
        left, right = [(lv.astype(dt), np.ones(8, bool))], [(rv.astype(dt), np.ones(5, bool))]
        assert _run(rdf, ctx, left, right, "left_semi", [8], [5]).tolist() == [0, 1, 2, 3, 4, 5]


@pytest.mark.gpu
def test_semi_row_appears_once_beside_a_hot_key(rdf, ctx):
    """One key with 10^5 right partners: its left rows appear once each, and SEMI and ANTI split the left side."""
    rng = np.random.default_rng(99)
    nl, nr = 400_000, 300_000
    lv = rng.integers(0, 2_000_000, nl).astype(np.int64)
    rv = rng.integers(0, 2_000_000, nr).astype(np.int64)
    lv[rng.permutation(nl)[:50_000]] = -7
    rv[rng.permutation(nr)[:100_000]] = -7
    left, right = [(lv, rng.random(nl) >= 0.01)], [(rv, np.ones(nr, bool))]
    _check(rdf, ctx, left, right, [nl], [nr])
    semi = _run(rdf, ctx, left, right, "left_semi", [nl], [nr])
    assert np.unique(semi).size == semi.size and np.count_nonzero(lv[semi] == -7) == np.count_nonzero((lv == -7) & left[0][1])


@pytest.mark.gpu
def test_semi_anti_ten_million_rows_and_same_bits_twice(rdf, ctx):
    rng = np.random.default_rng(21)
    left, right = _keys(rng, 10_000_000, ["int32"], 3_000_000, 0.05), _keys(rng, 1_000_000, ["int32"], 3_000_000, 0.05)
    _check(rdf, ctx, left, right, [10_000_000], [1_000_000])
    for how in ("left_semi", "left_anti"):
        a = _run(rdf, ctx, left, right, how, [10_000_000], [1_000_000])
        b = _run(rdf, ctx, left, right, how, [10_000_000], [1_000_000])
        assert np.array_equal(a, b)


@pytest.mark.gpu
def test_device_frame_semi_anti_keep_left_columns_and_lists(rdf, ctx):
    P = rdf.PrimitiveArray
    rng = np.random.default_rng(2)
    nl, nr = 3000, 800
    k, x = rng.integers(0, 100, nl).astype(np.int32), rng.random(nl)
    rk = rng.integers(0, 100, nr).astype(np.int32)
    a = rdf.DeviceFrame.from_host({"k": [P.from_numpy(k[:1000]), P.from_numpy(k[1000:])], "x": [P.from_numpy(x[:1000]), P.from_numpy(x[1000:])]}, ctx=ctx)
    lists = [[i] * (i % 3) if i % 5 else None for i in range(nl)]
    a = a.with_column("l", rdf.ListColumn.upload([rdf.ListArray.from_pylist(rdf.I32, lists[:1000]), rdf.ListArray.from_pylist(rdf.I32, lists[1000:])], ctx))
    b = rdf.DeviceFrame.from_host({"k": [P.from_numpy(rk)], "y": [P.from_numpy(rng.random(nr))]}, ctx=ctx)
    from rust_dataframe_b200.frame import join

    for how, anti in (("left_semi", False), ("left_anti", True)):
        g = a.join(b, [("k", "k")], how)
        assert list(g.schema.items()) == rdf.plan_join(a.schema, b.schema, [("k", "k")], how) == list(a.schema.items())
        rows = ao.join_exists([(k, np.ones(nl, bool))], [(rk, np.ones(nr, bool))], anti)
        h = g.to_host()
        assert np.array_equal(h["k"][0].value_slice(), k[rows]) and np.array_equal(h["x"][0].value_slice(), x[rows])
        assert h["l"][0].to_pylist() == [lists[r] for r in rows]
        lazy = a.evaluate([join(b, [("k", "k")], how)]).to_host()
        assert np.array_equal(lazy["x"][0].value_slice(), x[rows])


@pytest.mark.gpu
def test_semi_anti_errors_leak_nothing(rdf, ctx):
    P, N = rdf.PrimitiveArray, rdf.native
    a = rdf.Column.upload([P.from_numpy(np.arange(10, dtype=np.int64))], ctx=ctx)
    a11 = rdf.Column.upload([P.from_numpy(np.arange(11, dtype=np.int64))], ctx=ctx)
    f = rdf.Column.upload([P.from_numpy(np.arange(10, dtype=np.float64))], ctx=ctx)
    flag = rdf.Column.upload([rdf.BooleanArray.from_numpy(np.arange(10) % 2 == 0)], ctx=ctx)
    huge = rdf.Column.generate(rdf.I8, [2 ** 31, 2 ** 31], kind=2, ctx=ctx)
    one8 = rdf.Column.upload([P.from_numpy(np.zeros(1, np.int8))], ctx=ctx)

    def call(how, lk, rk, right=True):
        n = len(lk)
        l, r = (C.c_void_p * max(n, 1))(*[k.handle for k in lk]), (C.c_void_p * max(n, 1))(*[k.handle for k in rk])
        hl, hr = C.c_void_p(), C.c_void_p(12345)
        st = N.lib().bdf_join_indices_dev(ctx.handle, how, n, l, r, C.byref(hl), C.byref(hr) if right else None, None)
        assert hl.value is None
        return st, (N.lib().bdf_last_error() or b"").decode()

    ctx.synchronize()
    before = pool_used(ctx)
    for how in (N.JOIN_LEFT_SEMI, N.JOIN_LEFT_ANTI):
        assert call(how, [], []) == (N.INVALID, "Join criteria cannot be empty")
        assert call(how, [a] * 17, [a] * 17)[0] == N.INVALID
        assert call(how, [flag], [flag], False)[0] == N.UNSUPPORTED
        assert call(how, [a], [f]) == (N.UNSUPPORTED, "Join columns must have compatible types")
        assert call(how, [a, a11], [a, a])[0] == N.LENGTH_MISMATCH
        assert call(how, [huge], [one8])[0] == N.UNSUPPORTED
        assert call(how, [one8], [huge])[0] == N.UNSUPPORTED
    assert call(6, [a], [a])[0] == N.UNSUPPORTED
    assert call(N.JOIN_INNER, [a], [a], False)[0] == N.INVALID       # only the existence joins may leave out right_indices
    hl, hr, rows = C.c_void_p(), C.c_void_p(12345), C.c_int64(-1)
    lk = (C.c_void_p * 1)(a.handle)
    assert N.lib().bdf_join_indices_dev(ctx.handle, N.JOIN_LEFT_SEMI, 1, lk, lk, C.byref(hl), C.byref(hr), C.byref(rows)) == N.OK
    assert hr.value is None and rows.value == 10
    N.lib().bdf_col_free(ctx.handle, hl)
    assert N.lib().bdf_join_indices_dev(ctx.handle, N.JOIN_LEFT_ANTI, 1, lk, lk, C.byref(hl), None, C.byref(rows)) == N.OK
    assert rows.value == 0
    N.lib().bdf_col_free(ctx.handle, hl)
    ctx.synchronize()
    assert pool_used(ctx) == before
    fleet = rdf.Context.multi(0)
    try:
        fk = rdf.Column.upload([P.from_numpy(np.arange(10, dtype=np.int64))], ctx=fleet)
        with pytest.raises(rdf.UnsupportedType):
            rdf.join_indices([fk], [fk], "left_semi")
    finally:
        fleet.close()
