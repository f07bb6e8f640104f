"""Distinct rows and set operations on the GPU (bdf_duplicated_dev, bdf_set_op_dev, bdf_concat_dev, bdf_list_concat_dev and the
DeviceFrame methods over them), bit for bit against tests/setops_oracle.py, itself checked against pandas, SQLite and Counter
arithmetic in tests/test_setops.py."""
import ctypes as C
from collections import OrderedDict

import numpy as np
import pytest

import setops_oracle as so
from helpers import pool_used

DTYPES = ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "float32", "float64", "bool"]
TILE = 256   # positions per CTA of k_setop_mark


def _chunk(rdf, v, m, off=0):
    """One Arrow chunk of v / m; off > 0: a slice starting `off` slots into padded buffers (bitmaps start mid-byte)."""
    n = v.shape[0]
    if off:
        v = np.concatenate([np.zeros(off, v.dtype), v, np.zeros(5, v.dtype)])
        m = np.concatenate([np.zeros(off, bool), m, np.ones(5, bool)])
    if v.dtype == bool:
        whole = rdf.BooleanArray.from_numpy(v, m)
        return rdf.BooleanArray(whole.values, whole.validity, off, n, int((~m[off:off + n]).sum()))
    a = rdf.PrimitiveArray.from_numpy(v, m)
    return a.slice(off, n) if off else a


def _upload(rdf, ctx, v, m, lens, sliced=False):
    out, row = [], 0
    for k, n in enumerate(lens):
        out.append(_chunk(rdf, v[row:row + n], m[row:row + n], (3 + k % 5) if sliced else 0))
        row += n
    return rdf.Column.upload(out, ctx=ctx)


def _keys(rng, n, dtypes, card, null_frac=0.05):
    cols = []
    for dt in dtypes:
        if dt == "bool":
            v = rng.random(n) < 0.5
        else:
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


def _mask(col):
    """(mask bits, chunk lengths) of a Boolean result column, which must have no nulls."""
    chunks = col.download()
    for a in chunks:
        assert bool(a.valid_mask().all())
    bits = np.concatenate([a.value_bits() for a in chunks]) if chunks else np.zeros(0, bool)
    return bits, [len(a) for a in chunks]


def _dup(rdf, ctx, keys, lens, keep, sliced=False):
    cols = [_upload(rdf, ctx, v, m, lens, sliced) for v, m in keys]
    bits, got_lens = _mask(rdf.duplicated(cols, keep))
    assert got_lens == list(lens)
    return bits


def _setop(rdf, ctx, left, right, op, llens, rlens, sliced=(False, False)):
    lk = [_upload(rdf, ctx, v, m, llens, sliced[0]) for v, m in left]
    rk = [_upload(rdf, ctx, v, m, rlens, sliced[1]) for v, m in right]
    bits, got_lens = _mask(rdf.set_op_mask(lk, rk, op))
    assert got_lens == list(llens)
    return bits


def _ragged(rng, n, parts):
    cuts = np.sort(rng.integers(0, n + 1, parts - 1))
    lens = np.diff(np.r_[0, cuts, n]).tolist()
    lens.insert(len(lens) // 2, 0)   # an empty chunk
    return lens


# ---- duplicated ---------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("i,dt", list(enumerate(DTYPES)))
def test_duplicated_every_key_type(rdf, ctx, i, dt):
    rng = np.random.default_rng(10 + i)
    n = 20_000
    dtypes = [dt, "int16", "float64"][: 1 + i % 3]
    keys = _keys(rng, n, dtypes, 40 if dt != "bool" else 2)
    lens = _ragged(rng, n, 7)
    for keep in so.KEEPS:
        assert np.array_equal(_dup(rdf, ctx, keys, lens, keep), so.duplicated(keys, keep)), keep


@pytest.mark.gpu
@pytest.mark.parametrize("n_keys", [1, 2, 16])
def test_duplicated_key_counts_and_sliced_chunks(rdf, ctx, n_keys):
    rng = np.random.default_rng(n_keys)
    dtypes = [DTYPES[j % len(DTYPES)] for j in range(n_keys)]
    lens = [int(x) for x in rng.integers(0, 90, 300)]
    keys = _keys(rng, sum(lens), dtypes, 3 if n_keys == 16 else 20, 0.1)
    for keep in so.KEEPS:
        for sliced in (False, True):
            assert np.array_equal(_dup(rdf, ctx, keys, lens, keep, sliced), so.duplicated(keys, keep)), (keep, sliced)


@pytest.mark.gpu
def test_runs_across_chunks_and_tiles(rdf, ctx):
    sizes = [1, TILE - 1, TILE, TILE + 1, 2 * TILE + 3, 31, 32, 33, 5 * TILE]
    v = np.concatenate([np.full(s, j, np.int32) for j, s in enumerate(sizes)])
    rng = np.random.default_rng(3)
    perm_blocks = [np.flatnonzero(v == j) for j in rng.permutation(len(sizes))]
    v = v[np.concatenate(perm_blocks)]   # runs stay contiguous in row order, in a shuffled order of runs
    keys = [(v, np.ones(v.size, bool))]
    for lens in ([v.size], [100] * (v.size // 100) + [v.size % 100], [TILE] * (v.size // TILE) + [v.size % TILE]):
        for keep in so.KEEPS:
            assert np.array_equal(_dup(rdf, ctx, keys, lens, keep), so.duplicated(keys, keep))
    other = [(np.arange(len(sizes), dtype=np.int32).repeat(2), np.ones(2 * len(sizes), bool))]
    for op in so.OPS:
        assert np.array_equal(_setop(rdf, ctx, keys, other, op, [777, v.size - 777], [3, 2 * len(sizes) - 3]), so.set_op(keys, other, op))


@pytest.mark.gpu
def test_hot_run_all_distinct_empty_and_one_row(rdf, ctx):
    n = 1_000_000
    hot = np.zeros(n, np.int64)
    hot[::100_003] = np.arange(hot[::100_003].size) + 1
    keys = [(hot, np.ones(n, bool))]
    for keep in so.KEEPS:
        assert np.array_equal(_dup(rdf, ctx, keys, [400_000, 600_000], keep), so.duplicated(keys, keep))
    distinct = [(np.random.default_rng(1).permutation(n).astype(np.uint32), np.ones(n, bool))]
    assert not _dup(rdf, ctx, distinct, [n], "first").any()
    assert not _dup(rdf, ctx, distinct, [n], False).any()
    e = [(np.zeros(0, np.float32), np.zeros(0, bool))]
    assert _dup(rdf, ctx, e, [0], "first").size == 0
    one = [(np.array([np.nan], np.float32), np.ones(1, bool))]
    assert _dup(rdf, ctx, one, [1], False).tolist() == [False]
    for op in so.OPS:
        assert _setop(rdf, ctx, e, one, op, [0], [1]).size == 0
        assert _setop(rdf, ctx, one, e, op, [1], [0]).tolist() == so.set_op(one, e, op).tolist()
        assert _setop(rdf, ctx, one, one, op, [1], [1]).tolist() == so.set_op(one, one, op).tolist()


# ---- set operations -----------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("i,dt", list(enumerate(DTYPES)))
def test_set_ops_every_key_type(rdf, ctx, i, dt):
    rng = np.random.default_rng(50 + i)
    dtypes = [dt, "int32", "float32"][: 1 + i % 3]
    card = 2 if dt == "bool" else 30
    left, right = _keys(rng, 15_000, dtypes, card), _keys(rng, 6_000, dtypes, card)
    llens, rlens = _ragged(rng, 15_000, 5), _ragged(rng, 6_000, 3)
    for op in so.OPS:
        for sliced in ((False, False), (True, False), (False, True)):
            got = _setop(rdf, ctx, left, right, op, llens, rlens, sliced)
            assert np.array_equal(got, so.set_op(left, right, op)), (op, sliced)


@pytest.mark.gpu
@pytest.mark.parametrize("op", so.OPS)
def test_every_run_shape(rdf, ctx, op):
    lv, rv = [], []
    for cl in range(6):
        for cr in range(6):
            lv += [cl * 6 + cr] * cl
            rv += [cl * 6 + cr] * cr
    rng = np.random.default_rng(8)
    lv, rv = rng.permutation(np.array(lv, np.int16)), rng.permutation(np.array(rv, np.int16))
    left, right = [(lv, np.ones(lv.size, bool))], [(rv, np.ones(rv.size, bool))]
    got = _setop(rdf, ctx, left, right, op, [10, lv.size - 10], [rv.size])
    assert np.array_equal(got, so.set_op(left, right, op))
    for key in range(36):   # every run keeps exactly its first q left rows
        cl, cr = int((lv == key).sum()), int((rv == key).sum())
        q = min(int(so.q_of(op, cl, cr)), cl)   # a run without left rows keeps nothing
        assert got[lv == key].tolist() == [True] * q + [False] * (cl - q)


@pytest.mark.gpu
def test_sixteen_key_set_ops_and_determinism(rdf, ctx):
    rng = np.random.default_rng(16)
    dtypes = [DTYPES[j % len(DTYPES)] for j in range(16)]
    left, right = _keys(rng, 8_000, dtypes, 2, 0.2), _keys(rng, 8_000, dtypes, 2, 0.2)
    for op in so.OPS:
        a = _setop(rdf, ctx, left, right, op, [3000, 5000], [8000], (True, True))
        b = _setop(rdf, ctx, left, right, op, [3000, 5000], [8000], (True, True))
        assert np.array_equal(a, b) and np.array_equal(a, so.set_op(left, right, op))


# ---- frames ---------------------------------------------------------------------------------------------------------------------

def _frame(rdf, ctx, cols, lens):
    out = OrderedDict()
    for name, (v, m, tag) in cols.items():
        c = _upload(rdf, ctx, v, m, lens)
        out[name] = c.with_temporal(tag) if tag is not None else c
    return rdf.DeviceFrame(out)


def _list_col(rdf, ctx, lens, seed):
    rng = np.random.default_rng(seed)
    arrays = []
    for n in lens:
        rows = [None if rng.random() < 0.1 else [int(x) for x in rng.integers(0, 9, rng.integers(0, 4))] for _ in range(n)]
        arrays.append(rdf.ListArray.from_pylist(rdf.I32, rows))
    return rdf.ListColumn.upload(arrays, ctx), [r for a in arrays for r in a.to_pylist()]


def _values(col):
    out = []
    for a in col.download():
        if hasattr(a, "value_bits"):
            out += [bool(b) if ok else None for b, ok in zip(a.value_bits(), a.valid_mask())]
        else:
            vals = a.value_slice()
            out += [vals[j].tobytes() if ok else None for j, ok in enumerate(a.valid_mask())]
    return out


@pytest.mark.gpu
def test_frame_methods_carry_every_payload(rdf, ctx):
    rng = np.random.default_rng(21)
    lens = [700, 0, 1300, 500]
    n = sum(lens)
    k = (rng.integers(0, 50, n).astype(np.int32), rng.random(n) >= 0.05)
    t = (rng.integers(0, 30, n).astype(np.int64) * 3_600_000_000, rng.random(n) >= 0.05)
    flag, flag_m = rng.random(n) < 0.5, rng.random(n) >= 0.1
    pay = rng.standard_normal(n)
    ts = rdf.TemporalType.timestamp("us")
    left = _frame(rdf, ctx, OrderedDict(k=(*k, None), t=(*t, ts), flag=(flag, flag_m, None), pay=(pay, np.ones(n, bool), None)), lens)
    lst, lrows = _list_col(rdf, ctx, lens, 5)
    left = left.with_column("lst", lst)
    bounds = np.cumsum([0] + lens)
    for keep in so.KEEPS:
        out = left.drop_duplicates(["k", "t"], keep)
        rows = np.flatnonzero(~so.duplicated([k, t], keep))
        assert [out.columns["k"].chunk_len(j) for j in range(4)] == [int(((rows >= bounds[j]) & (rows < bounds[j + 1])).sum()) for j in range(4)]
        for name in ("k", "t", "flag", "pay"):
            src = _values(left.columns[name])
            assert _values(out.columns[name]) == [src[r] for r in rows], (keep, name)
        assert [r for a in out.columns["lst"].download() for r in a.to_pylist()] == [lrows[r] for r in rows]
        assert out.columns["t"].temporal == ts
    rn = 1500
    rev = np.r_[np.arange(rn)[::-1][: rn // 2], np.arange(rn // 2)]   # left rows, some twice: repeats on both sides
    rcols = OrderedDict(k=(k[0][rev], k[1][rev], None), t=(t[0][rev], t[1][rev], ts), flag=(flag[rev], flag_m[rev], None),
                        pay=(pay[rev], np.ones(rn, bool), None))
    right = _frame(rdf, ctx, rcols, [rn])
    lsmall = left.select(["k", "t", "flag", "pay"])
    lkeys = [k, t, (flag, flag_m), (pay, np.ones(n, bool))]
    rkeys = [(v, m) for v, m, _ in rcols.values()]
    for meth, op in (("intersect", "intersect"), ("intersect_all", "intersect_all"), ("subtract", "except"), ("except_all", "except_all")):
        out = getattr(lsmall, meth)(right)
        rows = np.flatnonzero(so.set_op(lkeys, rkeys, op))
        for name in ("k", "t", "flag", "pay"):
            src = _values(lsmall.columns[name])
            assert _values(out.columns[name]) == [src[r] for r in rows], (meth, name)
    assert len(lsmall.intersect_all(right).columns["k"]) > 0


@pytest.mark.gpu
def test_date32_keys_through_frames(rdf, ctx):
    rng = np.random.default_rng(32)
    n, d32 = 5000, rdf.TemporalType.date32()
    day = (rng.integers(18_000, 18_040, n).astype(np.int32), rng.random(n) >= 0.1)
    f = _frame(rdf, ctx, OrderedDict(day=(*day, d32)), [2000, 3000])
    g = _frame(rdf, ctx, OrderedDict(day=(day[0][:700].copy(), day[1][:700].copy(), d32)), [700])
    for keep in so.KEEPS:
        out = f.drop_duplicates(keep=keep)
        src = _values(f.columns["day"])
        assert _values(out.columns["day"]) == [src[r] for r in np.flatnonzero(~so.duplicated([day], keep))]
        assert out.columns["day"].temporal == d32
    out = f.except_all(g)
    src = _values(f.columns["day"])
    assert _values(out.columns["day"]) == [src[r] for r in np.flatnonzero(so.set_op([day], [(day[0][:700], day[1][:700])], "except_all"))]


@pytest.mark.gpu
def test_kept_rows_keep_their_bits(rdf, ctx):
    neg_nan = np.frombuffer(np.uint64(0xfff8000000000abc).tobytes(), np.float64)[0]
    key = np.array([-0.0, 0.0, neg_nan, np.nan, 1.0], np.float64)
    pay = np.array([-0.0, 1.0, neg_nan, 2.0, 3.0], np.float64)
    f = _frame(rdf, ctx, OrderedDict(key=(key, np.ones(5, bool), None), pay=(pay, np.ones(5, bool), None)), [2, 3])
    out = f.drop_duplicates(["key"])
    got = np.concatenate([a.value_slice() for a in out.columns["key"].download()])
    assert got.view(np.uint64).tolist() == key[[0, 2, 4]].view(np.uint64).tolist()
    got = np.concatenate([a.value_slice() for a in out.columns["pay"].download()])
    assert got.view(np.uint64).tolist() == pay[[0, 2, 4]].view(np.uint64).tolist()
    g = _frame(rdf, ctx, OrderedDict(key=(np.array([0.0, np.nan]), np.ones(2, bool), None), pay=(np.array([-0.0, neg_nan]), np.ones(2, bool), None)), [2])
    h = _frame(rdf, ctx, OrderedDict(key=(key, np.ones(5, bool), None), pay=(pay, np.ones(5, bool), None)), [5])
    out = h.intersect(g)   # pay must match too: rows 0 (-0.0, -0.0) and 2 (NaN, NaN) are in g
    got = np.concatenate([a.value_slice() for a in out.columns["key"].download()])
    assert got.view(np.uint64).tolist() == key[[0, 2]].view(np.uint64).tolist()


@pytest.mark.gpu
def test_union_and_concat_keep_chunks_types_and_lists(rdf, ctx):
    ts = rdf.TemporalType.timestamp("ms")
    a = _frame(rdf, ctx, OrderedDict(x=(np.arange(10, dtype=np.int64), np.arange(10) % 3 > 0, ts), b=(np.arange(10) % 2 == 0, np.ones(10, bool), None)), [4, 6])
    b = _frame(rdf, ctx, OrderedDict(x=(np.arange(5, dtype=np.int64) + 100, np.ones(5, bool), ts), b=(np.ones(5, bool), np.arange(5) > 1, None)), [0, 2, 3])
    la, ra = _list_col(rdf, ctx, [4, 6], 1)
    lb, rb = _list_col(rdf, ctx, [0, 2, 3], 2)
    a, b = a.with_column("l", la), b.with_column("l", lb)
    u = a.union(b)
    assert list(u.columns) == ["x", "b", "l"]
    assert [u.columns["x"].chunk_len(j) for j in range(5)] == [4, 6, 0, 2, 3]
    assert u.columns["x"].temporal == ts
    assert _values(u.columns["x"]) == _values(a.columns["x"]) + _values(b.columns["x"])
    assert _values(u.columns["b"]) == _values(a.columns["b"]) + _values(b.columns["b"])
    assert [r for x in u.columns["l"].download() for r in x.to_pylist()] == ra + rb
    swapped = rdf.DeviceFrame(OrderedDict([("l", b.columns["l"]), ("b", b.columns["b"]), ("x", b.columns["x"])]))
    v = a.union_by_name(swapped)
    assert _values(v.columns["b"]) == _values(u.columns["b"]) and _values(v.columns["x"]) == _values(u.columns["x"])
    c = rdf.concat([a.columns["x"], b.columns["x"], a.columns["x"]])
    assert c.n_chunks == 7 and c.temporal == ts and _values(c) == _values(a.columns["x"]) + _values(b.columns["x"]) + _values(a.columns["x"])
    sliced = rdf.Column.upload([_chunk(rdf, np.arange(20, dtype=np.int16), np.arange(20) % 4 > 0, 5),
                                _chunk(rdf, np.arange(7, dtype=np.int16), np.arange(7) % 2 > 0, 7)], ctx=ctx)
    assert _values(rdf.concat([sliced, sliced])) == _values(sliced) * 2
    bsl = rdf.Column.upload([_chunk(rdf, np.arange(20) % 3 == 0, np.arange(20) % 5 > 0, 3), _chunk(rdf, np.arange(9) % 2 == 0, np.ones(9, bool), 6)], ctx=ctx)
    assert _values(rdf.concat([bsl, bsl])) == _values(bsl) * 2


@pytest.mark.gpu
def test_lazy_steps_equal_eager_calls(rdf, ctx):
    rng = np.random.default_rng(31)
    n = 3000
    cols = OrderedDict(a=(rng.integers(0, 5, n).astype(np.int32), rng.random(n) > 0.1, None), b=(rng.integers(0, 3, n).astype(np.float64), np.ones(n, bool), None))
    f = _frame(rdf, ctx, cols, [1000, 2000])
    g = _frame(rdf, ctx, OrderedDict((k, (v[:900], m[:900], t)) for k, (v, m, t) in cols.items()), [900])
    F = rdf.frame
    lazy = f.evaluate([F.set_op(g, "except_all"), F.distinct(["a"], "last"), F.set_op(g, "union")])
    eager = f.except_all(g).drop_duplicates(["a"], "last").union(g)
    for name in ("a", "b"):
        assert _values(lazy.columns[name]) == _values(eager.columns[name])


# ---- errors ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_error_statuses_leak_nothing(rdf, ctx):
    N = rdf.native
    P = rdf.PrimitiveArray
    a = rdf.Column.upload([P.from_numpy(np.arange(10, dtype=np.int32))], ctx=ctx)
    b = rdf.Column.upload([P.from_numpy(np.arange(10, dtype=np.int64))], ctx=ctx)
    s = rdf.Column.upload([P.from_numpy(np.arange(7, dtype=np.int32))], ctx=ctx)
    lst, _ = _list_col(rdf, ctx, [3], 1)
    ctx.synchronize()
    before = pool_used(ctx)
    h = C.c_void_p()

    def arr(*cols):
        return (C.c_void_p * max(len(cols), 1))(*[c.handle for c in cols])

    lib = N.lib()
    cases = [
        (lambda: lib.bdf_duplicated_dev(ctx.handle, 0, arr(a), 0, C.byref(h)), N.INVALID),
        (lambda: lib.bdf_duplicated_dev(ctx.handle, 17, arr(*[a] * 17), 0, C.byref(h)), N.INVALID),
        (lambda: lib.bdf_duplicated_dev(ctx.handle, 1, None, 0, C.byref(h)), N.INVALID),
        (lambda: lib.bdf_duplicated_dev(ctx.handle, 1, arr(a), 3, C.byref(h)), N.INVALID),
        (lambda: lib.bdf_duplicated_dev(ctx.handle, 1, arr(a), 0, None), N.INVALID),
        (lambda: lib.bdf_duplicated_dev(ctx.handle, 2, arr(a, s), 0, C.byref(h)), N.LENGTH_MISMATCH),
        (lambda: lib.bdf_set_op_dev(ctx.handle, 4, 1, arr(a), arr(a), C.byref(h)), N.INVALID),
        (lambda: lib.bdf_set_op_dev(ctx.handle, 0, 1, arr(a), None, C.byref(h)), N.INVALID),
        (lambda: lib.bdf_set_op_dev(ctx.handle, 0, 1, arr(a), arr(b), C.byref(h)), N.UNSUPPORTED),
        (lambda: lib.bdf_set_op_dev(ctx.handle, 3, 2, arr(a, a), arr(a, s), C.byref(h)), N.LENGTH_MISMATCH),
        (lambda: lib.bdf_concat_dev(ctx.handle, 0, arr(a), C.byref(h)), N.INVALID),
        (lambda: lib.bdf_concat_dev(ctx.handle, 2, arr(a, b), C.byref(h)), N.UNSUPPORTED),
        (lambda: lib.bdf_list_concat_dev(ctx.handle, 0, arr(lst), C.byref(h)), N.INVALID),
        (lambda: lib.bdf_bool_widen_dev(ctx.handle, a.handle, C.byref(h)), N.UNSUPPORTED),
    ]
    for j, (call, want) in enumerate(cases):   # every error status, each leaving the pool as it was
        assert call() == want, (j, want)
        ctx.synchronize()
        assert pool_used(ctx) == before, j
    with pytest.raises(rdf.UnsupportedType):
        rdf.set_op_mask([lst], [lst], "intersect")
    ctx.synchronize()
    assert pool_used(ctx) == before
    fleet = rdf.Context.multi(0)
    try:
        fk = rdf.Column.upload([P.from_numpy(np.arange(10, dtype=np.int64))], ctx=fleet)
        for call in (lambda: rdf.duplicated([fk]), lambda: rdf.set_op_mask([fk], [fk], "intersect"), lambda: rdf.concat([fk, fk])):
            with pytest.raises(rdf.UnsupportedType):
                call()
    finally:
        fleet.close()


# ---- scale ----------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_ten_million_rows(rdf, ctx):
    rng = np.random.default_rng(10 ** 7)
    n, m = 10_000_000, 2_000_000
    left, right = _keys(rng, n, ["int32", "int8"], 60_000, 0.1), _keys(rng, m, ["int32", "int8"], 60_000, 0.1)
    for keep in ("first", False):
        assert np.array_equal(_dup(rdf, ctx, left, [4_000_000] * 2 + [2_000_000], keep), so.duplicated(left, keep))
    for op in ("intersect_all", "except"):
        assert np.array_equal(_setop(rdf, ctx, left, right, op, [n], [1_000_000] * 2), so.set_op(left, right, op))


# ---- null counts of computed inputs -------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_null_counts_of_computed_inputs(rdf, ctx):
    """Columns made by a kernel keep their null counts on the device until asked: concat, union, the Boolean widening and the Boolean
    payload of drop_duplicates must report the true counts, and count() / min() must see them."""
    rng = np.random.default_rng(41)
    lens = [3000, 0, 5000]
    n = sum(lens)
    v = rng.integers(-50, 50, n).astype(np.int32)
    m = rng.random(n) >= 0.3
    x = _upload(rdf, ctx, v, m, lens)
    nulls = [int((~m[:3000]).sum()), 0, int((~m[3000:]).sum())]
    wide = x.cast(rdf.I64)                       # null counts on the device
    srt = wide.take(rdf.sort_indices([(wide, False)]))   # one chunk, counts on the device
    flag = x.gt(0)                               # a Boolean with nulls, counts on the device
    for col, want in ((rdf.concat([wide, wide]), nulls * 2), (rdf.concat([srt, wide]), [sum(nulls)] + nulls),
                      (rdf.concat([flag, flag]), nulls * 2)):
        assert [col.chunk_info(j)["null_count"] for j in range(col.n_chunks)] == want
        assert [a.null_count for a in col.download()] == want
        assert sum(int((~a.valid_mask()).sum()) for a in col.download()) == sum(want)
    both = rdf.concat([wide, wide])
    assert both.count() == 2 * int(m.sum())
    h = C.c_void_p()
    rdf.native.raise_for_status(rdf.native.lib().bdf_bool_widen_dev(ctx.handle, flag.handle, C.byref(h)))
    w = rdf.Column(ctx, h)
    assert [w.chunk_info(j)["null_count"] for j in range(w.n_chunks)] == nulls and w.count() == int(m.sum())
    f = rdf.DeviceFrame(OrderedDict([("k", x), ("w", wide), ("flag", flag)]))
    u = f.union(f)
    assert [u.columns["w"].chunk_info(j)["null_count"] for j in range(6)] == nulls * 2
    assert u.columns["w"].count() == 2 * int(m.sum())
    assert [a.null_count for a in u.columns["flag"].download()] == nulls * 2
    d = f.drop_duplicates(["k"])
    keep = ~so.duplicated([(v, m)], "first")
    assert d.columns["w"].count() == int((keep & m).sum())
    assert sum(a.null_count for a in d.columns["flag"].download()) == int((keep & ~m).sum())
    assert [a.null_count for a in d.columns["flag"].download()] == [a.null_count for a in d.columns["k"].download()]
