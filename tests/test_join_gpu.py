"""The equi-join (bdf_join_indices_dev) on the GPU, element for element against the numpy restatement in tests/join_oracle.py
(itself checked against pyarrow and pandas in tests/test_join.py)."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import join_oracle as jo
from helpers import pool_used

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "float32", "float64"]


def _upload(rdf, ctx, values, mask, lens, sliced):
    """Chunks of the given lengths; `sliced`: every chunk is a slice at an odd offset of a larger array."""
    P = rdf.PrimitiveArray
    out, row = [], 0
    for k, n in enumerate(lens):
        v, m = values[row:row + n], None if mask is None else mask[row:row + n]
        if sliced:
            off = 3 + k
            pad_v = np.concatenate([np.zeros(off, v.dtype), v, np.zeros(5, v.dtype)])
            pad_m = np.concatenate([np.zeros(off, bool), np.ones(n, bool) if m is None else m, np.ones(5, bool)])
            out.append(P.from_numpy(pad_v, pad_m).slice(off, n))
        else:
            out.append(P.from_numpy(v, m))
        row += n
    return rdf.Column.upload(out, ctx=ctx)


def _indices(col):
    arrs = col.download()
    assert len(arrs) == 1
    v, m = arrs[0].value_slice(), arrs[0].valid_mask()
    return np.where(m, v.astype(np.int64), -1)


def _keys(rng, n, dtypes, card, null_fracs):
    cols = []
    for dt, nf in zip(dtypes, null_fracs):
        dt = np.dtype(dt)
        if dt.kind == "f":
            v = (rng.integers(0, card, n) - card // 2).astype(dt) * dt.type(0.5)
            v[rng.random(n) < 0.05] = np.nan
            v[rng.random(n) < 0.05] = -0.0
        elif dt.kind == "i":
            v = (rng.integers(0, card, n) - card // 2).astype(dt)
        else:
            v = rng.integers(0, card, n).astype(dt)
        cols.append((v, rng.random(n) >= nf))
    return cols


def _run(rdf, ctx, left, right, how, llens, rlens, sliced=(False, False)):
    lk = [_upload(rdf, ctx, v, m, llens, sliced[0]) for v, m in left]
    rk = [_upload(rdf, ctx, v, m, rlens, sliced[1]) for v, m in right]
    li, ri = rdf.join_indices(lk, rk, how)
    assert li.dtype == rdf.U32 and ri.dtype == rdf.U32 and li.n_chunks == 1 and ri.n_chunks == 1
    return _indices(li), _indices(ri)


def _check(rdf, ctx, left, right, llens, rlens, sliced=(False, False), hows=jo.HOWS):
    for how in hows:
        gl, gr = _run(rdf, ctx, left, right, how, llens, rlens, sliced)
        wl, wr = jo.join_indices(left, right, how)
        assert len(gl) == len(wl), how
        assert np.array_equal(gl, wl), how
        assert np.array_equal(gr, wr), how


# every numeric dtype in the first criterion, 1, 2 and 3 criteria; nulls on both sides, only in a later criterion for some
CASES = [(dt, [dt, "int16", "float64"][: 1 + i % 3], [0.05, 0.0, 0.1][i % 3]) for i, dt in enumerate(DTYPES)]


@pytest.mark.gpu
@pytest.mark.parametrize("dt,dtypes,nf", CASES)
def test_join_matches_the_oracle(rdf, ctx, dt, dtypes, nf):
    rng = np.random.default_rng(sum(map(ord, "".join(dtypes))) + int(nf * 100))
    card = 40 if np.dtype(dt).itemsize > 1 else 12
    nl, nr = 23_000, 7_000
    fracs = [nf] + [0.1] * (len(dtypes) - 1)   # with nf == 0: a null only in a later criterion
    left, right = _keys(rng, nl, dtypes, card, fracs), _keys(rng, nr, dtypes, card, fracs)
    _check(rdf, ctx, left, right, [10_000, 0, 1, 12_999], [4000, 3000])


@pytest.mark.gpu
@pytest.mark.parametrize("sliced", [(True, False), (False, True), (True, True)])
def test_join_sliced_and_ragged_chunks(rdf, ctx, sliced):
    rng = np.random.default_rng(7)
    left, right = _keys(rng, 9_000, ["int32", "float32"], 30, [0.1, 0.1]), _keys(rng, 6_500, ["int32", "float32"], 30, [0.1, 0.0])
    _check(rdf, ctx, left, right, [1, 33, 2047, 2049, 0, 4870], [5000, 1, 0, 1499], sliced)


@pytest.mark.gpu
def test_join_nan_and_signed_zero_keys(rdf, ctx):
    lv = np.array([0.0, -0.0, np.nan, -np.nan, 1.0, np.inf, -np.inf, 2.0], np.float64)
    rv = np.array([np.nan, -0.0, 0.0, np.inf, 1.0, 3.0, -np.inf], np.float64)
    for dt in (np.float64, np.float32):
        left, right = [(lv.astype(dt), np.ones(8, bool))], [(rv.astype(dt), np.ones(7, bool))]
        _check(rdf, ctx, left, right, [8], [3, 4])
        gl, gr = _run(rdf, ctx, left, right, "inner", [8], [7])
        assert list(zip(gl.tolist(), gr.tolist())) == [(0, 1), (0, 2), (1, 1), (1, 2), (2, 0), (3, 0), (4, 4), (5, 3), (6, 6)]


@pytest.mark.gpu
def test_join_edge_shapes(rdf, ctx):
    rng = np.random.default_rng(3)
    some = _keys(rng, 5000, ["int64"], 50, [0.1])
    empty = [(np.zeros(0, np.int64), np.ones(0, bool))]
    _check(rdf, ctx, some, empty, [5000], [0])                                        # an empty right side
    _check(rdf, ctx, empty, some, [0], [2000, 3000])                                  # an empty left side
    _check(rdf, ctx, empty, empty, [0], [0])
    far = [(np.arange(4000, dtype=np.int64) + 10_000, np.ones(4000, bool))]
    _check(rdf, ctx, some, far, [5000], [4000])                                       # no matches at all
    const_l = [(np.full(300, 9, np.uint16), np.ones(300, bool))]
    const_r = [(np.full(250, 9, np.uint16), np.ones(250, bool))]
    _check(rdf, ctx, const_l, const_r, [100, 200], [250])                             # a constant key: the full cross product
    gl, gr = _run(rdf, ctx, const_l, const_r, "inner", [300], [250])
    assert len(gl) == 75_000 and np.array_equal(gl, np.repeat(np.arange(300), 250)) and np.array_equal(gr, np.tile(np.arange(250), 300))
    nulls = [(np.zeros(100, np.int8), np.zeros(100, bool))]
    _check(rdf, ctx, nulls, nulls, [100], [100])                                      # null keys never match, not even each other


@pytest.mark.gpu
def test_join_hot_many_to_many_key(rdf, ctx):
    """About 10^8 output rows from one key held by 10^5 left and 10^3 right rows: counts per left row, and a seeded sample of
    positions, against the restatement (which is never materialised at this size)."""
    rng = np.random.default_rng(99)
    nl, nr = 150_000, 21_000
    lv = rng.integers(0, 1_000_000, nl).astype(np.int64)
    rv = rng.integers(0, 1_000_000, nr).astype(np.int64)
    lv[rng.permutation(nl)[:100_000]] = -7
    rv[rng.permutation(nr)[:1_000]] = -7
    lm, rm = rng.random(nl) >= 0.01, np.ones(nr, bool)
    left, right = [(lv, lm)], [(rv, rm)]
    for how in ("left", "inner"):
        gl, gr = _run(rdf, ctx, left, right, how, [nl], [nr])
        p = jo.plan(left, right, how)
        assert len(gl) == int(p["out_cnt"].sum()) > 95_000_000
        assert np.array_equal(np.bincount(gl, minlength=nl), p["out_cnt"])          # every left row once per output row it owns
        assert np.array_equal(gl, np.sort(gl))                                      # left rows in row order
        pos = np.sort(np.random.default_rng(5).integers(0, len(gl), 200_000))
        wl, wr = jo.pairs_at(p, pos)
        assert np.array_equal(gl[pos], wl) and np.array_equal(gr[pos], wr)
        del gl, gr


@pytest.mark.gpu
def test_join_same_bits_on_a_second_run(rdf, ctx):
    rng = np.random.default_rng(21)
    left, right = _keys(rng, 200_000, ["int32"], 3000, [0.05]), _keys(rng, 150_000, ["int32"], 3000, [0.05])
    for how in jo.HOWS:
        a = _run(rdf, ctx, left, right, how, [200_000], [150_000])
        b = _run(rdf, ctx, left, right, how, [200_000], [150_000])
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


@pytest.mark.gpu
def test_join_errors_leak_nothing(rdf, ctx):
    P, N = rdf.PrimitiveArray, rdf.native
    a = rdf.Column.upload([P.from_numpy(np.arange(10, dtype=np.int64))], ctx=ctx)
    a11 = rdf.Column.upload([P.from_numpy(np.arange(11, dtype=np.int64))], ctx=ctx)
    f = rdf.Column.upload([P.from_numpy(np.arange(10, dtype=np.float64))], ctx=ctx)
    flag = rdf.Column.upload([rdf.BooleanArray.from_numpy(np.arange(10) % 2 == 0)], ctx=ctx)
    big_l = rdf.Column.upload([P.from_numpy(np.zeros(300_000, np.int32))], ctx=ctx)   # 9e10 output rows: more than HBM holds
    big_r = rdf.Column.upload([P.from_numpy(np.zeros(300_000, np.int32))], ctx=ctx)
    huge = rdf.Column.generate(rdf.I8, [2 ** 31, 2 ** 31], kind=2, ctx=ctx)              # 2^32 rows: one too many for UInt32 indices
    one8 = rdf.Column.upload([P.from_numpy(np.zeros(1, np.int8))], ctx=ctx)

    def call(how, lk, rk):
        n = len(lk)
        l, r = (C.c_void_p * max(n, 1))(*[k.handle for k in lk]), (C.c_void_p * max(n, 1))(*[k.handle for k in rk])
        hl, hr = C.c_void_p(), C.c_void_p()
        st = N.lib().bdf_join_indices_dev(ctx.handle, how, n, l, r, C.byref(hl), C.byref(hr), None)
        assert hl.value is None and hr.value is None
        return st, (N.lib().bdf_last_error() or b"").decode()

    ctx.synchronize()
    before = pool_used(ctx)
    assert call(N.JOIN_INNER, [], []) == (N.INVALID, "Join criteria cannot be empty")
    assert call(N.JOIN_INNER, [a] * 17, [a] * 17)[0] == N.INVALID
    hl, hr = C.c_void_p(), C.c_void_p()
    assert N.lib().bdf_join_indices_dev(ctx.handle, N.JOIN_INNER, 1, None, None, C.byref(hl), C.byref(hr), None) == N.INVALID
    assert call(99, [a], [a])[0] == N.UNSUPPORTED
    assert call(N.JOIN_LEFT, [flag], [flag])[0] == N.UNSUPPORTED
    assert call(N.JOIN_LEFT, [a], [f]) == (N.UNSUPPORTED, "Join columns must have compatible types")
    assert call(N.JOIN_LEFT, [a, a11], [a, a])[0] == N.LENGTH_MISMATCH
    assert call(N.JOIN_LEFT, [huge], [one8])[0] == N.UNSUPPORTED
    assert call(N.JOIN_RIGHT, [one8], [huge])[0] == N.UNSUPPORTED
    assert call(N.JOIN_INNER, [big_l], [big_r])[0] == N.OOM
    with pytest.raises(MemoryError):
        rdf.join_indices([big_l], [big_r], "full")
    with pytest.raises(rdf.UnsupportedType):
        rdf.join_indices([a], [a], "outer")
    with pytest.raises(rdf.ComputeError, match="Join criteria cannot be empty"):
        rdf.join_indices([], [], "inner")
    ctx.synchronize()
    assert pool_used(ctx) == before
    fleet = rdf.Context.multi(0)
    try:
        fk = rdf.Column.upload([P.from_numpy(np.arange(10, dtype=np.int64))], ctx=fleet)
        with pytest.raises(rdf.UnsupportedType):
            rdf.join_indices([fk], [fk], "inner")
    finally:
        fleet.close()


def _fixture_frames(rdf, ctx):
    with open(os.path.join(ROOT, "tests", "golden", "join_tables.json")) as fh:
        d = json.load(fh)
    P = rdf.PrimitiveArray

    def arr(values):
        if any(isinstance(x, str) for x in values):
            v = np.array([0.0 if x is None else float.fromhex(x) for x in values])
        else:
            v = np.array([0 if x is None else x for x in values], np.int32)
        return [P.from_numpy(v, np.array([x is not None for x in values]))]

    j1, j2 = d["join_test_j1"], d["join_test_j2"]
    fa = rdf.DeviceFrame.from_host({"a": arr(j1["a"]), "b": arr(j1["b"])}, ctx=ctx)
    fb = rdf.DeviceFrame.from_host({"d": arr(j2["d"]), "f": arr(j2["f"])}, ctx=ctx)
    return fa, fb


@pytest.mark.gpu
def test_device_frame_join_on_the_reference_fixture(rdf, ctx):
    """The reference's three join tests (src/dataframe.rs:1005-1060) by row count, and FULL (13 rows where the reference gives 7)."""
    from rust_dataframe_b200.frame import join

    fa, fb = _fixture_frames(rdf, ctx)
    for how, crit, rows in (("left", [("b", "d")], 9), ("right", [("a", "d")], 10), ("inner", [("a", "d")], 4), ("full", [("a", "d")], 13)):
        g = fa.join(fb, crit, how)
        assert list(g.schema.items()) == rdf.plan_join(fa.schema, fb.schema, crit) == [("a", rdf.I32), ("b", rdf.I32), ("d", rdf.I32), ("f", rdf.F64)]
        h = g.to_host()
        assert all(len(v) == 1 and v[0].length == rows for v in h.values()), how
        assert len(fa.evaluate([join(fb, crit, how)]).columns["d"]) == rows
    h = fa.join(fb, [("b", "d")], "left").to_host()
    assert h["b"][0].value_slice().tolist() == [1, 2, 3, 4, 4, 4, 5, 6, 60]
    assert h["d"][0].valid_mask().tolist() == [True] * 8 + [False]
    f = h["f"][0]
    assert f.valid_mask().tolist() == [True, True, True, True, False, True, True, True, False]
    assert np.isnan(f.value_slice()[3]) and np.isinf(f.value_slice()[2])


@pytest.mark.gpu
def test_device_frame_self_join_uk_cities_against_pandas(rdf, ctx):
    """uk_cities joined with itself on the latitude rounded to a whole degree, against pandas' merge (same order: pandas keeps the
    left rows' order and, per left row, the right rows' order)."""
    import pandas as pd

    with open(os.path.join(ROOT, "tests", "golden", "uk_cities.json")) as fh:
        data = json.load(fh)
    lat, lng = np.asarray(data["lat"], np.float64), np.asarray(data["lng"], np.float64)
    key = np.round(lat).astype(np.int32)
    P = rdf.PrimitiveArray
    frame = rdf.DeviceFrame.from_host({"key": [P.from_numpy(key[:20]), P.from_numpy(key[20:])], "lat": [P.from_numpy(lat[:20]), P.from_numpy(lat[20:])],
                                       "lng": [P.from_numpy(lng[:20]), P.from_numpy(lng[20:])]}, ctx=ctx)
    df = pd.DataFrame({"key": key, "lat": lat, "lng": lng})
    for how in ("inner", "left", "right", "full"):
        g = frame.join(frame, [("key", "key")], how)
        assert list(g.schema) == ["a.key", "a.lat", "a.lng", "b.key", "b.lat", "b.lng"]
        h = {n: a[0].value_slice() for n, a in g.to_host().items()}
        want = df.merge(df, on="key", how={"full": "outer"}.get(how, how), suffixes=("_a", "_b"), sort=False)
        assert len(h["a.lat"]) == len(want)
        got = sorted(zip(h["a.lat"].tolist(), h["b.lat"].tolist(), h["a.lng"].tolist(), h["b.lng"].tolist()))
        assert got == sorted(zip(want["lat_a"], want["lat_b"], want["lng_a"], want["lng_b"]))
        if how in ("inner", "left"):
            assert np.array_equal(h["a.lat"], want["lat_a"].to_numpy()) and np.array_equal(h["b.lng"], want["lng_b"].to_numpy())
