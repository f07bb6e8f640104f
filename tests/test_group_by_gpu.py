"""Group-by over several key columns (bdf_group_by_dev) on the GPU, against the numpy restatement in tests/group_by_oracle.py
(itself checked against pyarrow and pandas in tests/test_group_by.py)."""
import json
import os

import numpy as np
import pytest

import group_by_oracle as gbo
from helpers import pool_used

FNS = ["sum", "max", "min", "avg", "count", "count_distinct", "first", "last"]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _chunks(rdf, values, mask, lens):
    out, row = [], 0
    for n in lens:
        out.append(rdf.PrimitiveArray.from_numpy(values[row:row + n], None if mask is None else mask[row:row + n]))
        row += n
    return out


def _one(col):
    arrs = col.download()
    assert len(arrs) == 1
    return arrs[0].value_slice(), arrs[0].valid_mask()


def _same_bits(got, want, valid):
    got, want = got[valid], np.asarray(want)[valid]
    if got.dtype.kind == "f":
        nan = np.isnan(got)
        assert np.array_equal(nan, np.isnan(want))
        got, want = got[~nan], want[~nan]
    u = np.dtype(f"u{got.dtype.itemsize}")
    assert np.array_equal(got.view(u), np.ascontiguousarray(want, dtype=got.dtype).view(u))


def _check(keys, res, okeys, ores, fns, value_dtypes):
    for col, (wv, wm) in zip(keys, okeys):
        gv, gm = _one(col)
        assert np.array_equal(gm, wm)
        if gv.dtype.kind == "f":   # a key's payload is any member of its class: compare classes (NaN, -0.0 == 0.0)
            assert np.array_equal(np.isnan(gv[gm]), np.isnan(wv[wm]))
            assert np.array_equal(np.nan_to_num(gv[gm]) + 0.0, np.nan_to_num(wv[wm]) + 0.0)
        else:
            assert np.array_equal(gv[gm], wv[wm])
    for r, o, fn, vd in zip(res, ores, fns, value_dtypes):
        gv, gm = _one(r)
        assert np.array_equal(gm, o["valid"]), fn
        if fn == "avg" or (fn == "sum" and np.dtype(vd).kind == "f"):
            # the sum bar 16 log2(n) eps sum|x| of the existing group tests; avg: that bar over the count (+ the division's rounding)
            exact, mag = o["exact"]
            eps = 2.0 ** -53 if (fn == "avg" or np.dtype(vd).itemsize == 8) else 2.0 ** -24
            cnt = np.maximum(o["count"], 1)
            bar = 16 * np.log2(np.maximum(o["count"], 2)) * eps * mag + 1e-300
            nan = np.isnan(exact)   # a NaN among the values makes the sum NaN
            assert np.array_equal(np.isnan(gv) & gm, nan & gm), fn
            ok = gm & ~nan
            if fn == "avg":
                want = exact / cnt
                assert np.all(np.abs(gv[ok] - want[ok]) <= bar[ok] / cnt[ok] + np.abs(want[ok]) * 2.0 ** -52), fn
            else:
                assert np.all(np.abs(gv[ok].astype(np.longdouble) - exact[ok]) <= bar[ok]), fn
        else:
            _same_bits(gv, o["values"], gm)


def _case(rng, n, kinds, card, knull):
    keys, masks = [], []
    for kd in kinds:
        kd = np.dtype(kd)
        if kd.kind == "f":
            k = (rng.integers(-card // 2, card // 2 + 1, n) * 0.5).astype(kd)
            k[rng.random(n) < 0.01] = np.nan
            k[rng.random(n) < 0.01] = -0.0
        elif kd.kind == "u":
            k = rng.integers(0, card, n).astype(kd)
        else:
            info = np.iinfo(kd)
            k = rng.integers(max(info.min, -card // 2), min(info.max, card // 2), n, endpoint=True).astype(kd)
        keys.append(k)
        masks.append(rng.random(n) >= knull if knull else None)
    return keys, masks


def _values(rng, n, vd, vnull):
    vd = np.dtype(vd)
    if vd.kind == "f":
        v = rng.uniform(-1e3, 1e3, n).astype(vd)
        v[rng.random(n) < 0.002] = np.nan
        v[rng.random(n) < 0.002] = -0.0
    else:
        info = np.iinfo(vd)
        v = rng.integers(info.min, info.max, n, dtype=vd, endpoint=True)
    return v, (rng.random(n) >= vnull if vnull else None)


# (key dtypes, value dtype, per-key cardinality, key null fraction, value null fraction, chunk lengths)
CASES = [
    (("int8", "float64"), "float64", 12, 0.05, 0.1, [50_000, 1, 0, 60_000, 64]),        # ~300 groups: 32 lanes
    (("uint64", "int32", "float32"), "int32", 6, 0.0, 0.2, [30_000, 17, 29_983]),          # three keys
    (("int32", "int16"), "float32", 300, 0.1, 0.3, [100_000]),                              # short groups: 8 lanes
    (("int64", "uint8"), "int16", 40_000, 0.02, 0.5, [70_000, 70_000]),                     # ~1-row groups: one lane
]


@pytest.mark.gpu
@pytest.mark.parametrize("kinds,vd,card,knull,vnull,lens", CASES)
def test_group_by_matches_the_oracle(rdf, ctx, kinds, vd, card, knull, vnull, lens):
    rng = np.random.default_rng(sum(map(ord, "".join(kinds) + vd)))
    n = sum(lens)
    keys, kms = _case(rng, n, kinds, card, knull)
    v, vm = _values(rng, n, vd, vnull)
    fns = [f for f in FNS if not (f == "avg" and np.dtype(vd).itemsize == 8 and np.dtype(vd).kind != "f")]
    kch = [_chunks(rdf, k, m, lens) for k, m in zip(keys, kms)]
    vch = _chunks(rdf, v, vm, lens)
    ck = [rdf.Column.upload(c, ctx=ctx) for c in kch]
    cv = rdf.Column.upload(vch, ctx=ctx)
    gk, res = rdf.group_by(ck, [(cv, f) for f in fns])
    ok, ores = gbo.group_by(kch, [(vch, f) for f in fns])
    _check(gk, res, ok, ores, fns, [vd] * len(fns))
    # the same bits on a second run
    gk2, res2 = rdf.group_by(ck, [(cv, f) for f in fns])
    for a, b in zip(res, res2):
        (x, xm), (y, ym) = _one(a), _one(b)
        u = np.dtype(f"u{x.dtype.itemsize}")
        assert np.array_equal(xm, ym) and np.array_equal(x.view(u), y.view(u))


@pytest.mark.gpu
def test_group_by_sliced_chunks(rdf, ctx):
    """Zero-copy slices (validity at a bit offset) as key and value chunks."""
    rng = np.random.default_rng(2)
    base_k = rng.integers(0, 9, 5000).astype(np.int32)
    base_k2 = rng.integers(0, 3, 5000).astype(np.uint16)
    base_v = rng.integers(-100, 100, 5000).astype(np.int64)
    mk, mv = rng.random(5000) > 0.1, rng.random(5000) > 0.3
    P = rdf.PrimitiveArray
    kch = [P.from_numpy(base_k, mk).slice(3, 2000), P.from_numpy(base_k, mk).slice(2100, 1500)]
    k2ch = [P.from_numpy(base_k2).slice(3, 2000), P.from_numpy(base_k2).slice(2100, 1500)]
    vch = [P.from_numpy(base_v, mv).slice(3, 2000), P.from_numpy(base_v, mv).slice(2100, 1500)]
    fns = ["sum", "min", "max", "count", "count_distinct", "first", "last"]
    gk, res = rdf.group_by([rdf.Column.upload(kch, ctx=ctx), rdf.Column.upload(k2ch, ctx=ctx)], [(rdf.Column.upload(vch, ctx=ctx), f) for f in fns])
    ok, ores = gbo.group_by([kch, k2ch], [(vch, f) for f in fns])
    _check(gk, res, ok, ores, fns, ["int64"] * len(fns))


@pytest.mark.gpu
def test_group_by_hot_keys(rdf, ctx):
    """Two keys with hundreds of thousands of rows each among many small groups (k_group_big), every aggregate, same bits twice."""
    rng = np.random.default_rng(21)
    n = 1_500_000
    k = rng.integers(0, 5000, n).astype(np.int64)
    hot = rng.random(n)
    k[hot < 0.45] = 17
    k[(hot >= 0.45) & (hot < 0.6)] = -3
    k2 = (k % 3).astype(np.int8)
    k2[hot < 0.45] = 1
    km = rng.random(n) >= 0.02
    vi = rng.integers(-2 ** 40, 2 ** 40, n).astype(np.int32)
    vf = rng.uniform(-1e3, 1e3, n)
    vf[rng.random(n) < 1e-4] = np.nan
    vm = rng.random(n) >= 0.1
    lens = [700_000, 800_000]
    kch, k2ch = _chunks(rdf, k, km, lens), _chunks(rdf, k2, None, lens)
    ich, fch = _chunks(rdf, vi, vm, lens), _chunks(rdf, vf, vm, lens)
    ck, ck2, ci, cf = (rdf.Column.upload(c, ctx=ctx) for c in (kch, k2ch, ich, fch))
    aggs = [(ci, f) for f in FNS] + [(cf, f) for f in FNS]
    gk, res = rdf.group_by([ck, ck2], aggs)
    ok, ores = gbo.group_by([kch, k2ch], [(ich, f) for f in FNS] + [(fch, f) for f in FNS])
    assert ores[FNS.index("count")]["values"].max() > 400_000
    _check(gk, res, ok, ores, FNS * 2, ["int32"] * len(FNS) + ["float64"] * len(FNS))
    gk2, res2 = rdf.group_by([ck, ck2], aggs)
    for a, b in zip(res, res2):
        (x, xm), (y, ym) = _one(a), _one(b)
        u = np.dtype(f"u{x.dtype.itemsize}")
        assert np.array_equal(xm, ym) and np.array_equal(x.view(u), y.view(u))


@pytest.mark.gpu
def test_one_key_group_by_equals_group_aggregate(rdf, ctx):
    rng = np.random.default_rng(8)
    n = 200_000
    k = rng.integers(0, 700, n).astype(np.int32)
    km = rng.random(n) > 0.05
    for vd in ("int64", "uint16", "float64", "float32"):
        v, vm = _values(rng, n, vd, 0.2)
        ck = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(k, km)], ctx=ctx)
        cv = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(v, vm)], ctx=ctx)
        keys, old = rdf.group_aggregate(ck, [cv])
        fns = ["sum", "count"] + (["min", "max"] if np.dtype(vd).kind != "f" else [])
        gk, res = rdf.group_by([ck], [(cv, f) for f in fns])
        for a, b in [(keys, gk[0])] + [(old[0][f], r) for f, r in zip(fns, res)]:
            (x, xm), (y, ym) = _one(a), _one(b)
            u = np.dtype(f"u{x.dtype.itemsize}")
            assert x.dtype == y.dtype and np.array_equal(xm, ym) and np.array_equal(x[xm].view(u), y[ym].view(u))


@pytest.mark.gpu
def test_group_by_edge_shapes(rdf, ctx):
    P = rdf.PrimitiveArray
    empty = rdf.Column.upload([P.from_numpy(np.zeros(0, np.int32))], ctx=ctx)
    gk, res = rdf.group_by([empty, empty], [(empty, f) for f in FNS])
    assert len(gk[0]) == 0 and all(len(r) == 0 for r in res)
    n = 100_000
    rng = np.random.default_rng(3)
    one = rdf.Column.upload([P.from_numpy(np.full(n, 5, np.int16))], ctx=ctx)
    v = rng.integers(-9, 9, n).astype(np.int32)
    cv = rdf.Column.upload([P.from_numpy(v)], ctx=ctx)
    gk, res = rdf.group_by([one, one], [(cv, "sum"), (cv, "count_distinct"), (cv, "first"), (cv, "last")])
    assert len(gk[0]) == 1 and [int(_one(r)[0][0]) for r in res] == [int(v.sum()), len(set(v.tolist())), int(v[0]), int(v[-1])]
    uniq = rdf.Column.upload([P.from_numpy(rng.permutation(n).astype(np.int64))], ctx=ctx)
    gk, res = rdf.group_by([uniq], [(cv, "first"), (cv, "count_distinct")])
    assert np.array_equal(_one(gk[0])[0], np.arange(n)) and (_one(res[1])[0] == 1).all()
    gk, res = rdf.group_by([uniq, one], [])                                     # distinct key tuples only
    assert len(gk[0]) == n and res == []
    gk, res = rdf.group_by([one], [(cv, FNS[j % 8]) for j in range(64)])          # 64 aggregations, duplicates included
    assert len(res) == 64 and int(_one(res[0])[0][0]) == int(v.sum()) and int(_one(res[8])[0][0]) == int(v.sum())
    # a group whose values are all null: avg / min / max / first / last NULL, sum 0, count / count_distinct 0
    k = np.array([1, 1, 2, 2, 2], np.int8)
    x = np.array([4.0, 5.0, 7.0, 8.0, 9.0])
    xm = np.array([True, True, False, False, False])
    ck = rdf.Column.upload([P.from_numpy(k)], ctx=ctx)
    cx = rdf.Column.upload([P.from_numpy(x, xm)], ctx=ctx)
    gk, res = rdf.group_by([ck], [(cx, f) for f in FNS])
    got = {f: _one(r) for f, r in zip(FNS, res)}
    for f in ("avg", "min", "max", "first", "last"):
        assert list(got[f][1]) == [True, False], f
    assert list(got["sum"][0]) == [9.0, 0.0] and list(got["count"][0]) == [2, 0] and list(got["count_distinct"][0]) == [2, 0]
    assert got["avg"][0][0] == 4.5 and got["first"][0][0] == 4.0 and got["last"][0][0] == 5.0


@pytest.mark.gpu
def test_group_by_errors(rdf, ctx):
    P = rdf.PrimitiveArray
    a = rdf.Column.upload([P.from_numpy(np.arange(10, dtype=np.int64))], ctx=ctx)
    b = rdf.Column.upload([P.from_numpy(np.arange(11, dtype=np.int64))], ctx=ctx)
    f = rdf.Column.upload([P.from_numpy(np.arange(10, dtype=np.float64))], ctx=ctx)
    flag = rdf.Column.upload([rdf.BooleanArray.from_numpy(np.arange(10) % 2 == 0)], ctx=ctx)
    rdf.group_by([a], [(f, fn) for fn in ("sum", "count_distinct", "first")])
    ctx.synchronize()
    before = pool_used(ctx)
    with pytest.raises(rdf.ComputeError):
        rdf.group_by([], [(a, "sum")])                                   # no key: BDF_INVALID
    with pytest.raises(rdf.ComputeError):
        rdf.group_by([a] * 17, [])                                       # more than 16 keys
    with pytest.raises(rdf.ComputeError):
        rdf.group_by([a], [(a, "sum")] * 65)                             # more than 64 aggregations
    with pytest.raises(rdf.UnsupportedType):
        rdf.group_by([flag], [(a, "sum")])
    with pytest.raises(rdf.UnsupportedType):
        rdf.group_by([a], [(flag, "count")])
    with pytest.raises(rdf.UnsupportedType):
        rdf.group_by([a], [(a, "median")])
    with pytest.raises(rdf.UnsupportedType, match="avg needs f64"):
        rdf.group_by([f], [(a, "avg")])
    with pytest.raises(rdf.ComputeError):
        rdf.group_by([a, b], [])                                         # keys of different lengths
    with pytest.raises(rdf.ComputeError):
        rdf.group_by([a], [(b, "sum")])
    import ctypes as C
    N = rdf.native
    aggs = (N.GroupAggC * 1)()
    aggs[0].column, aggs[0].function = f.handle.value, 99
    keys = (C.c_void_p * 1)(a.handle.value)
    out_k, out = (C.c_void_p * 1)(), (C.c_void_p * 1)()
    assert N.lib().bdf_group_by_dev(ctx.handle, 1, keys, 1, aggs, out_k, out, None) == N.UNSUPPORTED
    assert N.lib().bdf_group_by_dev(ctx.handle, 1, None, 0, None, out_k, out, None) == N.INVALID
    ctx.synchronize()
    assert pool_used(ctx) == before
    fleet = rdf.Context.multi(0)
    try:
        fk = rdf.Column.upload([P.from_numpy(np.arange(10, dtype=np.int64))], ctx=fleet)
        with pytest.raises(rdf.UnsupportedType):
            rdf.group_by([fk], [(fk, "sum")])
    finally:
        fleet.close()


@pytest.mark.gpu
def test_device_frame_aggregate_against_pandas(rdf, ctx):
    import pandas as pd

    rng = np.random.default_rng(12)
    n = 80_000
    k1 = rng.integers(0, 30, n).astype(np.int64)
    k2 = rng.integers(0, 4, n).astype(np.int8)
    x = rng.integers(-1000, 1000, n).astype(np.int32)
    y = rng.uniform(-1, 1, n)
    frame = rdf.DeviceFrame.from_host({"k1": [rdf.PrimitiveArray.from_numpy(k1)], "k2": [rdf.PrimitiveArray.from_numpy(k2)],
                                       "x": [rdf.PrimitiveArray.from_numpy(x)], "y": [rdf.PrimitiveArray.from_numpy(y)]}, ctx=ctx)
    aggr = [("sum", ["x"]), ("Max", ["y"]), ("avg", ["x", "y"]), ("count", ["y"]), ("CountDistinct", ["x"]), ("first", ["y"]), ("last", ["x"])]
    g = frame.aggregate(["k1", "k2"], aggr)
    assert list(g.schema.items()) == rdf.plan_aggregate(frame.schema, ["k1", "k2"], aggr)
    h = {name: arrs[0].value_slice() for name, arrs in g.to_host().items()}
    grp = pd.DataFrame({"k1": k1, "k2": k2, "x": x, "y": y}).groupby(["k1", "k2"], sort=True)
    want = grp.agg(sx=("x", "sum"), my=("y", "max"), ax=("x", "mean"), ay=("y", "mean"), cy=("y", "count"), dx=("x", "nunique"),
                   fy=("y", "first"), lx=("x", "last"))
    assert np.array_equal(h["k1"], want.index.get_level_values(0).to_numpy()) and np.array_equal(h["k2"], want.index.get_level_values(1).to_numpy())
    assert np.array_equal(h["sum(x)"], want["sx"].to_numpy().astype(np.int32)) and np.array_equal(h["max(y)"], want["my"].to_numpy())
    assert np.allclose(h["avg(x)"], want["ax"].to_numpy(), rtol=1e-14) and np.allclose(h["avg(y)"], want["ay"].to_numpy(), rtol=0, atol=1e-14)
    assert np.array_equal(h["count(y)"], want["cy"].to_numpy().astype(np.uint32))
    assert np.array_equal(h["count_distinct(x)"], want["dx"].to_numpy().astype(np.uint32))
    assert np.array_equal(h["first(y)"], want["fy"].to_numpy()) and np.array_equal(h["last(x)"], want["lx"].to_numpy())


@pytest.mark.gpu
def test_device_frame_aggregate_uk_cities_max(rdf, ctx):
    """The reference's only group-by test (lazyframe.rs:514-540): one Max aggregation over the Float64 lat / lng columns of
    uk_cities, here with a synthetic integer key (the row number mod 7)."""
    import pandas as pd

    with open(os.path.join(ROOT, "tests", "golden", "uk_cities.json")) as fh:
        data = json.load(fh)
    lat, lng = np.asarray(data["lat"], np.float64), np.asarray(data["lng"], np.float64)
    key = (np.arange(len(lat)) % 7).astype(np.int32)
    frame = rdf.DeviceFrame.from_host({"key": [rdf.PrimitiveArray.from_numpy(key)], "lat": [rdf.PrimitiveArray.from_numpy(lat)],
                                       "lng": [rdf.PrimitiveArray.from_numpy(lng)]}, ctx=ctx)
    g = frame.aggregate(["key"], [("Max", ["lat", "lng"])])
    assert list(g.schema.items()) == [("key", rdf.I32), ("max(lat)", rdf.F64), ("max(lng)", rdf.F64)]
    h = {name: arrs[0].value_slice() for name, arrs in g.to_host().items()}
    want = pd.DataFrame({"key": key, "lat": lat, "lng": lng}).groupby("key").max()
    assert np.array_equal(h["key"], want.index.to_numpy())
    assert np.array_equal(h["max(lat)"], want["lat"].to_numpy()) and np.array_equal(h["max(lng)"], want["lng"].to_numpy())


@pytest.mark.gpu
@pytest.mark.parametrize("vd", ["float64", "float32", "int16"])
def test_avg_without_min_max_and_long_groups_among_short(rdf, ctx, vd):
    """avg asked for alone, and beside sum / count / first / count_distinct only (no min / max of the same column), over
    mostly one-row groups (one lane per group) with one hot key (> 64 Ki rows), twenty groups of ~1 700 rows (a warp each,
    k_group_medium) and a group whose values are all null."""
    rng = np.random.default_rng(31 + len(vd))
    n = 700_000
    k = rng.permutation(n).astype(np.int64)
    k[rng.random(n) < 0.3] = 5
    sel = rng.random(n) < 0.05
    k[sel] = n + rng.integers(0, 20, int(sel.sum()))
    k[:3] = -1
    v, vm = _values(rng, n, vd, 0.1)
    vm = np.ones(n, bool) if vm is None else vm
    vm[:3] = False
    kch, vch = _chunks(rdf, k, None, [n]), _chunks(rdf, v, vm, [n])
    ck, cv = rdf.Column.upload(kch, ctx=ctx), rdf.Column.upload(vch, ctx=ctx)
    for fns in (["avg"], ["sum", "avg", "count", "first", "count_distinct"], ["min", "avg"]):
        gk, res = rdf.group_by([ck], [(cv, f) for f in fns])
        ok, ores = gbo.group_by([kch], [(vch, f) for f in fns])
        assert ores[0]["count"].max() > 100_000 and ((ores[0]["count"] > 1000) & (ores[0]["count"] < 3000)).sum() == 20   # valid values
        _check(gk, res, ok, ores, fns, [vd] * len(fns))
        avg, avg_valid = _one(res[fns.index("avg")])
        assert not avg_valid[0] and avg_valid[1:].sum() > 400_000   # key -1 sorts first: its group has no valid value
