"""The statistical aggregates on the GPU (include/b200df.h "statistical aggregates"): whole-column moment records against the exact
oracle (tests/stats_oracle.py), the statistics against bdf_moments_stat, group-by's new functions on every fold path, the distinct
values, multi-GPU contexts, errors and leaks."""
import ctypes as C
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest

import stats_oracle as so
from helpers import pool_used

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NUMERIC = ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "float32", "float64"]
STAT_FNS = ("variance", "var_pop", "stddev", "stddev_pop", "skewness", "kurtosis")


def _gpu_count():
    import torch

    return torch.cuda.device_count()


def _values(rng, name, n):
    dt = np.dtype(name)
    if dt.kind == "f":
        return rng.uniform(-1e3, 1e3, n).astype(dt)
    info = np.iinfo(dt)
    return rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)


def _sliced(rdf, v, mask, offset):
    """A chunk whose data starts `offset` elements into its buffers (an Arrow slice)."""
    pad = np.zeros(offset, dtype=v.dtype)
    full = np.concatenate([pad, v])
    fm = None if mask is None else np.concatenate([np.ones(offset, bool), mask])
    return rdf.PrimitiveArray.from_numpy(full, fm).slice(offset, v.shape[0])


def _chunks(rdf, name, seed, lens, null_frac, offsets=None):
    rng = np.random.default_rng(seed)
    out = []
    for i, n in enumerate(lens):
        v = _values(rng, name, n)
        m = None if null_frac == 0 else rng.random(n) >= null_frac
        off = offsets[i] if offsets else 0
        out.append(_sliced(rdf, v, m, off) if off else rdf.PrimitiveArray.from_numpy(v, m))
    return out


def _rec(d):
    return {k: d[k] for k in ("count", "mean", "m2", "m3", "m4")}


def _same(a, b):
    return (a is None and b is None) or (a is not None and b is not None and (np.float64(a).view(np.uint64) == np.float64(b).view(np.uint64)
                                                                              or (np.isnan(a) and np.isnan(b))))


LENS = [3000, 0, 1, 70_001, 64, 5, 200_000]
OFFSETS = [0, 0, 3, 7, 0, 13, 1]


@pytest.mark.parametrize("name", NUMERIC)
@pytest.mark.parametrize("null_frac", [0.0, 0.1, 1.0])
def test_record_within_bars_and_statistics_match_stat(rdf, ctx, name, null_frac):
    for offsets in (None, OFFSETS):
        chunks = _chunks(rdf, name, 7, LENS, null_frac, offsets)
        rec = rdf.AggregateFunctions.moments(chunks, ctx=ctx)
        ref = so.exact_moments(so.valid_values(chunks))
        err = so.within_bars(rec, ref)
        assert err is None, (name, null_frac, offsets, err)
        for stat in STAT_FNS:
            got = getattr(rdf.AggregateFunctions, {"var_pop": "variance_pop"}.get(stat, stat))(chunks, ctx=ctx)
            assert _same(got, rdf.moments_stat(rec, stat)), (stat, got)
            assert _same(got, so.stat_np(rec, stat)), (stat, got)
        dev = rdf.Column.upload(chunks, ctx=ctx)
        assert _rec(dev.moments()) == rec   # the device entry gives the host-in entry's bits
        dev.free()


@pytest.mark.parametrize("c", [1e6, 1e8])
def test_ill_conditioned_columns(rdf, ctx, c):
    rng = np.random.default_rng(int(c))
    x = c + rng.uniform(-1, 1, 1 << 20)
    chunks = [rdf.PrimitiveArray.from_numpy(p) for p in np.array_split(x, 5)]
    rec = rdf.AggregateFunctions.moments(chunks, ctx=ctx)
    ref = so.exact_moments(x)
    assert so.within_bars(rec, ref) is None, so.within_bars(rec, ref)
    if c == 1e6:   # the bars are tight enough to reject the power-sum formula
        assert so.within_bars(so.naive_moments(x), ref) is not None


def test_special_columns(rdf, ctx):
    A = rdf.AggregateFunctions
    tenth = [rdf.PrimitiveArray.from_numpy(np.full(3, 0.1))]
    rec = A.moments(tenth, ctx=ctx)
    assert (rec["mean"], rec["m2"], rec["m3"], rec["m4"]) == (0.1, 0.0, 0.0, 0.0)
    assert A.stddev(tenth, ctx=ctx) == 0.0 and A.variance(tenth, ctx=ctx) == 0.0
    assert A.skewness(tenth, ctx=ctx) is None and A.kurtosis(tenth, ctx=ctx) is None
    big = [rdf.PrimitiveArray.from_numpy(np.full(n, 123456789012345, dtype=np.int64)) for n in (100_000, 1, 4097)]
    rec = A.moments(big, ctx=ctx)
    assert rec["mean"] == 123456789012345.0 and rec["m2"] == rec["m3"] == rec["m4"] == 0.0
    long_tenth = [rdf.PrimitiveArray.from_numpy(np.full(1_000_003, 0.1))]
    rec = A.moments(long_tenth, ctx=ctx)
    assert rec["mean"] == 0.1 and rec["m2"] == 0.0
    for bad in (np.nan, np.inf, -np.inf):
        v = np.arange(10_000, dtype=np.float64)
        v[4321] = bad
        m = np.ones(10_000, bool)
        m[5] = False
        rec = A.moments([rdf.PrimitiveArray.from_numpy(v, m)], ctx=ctx)
        assert rec["count"] == 9_999 and all(np.isnan(rec[k]) for k in ("mean", "m2", "m3", "m4"))
        assert np.isnan(A.variance([rdf.PrimitiveArray.from_numpy(v, m)], ctx=ctx))
    # None rules
    assert A.variance([rdf.PrimitiveArray.from_numpy(np.zeros(0))], ctx=ctx) is None
    one = [rdf.PrimitiveArray.from_numpy(np.array([5.0]))]
    assert A.variance(one, ctx=ctx) is None and A.stddev(one, ctx=ctx) is None and A.variance_pop(one, ctx=ctx) == 0.0
    allnull = [rdf.PrimitiveArray.from_numpy(np.array([1.0, 2.0]), np.array([False, False]))]
    assert all(getattr(A, f)(allnull, ctx=ctx) is None for f in ("variance", "variance_pop", "stddev", "stddev_pop", "skewness", "kurtosis"))
    # Float32 is exact as f64; Int64 / UInt64 beyond 2^53 round to nearest
    f32 = np.random.default_rng(1).uniform(-10, 10, 50_001).astype(np.float32)
    rec = A.moments([rdf.PrimitiveArray.from_numpy(f32)], ctx=ctx)
    assert so.within_bars(rec, so.exact_moments(f32.astype(np.float64))) is None
    for dt in (np.int64, np.uint64):
        info = np.iinfo(dt)
        v = np.random.default_rng(2).integers(info.max // 2, info.max, 30_000, dtype=dt, endpoint=True)
        rec = A.moments([rdf.PrimitiveArray.from_numpy(v)], ctx=ctx)
        assert so.within_bars(rec, so.exact_moments(v.astype(np.float64))) is None


def test_determinism_and_a_generated_column(rdf, oracle, ctx):
    lens = [1 << 22] * 4
    col = rdf.Column.generate(rdf.F64, lens, kind=0, lo=-5.0, hi=7.0, seed=99, col_id=3, null_mod=7, ctx=ctx)
    first = col.moments()
    for _ in range(3):
        assert col.moments() == first
    parts, row0 = [], 0
    for n in lens:
        parts.append(oracle.generate(oracle.F64, 0, -5.0, 7.0, 99, 3, row0, n, 7))
        row0 += n
    got = col.download()
    for g, w in zip(got, parts):   # the regeneration is bit-identical
        assert np.array_equal(g.valid_mask(), w.valid_mask()) and g.value_slice().tobytes() == np.asarray(w.values).tobytes()
    assert so.within_bars(first, _longdouble_moments(so.valid_values(parts))) is None
    col.free()


def _longdouble_moments(x):
    """Two passes in 80-bit long double (pairwise sums): far inside the bars, and fast enough for 2^24 rows."""
    L = np.longdouble
    xl = x.astype(L)
    n = xl.shape[0]
    mean = xl.sum() / n
    d = xl - mean
    d2 = d * d
    m2 = d2.sum()
    return {"count": n, "mean": float(mean), "m2": float(m2), "m3": float((d2 * d).sum()), "m4": float((d2 * d2).sum()),
            "abs3": float((d2 * np.abs(d)).sum()), "mean_abs": float(np.abs(xl).sum() / n), "sigma": float(np.sqrt(m2 / n))}


def test_multi_gpu_fleets(rdf, ctx):
    n = _gpu_count()
    chunks = _chunks(rdf, "float64", 21, LENS, 0.1)
    one = rdf.AggregateFunctions.moments(chunks, ctx=ctx)
    ref = so.exact_moments(so.valid_values(chunks))
    for size in [0] + [k for k in (1, 2, 3, 4, 8) if k <= n]:
        fleet = rdf.Context.multi(size)
        try:
            rec = rdf.AggregateFunctions.moments(chunks, ctx=fleet)
            if fleet.n_gpus == 1:
                assert rec == one, (size, rec, one)
            assert so.within_bars(rec, ref) is None
            dev = rdf.Column.upload(chunks, ctx=fleet)
            assert dev.moments() == rec
            with pytest.raises(rdf.UnsupportedType):
                dev.count_distinct()
            with pytest.raises(rdf.UnsupportedType):
                rdf.AggregateFunctions.sum_distinct(chunks, ctx=fleet)
            dev.free()
        finally:
            fleet.close()


def test_single_rank_communicator_gives_one_gpu_bits(rdf, ctx):
    chunks = _chunks(rdf, "int32", 22, LENS, 0.1)
    one = rdf.AggregateFunctions.moments(chunks, ctx=ctx)
    c = rdf.Context(0)
    try:
        c.comm_attach(rdf.Context.comm_unique_id(), 0, 1)
        assert rdf.AggregateFunctions.moments(chunks, ctx=c) == one
        with pytest.raises(rdf.UnsupportedType):
            rdf.AggregateFunctions.count_distinct(chunks, ctx=c)
        c.comm_detach()
    finally:
        c.close()


def test_two_rank_communicator(rdf):
    if _gpu_count() < 2:
        pytest.skip("needs 2 GPUs")
    uid = rdf.Context.comm_unique_id().hex()
    env = dict(os.environ)
    procs = [subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "stats_comm_worker.py"), uid, str(r), "2"], env=env,
                              stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True) for r in range(2)]
    outs = [p.communicate(timeout=300) for p in procs]
    for p, (o, e) in zip(procs, outs):
        assert p.returncode == 0, e[-2000:]
    assert outs[0][0].strip().splitlines()[-1] == outs[1][0].strip().splitlines()[-1]


# ---- group-by ----

def _group_case(rdf, rng, shape, name="float64", null_frac=0.1):
    if shape == "singletons":
        k = np.arange(20_000, dtype=np.int32)
    elif shape == "medium":   # ~50 000-row groups among singletons
        k = np.concatenate([np.arange(40_000, dtype=np.int32), np.full(50_000, -1, np.int32), np.full(49_000, -2, np.int32)])
    elif shape == "hot":      # one group above 64 Ki rows, and small ones
        k = np.concatenate([np.full(300_000, 7, np.int32), rng.integers(0, 500, 30_000).astype(np.int32)])
    else:                     # mid-sized groups: the 32-lane fold
        k = rng.integers(0, 300, 60_000).astype(np.int32)
    rng.shuffle(k)
    n = k.shape[0]
    v = _values(rng, name, n)
    if np.dtype(name).kind == "f":
        v = (1e3 + v).astype(name)
    m = rng.random(n) >= null_frac
    cut = [0, n // 3, n // 3 + 1, n]
    kc = [rdf.PrimitiveArray.from_numpy(k[a:b]) for a, b in zip(cut, cut[1:])]
    vc = [rdf.PrimitiveArray.from_numpy(v[a:b], m[a:b]) for a, b in zip(cut, cut[1:])]
    return k, v, m, kc, vc


@pytest.mark.parametrize("shape", ["singletons", "medium", "hot", "mixed"])
@pytest.mark.parametrize("name", ["float64", "int64", "int16", "float32"])
def test_group_statistics_against_the_oracle(rdf, ctx, shape, name):
    rng = np.random.default_rng(zlib.crc32(f"{shape}/{name}".encode()))
    k, v, m, kc, vc = _group_case(rdf, rng, shape, name)
    key, val = rdf.Column.upload(kc, ctx=ctx), rdf.Column.upload(vc, ctx=ctx)
    old = [(val, "sum"), (val, "count"), (val, "max")] + ([(val, "avg")] if name not in ("int64",) else [])
    new = [(val, f) for f in STAT_FNS] + [(val, "sum_distinct")]
    keys_a, res_a = rdf.group_by([key], old)
    keys_b, res_b = rdf.group_by([key], old[:2] + new + old[2:])
    got_old = [r.download()[0] for r in res_a]
    got_mix = [r.download()[0] for r in res_b]
    # old functions in the same call are bit-identical to a call without the new ones
    for a, b in zip(got_old, got_mix[:2] + got_mix[2 + len(new):]):
        assert np.array_equal(a.valid_mask(), b.valid_mask())
        assert a.value_slice().tobytes() == b.value_slice().tobytes()
    gkeys = keys_b[0].download()[0].value_slice()
    order = {kk: i for i, kk in enumerate(gkeys)}
    rows = {}
    for i, kk in enumerate(k):
        rows.setdefault(kk, []).append(i)
    stats = got_mix[2:2 + len(STAT_FNS)]
    sdist = got_mix[2 + len(STAT_FNS)]
    checked = 0
    for kk, idx in rows.items():
        g = order[kk]
        idx = np.asarray(idx)
        x = v[idx][m[idx]].astype(np.float64)
        ref = so.exact_moments(x)
        for stat, col in zip(STAT_FNS, stats):
            want = so.stat_np(ref, stat)
            valid = bool(col.valid_mask()[g])
            assert valid == (want is not None), (kk, stat, ref["count"])
            if want is not None and ref["count"] > 1 and ref["m2"] > 0:
                got = col.value_slice()[g]
                tol = 1e-9 if stat in ("variance", "var_pop", "stddev", "stddev_pop") else 1e-6
                assert abs(got - want) <= tol * max(1.0, abs(want)), (kk, stat, got, want)
        c, s = so.count_sum_distinct(v[idx][m[idx]])
        got_s = sdist.value_slice()[g]
        if np.dtype(name).kind == "f":   # a different fold of the same double sum, rounded once to the column type
            tol = 1e-12 * max(1.0, float(np.abs(so.distinct_values(v[idx][m[idx]])).sum())) + float(np.spacing(np.abs(s)))
            assert abs(float(got_s) - float(s)) <= tol, (kk, got_s, s)
        else:
            assert got_s == s, (kk, got_s, s)
        checked += 1
    assert checked == len(gkeys)
    assert sdist.validity is None or sdist.valid_mask().all()
    for col in [key, val] + keys_a + res_a + keys_b + res_b:
        col.free()


def test_group_statistics_cross_check_pandas_and_scipy(rdf, ctx):
    import pandas as pd
    import scipy.stats

    rng = np.random.default_rng(31)
    k = rng.integers(0, 50, 40_000).astype(np.int32)
    v = rng.normal(5.0, 2.0, 40_000)
    key, val = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(k)], ctx=ctx), rdf.Column.upload([rdf.PrimitiveArray.from_numpy(v)], ctx=ctx)
    keys, res = rdf.group_by([key], [(val, f) for f in ("variance", "stddev", "skewness", "kurtosis", "var_pop")])
    got = [r.download()[0].value_slice() for r in res]
    gk = keys[0].download()[0].value_slice()
    s = pd.Series(v).groupby(k)
    assert np.allclose(got[0], s.var().loc[gk].to_numpy(), rtol=1e-12)
    assert np.allclose(got[1], s.std().loc[gk].to_numpy(), rtol=1e-12)
    assert np.allclose(got[4], s.var(ddof=0).loc[gk].to_numpy(), rtol=1e-12)
    for i, kk in enumerate(gk):
        x = v[k == kk]
        assert np.isclose(got[2][i], scipy.stats.skew(x, bias=True), rtol=1e-9, atol=1e-12)
        assert np.isclose(got[3][i], scipy.stats.kurtosis(x, bias=True, fisher=True), rtol=1e-9, atol=1e-12)
    for col in [key, val] + keys + res:
        col.free()


def test_group_sum_distinct_rules(rdf, ctx):
    k = np.array([1, 1, 1, 1, 2, 2, 2, 3, 3, 4], dtype=np.int32)
    v = np.array([-0.0, 0.0, 2.5, 2.5, np.nan, -np.nan, 1.0, 5.0, 5.0, 9.0])
    m = np.array([1, 1, 1, 1, 1, 1, 1, 1, 1, 0], bool)
    key, val = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(k)], ctx=ctx), rdf.Column.upload([rdf.PrimitiveArray.from_numpy(v, m)], ctx=ctx)
    _, res = rdf.group_by([key], [(val, "sum_distinct"), (val, "count_distinct")])
    s, c = res[0].download()[0], res[1].download()[0].value_slice()
    sv = s.value_slice()
    assert sv[0] == 2.5 and np.isnan(sv[1]) and sv[2] == 5.0 and sv[3] == 0.0 and not np.signbit(sv[3])
    assert list(c) == [2, 2, 1, 0]
    assert s.validity is None or s.valid_mask().all()
    for col in [key, val] + res:
        col.free()


def test_whole_column_distinct_against_numpy(rdf, ctx):
    rng = np.random.default_rng(41)
    for name in NUMERIC:
        chunks = _chunks(rdf, name, 5, [5000, 0, 1, 20_000], 0.1)
        if np.dtype(name).kind == "f":   # repeats, signed zeros and NaNs
            chunks = [rdf.PrimitiveArray.from_numpy(np.round(np.asarray(c.value_slice()) / 100).astype(name) * np.where(rng.random(c.length) < .5, 1, -1).astype(name),
                                                    c.valid_mask()) for c in chunks]
            v = np.asarray(chunks[0].values)
            v[:5] = np.nan
        x = np.concatenate([np.asarray(c.value_slice())[c.valid_mask()] for c in chunks])
        c, s = so.count_sum_distinct(x)
        assert rdf.AggregateFunctions.count_distinct(chunks, ctx=ctx) == c, name
        got = rdf.AggregateFunctions.sum_distinct(chunks, ctx=ctx)
        if np.dtype(name).kind == "f":
            assert np.isnan(got) and np.isnan(s), (name, got, s)   # the column holds NaNs
        else:
            assert got == s, (name, got, s)
    assert rdf.AggregateFunctions.sum_distinct([rdf.PrimitiveArray.from_numpy(np.array([1], np.int16), np.array([False]))], ctx=ctx) == 0
    assert rdf.AggregateFunctions.count_distinct([rdf.PrimitiveArray.from_numpy(np.zeros(0, np.int16))], ctx=ctx) == 0


def test_errors_and_no_leak(rdf, ctx):
    N = rdf.native
    L = N.lib()
    r, d = N.MomentRec(), N.DistinctRec()
    b = rdf.BooleanArray.from_numpy(np.array([True, False]))
    bcol = rdf.Column.upload([b], ctx=ctx)
    f = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.arange(10.0))], ctx=ctx)
    ctx.synchronize()
    before = pool_used(ctx)
    assert L.bdf_moments_dev(ctx.handle, bcol.handle, C.byref(r)) == N.UNSUPPORTED
    assert L.bdf_distinct_dev(ctx.handle, bcol.handle, C.byref(d)) == N.UNSUPPORTED
    assert L.bdf_moments(ctx.handle, N.BOOL, 1, N.make_views([b]), C.byref(r)) == N.UNSUPPORTED
    assert L.bdf_moments_dev(ctx.handle, None, C.byref(r)) == N.INVALID
    assert L.bdf_moments_dev(ctx.handle, f.handle, None) == N.INVALID
    assert L.bdf_distinct_dev(None, f.handle, C.byref(d)) == N.INVALID
    assert L.bdf_moments(ctx.handle, rdf.F64, 1, None, C.byref(r)) == N.INVALID
    aggs = (N.GroupAggC * 1)()
    aggs[0].column, aggs[0].function = bcol.handle.value, N.GROUP_VARIANCE
    hk, out, ng = (C.c_void_p * 1)(), (C.c_void_p * 1)(), C.c_int64()
    kc = (C.c_void_p * 1)(f.handle.value)
    assert L.bdf_group_by_dev(ctx.handle, 1, kc, 1, aggs, hk, out, C.byref(ng)) == N.UNSUPPORTED
    aggs[0].column, aggs[0].function = f.handle.value, 15
    assert L.bdf_group_by_dev(ctx.handle, 1, kc, 1, aggs, hk, out, C.byref(ng)) == N.UNSUPPORTED
    # successful calls leave nothing behind either
    for _ in range(2):
        f.moments(), f.count_distinct(), f.sum_distinct()
        ks, res = rdf.group_by([f], [(f, "variance"), (f, "sum_distinct"), (f, "kurtosis")])
        for col in ks + res:
            col.free()
    ctx.synchronize()
    assert pool_used(ctx) == before
    bcol.free()
    f.free()


def test_cpp_mirror_statistics(rdf):
    host = os.path.join(ROOT, "rust-dataframe_b200", "host")
    subprocess.check_call(["make", "-C", host, "test_stats_host"], stdout=subprocess.DEVNULL)
    env = dict(os.environ, BDF_ONE_GPU="1")
    r = subprocess.run([os.path.join(host, "test_stats_host")], capture_output=True, text=True, timeout=300, env=env)
    print(r.stdout[-3000:], r.stderr[-2000:])
    assert r.returncode == 0 and "STATS OK" in r.stdout
