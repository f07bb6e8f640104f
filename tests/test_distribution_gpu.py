"""The column distributions on the GPU (include/b200df.h "distributions"): percentile, median, mode, uniques, value counts and the
histogram over whole columns, median and mode per group, against the numpy restatements of tests/distribution_oracle.py bit for bit."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import distribution_oracle as do
from helpers import pool_used

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NUMERIC = ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "float32", "float64"]
PS = [0.0, 0.1, 0.25, 0.5, 0.75, 0.9, 1.0, 0.3333]
HIST_SMEM_BINS = 2048   # k_dist.cu kHistSmemBins: bins counted per CTA in shared memory (the header states it too)


def _bits(x):
    return None if x is None else int(np.float64(x).view(np.uint64))


def _np(a):
    return np.asarray(a.values[a.offset:a.offset + a.length])


def _valid(chunks):
    return np.concatenate([_np(a)[a.valid_mask()] for a in chunks]) if chunks else np.array([])


def _values(rng, name, n, distinct=None):
    dt = np.dtype(name)
    if distinct:
        return rng.integers(0, distinct, n).astype(dt)
    if dt.kind == "f":
        return rng.normal(0, 1e3, n).astype(dt)
    info = np.iinfo(dt)
    return rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)


def _chunks(rdf, name, seed, lens, null_frac, offsets=None, distinct=None):
    rng = np.random.default_rng(seed)
    out = []
    for i, n in enumerate(lens):
        v = _values(rng, name, n, distinct)
        m = None if null_frac == 0 else rng.random(n) >= null_frac
        off = offsets[i] if offsets else 0
        if off:
            full = np.concatenate([np.zeros(off, v.dtype), v])
            fm = None if m is None else np.concatenate([np.ones(off, bool), m])
            out.append(rdf.PrimitiveArray.from_numpy(full, fm).slice(off, n))
        else:
            out.append(rdf.PrimitiveArray.from_numpy(v, m))
    return out


def _download(col):
    return _valid(col.download())


def _check_column(rdf, ctx, chunks, name, nbins=(1, 10)):
    """Every whole-column entry of one column against the oracle, bit for bit."""
    col = rdf.Column.upload(chunks, ctx=ctx)
    v = _valid(chunks).astype(name)
    got = col.percentile(PS)
    want = [do.percentile(v, p) for p in PS]
    assert [_bits(g) for g in got] == [_bits(w) for w in want], (name, got, want)
    host = rdf.AggregateFunctions.percentile(chunks, PS, ctx=ctx)
    assert [_bits(g) for g in host] == [_bits(w) for w in want]
    m, f = col._mode()
    wm, wf = do.mode(v)
    assert f == wf and (m is None) == (wm is None)
    if m is not None:
        assert np.asarray(m).tobytes() == np.asarray(wm).tobytes(), (name, m, wm)
    vals, cnts = col.value_counts()
    uv, uc = do.uniques(v)
    assert _download(vals).tobytes() == uv.tobytes() and (_download(cnts) == uc).all()
    for nb in nbins:
        e, c = col.hist(nb)
        we, wc = do.histogram(v, nb)
        assert e.tobytes() == we.tobytes() and (c == wc).all(), (name, nb)
    for x in (vals, cnts, col):
        x.free()


@pytest.mark.parametrize("name", NUMERIC)
@pytest.mark.parametrize("null_frac", [0.0, 0.1, 1.0])
def test_every_dtype_and_null_fraction(rdf, ctx, name, null_frac):
    _check_column(rdf, ctx, _chunks(rdf, name, 11, [1000, 7, 4099, 1], null_frac), name)
    _check_column(rdf, ctx, _chunks(rdf, name, 12, [3000, 200], null_frac, distinct=50), name)


@pytest.mark.parametrize("name", ["int8", "int32", "uint64", "float32", "float64"])
def test_many_chunks_and_offset_arrays(rdf, ctx, name):
    rng = np.random.default_rng(5)
    lens = list(rng.integers(0, 300, 300))
    _check_column(rdf, ctx, _chunks(rdf, name, 21, lens, 0.1, offsets=[int(i % 8) for i in range(len(lens))]), name)


def test_filter_and_take_outputs(rdf, ctx):
    chunks = _chunks(rdf, "float64", 31, [5000, 3000], 0.1)
    col = rdf.Column.upload(chunks, ctx=ctx)
    mask = col.gt(0.0)
    f = col.filter(mask)
    idx = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.random.default_rng(1).integers(0, 8000, 6000).astype(np.uint32))], ctx=ctx)
    t = col.take(idx)
    for c in (f, t):
        v = _download(c)
        assert _bits(c.median()) == _bits(do.percentile(v, 0.5))
        assert c.mode() == do.mode(v)[0]
        e, k = c.hist(10)
        we, wk = do.histogram(v, 10)
        assert e.tobytes() == we.tobytes() and (k == wk).all()
    for c in (f, t, idx, mask, col):
        c.free()


def test_rechunking_and_repeated_calls_are_identical(rdf, ctx):
    rng = np.random.default_rng(8)
    v = rng.normal(0, 1, 100000)
    m = rng.random(100000) > 0.1
    one = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(v, m)], ctx=ctx)
    cuts = np.sort(rng.integers(0, 100000, 40))
    parts = np.split(np.arange(100000), cuts)
    many = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(v[p], m[p]) for p in parts], ctx=ctx)
    ref = (one.percentile(PS), one._mode(), one.hist(2 ** 20)[1].tobytes(), one.hist(37)[1].tobytes())
    for c in (one, many, one):
        assert (c.percentile(PS), c._mode(), c.hist(2 ** 20)[1].tobytes(), c.hist(37)[1].tobytes()) == ref
    one.free()
    many.free()


def test_planted_columns(rdf, ctx):
    def check(v, mask=None, nb=(1, 10)):
        _check_column(rdf, ctx, [rdf.PrimitiveArray.from_numpy(v, mask)], v.dtype.name, nb)

    n = 1 << 20
    check(np.full(n, 3.25))                                  # one value: the hot bin, candidates that never shrink
    check(np.full(n, -7, dtype=np.int64))
    check(np.where(np.arange(n) % 3 == 0, 1.5, -2.0))          # two values
    tile = 4096   # an f64 tile: the wanted rank at a tile edge and at a chunk edge
    for k in (tile - 1, tile, tile + 1):
        v = np.concatenate([np.zeros(k), np.ones(2 * k + 1)])
        check(v)
        _check_column(rdf, ctx, [rdf.PrimitiveArray.from_numpy(v[:k]), rdf.PrimitiveArray.from_numpy(v[k:])], "float64")
    i64 = np.iinfo(np.int64)
    check(np.array([i64.min, i64.max, i64.min, 2 ** 53 + 1, 2 ** 60 + 3, -(2 ** 62) - 1], dtype=np.int64))
    check(np.array([0, 2 ** 64 - 1, 2 ** 64 - 2, 2 ** 63, 2 ** 53 + 1], dtype=np.uint64))
    check(np.array([-0.0, 0.0, -0.0, 1.0, 0.0]))             # one class of zeros
    check(np.array([np.nan] * 6 + [1.0, 2.0, -np.nan]))      # a NaN majority: the median is NaN
    check(np.array([-np.inf, np.inf]), nb=())                # NaN by interpolation; an infinite range is refused below
    check(np.array([-np.inf, np.inf, np.inf]), nb=())
    check(np.array([1e-45, 3e-45, -1e-45, 1e-40, 0.0], dtype=np.float32))   # Float32 subnormals
    v = np.array([0.0, 1.0, 2.0, 3.0, 4.0, 5.0, 6.0, 7.0, 8.0, 9.0])
    col = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(v)], ctx=ctx)
    assert col.median() == 4.5 and col.percentile(1.0) == 9.0   # p * (n - 1), not p * n
    col.free()
    nulls = np.array([5.0, 0.0, 0.0, 0.0, 7.0])
    col = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(nulls, np.array([1, 0, 0, 0, 1], bool))], ctx=ctx)
    assert col.median() == 6.0 and col.mode() == 5.0   # nulls are skipped, not read as 0
    col.free()
    col = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.array([9, 4, 9, 4, 1], dtype=np.int32))], ctx=ctx)
    assert col.mode() == 4   # a tie goes to the smallest value
    col.free()
    col = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.array([-0.0, 0.0, 0.0, 2.0, 2.0]))], ctx=ctx)
    assert col.mode() == 0.0 and col.uniques().download()[0].length == 2   # -0.0 and 0.0 are one key
    col.free()


@pytest.mark.parametrize("nbins", [1, 10, HIST_SMEM_BINS - 1, HIST_SMEM_BINS, HIST_SMEM_BINS + 1, 2 ** 20])
@pytest.mark.parametrize("name", ["int16", "float32", "float64"])
def test_hist_bins_and_ranges(rdf, ctx, nbins, name):
    chunks = _chunks(rdf, name, nbins, [70000, 3], 0.1)
    col = rdf.Column.upload(chunks, ctx=ctx)
    v = _valid(chunks)
    for rng in (None, (-500.0, 700.0), (3.0, 3.0)):
        e, c = col.hist(nbins, range=rng)
        we, wc = do.histogram(v, nbins, rng)
        assert e.tobytes() == we.tobytes() and (c == wc).all(), rng
    on_edges = do.edges_restated(-2.0, 5.0, nbins)   # every edge, exactly
    ec = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(on_edges.astype(np.float64))], ctx=ctx)
    e, c = ec.hist(nbins)
    we, wc = do.histogram(on_edges, nbins)
    assert e.tobytes() == we.tobytes() and (c == wc).all()
    d = ec.hist(nbins, density=True)[1]
    assert d.tobytes() == np.histogram(on_edges, nbins, density=True)[0].tobytes()
    col.free()
    ec.free()


def test_hist_edge_correction(rdf, ctx):
    """Values on the edges of ranges where the formula alone misplaces some of them: numpy's one-step correction decides their bins."""
    rng = np.random.default_rng(7)
    cases = 0
    for _ in range(400):
        lo, hi = sorted(rng.normal(0, 1e3, 2))
        nb = int(rng.integers(3, 50))
        e = do.edges_restated(lo, hi, nb)
        x = e.copy()
        raw = np.minimum(((x - lo) / (hi - lo) * nb).astype(np.int64), nb - 1)
        if (np.bincount(raw, minlength=nb) == do.bins_restated(x, e)).all():
            continue
        col = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(x)], ctx=ctx)
        ge, gc = col.hist(nb, range=(lo, hi))
        assert ge.tobytes() == e.tobytes() and (gc == do.bins_restated(x, e)).all()
        col.free()
        cases += 1
    assert cases >= 3


@pytest.mark.parametrize("shape", ["two_keys", "hot", "one_row", "null_key"])
@pytest.mark.parametrize("name", ["int32", "float64", "uint8"])
def test_group_median_and_mode(rdf, ctx, shape, name):
    rng = np.random.default_rng(hash(shape) % 1000)
    n = 20000
    if shape == "two_keys":
        k1, k2 = rng.integers(0, 30, n), rng.integers(0, 7, n)
    elif shape == "hot":
        k1, k2 = np.where(rng.random(n) < 0.9, 5, rng.integers(0, 1000, n)), np.zeros(n, int)
    elif shape == "one_row":
        k1, k2 = np.arange(n), np.zeros(n, int)
    else:
        k1, k2 = rng.integers(0, 10, n), np.zeros(n, int)
    kmask = rng.random(n) > 0.2 if shape == "null_key" else None
    v = _values(rng, name, n, distinct=40)
    vm = rng.random(n) > 0.1
    kc1 = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(k1.astype(np.int32), kmask)], ctx=ctx)
    kc2 = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(k2.astype(np.int16))], ctx=ctx)
    vc = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(v, vm)], ctx=ctx)
    ks, res = rdf.group_by([kc1, kc2], [(vc, "exact_median"), (vc, "mode"), (vc, "avg")])
    a1, a2 = ks[0].download()[0], ks[1].download()[0]
    med, mod = res[0].download()[0], res[1].download()[0]
    key_of = (np.where(kmask, k1, -1) if kmask is not None else k1) * 10 + k2
    gk = np.where(a1.valid_mask(), _np(a1).astype(np.int64), -1) * 10 + _np(a2)
    for i, g in enumerate(gk):
        sel = (key_of == g) & vm
        vals = v[sel]
        wm = do.percentile(vals, 0.5)
        wmode = do.mode(vals)[0]
        assert med.is_valid(i) == (wm is not None) and mod.is_valid(i) == (wmode is not None)
        if wm is not None:
            assert _bits(_np(med)[i]) == _bits(wm) and _np(mod)[i] == wmode
    for c in ks + res + [kc1, kc2, vc]:
        c.free()


@pytest.mark.parametrize("name", ["int64", "float32", "float64"])
def test_group_of_one_key_is_the_whole_column(rdf, ctx, name):
    chunks = _chunks(rdf, name, 41, [5000, 123], 0.1, distinct=None)
    vc = rdf.Column.upload(chunks, ctx=ctx)
    kc = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.zeros(5123, np.int8))], ctx=ctx)
    ks, res = rdf.group_by([kc], [(vc, "exact_median"), (vc, "mode")])
    assert _bits(_np(res[0].download()[0])[0]) == _bits(vc.median())
    assert np.asarray(_np(res[1].download()[0])[0]).tobytes() == np.asarray(vc.mode()).tobytes()
    for c in ks + res + [vc, kc]:
        c.free()


def test_reference_uk_cities(rdf):
    df = rdf.DeviceFrame.from_csv(os.path.join(ROOT, "tests", "golden", "uk_cities_with_headers.csv"))
    e, d = df.column("lng").hist(10, density=True)
    _, c = df.column("lng").hist(10)
    assert len(d) == 10 and len(e) == 11 and c.sum() == 37
    assert df.column("lat").uniques().download()[0].length == 37


def test_errors_and_no_leak(rdf, ctx):
    N = rdf.native
    L = N.lib()
    b = rdf.BooleanArray.from_numpy(np.array([True, False]))
    bcol = rdf.Column.upload([b], ctx=ctx)
    f = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.array([1.0, np.inf, 2.0]))], ctx=ctx)
    ctx.synchronize()
    before = pool_used(ctx)
    out, some = (C.c_double * 4)(), (C.c_int32 * 4)()
    p = (C.c_double * 4)(0.5, 0.5, 0.5, 0.5)
    bits, freq = C.c_uint64(), C.c_int64()
    e, cnt = (C.c_double * 11)(), (C.c_int64 * 10)()
    h = C.c_void_p()
    assert L.bdf_percentile_dev(ctx.handle, bcol.handle, 1, p, out, some) == N.UNSUPPORTED
    assert L.bdf_mode_dev(ctx.handle, bcol.handle, C.byref(bits), C.byref(freq), some) == N.UNSUPPORTED
    assert L.bdf_uniques_dev(ctx.handle, bcol.handle, C.byref(h), None) == N.UNSUPPORTED
    assert L.bdf_hist_dev(ctx.handle, bcol.handle, 10, None, e, cnt) == N.UNSUPPORTED
    assert L.bdf_percentile(ctx.handle, N.BOOL, 1, N.make_views([b]), 1, p, out, some) == N.UNSUPPORTED
    for bad in (-0.1, 1.5, float("nan")):
        q = (C.c_double * 1)(bad)
        assert L.bdf_percentile_dev(ctx.handle, f.handle, 1, q, out, some) == N.INVALID
    assert L.bdf_percentile_dev(ctx.handle, f.handle, 0, p, out, some) == N.INVALID
    assert L.bdf_percentile_dev(ctx.handle, f.handle, 1025, p, out, some) == N.INVALID
    assert L.bdf_percentile_dev(ctx.handle, None, 1, p, out, some) == N.INVALID
    assert L.bdf_mode_dev(ctx.handle, f.handle, None, C.byref(freq), some) == N.INVALID
    assert L.bdf_hist_dev(ctx.handle, f.handle, 0, None, e, cnt) == N.INVALID
    assert L.bdf_hist_dev(ctx.handle, f.handle, (1 << 24) + 1, None, e, cnt) == N.INVALID
    assert L.bdf_hist_dev(ctx.handle, f.handle, 10, None, e, cnt) == N.INVALID
    assert "autodetected range" in N.lib().bdf_last_error().decode()
    assert L.bdf_hist_dev(ctx.handle, f.handle, 10, (C.c_double * 2)(2.0, 1.0), e, cnt) == N.INVALID
    assert "max must be larger than min" in N.lib().bdf_last_error().decode()
    assert L.bdf_hist_dev(ctx.handle, f.handle, 10, (C.c_double * 2)(0.0, float("inf")), e, cnt) == N.INVALID
    assert "supplied range" in N.lib().bdf_last_error().decode()
    assert list(e) == [0.0] * 11 and list(cnt) == [0] * 10   # nothing written on failure
    aggs = (N.GroupAggC * 1)()
    hk, ro, ng = (C.c_void_p * 1)(), (C.c_void_p * 1)(), C.c_int64()
    kc = (C.c_void_p * 1)(f.handle.value)
    for unknown in (15, 31, 34, -1):   # the ids around the distribution block stay unknown
        aggs[0].column, aggs[0].function = f.handle.value, unknown
        assert L.bdf_group_by_dev(ctx.handle, 1, kc, 1, aggs, hk, ro, C.byref(ng)) == N.UNSUPPORTED
    with pytest.raises(rdf.UnsupportedType):
        rdf.group_by([f], [(f, "median")])   # the group-by name is "exact_median"
    for _ in range(2):   # successful calls leave nothing behind either
        f.median(), f.mode(), f.hist(4, range=(0.0, 3.0)), f.uniques().free()
        ks, res = rdf.group_by([f], [(f, "exact_median"), (f, "mode")])
        for col in ks + res:
            col.free()
    ctx.synchronize()
    assert pool_used(ctx) == before
    bcol.free()
    f.free()


def test_multi_gpu_context_is_refused(rdf):
    N = rdf.native
    L = N.lib()
    fleet = rdf.Context.multi(0)
    h = fleet.handle
    try:
        a = rdf.PrimitiveArray.from_numpy(np.arange(10.0))
        out, some, p = (C.c_double * 1)(), (C.c_int32 * 1)(), (C.c_double * 1)(0.5)
        bits, freq = C.c_uint64(), C.c_int64()
        assert L.bdf_percentile(h, rdf.F64, 1, N.make_views([a]), 1, p, out, some) == N.UNSUPPORTED
        assert L.bdf_mode(h, rdf.F64, 1, N.make_views([a]), C.byref(bits), C.byref(freq), some) == N.UNSUPPORTED
        assert L.bdf_percentile_dev(h, None, 1, p, out, some) == N.UNSUPPORTED
        assert L.bdf_hist_dev(h, None, 1, None, (C.c_double * 2)(), (C.c_int64 * 1)()) == N.UNSUPPORTED
        assert L.bdf_uniques_dev(h, None, C.byref(C.c_void_p()), None) == N.UNSUPPORTED
        assert L.bdf_mode_dev(h, None, C.byref(bits), C.byref(freq), some) == N.UNSUPPORTED
    finally:
        fleet.close()


def test_launch_records(rdf, ctx):
    col = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.random.default_rng(2).normal(0, 1, 100000))], ctx=ctx)
    ctx.profile_enable(True)
    col.median()
    col.hist(10)
    recs = ctx.profile_read()
    ctx.profile_enable(False)
    kinds = {r["kernel"] for r in recs}
    assert {"select", "hist"} <= kinds
    col.free()


def test_cpp_mirror_distributions(rdf):
    host = os.path.join(ROOT, "rust-dataframe_b200", "host")
    subprocess.check_call(["make", "-C", host, "test_dist_host"], stdout=subprocess.DEVNULL)
    env = dict(os.environ, BDF_ONE_GPU="1")
    r = subprocess.run([os.path.join(host, "test_dist_host")], capture_output=True, text=True, timeout=300, env=env)
    print(r.stdout[-3000:], r.stderr[-2000:])
    assert r.returncode == 0 and "DIST OK" in r.stdout
