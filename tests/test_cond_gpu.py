"""Null handling and conditional selection on the GPU (k_cond.cu), compared bit for bit with cond_oracle.py.

Every case runs over chunks of the lengths where the kernels change shape -- 0, 1, 31, 32, 33, the tiles +-1 (2048 rows for
the value kernels, 32768 for the word kernels) and 100 001 -- cut out of larger arrays at odd offsets, so that values and
validity (and Boolean values) start at bit offsets.  Null counts must be exact and the chunk structure kept."""
import ctypes as C
import os
import subprocess
import zlib

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import cond_oracle as co
from helpers import pool_used

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

NUMERIC = ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "float32", "float64"]
VALUE_TILE = 8 * 8 * 32     # k_cond.cu kCondTile
WORD_TILE = 256 * 4 * 32    # k_cond.cu kCondBoolTile
LENS = [0, 1, 31, 32, 33, VALUE_TILE - 1, VALUE_TILE, VALUE_TILE + 1, 100_001]
BOOL_LENS = [0, 1, 31, 33, WORD_TILE - 1, WORD_TILE, WORD_TILE + 1, 100_001]


def _seed(*names) -> int:
    """A fixed seed per case (str hashes change from process to process)."""
    return zlib.crc32("/".join(names).encode())


def _values(rng, name, n):
    if name == "bool":
        return rng.random(n) < 0.5
    npdt = np.dtype(name)
    if npdt.kind == "f":   # few distinct values, so greatest / least meet ties, signed zeros, infinities and NaN
        pool = np.array([0.0, -0.0, 1.5, -1.5, np.inf, -np.inf, np.nan, 3.25, -7.0, 1e30], dtype=npdt)
        v = pool[rng.integers(0, len(pool), n)]
        nan2 = np.array([0x7FC00123 if npdt.itemsize == 4 else 0x7FF8000000000123], dtype=f"u{npdt.itemsize}").view(npdt)
        v[rng.random(n) < 0.02] = nan2[0]
        return v
    info = np.iinfo(npdt)
    return rng.integers(max(info.min, -40), min(info.max, 40), n, endpoint=True).astype(npdt)


class Arg:
    """One column argument: the host arrays (the oracle's view) and the chunks that are uploaded."""

    def __init__(self, rdf, rng, name, lens, null_frac, bitmap=True):
        self.name = name
        n = sum(lens)
        self.v = _values(rng, name, n)
        self.m = rng.random(n) >= null_frac if bitmap else np.ones(n, dtype=bool)
        self.chunks, pos = [], 0
        for i, ln in enumerate(lens):
            off = (i * 3 + 1) % 8   # a bit offset on values and validity
            vv = np.concatenate([_values(rng, name, off), self.v[pos:pos + ln]])
            mm = np.concatenate([np.ones(off, dtype=bool), self.m[pos:pos + ln]])
            if name == "bool":
                arr = rdf.BooleanArray.from_numpy(vv, mm if bitmap else None).slice(off, ln)
                arr.null_count = int((~mm[off:]).sum()) if bitmap else 0
            else:
                arr = rdf.PrimitiveArray.from_numpy(vv, mm if bitmap else None).slice(off, ln)
            self.chunks.append(arr)
            pos += ln

    def column(self, rdf, ctx, temporal=None):
        dtype = rdf.native.BOOL if self.name == "bool" else rdf.dtype_of(self.name)
        col = rdf.Column.upload(self.chunks, ctx, dtype=dtype)
        return col.with_temporal(temporal) if temporal is not None else col

    @property
    def host(self):
        return self.v, self.m


def _download(rdf, col):
    res = col.download()
    if not res:
        return np.zeros(0), np.zeros(0, dtype=bool), []
    if col.dtype == rdf.native.BOOL:
        v = np.concatenate([r.value_bits() for r in res])
    else:
        v = np.concatenate([r.value_slice() for r in res])
    m = np.concatenate([r.valid_mask() for r in res])
    return v, m, res


def _check(rdf, col, want, lens):
    v, m, _ = _download(rdf, col)
    assert col.n_chunks == len(lens)
    assert co.same((v, m), want)
    pos = 0
    for i, ln in enumerate(lens):
        info = col.chunk_info(i)
        assert info["len"] == ln
        assert info["null_count"] == int((~want[1][pos:pos + ln]).sum()), i
        pos += ln


def _scalar_host(rdf, name, value, n):
    npdt = bool if name == "bool" else np.dtype(name)
    return co.scalar(value, n, npdt)


ORACLE = {"coalesce": co.coalesce, "greatest": co.greatest, "least": co.least}


@pytest.mark.parametrize("name", NUMERIC + ["bool"])
@pytest.mark.parametrize("fn", ["coalesce", "greatest", "least", "nanvl"])
def test_rowwise_functions(rdf, ctx, name, fn):
    if name == "bool" and fn != "coalesce":
        pytest.skip("Boolean values are only selected by coalesce / case_when")
    if fn == "nanvl" and name not in ("float32", "float64"):
        pytest.skip("nanvl is a float function")
    lens = BOOL_LENS if name == "bool" else LENS
    n = sum(lens)
    rng = np.random.default_rng(_seed(name, fn))
    counts = [2] if fn == "nanvl" else ([1, 2, 3, 64] if fn == "coalesce" else [2, 3, 64])
    for k in counts:
        for null_frac in ((0.1,) if k == 64 else (0.0, 0.1, 1.0)):
            args = [Arg(rdf, rng, name, lens, null_frac, bitmap=(j % 3 != 2)) for j in range(k)]
            cols = [a.column(rdf, ctx) for a in args]
            if fn == "nanvl":
                got, want = cols[0].nanvl(cols[1]), co.nanvl(args[0].host, args[1].host)
            else:
                got, want = getattr(rdf, fn)(*cols), ORACLE[fn]([a.host for a in args])
            _check(rdf, got, want, lens)
            if k >= 2:   # valid and NULL scalars next to columns with and without a bitmap
                sval = True if name == "bool" else (1 if name[0] != "f" else -0.0)
                vals = [cols[0], sval, None, cols[1]] if fn != "nanvl" else [cols[0], sval]
                host = [args[0].host, _scalar_host(rdf, name, sval, n), _scalar_host(rdf, name, None, n), args[1].host]
                if fn == "nanvl":
                    got, want = cols[0].nanvl(sval), co.nanvl(args[0].host, host[1])
                else:
                    got, want = getattr(rdf, fn)(*vals), ORACLE[fn](host)
                _check(rdf, got, want, lens)
            for c in cols:
                c.free()


@pytest.mark.parametrize("name", NUMERIC + ["bool"])
def test_case_when(rdf, ctx, name):
    lens = BOOL_LENS if name == "bool" else LENS
    n = sum(lens)
    rng = np.random.default_rng(_seed("case", name))
    for branches in (1, 2, 3, 64):
        for null_frac in ((0.1,) if branches == 64 else (0.0, 0.1, 1.0)):
            conds = [Arg(rdf, rng, "bool", lens, null_frac, bitmap=(j % 2 == 0)) for j in range(branches)]
            vals = [Arg(rdf, rng, name, lens, null_frac, bitmap=(j % 3 != 1)) for j in range(branches + 1)]
            cc = [c.column(rdf, ctx) for c in conds]
            vc = [v.column(rdf, ctx) for v in vals]
            chain = rdf.when(cc[0], vc[0])
            for c, v in zip(cc[1:], vc[1:branches]):
                chain = chain.when(c, v)
            cond_host = [c.host for c in conds]
            _check(rdf, chain.otherwise(vc[-1]), co.case_when(cond_host, [v.host for v in vals]), lens)
            _check(rdf, chain.end(), co.case_when(cond_host, [v.host for v in vals[:-1]] + [_scalar_host(rdf, name, None, n)]), lens)
            sval = False if name == "bool" else 5
            _check(rdf, chain.otherwise(sval), co.case_when(cond_host, [v.host for v in vals[:-1]] + [_scalar_host(rdf, name, sval, n)]), lens)
            if branches == 2:   # every value a scalar but one: the conditions give the length
                only = rdf.when(cc[0], sval).when(cc[1], vc[1]).otherwise(None)
                want = co.case_when(cond_host, [_scalar_host(rdf, name, sval, n), vals[1].host, _scalar_host(rdf, name, None, n)])
                _check(rdf, only, want, lens)
            for c in cc + vc:
                c.free()


@pytest.mark.parametrize("name", NUMERIC + ["bool"])
def test_null_tests(rdf, ctx, name):
    lens = BOOL_LENS
    rng = np.random.default_rng(_seed("test", name))
    for null_frac in (0.0, 0.1, 1.0):
        for bitmap in (True, False):
            a = Arg(rdf, rng, name, lens, null_frac, bitmap=bitmap)
            col = a.column(rdf, ctx)
            _check(rdf, col.is_null(), co.is_null(a.host), lens)
            _check(rdf, col.is_not_null(), co.is_not_null(a.host), lens)
            want = co.is_nan(a.host) if name != "bool" else (np.zeros(sum(lens), bool), np.ones(sum(lens), bool))
            got = col.is_nan()
            _check(rdf, got, want, lens)
            for i in range(len(lens)):
                assert not got.chunk_info(i)["has_validity"]
            col.free()


def test_timestamp_tag_passes_through(rdf, ctx):
    rng = np.random.default_rng(5)
    ts = rdf.TemporalType.timestamp("us")
    a, b = Arg(rdf, rng, "int64", LENS, 0.3), Arg(rdf, rng, "int64", LENS, 0.2)
    ca, cb = a.column(rdf, ctx, ts), b.column(rdf, ctx, ts)
    for got, want in ((rdf.coalesce(ca, cb), co.coalesce([a.host, b.host])), (rdf.greatest(ca, cb), co.greatest([a.host, b.host])),
                      (ca.fill_null(0), co.coalesce([a.host, co.scalar(0, sum(LENS), np.int64)]))):
        assert got.temporal == ts
        _check(rdf, got, want, LENS)
    plain = b.column(rdf, ctx)
    with pytest.raises(rdf.UnsupportedType):
        rdf.coalesce(ca, plain)


def test_errors_leak_nothing(rdf, ctx):
    N = rdf.native
    lib = N.lib()
    rng = np.random.default_rng(9)
    i32 = Arg(rdf, rng, "int32", [10, 20], 0.2).column(rdf, ctx)
    i32b = Arg(rdf, rng, "int32", [10, 20], 0.2).column(rdf, ctx)
    f64 = Arg(rdf, rng, "float64", [10, 20], 0.2).column(rdf, ctx)
    short = Arg(rdf, rng, "int32", [10, 21], 0.2).column(rdf, ctx)
    bl = Arg(rdf, rng, "bool", [10, 20], 0.2).column(rdf, ctx)
    bl2 = Arg(rdf, rng, "bool", [10, 20], 0.0).column(rdf, ctx)
    ctx.synchronize()
    before = pool_used(ctx)

    def args(*vals):
        a = (N.Arg * max(len(vals), 1))()
        for j, v in enumerate(vals):
            if v is None:
                a[j].valid = 0
            elif isinstance(v, int):
                a[j].bits, a[j].valid = v, 1
            else:
                a[j].column, a[j].valid = v.handle, 1
        return a

    h = C.c_void_p()
    rw = lambda fn, *v: lib.bdf_rowwise_dev(ctx.handle, fn, len(v), args(*v), C.byref(h))
    assert rw(N.ROW_COALESCE, i32, f64) == N.INVALID                  # mixed types
    assert rw(N.ROW_COALESCE, i32, short) == N.LENGTH_MISMATCH
    assert rw(N.ROW_GREATEST, bl, bl2) == N.UNSUPPORTED               # Boolean greatest
    assert rw(N.ROW_NANVL, i32, i32b) == N.UNSUPPORTED                # nanvl of integers
    assert rw(N.ROW_COALESCE, 1, None) == N.INVALID                   # no column argument
    assert rw(N.ROW_GREATEST, i32) == N.INVALID                       # too few arguments
    assert rw(N.ROW_NANVL, f64, f64, f64) == N.INVALID
    assert lib.bdf_rowwise_dev(ctx.handle, N.ROW_COALESCE, 65, args(*([i32] * 65)), C.byref(h)) == N.INVALID
    assert rw(7, i32, i32b) == N.INVALID
    assert rw(N.ROW_COALESCE, bl, 2) == N.INVALID                     # a Boolean scalar is 0 or 1
    conds = (C.c_void_p * 2)(i32.handle, bl.handle)
    assert lib.bdf_case_when_dev(ctx.handle, 1, conds, args(i32, i32b), C.byref(h)) == N.INVALID   # a condition must be Boolean
    conds = (C.c_void_p * 1)(bl.handle)
    assert lib.bdf_case_when_dev(ctx.handle, 1, conds, args(short, None), C.byref(h)) == N.LENGTH_MISMATCH
    assert lib.bdf_case_when_dev(ctx.handle, 1, conds, args(1, None), C.byref(h)) == N.INVALID      # nothing gives the type
    assert lib.bdf_case_when_dev(ctx.handle, 0, conds, args(i32), C.byref(h)) == N.INVALID
    assert lib.bdf_null_test_dev(ctx.handle, 3, i32.handle, C.byref(h)) == N.INVALID
    with pytest.raises(rdf.UnsupportedType):
        i32.fill_null(1.5)
    ctx.synchronize()
    assert pool_used(ctx) == before


@pytest.fixture(scope="module")
def fleet(rdf):
    import torch

    if not torch.cuda.device_count():
        pytest.skip("no GPU")
    ctx = rdf.Context.multi(0)
    yield ctx
    ctx.close()


def test_multi_gpu_matches_one_gpu(rdf, ctx, fleet):
    lens = [100_001, 0, 1, 70_000, 64, 33_333, 4097]
    rng = np.random.default_rng(21)
    for name in ("float64", "int32", "uint8", "bool"):
        args = [Arg(rdf, rng, name, lens, 0.2, bitmap=(j != 1)) for j in range(3)]
        conds = [Arg(rdf, rng, "bool", lens, 0.1) for _ in range(2)]
        one = [a.column(rdf, ctx) for a in args]
        many = [a.column(rdf, fleet) for a in args]
        c_one = [c.column(rdf, ctx) for c in conds]
        c_many = [c.column(rdf, fleet) for c in conds]
        calls = [lambda cs, ks: rdf.coalesce(*cs), lambda cs, ks: rdf.when(ks[0], cs[0]).when(ks[1], cs[1]).otherwise(cs[2]),
                 lambda cs, ks: cs[0].is_null(), lambda cs, ks: cs[1].is_nan()]
        if name != "bool":
            calls += [lambda cs, ks: rdf.greatest(*cs), lambda cs, ks: rdf.least(cs[0], cs[2])]
        if name == "float64":
            calls.append(lambda cs, ks: cs[0].nanvl(cs[1]))
        for call in calls:
            a, b = call(one, c_one), call(many, c_many)
            va, ma, ra = _download(rdf, a)
            vb, mb, rb = _download(rdf, b)
            assert co.same((vb, mb), (va, ma)) and len(ra) == len(rb) == len(lens)
            for i in range(len(lens)):
                assert a.chunk_info(i) == b.chunk_info(i)


def test_frame_left_join_fill_null_and_coalesce(rdf, ctx):
    rng = np.random.default_rng(4)
    ka = rng.integers(0, 50, 300).astype(np.int64)
    kb = rng.permutation(np.arange(0, 100, 2)).astype(np.int64)
    xb = rng.uniform(-5, 5, kb.shape[0])
    ya = rng.uniform(-5, 5, 300)
    fa = rdf.DeviceFrame.from_host({"k": [rdf.PrimitiveArray.from_numpy(ka)], "y": [rdf.PrimitiveArray.from_numpy(ya)]}, ctx=ctx)
    fb = rdf.DeviceFrame.from_host({"kb": [rdf.PrimitiveArray.from_numpy(kb)], "x": [rdf.PrimitiveArray.from_numpy(xb)]}, ctx=ctx)
    joined = fa.join(fb, [("k", "kb")], "left")
    host = joined.to_host()
    t = pa.table({n: pa.array(c[0].value_slice(), mask=~c[0].valid_mask()) for n, c in host.items()})
    filled = joined.fill_null(0)
    got = filled.to_host()
    assert np.array_equal(got["x"][0].value_slice(), np.asarray(pc.fill_null(t["x"], 0.0)).astype(np.float64))
    assert got["x"][0].valid_mask().all() and got["kb"][0].valid_mask().all()
    assert np.array_equal(got["kb"][0].value_slice(), np.asarray(pc.fill_null(t["kb"], 0)))
    co_col = rdf.coalesce(joined.column("x"), joined.column("y"))
    v, m, _ = _download(rdf, co_col)
    want = pc.coalesce(t["x"], t["y"]).combine_chunks()
    assert m.all() and np.array_equal(v, np.asarray(want))
    only = joined.fill_null({"x": -1.0})
    assert only.column("kb").chunk_info(0)["null_count"] == joined.column("kb").chunk_info(0)["null_count"]
    with pytest.raises(rdf.UnsupportedType):
        joined.fill_null({"k": 0.5})


def test_frame_drop_nulls_and_null_filters(rdf, ctx):
    P = rdf.PrimitiveArray
    a = [P.from_pylist(rdf.I32, [1, None, 3, None, 5]), P.from_pylist(rdf.I32, [None, 7])]
    b = [P.from_pylist(rdf.F64, [1.0, 2.0, None, None, float("nan")]), P.from_pylist(rdf.F64, [None, 8.0])]
    c = [P.from_pylist(rdf.I64, [1, 2, 3, 4, 5]), P.from_pylist(rdf.I64, [6, 7])]
    d = [P.from_pylist(rdf.U8, [None, 2, 3, 4, 5]), P.from_pylist(rdf.U8, [6, None])]
    f = rdf.DeviceFrame.from_host({"a": a, "b": b, "c": c, "d": d}, ctx=ctx)
    rows = lambda fr, n: [x for ch in fr.to_host()[n] for x in ch.to_pylist()]
    assert rows(f.drop_nulls(), "c") == [5]
    assert rows(f.drop_nulls(how="all", subset=["a", "b"]), "c") == [1, 2, 3, 5, 7]
    assert rows(f.drop_nulls(subset=["a"]), "c") == [1, 3, 5, 7]
    assert rows(f.filter(rdf.frame.is_null("a")), "c") == [2, 4, 6]
    assert rows(f.filter(rdf.frame.is_nan("b")), "c") == [5]
    assert rows(f.filter(("and", rdf.frame.is_not_null("a"), rdf.frame.is_not_null("d"))), "c") == [3, 5]
    assert f.drop_nulls().column("c").n_chunks == 2


def test_frame_when_over_a_lag_column(rdf, ctx):
    P = rdf.PrimitiveArray
    x = np.array([3.0, 1.0, 4.0, 1.0, 5.0, 9.0, 2.0, 6.0])
    f = rdf.DeviceFrame.from_host({"i": [P.from_numpy(np.arange(8, dtype=np.int64))], "x": [P.from_numpy(x)]}, ctx=ctx)
    f = f.window([], [("i", False)], [("prev", "lag", "x", 1)])
    prev = f.column("prev")
    up = prev.lt(f.column("x"))
    res = rdf.when(up, f.column("x")).when(prev.is_null(), -1.0).otherwise(0.0)
    v, m, _ = _download(rdf, res)
    want = [-1.0] + [x[i] if x[i - 1] < x[i] else 0.0 for i in range(1, 8)]
    assert m.all() and list(v) == want


@pytest.mark.parametrize("name", ["int8", "uint32", "int64", "float32", "float64"])
def test_scalar_functions_over_host_chunks(rdf, ctx, name):
    """ScalarFunctions.coalesce / greatest / least / nanvl: lists of chunks (sliced, with and without bitmaps) and scalars, uploaded,
    computed and downloaded; the chunk structure, values and null counts as the oracle says."""
    rng = np.random.default_rng(_seed("host", name))
    n = sum(LENS)
    a, b, c = (Arg(rdf, rng, name, LENS, f, bitmap=bm) for f, bm in ((0.3, True), (0.2, True), (0.0, False)))
    sval = 3 if name[0] != "f" else 0.5

    def check(res, want):
        assert len(res) == len(LENS) and [r.length for r in res] == LENS
        v = np.concatenate([r.value_slice() for r in res])
        m = np.concatenate([r.valid_mask() for r in res])
        assert co.same((v, m), want)
        pos = 0
        for r, ln in zip(res, LENS):
            assert r.compute_null_count() == int((~want[1][pos:pos + ln]).sum())
            pos += ln

    SF = rdf.ScalarFunctions
    check(SF.coalesce(a.chunks, b.chunks, ctx=ctx), co.coalesce([a.host, b.host]))
    check(SF.coalesce(a.chunks, None, sval, ctx=ctx), co.coalesce([a.host, _scalar_host(rdf, name, None, n), _scalar_host(rdf, name, sval, n)]))
    check(SF.greatest(a.chunks, b.chunks, c.chunks, ctx=ctx), co.greatest([a.host, b.host, c.host]))
    check(SF.least(a.chunks, sval, ctx=ctx), co.least([a.host, _scalar_host(rdf, name, sval, n)]))
    if name[0] == "f":
        check(SF.nanvl(a.chunks, b.chunks, ctx=ctx), co.nanvl(a.host, b.host))
    else:
        with pytest.raises(rdf.UnsupportedType):
            SF.nanvl(a.chunks, b.chunks, ctx=ctx)


def test_cpp_mirror_null_functions(rdf):
    host = os.path.join(ROOT, "rust-dataframe_b200", "host")
    subprocess.check_call(["make", "-C", host, "test_cond_host"], stdout=subprocess.DEVNULL)
    env = dict(os.environ, BDF_ONE_GPU="1")
    r = subprocess.run([os.path.join(host, "test_cond_host")], capture_output=True, text=True, timeout=300, env=env)
    print(r.stdout[-3000:], r.stderr[-2000:])
    assert r.returncode == 0 and "COND OK" in r.stdout
