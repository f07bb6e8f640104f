"""DataFrame::to_csv on the device: every file byte for byte against tests/csv_write_oracle.py, round trips through the library's own
reader and pyarrow, the reference's end-to-end pipeline, a multi-GB write in bounded memory, and the errors."""
import ctypes as C
import hashlib
import os
import shutil
from collections import OrderedDict

import numpy as np
import pytest

import csv_write_oracle as wo
from helpers import pool_used

HERE = os.path.dirname(os.path.abspath(__file__))
UK = os.path.join(HERE, "golden", "uk_cities_with_headers.csv")
NP = {0: np.int8, 1: np.int16, 2: np.int32, 3: np.int64, 4: np.uint8, 5: np.uint16, 6: np.uint32, 7: np.uint64, 8: np.float32, 9: np.float64}
DTYPES = list(range(11))


def _values(rng, dt, n):
    if dt == wo.BOOL:
        return rng.random(n) < 0.5
    t = NP[dt]
    if dt == 8:
        return rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32).view(np.float32)
    if dt == 9:
        return rng.integers(0, 2 ** 64, n, dtype=np.uint64).view(np.float64)
    info = np.iinfo(t)
    return rng.integers(info.min, info.max, n, dtype=t, endpoint=True)


def _upload(rdf, ctx, dt, vals, valid, lens=None):
    """One column in chunks of `lens` rows, each a slice at bit offset 1..7 of a larger host array (offset 0 for the first)."""
    lens = [len(vals)] if lens is None else lens
    chunks, s = [], 0
    for i, n in enumerate(lens):
        off = i % 8
        v = vals[s:s + n]
        m = None if valid is None else valid[s:s + n]
        if dt == wo.BOOL:
            a = rdf.BooleanArray.from_numpy(np.concatenate([np.zeros(off, bool), v]), None if m is None else np.concatenate([np.ones(off, bool), m]))
        else:
            a = rdf.PrimitiveArray.from_numpy(np.concatenate([np.zeros(off, v.dtype), v]), None if m is None else np.concatenate([np.ones(off, bool), m]))
        a = a.slice(off, n)
        a.null_count = 0 if m is None else int((~m).sum())
        chunks.append(a)
        s += n
    return rdf.Column.upload(chunks, ctx=ctx, dtype=dt)


def _write_and_compare(rdf, ctx, tmp_path, cols, lens=None, has_header=True, delimiter=","):
    dev = OrderedDict((name, _upload(rdf, ctx, dt, v, m, lens)) for name, dt, v, m in cols)
    p = tmp_path / "w.csv"
    rdf.write_csv(str(p), dev, has_header=has_header, delimiter=delimiter)
    got, want = p.read_bytes(), wo.write(cols, has_header, delimiter)
    if got != want:
        gl, wl = got.split(b"\n"), want.split(b"\n")
        bad = [i for i in range(min(len(gl), len(wl))) if gl[i] != wl[i]][:5]
        raise AssertionError(f"{len(got)} vs {len(want)} bytes; first differing lines {[(i, gl[i][:120], wl[i][:120]) for i in bad]}")
    return dev, p


@pytest.mark.gpu
@pytest.mark.parametrize("nullable", [False, True])
@pytest.mark.parametrize("dt", DTYPES)
def test_every_dtype_in_sliced_chunks(rdf, ctx, tmp_path, dt, nullable):
    rng = np.random.default_rng(100 + dt)
    n = 6000
    vals = _values(rng, dt, n)
    valid = rng.random(n) >= 0.2 if nullable else None
    lens = [1000, 1, 2500, 7, 1492, 1000]
    _write_and_compare(rdf, ctx, tmp_path, [("v", dt, vals, valid), ("k", 2, np.arange(n, dtype=np.int32), None)], lens)
    _write_and_compare(rdf, ctx, tmp_path, [("v", dt, vals, valid)], lens)   # alone: a NULL row is ""


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 2, 16, 64])
def test_column_counts(rdf, ctx, tmp_path, k):
    rng = np.random.default_rng(k)
    n = 3000
    cols = []
    for j in range(k):
        dt = DTYPES[(j * 7) % 11]
        cols.append((f"c{j}", dt, _values(rng, dt, n), rng.random(n) >= 0.1 if j % 3 == 0 else None))
    _write_and_compare(rdf, ctx, tmp_path, cols, [1200, 1800])


@pytest.mark.gpu
@pytest.mark.parametrize("has_header", [True, False])
def test_zero_and_one_row(rdf, ctx, tmp_path, has_header):
    one = [("a", 3, np.array([-5], np.int64), None), ("b", 9, np.array([0.5]), np.array([False]))]
    _write_and_compare(rdf, ctx, tmp_path, one, has_header=has_header)
    _write_and_compare(rdf, ctx, tmp_path, [("a", 9, np.array([np.nan]), np.array([False]))], has_header=has_header)
    zero = [("a", 3, np.zeros(0, np.int64), None), ("b", 8, np.zeros(0, np.float32), None)]
    _write_and_compare(rdf, ctx, tmp_path, zero, has_header=has_header)
    assert (tmp_path / "w.csv").read_bytes() == (b"a,b\n" if has_header else b"")


@pytest.mark.gpu
def test_one_nullable_column_and_quoted_names(rdf, ctx, tmp_path):
    _, p = _write_and_compare(rdf, ctx, tmp_path, [("x", 2, np.array([1, 2, 3], np.int32), np.array([True, False, True]))])
    assert p.read_bytes() == b'x\n1\n""\n3\n'
    names = ["plain", "with,comma", 'with"quote', "with\nnewline", "with\rcr", "semi;colon"]
    cols = [(nm, 2, np.arange(4, dtype=np.int32) * j, None) for j, nm in enumerate(names)]
    _, p = _write_and_compare(rdf, ctx, tmp_path, cols)
    assert p.read_bytes().startswith(b'plain,"with,comma","with""quote","with\nnewline","with\rcr",semi;colon\n')
    _, p = _write_and_compare(rdf, ctx, tmp_path, cols, delimiter=";")
    assert p.read_bytes().startswith(b'plain;with,comma;"with""quote";"with\nnewline";"with\rcr";"semi;colon"\n')


@pytest.mark.gpu
def test_delimiters(rdf, ctx, tmp_path):
    rng = np.random.default_rng(9)
    cols = [(f"c{dt}", dt, _values(rng, dt, 500), rng.random(500) >= 0.3) for dt in DTYPES]
    for d in [";", "\t", "|"]:
        _write_and_compare(rdf, ctx, tmp_path, cols, [200, 300], delimiter=d)
    dev = OrderedDict((name, _upload(rdf, ctx, dt, v, m)) for name, dt, v, m in cols[:2])
    before = pool_used(ctx)
    for d in wo.REFUSED_DELIMITERS:
        with pytest.raises(rdf.ComputeError, match=r"\[bdf status 8\]"):
            rdf.write_csv(str(tmp_path / "r.csv"), dev, delimiter=bytes([d]))
    assert pool_used(ctx) == before


def _float_cases(width):
    rng = np.random.default_rng(width)
    n = 2_000_000
    if width == 64:
        ut, ft, mbits, ebits = np.uint64, np.float64, 52, 11
        rand = rng.integers(0, 2 ** 64, n, dtype=np.uint64)
    else:
        ut, ft, mbits, ebits = np.uint32, np.float32, 23, 8
        rand = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32)
    # every exponent (subnormals included) with random mantissas, NaN payloads, +-inf, +-0
    e = np.arange(2 ** ebits, dtype=np.uint64)
    mant = rng.integers(0, 2 ** mbits, (2 ** ebits, 8), dtype=np.uint64)
    every_exp = ((e[:, None] << np.uint64(mbits)) | mant).ravel()
    pow2 = e << np.uint64(mbits)                      # every power of two (and 0, inf)
    sub_pow2 = np.uint64(1) << np.arange(mbits, dtype=np.uint64)   # the subnormal powers of two
    ten = []
    lo, hi = (-324, 309) if width == 64 else (-46, 39)
    for k in range(lo, hi):
        b = int(np.array(ft(float(f"1e{k}"))).view(ut))
        ten += [b + d for d in range(-3, 4) if 0 <= b + d < (2 ** (mbits + ebits) - 2 ** mbits)]
    fin = np.finfo(ft)
    extremes = np.array([fin.max, fin.tiny, fin.smallest_subnormal, fin.eps, 1.0], ft).view(ut)
    allb = np.concatenate([rand.astype(np.uint64), every_exp, pow2, sub_pow2, np.array(ten, np.uint64), extremes.astype(np.uint64)])
    sign = np.uint64(1) << np.uint64(width - 1)
    allb = np.concatenate([allb, allb | sign])
    return allb.astype(ut).view(ft)


@pytest.mark.gpu
@pytest.mark.parametrize("width", [64, 32])
def test_floats_byte_for_byte(rdf, ctx, tmp_path, width):
    vals = _float_cases(width)
    assert vals.size >= 4_000_000
    dt = 9 if width == 64 else 8
    _write_and_compare(rdf, ctx, tmp_path, [("x", dt, vals, None)], [vals.size // 3, vals.size - vals.size // 3])


def _device_bits(col):
    out = []
    for a in col.download():
        m = a.valid_mask()
        v = np.asarray(a.value_bits()) if hasattr(a, "value_bits") else np.asarray(a.value_slice())
        out.append((v, m))
    return np.concatenate([v for v, _ in out]), np.concatenate([m for _, m in out])


@pytest.mark.gpu
def test_round_trip_through_the_reader_and_pyarrow(rdf, ctx, tmp_path):
    rng = np.random.default_rng(77)
    n = 20000
    cols = [(f"c{dt}", dt, _values(rng, dt, n), rng.random(n) >= 0.15) for dt in DTYPES]
    _, p = _write_and_compare(rdf, ctx, tmp_path, cols, [7000, 13000])
    back = rdf.DeviceFrame.from_csv(str(p), schema=DTYPES, batch_size=4096, ctx=ctx)
    for name, dt, vals, valid in cols:
        v, m = _device_bits(back.column(name))
        assert np.array_equal(m, valid), name
        if dt in (8, 9):
            u = f"u{vals.itemsize}"
            same = (v.view(u) == vals.view(u)) | (np.isnan(v) & np.isnan(vals))
            assert same[m].all(), name
        else:
            assert np.array_equal(v[m], vals[m]), name
    pa = pytest.importorskip("pyarrow")
    pcsv = pytest.importorskip("pyarrow.csv")
    pat = {0: pa.int8(), 1: pa.int16(), 2: pa.int32(), 3: pa.int64(), 4: pa.uint8(), 5: pa.uint16(), 6: pa.uint32(), 7: pa.uint64(),
           8: pa.float32(), 9: pa.float64(), 10: pa.bool_()}
    t = pcsv.read_csv(str(p), convert_options=pcsv.ConvertOptions(column_types={f"c{dt}": pat[dt] for dt in DTYPES}, null_values=[""]))
    for name, dt, vals, valid in cols:
        c = t.column(name).combine_chunks()
        assert np.array_equal(~np.asarray(c.is_null()), valid), name
        got = [x for x, ok in zip(c.to_pylist(), valid) if ok]
        want = vals[valid]
        if dt in (8, 9):
            g = np.array(got, dtype=want.dtype)
            u = f"u{want.itemsize}"
            assert ((g.view(u) == want.view(u)) | (np.isnan(g) & np.isnan(want))).all(), name
        else:
            assert got == want.tolist(), name


@pytest.mark.gpu
def test_uk_cities(rdf, ctx, tmp_path):
    df = rdf.DeviceFrame.from_csv(UK, ctx=ctx)
    p = tmp_path / "uk.csv"
    df.to_csv(str(p))
    lines = open(UK).read().splitlines()
    want = ["lat,lng"]
    for ln in lines[1:]:
        f = ln.rsplit(",", 2)
        want.append(",".join(x.rstrip("0").rstrip(".") for x in f[1:]))
    assert p.read_text().splitlines() == want
    assert "-3.17909" in p.read_text()
    # test_lazy_evaluation (src/evaluation.rs:359-434): CSV -> rename -> sin(lat), sin(lng) -> limit 25 -> to_csv
    ren = rdf.DeviceFrame(OrderedDict([("latitude", df.column("lat")), ("longitude", df.column("lng"))]))
    ren = ren.with_column("sin_lat", ren.column("latitude").sin()).with_column("sin_lng", ren.column("longitude").sin()).limit(25)
    q = tmp_path / "lazy.csv"
    ren.to_csv(str(q))
    host = [(n, 9, np.concatenate([a.value_slice() for a in c.download()]), None) for n, c in ren.columns.items()]
    assert q.read_bytes() == wo.write(host)
    assert len(q.read_text().splitlines()) == 26


def _pool_high(ctx, reset=False):
    cu = C.CDLL("libcuda.so.1")
    dev, pool, v = C.c_int(), C.c_void_p(), C.c_uint64(0)
    assert cu.cuDeviceGet(C.byref(dev), ctx.device) == 0 and cu.cuDeviceGetDefaultMemPool(C.byref(pool), dev) == 0
    if reset:
        assert cu.cuMemPoolSetAttribute(pool, 8, C.byref(v)) == 0   # CU_MEMPOOL_ATTR_USED_MEM_HIGH
        return 0
    assert cu.cuMemPoolGetAttribute(pool, 8, C.byref(v)) == 0
    return v.value


@pytest.mark.gpu
def test_full_size_write_in_bounded_memory(rdf, ctx, tmp_path):
    n = 100_000_000
    if shutil.disk_usage(str(tmp_path)).free < 16 << 30:
        pytest.skip("needs 16 GB of free disk for a 6 GB file")
    lens = [n // 4] * 4
    i64 = rdf.Column.generate(rdf.I64, lens, kind=3, col_id=1, null_mod=10, ctx=ctx)
    f64 = rdf.Column.generate(rdf.F64, lens, kind=0, lo=-1e3, hi=1e3, col_id=2, null_mod=10, ctx=ctx)
    f32 = rdf.Column.generate(rdf.F32, lens, kind=0, lo=-1.0, hi=1.0, col_id=3, null_mod=10, ctx=ctx)
    b = rdf.Column.generate(rdf.F64, lens, kind=0, col_id=4, ctx=ctx).gt(0.5)
    frame = OrderedDict([("i", i64), ("d", f64), ("f", f32), ("b", b)])
    p = tmp_path / "big.csv"
    ctx.synchronize()
    used = pool_used(ctx)
    _pool_high(ctx, reset=True)
    rdf.write_csv(str(p), frame)
    high = _pool_high(ctx) - used
    size = p.stat().st_size
    assert size > 4 << 30
    assert high <= (2 * 64 + 16 + 2) << 20, high   # two text buffers, offsets, scan sums and the column table
    assert pool_used(ctx) == used
    h1 = hashlib.sha256(p.read_bytes()).hexdigest()
    rdf.write_csv(str(p), frame)
    assert hashlib.sha256(p.read_bytes()).hexdigest() == h1
    back = rdf.DeviceFrame.from_csv(str(p), schema=[rdf.I64, rdf.F64, rdf.F32, wo.BOOL], batch_size=1 << 22, ctx=ctx)
    for name, col in frame.items():
        gv, gm = _device_bits(back.column(name))
        wv, wm = _device_bits(col)
        assert np.array_equal(gm, wm), name
        u = f"u{wv.itemsize}"
        assert np.array_equal(gv[gm].view(u) if wv.dtype.kind == "f" else gv[gm], wv[wm].view(u) if wv.dtype.kind == "f" else wv[wm]), name
        del gv, gm, wv, wm
    del back
    os.unlink(p)


@pytest.mark.gpu
def test_errors_leak_nothing(rdf, ctx, tmp_path):
    N = rdf.native
    lib = N.lib()
    a = _upload(rdf, ctx, 2, np.arange(10, dtype=np.int32), None, [4, 6])
    b = _upload(rdf, ctx, 2, np.arange(10, dtype=np.int32), None, [5, 5])
    names = (C.c_char_p * 2)(b"a", b"b")
    ctx.synchronize()
    before = pool_used(ctx)

    def call(path, k, cols, ctxh=ctx.handle):
        return lib.bdf_csv_write(ctxh, str(path).encode(), k, names, (C.c_void_p * 2)(*[c.handle for c in cols]), None)

    assert call("/nonexistent-dir/x.csv", 1, [a]) == N.INVALID
    assert "nonexistent" in lib.bdf_last_error().decode()
    assert call(tmp_path / "m.csv", 2, [a, b]) == N.LENGTH_MISMATCH
    assert call(tmp_path / "e.csv", 0, [a]) == N.INVALID
    fleet = N.Context.multi(1)
    try:
        assert call(tmp_path / "f.csv", 1, [a], fleet.handle) == N.UNSUPPORTED
    finally:
        fleet.close()
    ctx.synchronize()
    assert pool_used(ctx) == before
    assert call(tmp_path / "ok.csv", 1, [a]) == N.OK
    assert (tmp_path / "ok.csv").read_bytes() == b"a\n" + b"".join(b"%d\n" % i for i in range(10))
