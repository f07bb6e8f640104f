"""DataFrame::to_json on the device: every file byte for byte against tests/json_write_oracle.py (every dtype, nulls, sliced chunks,
escaped names, temporal kinds at their range ends, list columns up to one list longer than a text buffer), round trips through the
library's own reader, the refusals, and a 1e8-row write in bounded memory."""
import ctypes as C
import hashlib
import os
import shutil
from collections import OrderedDict

import numpy as np
import pytest

import json_write_oracle as wo
from helpers import pool_used

NP = {0: np.int8, 1: np.int16, 2: np.int32, 3: np.int64, 4: np.uint8, 5: np.uint16, 6: np.uint32, 7: np.uint64, 8: np.float32, 9: np.float64}
DTYPES = list(range(11))


def _values(rng, dt, n):
    if dt == wo.BOOL:
        return rng.random(n) < 0.5
    if dt == 8:
        v = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32).view(np.float32)
        v[::97] = np.array([np.nan, np.inf, -np.inf, 1e13, 1e12, 1e-6, 1e-7, -0.0], np.float32)[np.arange(len(v[::97])) % 8]
        return v
    if dt == 9:
        v = rng.integers(0, 2 ** 64, n, dtype=np.uint64).view(np.float64)
        v[::89] = np.array([np.nan, np.inf, -np.inf, 1e16, 1e15, 1e-5, 1e-4, -0.0, 5e-324, 1.0])[np.arange(len(v[::89])) % 10]
        return v
    info = np.iinfo(NP[dt])
    v = rng.integers(info.min, info.max, n, dtype=NP[dt], endpoint=True)
    v[:2] = [info.min, info.max][:len(v[:2])]
    return v


def _upload(rdf, ctx, dt, vals, valid, lens=None, temporal=None):
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
    col = rdf.Column.upload(chunks, ctx=ctx, dtype=dt)
    if temporal is not None:
        col.temporal = rdf.TemporalType(*temporal)
    return col


def _upload_list(rdf, ctx, dt, rows, lens=None):
    lens = [len(rows)] if lens is None else lens
    chunks, s = [], 0
    for n in lens:
        chunks.append(rdf.ListArray.from_pylist(dt, rows[s:s + n]))
        s += n
    return rdf.ListColumn.upload(chunks, ctx=ctx, dtype=dt)


def _device(rdf, ctx, cols, lens=None):
    dev = OrderedDict()
    for c in cols:
        if c.get("lists") is not None:
            dev[c["name"]] = _upload_list(rdf, ctx, c["dtype"], c["lists"], lens)
        else:
            dev[c["name"]] = _upload(rdf, ctx, c["dtype"], c["values"], c.get("valid"), lens, c.get("temporal"))
    return dev


def _compare(got, want):
    if got != want:
        gl, wl = got.split(b"\n"), want.split(b"\n")
        bad = [i for i in range(min(len(gl), len(wl))) if gl[i] != wl[i]][:5]
        raise AssertionError(f"{len(got)} vs {len(want)} bytes; first differing lines {[(i, gl[i][:160], wl[i][:160]) for i in bad]}")


def _write_and_compare(rdf, ctx, tmp_path, cols, lens=None, explicit_nulls=False, want=None):
    dev = _device(rdf, ctx, cols, lens)
    p = tmp_path / "w.json"
    rdf.write_json(str(p), dev, explicit_nulls=explicit_nulls)
    _compare(p.read_bytes(), wo.write(cols, explicit_nulls) if want is None else want)
    return dev, p


@pytest.mark.gpu
@pytest.mark.parametrize("explicit", [False, True])
@pytest.mark.parametrize("nullable", [False, True])
@pytest.mark.parametrize("dt", DTYPES)
def test_every_dtype_in_sliced_chunks(rdf, ctx, tmp_path, dt, nullable, explicit):
    rng = np.random.default_rng(100 + dt)
    n = 6000
    vals = _values(rng, dt, n)
    valid = rng.random(n) >= 0.2 if nullable else None
    lens = [1000, 1, 2500, 7, 1492, 1000]
    cols = [{"name": "v", "dtype": dt, "values": vals, "valid": valid}, {"name": "k", "dtype": 2, "values": np.arange(n, dtype=np.int32)}]
    _write_and_compare(rdf, ctx, tmp_path, cols, lens, explicit)
    _write_and_compare(rdf, ctx, tmp_path, cols[:1], lens, explicit)   # alone: a NULL row is {}


@pytest.mark.gpu
def test_many_uneven_chunks_and_tiny_frames(rdf, ctx, tmp_path):
    rng = np.random.default_rng(7)
    lens = [int(x) for x in rng.integers(0, 40, 300)] + [0, 0, 5000, 0]
    n = sum(lens)
    cols = [{"name": "a", "dtype": 3, "values": _values(rng, 3, n), "valid": rng.random(n) > 0.3},
            {"name": "b", "dtype": 9, "values": _values(rng, 9, n)},
            {"name": "l", "dtype": 6, "lists": [None if rng.random() < 0.2 else [int(x) for x in rng.integers(0, 9, rng.integers(0, 4))] for _ in range(n)]}]
    _write_and_compare(rdf, ctx, tmp_path, cols, lens)
    _write_and_compare(rdf, ctx, tmp_path, cols, lens, explicit_nulls=True)
    for m in (0, 1):
        small = [dict(c, values=c["values"][:m], valid=None if c.get("valid") is None else c["valid"][:m]) if "values" in c else dict(c, lists=c["lists"][:m])
                 for c in cols]
        _, p = _write_and_compare(rdf, ctx, tmp_path, small, [m])
        assert (p.stat().st_size == 0) == (m == 0)


@pytest.mark.gpu
def test_names_that_need_escapes(rdf, ctx, tmp_path):
    names = ['q"uote', "back\\slash", "tab\tnl\nbs\bff\fcr\r", "\x01\x1f", "é ü", ""]
    cols = [{"name": nm, "dtype": 2, "values": np.arange(50, dtype=np.int32) * (i + 1)} for i, nm in enumerate(names)]
    _write_and_compare(rdf, ctx, tmp_path, cols, [20, 30])


@pytest.mark.gpu
def test_every_temporal_kind_unit_and_tz_at_the_range_ends(rdf, ctx, tmp_path):
    rng = np.random.default_rng(21)
    cols = []
    n = 4000
    for kind, unit, tz in [(wo.DATE32, 0, None), (wo.DATE64, 1, None), (wo.TIME32, 0, None), (wo.TIME32, 1, None), (wo.TIME64, 2, None),
                           (wo.TIME64, 3, None)] + [(wo.TIMESTAMP, u, tz) for u in range(4) for tz in (None, "UTC", "+00:00", "+05:30", "-23:59")]:
        ups = 1000 if kind == wo.DATE64 else wo.PER_SEC[unit]
        off = wo.tz_suffix(tz)[0] * ups if kind == wo.TIMESTAMP else 0
        if kind in (wo.TIME32, wo.TIME64):
            lo, hi = 0, 86400 * ups - 1
        elif kind == wo.DATE32:
            lo, hi = wo.MIN_DAY, wo.MAX_DAY
        else:   # the local day of every value in chrono's range, and inside Int64
            lo = max(wo.MIN_DAY * 86400 * ups - off, -2 ** 63)
            hi = min((wo.MAX_DAY + 1) * 86400 * ups - 1 - off, 2 ** 63 - 1)
        dt = 2 if kind in (wo.DATE32, wo.TIME32) else 3
        v = rng.integers(lo, hi, n, dtype=np.int64, endpoint=True)
        v[:4] = [lo, hi, 0, -1 if lo < 0 else 1]
        cols.append({"name": f"t{len(cols)}", "dtype": dt, "values": v.astype(NP[dt]), "valid": rng.random(n) > 0.1, "temporal": (kind, unit, tz)})
    _write_and_compare(rdf, ctx, tmp_path, cols, [1000, 3, 2997])
    _write_and_compare(rdf, ctx, tmp_path, cols, [4000], explicit_nulls=True)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", list(range(10)))
def test_list_columns(rdf, ctx, tmp_path, dt):
    rng = np.random.default_rng(50 + dt)
    n = 3000
    pool = _values(rng, dt, 20000)
    rows, k = [], 0
    for _ in range(n):
        r = rng.random()
        if r < 0.1:
            rows.append(None)
        elif r < 0.2:
            rows.append([])
        else:
            m = int(rng.integers(1, 8))
            rows.append([None if rng.random() < 0.15 else pool[(k + i) % len(pool)].item() for i in range(m)])
            k += m
    cols = [{"name": "l", "dtype": dt, "lists": rows}, {"name": "x", "dtype": 2, "values": np.arange(n, dtype=np.int32), "valid": rng.random(n) > 0.5}]
    _write_and_compare(rdf, ctx, tmp_path, cols, [1000, 0, 1, 1999])
    _write_and_compare(rdf, ctx, tmp_path, cols, [3000], explicit_nulls=True)


@pytest.mark.gpu
def test_a_hot_list_beside_a_million_one_element_lists(rdf, ctx, tmp_path):
    rng = np.random.default_rng(61)
    n = 1_000_000
    rows = [[int(x)] for x in rng.integers(-1000, 1000, n)]
    rows[n // 2] = [int(x) for x in rng.integers(-10 ** 9, 10 ** 9, 3_000_000)]
    cols = [{"name": "l", "dtype": 3, "lists": rows}, {"name": "i", "dtype": 2, "values": np.arange(n, dtype=np.int32)}]
    _write_and_compare(rdf, ctx, tmp_path, cols, [n // 3, n - n // 3])


@pytest.mark.gpu
def test_one_list_longer_than_a_text_buffer(rdf, ctx, tmp_path):
    rng = np.random.default_rng(62)
    big = rng.normal(size=12_000_000) * 1e3
    rows = [[1.5], big.tolist(), [], None, [2.0]]
    dev = OrderedDict([("l", _upload_list(rdf, ctx, 9, rows)), ("i", _upload(rdf, ctx, 2, np.arange(5, dtype=np.int32), None))])
    p = tmp_path / "big.json"
    rdf.write_json(str(p), dev)
    want = (b'{"l":[1.5],"i":0}\n{"l":[' + ",".join(wo.format_f64_repr(x) for x in big.tolist()).encode() + b'],"i":1}\n'
            b'{"l":[],"i":2}\n{"i":3}\n{"l":[2.0],"i":4}\n')
    assert len(want) > 64 << 20
    _compare(p.read_bytes(), want)


@pytest.mark.gpu
@pytest.mark.parametrize("m", [4_000_000, 12_000_000])
def test_consecutive_lists_longer_than_a_text_buffer(rdf, ctx, tmp_path, m):
    """Three adjacent rows whose text each outgrows a text buffer, then short ones.  With 4e6 elements the first two share a window
    (2^23 elements) and the third starts the next; with 1.2e7 each row is a window of its own.  Each row holds the same values in a
    different rotation, so text left over from another row cannot match."""
    rng = np.random.default_rng(63)
    pool = rng.normal(size=100_003) * 1e3
    strs = [wo.format_f64_repr(x) for x in pool.tolist()]
    shifts = [0, 33_331, 66_662]
    vals = np.concatenate([np.roll(pool, -sh)[np.arange(m) % len(pool)] for sh in shifts] + [np.array([1.5, 2.5])])
    offs = np.array([0, m, 2 * m, 3 * m, 3 * m + 1, 3 * m + 2], np.int32)
    lst = rdf.ListColumn.upload([rdf.ListArray(9, offs, None, 0, 5, 0, rdf.PrimitiveArray.from_numpy(vals))], ctx=ctx, dtype=9)
    dev = OrderedDict([("l", lst), ("i", _upload(rdf, ctx, 2, np.arange(5, dtype=np.int32), None))])
    p = tmp_path / "long.json"
    rdf.write_json(str(p), dev)
    want = []
    for r, sh in enumerate(shifts):
        rot = strs[sh:] + strs[:sh]
        body = ",".join((rot * (m // len(rot) + 1))[:m]).encode()
        assert len(body) > 64 << 20
        want.append(b'{"l":[' + body + b'],"i":%d}\n' % r)
    want.append(b'{"l":[1.5],"i":3}\n{"l":[2.5],"i":4}\n')
    _compare(p.read_bytes(), b"".join(want))


@pytest.mark.gpu
def test_round_trip_through_the_reader(rdf, ctx, tmp_path):
    rng = np.random.default_rng(70)
    n = 5000
    cols, schema = [], []
    for dt in DTYPES:
        cols.append({"name": f"c{dt}", "dtype": dt, "values": _values(rng, dt, n), "valid": rng.random(n) > 0.2})
        schema.append((f"c{dt}", dt))
    rows = [None if rng.random() < 0.1 else [None if rng.random() < 0.1 else float(x) for x in rng.normal(size=rng.integers(0, 5))] for _ in range(n)]
    cols.append({"name": "l", "dtype": 9, "lists": rows})
    schema.append(("l", rdf.native.LIST_BASE + 9))
    dev, p = _write_and_compare(rdf, ctx, tmp_path, cols, [2000, 3000])
    with rdf.JsonFile(str(p), schema=schema, batch_size=1000) as f:
        back = f.read([f"c{dt}" for dt in DTYPES])
        lst = f.read_list("l")
    for c in cols[:-1]:
        got = [x for a in back[c["name"]].download() for x in a.to_pylist()]
        v, m = c["values"], c["valid"]
        fin = np.isfinite(v) if c["dtype"] in (8, 9) else np.ones(n, bool)
        for r in range(n):
            if not m[r] or not fin[r]:
                assert got[r] is None, (c["name"], r)   # NaN and infinities come back NULL, as documented
            elif c["dtype"] in (8, 9):
                assert np.array([got[r]], NP[c["dtype"]]).view(f"u{v.itemsize}")[0] == v[r:r + 1].view(f"u{v.itemsize}")[0]
            else:
                assert got[r] == v[r].item(), (c["name"], r)
    got_rows = [x for a in lst.download() for x in a.to_pylist()]
    assert got_rows == rows


@pytest.mark.gpu
def test_integral_float64_reads_back_as_float64_under_inference(rdf, ctx, tmp_path):
    col = _upload(rdf, ctx, 9, np.array([1.0, 2.0, -3.0, 0.0]), None)
    p = tmp_path / "f.json"
    rdf.DeviceFrame(OrderedDict([("x", col)])).to_json(str(p))
    assert p.read_bytes() == b'{"x":1.0}\n{"x":2.0}\n{"x":-3.0}\n{"x":0.0}\n'
    back = rdf.DeviceFrame.from_json(str(p))
    assert back.schema["x"] == 9


@pytest.mark.gpu
def test_frame_to_json_writes_every_column_kind(rdf, ctx, tmp_path):
    rng = np.random.default_rng(80)
    n = 1000
    cols = [{"name": "i", "dtype": 3, "values": _values(rng, 3, n)},
            {"name": "t", "dtype": 3, "values": rng.integers(0, 2 * 10 ** 12, n), "temporal": (wo.TIMESTAMP, 1, "+05:30")},
            {"name": "b", "dtype": wo.BOOL, "values": rng.random(n) < 0.5},
            {"name": "l", "dtype": 8, "lists": [[float(np.float32(x)) for x in rng.normal(size=3)] for _ in range(n)]}]
    dev = _device(rdf, ctx, cols)
    p = tmp_path / "fr.json"
    rdf.DeviceFrame(dev).to_json(str(p), explicit_nulls=True)
    _compare(p.read_bytes(), wo.write(cols, True))


@pytest.mark.gpu
def test_refusals_write_nothing_and_leak_nothing(rdf, ctx, tmp_path):
    N = rdf.native
    lib = N.lib()
    a = _upload(rdf, ctx, 2, np.arange(10, dtype=np.int32), None, [4, 6])
    b = _upload(rdf, ctx, 2, np.arange(10, dtype=np.int32), None, [5, 5])
    ts = _upload(rdf, ctx, 3, np.arange(10, dtype=np.int64), None, [4, 6])
    bad_day = _upload(rdf, ctx, 2, np.array([0, wo.MAX_DAY + 1] + [0] * 8, np.int32), None, [4, 6])
    bad_tod = _upload(rdf, ctx, 3, np.array([0, -1] + [0] * 8, np.int64), None, [4, 6])
    lst = _upload_list(rdf, ctx, 3, [[1]] * 10, [4, 6])
    names = (C.c_char_p * 2)(b"a", b"b")
    ctx.synchronize()
    before = pool_used(ctx)

    def call(path, k, cols, types=None, lists=None, ctxh=ctx.handle):
        hs = (C.c_void_p * 2)(*[c.handle if c is not None else None for c in cols] + [None] * (2 - len(cols)))
        ts_ = None if types is None else (N.TemporalTypeC * 2)(*[N.TemporalTypeC(t[0], t[1], t[2]) for t in types] + [N.TemporalTypeC(0, 0, None)] * (2 - len(types)))
        ls = None if lists is None else (C.c_void_p * 2)(*[l.handle if l is not None else None for l in lists] + [None] * (2 - len(lists)))
        return lib.bdf_json_write(ctxh, str(path).encode(), k, names, hs, ts_, ls, None)

    cases = [
        (tmp_path / "a.json", 1, [ts], [(wo.TIMESTAMP, 0, b"Europe/Paris")], None, N.UNSUPPORTED),
        (tmp_path / "b.json", 1, [bad_day], [(wo.DATE32, 0, None)], None, N.INVALID),
        (tmp_path / "c.json", 1, [bad_tod], [(wo.TIME64, 2, None)], None, N.INVALID),
        (tmp_path / "d.json", 2, [a, b], None, None, N.LENGTH_MISMATCH),
        (tmp_path / "e.json", 2, [a, a], None, None, N.OK),
        (tmp_path / "f.json", 1, [a], [(wo.TIMESTAMP, 0, None)], None, N.INVALID),            # Int32 is not a Timestamp
        (tmp_path / "g.json", 1, [a], None, [lst], N.INVALID),                                 # both a column and a list
        (tmp_path / "h.json", 0, [a], None, None, N.INVALID),
        (tmp_path / "no" / "such" / "dir.json", 1, [a], None, None, N.INVALID),
    ]
    for path, k, cols, types, lists, want in cases:
        st = call(path, k, cols, types, lists)
        assert st == want, (path, st, lib.bdf_last_error())
        if want != N.OK:
            assert not os.path.exists(path), path
            if path.name == "dir.json":
                assert b"No such file" in lib.bdf_last_error()
    assert call(tmp_path / "b.json", 1, [bad_day], [(wo.DATE32, 0, None)]) == N.INVALID and b"95026602" in lib.bdf_last_error()
    assert call(tmp_path / "i.json", 1, [None], None, [lst]) == N.OK
    ctx.synchronize()
    assert pool_used(ctx) == before
    fleet = N.Context.multi(1)
    try:
        assert call(tmp_path / "m.json", 1, [a], ctxh=fleet.handle) == N.UNSUPPORTED
        assert not os.path.exists(tmp_path / "m.json")
    finally:
        fleet.close()


def _pool_high(ctx, reset=False):
    cu = C.CDLL("libcuda.so.1")
    dev, pool, v = C.c_int(), C.c_void_p(), C.c_uint64(0)
    assert cu.cuDeviceGet(C.byref(dev), ctx.device) == 0 and cu.cuDeviceGetDefaultMemPool(C.byref(pool), dev) == 0
    if reset:
        assert cu.cuMemPoolSetAttribute(pool, 8, C.byref(v)) == 0   # CU_MEMPOOL_ATTR_USED_MEM_HIGH
        return 0
    assert cu.cuMemPoolGetAttribute(pool, 8, C.byref(v)) == 0
    return v.value


def _bits(col):
    out = []
    for a in col.download():
        m = a.valid_mask()
        v = np.asarray(a.value_bits()) if hasattr(a, "value_bits") else np.asarray(a.value_slice())
        out.append((v, m))
    return np.concatenate([v for v, _ in out]), np.concatenate([m for _, m in out])


@pytest.mark.gpu
def test_full_size_write_in_bounded_memory(rdf, ctx, tmp_path):
    n = 100_000_000
    if shutil.disk_usage(str(tmp_path)).free < 48 << 30:
        pytest.skip("needs 48 GB of free disk for a 20 GB file")
    lens = [n // 4] * 4
    i64 = rdf.Column.generate(rdf.I64, lens, kind=3, col_id=1, null_mod=10, ctx=ctx)
    f64 = rdf.Column.generate(rdf.F64, lens, kind=0, lo=-1e3, hi=1e3, col_id=2, null_mod=10, ctx=ctx)
    f32 = rdf.Column.generate(rdf.F32, lens, kind=0, lo=-1.0, hi=1.0, col_id=3, null_mod=10, ctx=ctx)
    b = rdf.Column.generate(rdf.F64, lens, kind=0, col_id=4, ctx=ctx).gt(0.5)
    ts = rdf.Column.generate(rdf.I64, lens, kind=0, lo=0, hi=2e12, col_id=5, ctx=ctx)
    ts.temporal = rdf.TemporalType(wo.TIMESTAMP, 1)
    # List<Float64> of mean length 4 (0..8 elements per row), in chunks aligned with the columns' chunks
    rng = np.random.default_rng(90)
    chunks = []
    for ln in lens:
        offs = np.concatenate([[0], np.cumsum(rng.integers(0, 9, ln))]).astype(np.int32)
        vals = rdf.PrimitiveArray.from_numpy(rng.uniform(-1e6, 1e6, int(offs[-1])), None)
        chunks.append(rdf.ListArray(9, offs, None, 0, ln, 0, vals))
    lc = rdf.ListColumn.upload(chunks, ctx=ctx, dtype=9)
    del chunks, vals
    frame = OrderedDict([("i", i64), ("d", f64), ("f", f32), ("b", b), ("t", ts), ("l", lc)])
    p = tmp_path / "big.json"
    ctx.synchronize()
    used = pool_used(ctx)
    _pool_high(ctx, reset=True)
    rdf.write_json(str(p), frame)
    high = _pool_high(ctx) - used
    assert p.stat().st_size > 10 << 30
    # two text buffers, row and element offsets and scan sums, one list column's positions, the tables
    assert high <= (2 * 64 + 16 + 64 + 16 + 4) << 20, high
    assert pool_used(ctx) == used
    h1 = hashlib.sha256()
    with open(p, "rb") as fh:
        for blk in iter(lambda: fh.read(1 << 26), b""):
            h1.update(blk)
    rdf.write_json(str(p), frame)
    h2 = hashlib.sha256()
    with open(p, "rb") as fh:
        for blk in iter(lambda: fh.read(1 << 26), b""):
            h2.update(blk)
    assert h1.hexdigest() == h2.hexdigest()
    with rdf.JsonFile(str(p), schema=[("i", rdf.I64), ("d", rdf.F64), ("f", rdf.F32), ("b", wo.BOOL)], batch_size=1 << 22, ctx=ctx) as f:
        back = f.read(["i", "d", "f", "b"])
    for name in ("i", "d", "f", "b"):
        gv, gm = _bits(back[name])
        wv, wm = _bits(frame[name])
        assert np.array_equal(gm, wm), name
        if wv.dtype.kind == "f":
            u = f"u{wv.itemsize}"
            assert np.array_equal(gv[gm].view(u), wv[wm].view(u)), name
        else:
            assert np.array_equal(gv[gm], wv[wm]), name
        del gv, gm, wv, wm
    del back
    os.unlink(p)
