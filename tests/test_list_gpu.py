"""List columns on the GPU: every function against tests/list_oracle.py, bit for bit."""
import json
import math
import os

import numpy as np
import pyarrow as pa
import pytest

import list_oracle as lo
from helpers import pool_used


def _pool_attr(ctx, attr, value=None):
    import ctypes as C
    cu = C.CDLL("libcuda.so.1")
    dev, pool, v = C.c_int(), C.c_void_p(), C.c_uint64(0 if value is None else value)
    assert cu.cuInit(0) == 0 and cu.cuDeviceGet(C.byref(dev), ctx.device) == 0
    assert cu.cuDeviceGetDefaultMemPool(C.byref(pool), dev) == 0
    if value is None:
        assert cu.cuMemPoolGetAttribute(pool, attr, C.byref(v)) == 0
    else:
        assert cu.cuMemPoolSetAttribute(pool, attr, C.byref(v)) == 0
    return v.value


def reset_pool_peak(ctx):
    _pool_attr(ctx, 8, 0)   # CU_MEMPOOL_ATTR_USED_MEM_HIGH: reset to the current use


def pool_peak(ctx) -> int:
    return _pool_attr(ctx, 8)

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "array_functions.json")))
NP = [np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64, np.float32, np.float64]
PA = [pa.int8(), pa.int16(), pa.int32(), pa.int64(), pa.uint8(), pa.uint16(), pa.uint32(), pa.uint64(), pa.float32(), pa.float64()]


def bits(x, dt):
    if x is None:
        return None
    a = np.array([x], dtype=NP[dt])
    if dt >= 8 and math.isnan(float(a[0])):
        a = np.array([np.nan], dtype=NP[dt])
    return int(a.view(f"u{a.itemsize}")[0])


def lists_bits(lists, dt):
    return [None if l is None else [bits(x, dt) for x in l] for l in lists]


def make_chunk(rng, dt, n, spans=True, sliced=False, min_len=0):
    """A pyarrow ListArray of n lists: null lists (some spanning elements), empty lists, null elements, NaN / +-0.0.  sliced: the
    list array is a slice (list offset != 0) and so is its child (child offset != 0)."""
    is_f = dt >= 8
    lens = rng.integers(min_len, 9, n)
    total = int(lens.sum())
    if is_f:
        pool = np.array([0.0, -0.0, np.nan, 1.5, -2.0, 3.0, 2.0], dtype=NP[dt])
        vals = pool[rng.integers(0, len(pool), total)]
    else:
        vals = rng.integers(0, 6, total).astype(NP[dt])
    emask = rng.random(total) < 0.15
    child = pa.array(vals, type=PA[dt], mask=emask)
    if sliced:   # the same elements behind a child offset of 2
        pad = np.zeros(2, dtype=NP[dt])
        child = pa.array(np.concatenate([pad, vals, pad]), type=PA[dt], mask=np.concatenate([[True, False], emask, [False, True]])).slice(2, total)
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    lvalid = rng.random(n) >= 0.1
    if not spans:   # null lists without elements
        lens[~lvalid] = 0
        return make_from(lens, lvalid, vals, emask, dt)
    arr = pa.ListArray.from_buffers(pa.list_(PA[dt]), n, [pa.py_buffer(np.packbits(lvalid, bitorder="little")), pa.py_buffer(offsets)],
                                    null_count=int((~lvalid).sum()), children=[child]) if hasattr(pa.ListArray, "from_buffers") else \
        pa.Array.from_buffers(pa.list_(PA[dt]), n, [pa.py_buffer(np.packbits(lvalid, bitorder="little")), pa.py_buffer(offsets)],
                              null_count=int((~lvalid).sum()), children=[child])
    if sliced and n >= 10:
        arr = arr.slice(3, n - 5)
    return arr


def make_from(lens, lvalid, vals, emask, dt):
    lists, k = [], 0
    for ln, v in zip(lens, lvalid):
        items = [None if emask[k + i] else vals[k + i] for i in range(ln)]
        k += ln
        lists.append(items if v else None)
    return pa.array(lists, pa.list_(PA[dt]))


def to_lists(arr):
    return [None if x is None else [y for y in x] for x in arr.to_pylist()]


def upload(rdf, ctx, arrays):
    return rdf.ListColumn.upload([rdf.ListArray.from_arrow(a) for a in arrays], ctx)


def down_lists(lc):
    out = []
    for ch in lc.download():
        out.extend(ch.to_pylist())
    return out


def down_col(col):
    out = []
    for ch in col.download():
        m = ch.valid_mask()
        if hasattr(ch, "value_bits"):
            vb = ch.value_bits()
            out.extend(bool(vb[i]) if m[i] else None for i in range(len(m)))
        else:
            vs = ch.value_slice()
            out.extend(vs[i] if m[i] else None for i in range(len(m)))
    return out


@pytest.mark.parametrize("dt", range(10))
@pytest.mark.parametrize("shape", ["chunks", "sliced", "no_span"])
def test_every_function_against_the_oracle(rdf, ctx, dt, shape):
    rng = np.random.default_rng(dt * 7 + len(shape))
    mk = lambda m=0: [make_chunk(rng, dt, n, spans=shape != "no_span", sliced=shape == "sliced", min_len=m) for n in (40, 0, 300, 1)]
    A, B, M = mk(), mk(), mk(1)
    la, lb = sum((to_lists(a) for a in A), []), sum((to_lists(b) for b in B), [])
    ca, cb = upload(rdf, ctx, A), upload(rdf, ctx, B)
    # the search value's key is computed on the host: 0.0, -0.0 and NaN exercise its float rules
    for v in ([NP[dt](2), NP[dt](0), NP[dt](-0.0), NP[dt](np.nan)] if dt >= 8 else [NP[dt](2), NP[dt](0)]):
        assert down_col(ca.array_contains(v)) == [lo.array_contains(l, v) for l in la]
        assert [int(x) for x in down_col(ca.array_position(v))] == [lo.array_position(l, v) for l in la]
        assert lists_bits(down_lists(ca.array_remove(v)), dt) == lists_bits([lo.array_remove(l, v) for l in la], dt)
    assert [int(x) for x in down_col(ca.size())] == [lo.size(l) for l in la]
    # max / min over the same chunk shapes without a valid empty list (that one is ReferencePanic, test_pool_and_errors)
    lm = sum((to_lists(m) for m in M), [])
    cm = upload(rdf, ctx, M)
    assert [bits(x, dt) for x in down_col(cm.array_max())] == [bits(lo.array_max(l), dt) for l in lm]
    assert [bits(x, dt) for x in down_col(cm.array_min())] == [bits(lo.array_min(l), dt) for l in lm]
    assert lists_bits(down_lists(ca.array_sort()), dt) == lists_bits([lo.array_sort(l) for l in la], dt)
    assert lists_bits(down_lists(ca.array_distinct()), dt) == lists_bits([lo.array_distinct(l) for l in la], dt)
    for k in (0, 1, 3):
        assert lists_bits(down_lists(ca.array_repeat(k)), dt) == lists_bits([lo.array_repeat(l, k) for l in la], dt)
    assert lists_bits(down_lists(ca.array_except(cb)), dt) == lists_bits([lo.array_except(a, b) for a, b in zip(la, lb)], dt)
    assert lists_bits(down_lists(ca.array_intersect(cb)), dt) == lists_bits([lo.array_intersect(a, b) for a, b in zip(la, lb)], dt)
    assert lists_bits(down_lists(ca.array_union(cb)), dt) == lists_bits([lo.array_union(a, b) for a, b in zip(la, lb)], dt)
    rows, vals = ca.explode()
    wr, wv = lo.explode(la)
    assert [int(x) for x in down_col(rows)] == wr
    assert [bits(x, dt) for x in down_col(vals)] == [bits(x, dt) for x in wv]
    assert lists_bits(down_lists(ca), dt) == lists_bits(la, dt)   # download of the uploaded list


def test_the_reference_tests_through_the_device(rdf, ctx):
    v, o = GOLDEN["values"], GOLDEN["offsets"]
    def col(dt):
        return rdf.ListColumn.upload([rdf.ListArray(dt, np.array(o, np.int32), None, 0, len(o) - 1, 0,
                                                    rdf.PrimitiveArray.from_numpy(np.array(v, dtype=NP[dt])))], ctx)
    for dt in (rdf.I32, rdf.I64, rdf.F64):
        assert down_col(col(dt).array_contains(NP[dt](2))) == GOLDEN["contains"]["expected"]
    c = col(rdf.I64)
    assert [int(x) for x in down_col(c.array_position(2))] == GOLDEN["position"]["expected"]
    r = c.array_remove(2).download()[0]
    assert len(r) == 6 and len(r.values) == GOLDEN["remove"]["values_len"] and list(r.offsets[:-1]) == GOLDEN["remove"]["offsets"]
    s = c.array_sort().download()[0]
    assert len(s) == 6 and list(s.offsets[:-1]) == GOLDEN["sort"]["offsets"]
    assert list(s.values.value_slice()) == GOLDEN["sort"]["values"]


def test_hot_list(rdf, ctx):
    """One list of 1e7 elements among 1e7 one-element lists: the long-list search, the fold's big-group path, the sort."""
    rng = np.random.default_rng(3)
    hot = 10_000_000
    n_small = 10_000_000
    vals = rng.integers(0, 1000, hot + n_small).astype(np.int64)
    vals[hot - 5] = 77777
    offsets = np.concatenate([[0], [hot], hot + np.arange(1, n_small + 1)]).astype(np.int32)
    a = rdf.ListArray(rdf.I64, offsets, None, 0, n_small + 1, 0, rdf.PrimitiveArray.from_numpy(vals))
    c = rdf.ListColumn.upload([a], ctx)
    pos = c.array_position(77777).download()[0].value_slice()
    assert pos[0] == hot - 4 and np.array_equal(pos[1:], (vals[hot:] == 77777).astype(np.int32))
    con = down_col(c.array_contains(77777))
    assert con[0] is True
    mx = c.array_max().download()[0].value_slice()
    assert mx[0] == vals[:hot].max() and np.array_equal(mx[1:], vals[hot:])
    s = c.array_sort().download()[0]
    assert np.array_equal(s.values.value_slice()[:hot], np.sort(vals[:hot], kind="stable")) and np.array_equal(s.values.value_slice()[hot:], vals[hot:])
    d = c.array_distinct().download()[0]
    _, first = np.unique(vals[:hot], return_index=True)
    assert np.array_equal(d.values.value_slice()[:len(first)], vals[:hot][np.sort(first)])
    r = c.array_repeat(2).download()[0]
    assert np.array_equal(r.values.value_slice()[:2 * hot], np.tile(vals[:hot], 2))


def test_large_int64_column(rdf, ctx):
    """1e8 Int64 elements in 25 chunks of lists of mean length 32 through contains, sort and explode."""
    n_chunks, per = 25, 4_000_000
    rng = np.random.default_rng(11)
    chunks = []
    for k in range(n_chunks):
        lens = rng.integers(0, 65, per // 32)
        lens[-1] += per - lens.sum()
        lens = np.maximum(lens, 0)
        off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
        vals = rng.integers(-1000, 1000, int(off[-1])).astype(np.int64)
        chunks.append(rdf.ListArray(rdf.I64, off, None, 0, len(lens), 0, rdf.PrimitiveArray.from_numpy(vals)))
    ctx.synchronize()
    base = pool_used(ctx)
    reset_pool_peak(ctx)
    c = rdf.ListColumn.upload(chunks, ctx)
    E = sum(len(ch.values) for ch in chunks)
    con = c.array_contains(5).download()
    for ch, got in zip(chunks, con):   # every list: a count of matches per list from a cumulative sum
        cs = np.concatenate([[0], np.cumsum(ch.values.values == 5)])
        assert np.array_equal(got.value_bits()[:len(ch)].astype(bool), (cs[ch.offsets[1:]] - cs[ch.offsets[:-1]]) > 0)
    k0 = chunks[0]
    s = c.array_sort()
    got = s.download()[0]
    n0 = len(k0.values)
    parent0 = np.repeat(np.arange(len(k0)), np.diff(k0.offsets))
    assert np.array_equal(got.offsets[:len(k0) + 1], k0.offsets)
    assert np.array_equal(got.values.value_slice()[:n0], k0.values.values[np.lexsort((k0.values.values, parent0))])
    s.free()
    rows, vals = c.explode()
    assert len(vals) == sum(len(ch.values) for ch in chunks)
    assert np.array_equal(vals.download()[0].value_slice()[:n0], chunks[0].values.values)
    assert np.array_equal(rows.download()[0].value_slice()[:n0], parent0)
    # bounded device memory: the elements and every temporary of the sort stay under 64 bytes per element
    assert pool_peak(ctx) - base < 64 * E


def test_ipc_read_of_list_columns(rdf, ctx, tmp_path):
    rng = np.random.default_rng(4)
    batches = [pa.record_batch([make_chunk(rng, 3, n), make_chunk(rng, 9, n)], names=["a", "b"]) for n in (10, 0, 77)]
    path = str(tmp_path / "l.arrow")
    with pa.OSFile(path, "wb") as sink, pa.ipc.new_file(sink, batches[0].schema) as w:
        for b in batches:
            w.write_batch(b)
    with rdf.IpcFile(path) as f:
        cols = f.read(["a", "b"], ctx=ctx)
        for name, dt in (("a", 3), ("b", 9)):
            want = sum((to_lists(b.column(name)) for b in batches), [])
            assert lists_bits(down_lists(cols[name]), dt) == lists_bits(want, dt)


def test_pool_and_errors(rdf, ctx):
    N = rdf.native
    a = rdf.ListColumn.upload([rdf.ListArray.from_pylist(rdf.I32, [[1, 2], [], None])], ctx)
    b = rdf.ListColumn.upload([rdf.ListArray.from_pylist(rdf.I32, [[1], [2]])], ctx)
    f = rdf.ListColumn.upload([rdf.ListArray.from_pylist(rdf.F64, [[1.0], [2.0], [3.0]])], ctx)
    ctx.synchronize()
    before = pool_used(ctx)
    with pytest.raises(rdf.ComputeError):
        a.array_union(b)
    with pytest.raises(rdf.UnsupportedType):
        a.array_union(f)
    with pytest.raises(rdf.ComputeError):
        a.array_repeat(-1)
    with pytest.raises(rdf.ReferencePanic):
        a.array_max()
    with pytest.raises(rdf.UnsupportedType):
        rdf.ListColumn.upload([rdf.ListArray.from_pylist(rdf.I32, [[1]])], ctx, dtype=N.BOOL)
    r = a.array_sort()
    r.free()
    ctx.synchronize()
    assert pool_used(ctx) == before
    fleet = rdf.Context.multi(1)
    with pytest.raises(rdf.UnsupportedType):
        rdf.ListColumn.upload([rdf.ListArray.from_pylist(rdf.I32, [[1]])], fleet)
    fleet.close()
