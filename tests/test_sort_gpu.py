"""DataFrame::sort on the device (bdf_sort_indices_dev + bdf_take_dev) against the oracle's restatement of
lexsort_to_indices / take (src/dataframe.rs:194-222, src/table.rs:218-241; pinned by the reference's test_sort vector
and pyarrow in tests/test_oracle_golden.py).  A stable sort has exactly one right answer: indices are compared
for EQUALITY, taken columns bit for bit."""
import numpy as np
import pytest

from helpers import assert_same_array, pool_used, random_mask

pytestmark = pytest.mark.gpu

RAGGED = [0, 1, 31, 2047, 2048, 2049, 0, 10_007, 70_001]


def make_key(rdf, rng, dtype, lens, null_frac, sliced, small_range=True, specials=False):
    npdt = np.dtype(rdf.NP_DTYPES[dtype])
    out = []
    for k, n in enumerate(lens):
        pad = (3 + 5 * k) % 23 if sliced else 0
        if npdt.kind == "f":
            v = (np.round(rng.normal(0, 3, n + pad + 2)) if small_range else rng.normal(0, 1e6, n + pad + 2)).astype(npdt)
            if specials and n > 64:
                v[pad:pad + 8] = [np.nan, -0.0, 0.0, np.inf, -np.inf, np.nan, 1.5, -1.5]
        else:
            info = np.iinfo(npdt)
            lo, hi = (max(info.min, -5), min(info.max, 5)) if small_range else (info.min, info.max)
            v = rng.integers(lo, hi, n + pad + 2, dtype=npdt, endpoint=True)
        a = rdf.PrimitiveArray.from_numpy(v, random_mask(rng, n + pad + 2, null_frac) if null_frac else None)
        a.null_count = -1 if a.validity is not None else 0
        out.append(a.slice(pad, n))
    return out


def check_sort(rdf, oracle, criteria_host, payload_host=()):
    """criteria_host: [(chunks, descending)]; returns the device index column after comparing it with the oracle's."""
    cols = [rdf.Column.upload(ch) for ch, _ in criteria_host]
    idx = rdf.sort_indices([(c, d) for c, (_, d) in zip(cols, criteria_host)])
    got = idx.download()
    assert len(got) == 1 and got[0].validity is None
    st, want = oracle.lexsort_indices(criteria_host)
    assert st == oracle.OK
    g = got[0].value_slice()
    bad = np.nonzero(g != want)[0]
    assert bad.size == 0, f"indices differ at {bad[:5]}: got {g[bad[:5]]}, want {want[bad[:5]]}"
    for chunks in list(ch for ch, _ in criteria_host) + list(payload_host):
        taken = rdf.Column.upload(chunks).take(idx).download()
        assert len(taken) == 1
        _, wt = oracle.take(chunks, want)
        assert_same_array(taken[0], wt, what="take by sort indices")
    return idx


def test_reference_sort_golden_on_gpu(rdf, ctx, oracle):
    """src/dataframe.rs:963-1002: a Int32 descending (one null), b UInt8 ascending."""
    a = [rdf.PrimitiveArray.from_pylist(rdf.I32, [1, 1, None, 3, 3, 4])]
    b = [rdf.PrimitiveArray.from_pylist(rdf.U8, [9, 5, 6, 7, 4, 8])]
    ca, cb = rdf.Column.upload(a), rdf.Column.upload(b)
    sa, sb = rdf.sort_columns([(ca, True), (cb, False)], [ca, cb])
    assert sa.download()[0].to_pylist() == [4, 3, 3, 1, 1, None]
    assert sb.download()[0].to_pylist() == [8, 4, 7, 5, 9, 6]
    with pytest.raises(rdf.ComputeError):
        rdf.sort_indices([])


@pytest.mark.parametrize("tname", ["I8", "I16", "I32", "I64", "U8", "U16", "U32", "U64", "F32", "F64"])
def test_single_key_every_type(rdf, ctx, oracle, tname):
    dtype = getattr(rdf, tname)
    rng = np.random.default_rng(100 + dtype)
    for null_frac, sliced, small, desc in ((0, False, True, False), (0.2, True, True, True), (0.1, True, False, False), (0.1, False, False, True)):
        key = make_key(rdf, rng, dtype, RAGGED, null_frac, sliced, small_range=small, specials=True)
        check_sort(rdf, oracle, [(key, desc)])


def test_multi_key_mixed_types_and_payload(rdf, ctx, oracle):
    rng = np.random.default_rng(5)
    lens = [5000, 0, 33, 120_000]
    k1 = make_key(rdf, rng, rdf.I8, lens, 0.1, True)
    k2 = make_key(rdf, rng, rdf.F64, lens, 0.2, True, specials=True)
    k3 = make_key(rdf, rng, rdf.U32, lens, 0.0, False)
    payload = make_key(rdf, rng, rdf.I64, lens, 0.3, True, small_range=False)
    flags = [rdf.BooleanArray.from_numpy(rng.random(n) > 0.5, rng.random(n) > 0.2) for n in lens]
    for desc in ((False, False, False), (True, False, True), (False, True, True)):
        idx = check_sort(rdf, oracle, [(k1, desc[0]), (k2, desc[1]), (k3, desc[2])], payload_host=[payload])
        # a boolean column rides along too (DataFrame::sort_by_indices takes EVERY column)
        tb = rdf.Column.upload(flags).take(idx).download()[0]
        _, want_idx = oracle.lexsort_indices([(k1, desc[0]), (k2, desc[1]), (k3, desc[2])])
        _, wb = oracle.take(flags, want_idx)
        assert np.array_equal(tb.valid_mask(), wb.valid_mask())
        assert np.array_equal(tb.value_bits()[wb.valid_mask()], wb.value_bits()[wb.valid_mask()])
    # criteria with differently chunked columns: the row space is the concatenation, not the chunking
    flat = [rdf.PrimitiveArray.from_numpy(np.concatenate([c.value_slice() for c in k3]))]
    i1 = rdf.sort_indices([(rdf.Column.upload(k1), False), (rdf.Column.upload(flat), True)]).download()[0].value_slice()
    _, w1 = oracle.lexsort_indices([(k1, False), (k3, True)])
    assert np.array_equal(i1, w1)


def test_take_rules(rdf, ctx, oracle):
    rng = np.random.default_rng(9)
    lens = [100, 0, 4000, 1]
    vals = make_key(rdf, rng, rdf.F32, lens, 0.2, True, small_range=False)
    total = sum(lens)
    cv = rdf.Column.upload(vals)
    # multi-chunk indices with nulls
    ix = [rng.integers(0, total, n).astype(np.uint32) for n in (0, 5, 3000, 64)]
    im = [rng.random(len(x)) > 0.25 for x in ix]
    ci = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(x, m) for x, m in zip(ix, im)])
    got = cv.take(ci).download()
    assert len(got) == 1
    _, want = oracle.take(vals, np.concatenate(ix), np.concatenate(im))
    assert_same_array(got[0], want, what="take with null indices")
    assert cv.take(ci).count() == want.length - want.null_count
    # no validity anywhere -> no validity on the result
    dense = [rdf.PrimitiveArray.from_numpy(np.arange(1000, dtype=np.int64))]
    out = rdf.Column.upload(dense).take(rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.array([999, 0, 5], np.uint32))])).download()[0]
    assert out.validity is None and out.value_slice().tolist() == [999, 0, 5]
    # index past the end: found by the kernel, after the output column was made, which is dropped again
    cd = rdf.Column.upload(dense)
    past_end = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.array([1000], np.uint32))])
    ctx.synchronize()
    before = pool_used(ctx)
    with pytest.raises(rdf.ArrowError, match="take: index out of bounds$"):
        cd.take(past_end)
    ctx.synchronize()
    assert pool_used(ctx) == before
    with pytest.raises(rdf.UnsupportedType):  # indices must be UInt32
        cv.take(rdf.Column.upload(dense))
    with pytest.raises(rdf.UnsupportedType):  # boolean sort criterion
        rdf.sort_indices([(rdf.Column.upload([rdf.BooleanArray.from_numpy(np.ones(4, bool))]), False)])
    with pytest.raises(rdf.ComputeError):     # criteria of different lengths
        rdf.sort_indices([(cv, False), (rdf.Column.upload(dense), False)])
    empty = rdf.sort_indices([(rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.zeros(0))]), False)]).download()
    assert empty[0].length == 0


def test_two_keys_1e7_against_oracle(rdf, ctx, oracle):
    """1e7 rows in 10 chunks: Int64 key with few distinct values (ties -> stability matters), then Float64 descending."""
    CH, NCH = 1_000_000, 10
    lens = [CH] * NCH
    k1 = rdf.Column.generate(rdf.F64, lens, 0, -100.0, 100.0, col_id=70, null_mod=10).cast(rdf.I8)   # ~200 distinct values, ~10 % nulls
    k2 = rdf.Column.generate(rdf.F64, lens, 0, -1e3, 1e3, col_id=71)
    idx = rdf.sort_indices([(k1, False), (k2, True)])
    h1, h2 = k1.download(), k2.download()
    st, want = oracle.lexsort_indices([(h1, False), (h2, True)])
    assert st == oracle.OK
    assert np.array_equal(idx.download()[0].value_slice(), want)
    t2 = k2.take(idx).download()[0]
    _, w2 = oracle.take(h2, want)
    assert_same_array(t2, w2, what="1e7 take")


def test_full_size_sort_1e8_properties(rdf, ctx):
    """1e8 Float64 rows (config-1 column): size-independent properties -- the result is a permutation, the taken
    column is non-decreasing, and equal neighbours keep their original order (stability)."""
    lens = [4_000_000] * 25
    a = rdf.Column.generate(rdf.F64, lens, 0, -1e3, 1e3, col_id=80)
    q = a.multiply(rdf.Column.generate(rdf.F64, lens, 1, col_id=81)).cast(rdf.I16)   # many ties
    for col in (a, q):
        idx = rdf.sort_indices([(col, False)])
        taken = col.take(idx)
        v = taken.download()[0].value_slice()
        i = idx.download()[0].value_slice()
        assert v.shape[0] == 100_000_000
        assert bool(np.all(v[1:] >= v[:-1]))
        seen = np.zeros(100_000_000, dtype=bool)
        seen[i] = True
        assert bool(seen.all())
        ties = v[1:] == v[:-1]
        assert bool(np.all(i[1:][ties] > i[:-1][ties]))
        src = np.concatenate([c.value_slice() for c in col.download()])
        assert np.array_equal(v[::9973], src[i[::9973]])
