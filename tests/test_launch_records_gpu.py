"""Launch counts and profile records of the one-GPU element-wise operators: for every call the launch_count() delta and the
profile_read() list of (kernel, dtype, rows, bytes), worked out here from the input shapes.  bench.py reports both, so they
must not move when the host code around the launches changes."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LENS = [5000, 1, 0, 4097, 70001]   # ragged, with an empty chunk
BIG = 2 << 20                      # rows per chunk of the asynchronous uploads (16 MiB of Float64)

F64, I32, I64, U32, BOOL = 9, 2, 3, 6, 10
WIDTH = {2: 4, 3: 8, 6: 4, 9: 8}


def bm(n):
    return (n + 7) // 8


def host_chunks(rdf, rng, dtype, kind, lens=LENS):
    """kind: 'plain' (no bitmap), 'nullable' (bitmap at bit 0) or 'sliced' (a slice whose bitmap starts at bit 3 + k)."""
    out = []
    for k, n in enumerate(lens):
        pad = 3 + k if kind == "sliced" else 0
        m = n + pad
        if dtype == F64:
            v = rng.uniform(1.0, 100.0, m)
        elif dtype == I32:
            v = rng.integers(1, 20000, m, dtype=np.int32)
        else:
            v = rng.integers(1, 2 ** 40, m, dtype=np.int64)
        mask = None if kind == "plain" else rng.random(m) > 0.2
        out.append(rdf.PrimitiveArray.from_numpy(v, mask).slice(pad, n))
    return out


def shape(chunks):
    return [(c.length, c.validity is not None) for c in chunks]


def measure(ctx, fn, settle=True):
    """settle=False leaves uploads in flight: fn then uploads its inputs itself, asynchronously."""
    if settle:
        ctx.synchronize()
    ctx.profile_read()
    l0 = ctx.launch_count()
    res = fn()
    ctx.synchronize()
    recs = [(r["kernel"], r["dtype"], r["rows"], r["bytes"]) for r in ctx.profile_read()]
    return ctx.launch_count() - l0, recs, res


@pytest.fixture(scope="module")
def pctx(ctx):
    ctx.profile_enable(True)
    yield ctx
    ctx.profile_enable(False)


@pytest.fixture(scope="module")
def cols(rdf, pctx):
    """Resident columns: {(dtype, kind): (host chunks, Column)}."""
    rng = np.random.default_rng(11)
    out = {}
    for dtype in (F64, I32, I64):
        for kind in ("plain", "nullable", "sliced"):
            h = host_chunks(rdf, rng, dtype, kind)
            out[(dtype, kind)] = (h, rdf.Column.upload(h, pctx))
    return out


PAIRS = [("plain", "plain"), ("nullable", "sliced"), ("sliced", "plain")]


@pytest.mark.parametrize("op,dtype", [(op, F64) for op in range(7)] + [(op, I32) for op in range(4)])   # atan2 / hypot / log take floats
@pytest.mark.parametrize("pair", PAIRS)
def test_binary(rdf, pctx, cols, op, dtype, pair):
    (ha, a), (hb, b) = cols[(dtype, pair[0])], cols[(dtype, pair[1])]
    w = WIDTH[dtype]
    rows = sum(LENS)
    nbytes = sum(3 * n * w + (va + vb + (op > rdf.native.DIV or va or vb)) * bm(n)
                 for (n, va), (_, vb) in zip(shape(ha), shape(hb)))
    launches, recs, _ = measure(pctx, lambda: a._bin(op, b))
    assert launches == 1
    assert recs == [("binary", dtype, rows, nbytes)]


@pytest.mark.parametrize("dtype", [F64, I64])
@pytest.mark.parametrize("pair", PAIRS)
def test_binary_agg_fused(rdf, pctx, cols, dtype, pair):
    (ha, a), (hb, b) = cols[(dtype, pair[0])], cols[(dtype, pair[1])]
    w = WIDTH[dtype]
    nbytes = sum(3 * n * w + (va + vb + (va or vb)) * bm(n) for (n, va), (_, vb) in zip(shape(ha), shape(hb)))
    launches, recs, _ = measure(pctx, lambda: a.binary_agg(rdf.native.ADD, b))
    assert launches == 2   # the fused pass and the fold of its per-tile partials
    assert recs == [("binary", dtype, sum(LENS), nbytes)]


@pytest.mark.parametrize("kind", ["plain", "nullable", "sliced"])
@pytest.mark.parametrize("op,dtype", [("sin", F64), ("abs", F64), ("abs", I32)])
def test_unary(rdf, pctx, cols, kind, op, dtype):
    h, a = cols[(dtype, kind)]
    w = WIDTH[dtype]
    nbytes = sum(2 * n * w + 2 * v * bm(n) for n, v in shape(h))
    launches, recs, _ = measure(pctx, lambda: getattr(a, op)())
    assert launches == 1
    assert recs == [("unary", dtype, sum(LENS), nbytes)]


@pytest.mark.parametrize("kind", ["plain", "nullable", "sliced"])
@pytest.mark.parametrize("src,dst,fallible", [(F64, I32, True), (I64, I32, True), (I32, F64, False), (I32, I64, False)])
def test_cast(rdf, pctx, cols, kind, src, dst, fallible):
    h, a = cols[(src, kind)]
    nbytes = sum(n * (WIDTH[src] + WIDTH[dst]) + (v + (v or fallible)) * bm(n) for n, v in shape(h))
    launches, recs, _ = measure(pctx, lambda: a.cast(dst))
    assert launches == 1
    assert recs == [("cast", dst, sum(LENS), nbytes)]


@pytest.mark.parametrize("kind", ["plain", "nullable", "sliced"])
@pytest.mark.parametrize("typ,fn,out_dtype", [("date32", "year", I32), ("date32", "date_add", I32), ("ts", "to_date", I32),
                                              ("ts", "unix_timestamp", I64)])
def test_temporal(rdf, pctx, cols, kind, typ, fn, out_dtype):
    t = rdf.TemporalType.date32() if typ == "date32" else rdf.TemporalType.timestamp("us")
    h, a = cols[(t.dtype, kind)]
    nbytes = sum(n * (WIDTH[t.dtype] + WIDTH[out_dtype]) + (v + 1) * bm(n) for n, v in shape(h))
    call = (lambda: a.date_add(3)) if fn == "date_add" else (lambda: getattr(a, fn)())
    try:
        a.with_temporal(t)
        launches, recs, _ = measure(pctx, call)
    finally:
        a.with_temporal(None)
    assert launches == 1
    assert recs == [("temporal", out_dtype, sum(LENS), nbytes)]


@pytest.mark.parametrize("fn,out_dtype", [("date_diff", I32), ("months_between", F64)])
@pytest.mark.parametrize("pair", PAIRS)
def test_temporal_binary(rdf, pctx, cols, fn, out_dtype, pair):
    (ha, a), (hb, b) = cols[(I32, pair[0])], cols[(I32, pair[1])]
    nbytes = sum(n * (4 + 4 + WIDTH[out_dtype]) + (va + vb + 1) * bm(n) for (n, va), (_, vb) in zip(shape(ha), shape(hb)))
    try:
        a.with_temporal(rdf.TemporalType.date32())
        b.with_temporal(rdf.TemporalType.date32())
        launches, recs, _ = measure(pctx, lambda: getattr(a, fn)(b))
    finally:
        a.with_temporal(None)
        b.with_temporal(None)
    assert launches == 1
    assert recs == [("temporal", out_dtype, sum(LENS), nbytes)]


@pytest.mark.parametrize("rhs", ["column_f64", "column_i32", "scalar", "int_scalar"])
@pytest.mark.parametrize("pair", PAIRS)
def test_compare(rdf, pctx, cols, rhs, pair):
    ldt = I32 if rhs == "int_scalar" else F64
    ha, a = cols[(ldt, pair[0])]
    if rhs.startswith("column"):
        rdt = F64 if rhs == "column_f64" else I32
        hb, b = cols[(rdt, pair[1])]
        sb, wr = shape(hb), WIDTH[rdt]
    else:
        b = 50.0 if rhs == "scalar" else 7.0   # an integral scalar against an Int32 column
        sb, wr = [(n, False) for n in LENS], 0
    nbytes = sum((WIDTH[ldt] + wr) * n + bm(n) * (1 + va + vb + (va or vb)) for (n, va), (_, vb) in zip(shape(ha), sb))
    launches, recs, _ = measure(pctx, lambda: a.gt(b))
    assert launches == 1
    assert recs == [("compare", BOOL, sum(LENS), nbytes)]


@pytest.fixture(scope="module")
def masks(rdf, pctx, cols):
    """Boolean columns: two compare results (with and without a bitmap) and an uploaded slice at bit offset 5."""
    m_plain = cols[(F64, "plain")][1].gt(50.0)
    m_null = cols[(F64, "sliced")][1].lt(30.0)
    rng = np.random.default_rng(5)
    up = []
    for n in LENS:
        bits, valid = rng.random(n + 5) > 0.5, rng.random(n + 5) > 0.3
        up.append(rdf.BooleanArray.from_numpy(bits, valid).slice(5, n))
    return {"plain": m_plain, "nullable": m_null, "sliced": rdf.Column.upload(up, pctx, dtype=BOOL)}


@pytest.mark.parametrize("op", ["and", "or", "not"])
@pytest.mark.parametrize("pair", PAIRS)
def test_boolean(rdf, pctx, masks, op, pair):
    a, b = masks[pair[0]], masks[pair[1]]
    rows = sum(LENS)
    call = {"and": lambda: a.logical_and(b), "or": lambda: a.logical_or(b), "not": lambda: a.logical_not()}[op]
    launches, recs, _ = measure(pctx, call)
    assert launches == 1
    assert recs == [("compare", BOOL, rows, rows // 8 * (2 if op == "not" else 3))]


@pytest.mark.parametrize("dtype", [F64, I32, I64])
@pytest.mark.parametrize("null_mod", [0, 7])
def test_generate(rdf, pctx, dtype, null_mod):
    launches, recs, _ = measure(pctx, lambda: rdf.Column.generate(dtype, LENS, null_mod=null_mod, ctx=pctx))
    assert launches == 1
    assert recs == [("generate", dtype, sum(LENS), sum(LENS) * WIDTH[dtype])]


@pytest.mark.parametrize("mode", ["column", "agg", "agg_only"])
@pytest.mark.parametrize("pair", PAIRS)
def test_expr(rdf, pctx, cols, mode, pair):
    (ha, a), (hb, b) = cols[(F64, pair[0])], cols[(F64, pair[1])]
    nodes = [(rdf.native.ADD, 0, 1), (rdf.native.DIV, 2, 0)]
    out = mode != "agg_only"
    nbytes = sum(8 * n * 2 + (va + vb) * bm(n) + (8 * n + (va or vb) * bm(n) if out else 0)
                 for (n, va), (_, vb) in zip(shape(ha), shape(hb)))
    if mode == "column":
        call = lambda: rdf.eval_expr([a, b], nodes)
    else:
        call = lambda: rdf.eval_expr_agg([a, b], nodes, materialise=out)
    launches, recs, _ = measure(pctx, call)
    assert launches == (1 if mode == "column" else 2)
    assert recs == [("expr", F64, sum(LENS), nbytes)]


@pytest.mark.parametrize("dtype,kind", [(F64, "plain"), (F64, "sliced"), (I32, "nullable")])
def test_take(rdf, pctx, cols, dtype, kind):
    _, v = cols[(dtype, kind)]
    rng = np.random.default_rng(3)
    idx_lens = [300, 0, 4000]
    idx = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(rng.integers(0, sum(LENS), n, dtype=np.uint32)) for n in idx_lens], pctx)
    n = sum(idx_lens)
    launches, recs, _ = measure(pctx, lambda: v.take(idx))
    assert launches == 1
    assert recs == [("take", dtype, n, n * (4 + 2 * WIDTH[dtype]))]


def _check_split(recs, launches, kernel, dtype, rows, nbytes, groups):
    """Uploads still in flight: how many launches depends on timing, what they cover does not."""
    assert 1 <= len(recs) <= groups
    assert launches == len(recs)
    assert all(r[0] == kernel and r[1] == dtype for r in recs)
    assert sum(r[2] for r in recs) == rows
    assert sum(r[3] for r in recs) == nbytes


def test_binary_async_upload(rdf, pctx):
    rng = np.random.default_rng(17)
    lens = [BIG] * 4    # two Float64 columns: every chunk pair is one 32 MiB upload group
    ha = [rdf.PrimitiveArray.from_numpy(rng.uniform(1, 2, n)) for n in lens]
    hb = [rdf.PrimitiveArray.from_numpy(rng.uniform(1, 2, n), rng.random(n) > 0.5) for n in lens]
    pctx.synchronize()
    launches, recs, _ = measure(pctx, lambda: (lambda a, b: a.add(b))(*rdf.Column.upload_many([ha, hb], pctx, asynchronous=True)), settle=False)
    _check_split(recs, launches, "binary", F64, sum(lens), sum(3 * n * 8 + 2 * bm(n) for n in lens), len(lens))


def test_unary_async_upload(rdf, pctx):
    rng = np.random.default_rng(19)
    lens = [2 * BIG] * 4    # one Float64 column: every chunk is one 32 MiB upload group
    h = [rdf.PrimitiveArray.from_numpy(rng.uniform(-1, 1, n), rng.random(n) > 0.5) for n in lens]
    pctx.synchronize()
    launches, recs, _ = measure(pctx, lambda: rdf.Column.upload(h, pctx, asynchronous=True).sin(), settle=False)
    _check_split(recs, launches, "unary", F64, sum(lens), sum(2 * n * 8 + 2 * bm(n) for n in lens), len(lens))


def test_temporal_async_upload(rdf, pctx):
    rng = np.random.default_rng(23)
    lens = [2 * BIG] * 4    # one Int64 timestamp column: every chunk is one 32 MiB upload group
    h = [rdf.PrimitiveArray.from_numpy(rng.integers(0, 2 ** 50, n, dtype=np.int64)) for n in lens]
    t = rdf.TemporalType.timestamp("us")
    pctx.synchronize()
    launches, recs, _ = measure(pctx, lambda: rdf.Column.upload(h, pctx, asynchronous=True).with_temporal(t).year(), settle=False)
    _check_split(recs, launches, "temporal", I32, sum(lens), sum(n * 12 + bm(n) for n in lens), len(lens))


@pytest.mark.parametrize("body", ["binary", "unary", "cast", "temporal", "temporal_binary", "compare", "boolean", "generate"])
def test_no_chunks_no_launch(rdf, pctx, body):
    """Every element-wise body over a column without chunks makes an empty column and neither launches nor records."""
    e64 = rdf.Column.upload([], pctx, dtype=F64)
    e32 = rdf.Column.upload([], pctx, dtype=I32).with_temporal(rdf.TemporalType.date32())
    ebool = e64.gt(0.0)
    call = {
        "binary": lambda: e64.add(e64),
        "unary": lambda: e64.sin(),
        "cast": lambda: e64.cast(I32),
        "temporal": lambda: e32.year(),
        "temporal_binary": lambda: e32.date_diff(e32),
        "compare": lambda: e64.gt(e64),
        "boolean": lambda: ebool.logical_and(ebool),
        "generate": lambda: rdf.Column.generate(F64, [], ctx=pctx),
    }[body]
    launches, recs, out = measure(pctx, call)
    assert out.n_chunks == 0
    assert launches == 0
    assert recs == []
