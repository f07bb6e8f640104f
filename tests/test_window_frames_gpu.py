"""Bounded window frames (ROWS / RANGE BETWEEN) and first_value / last_value / nth_value on the GPU, against the numpy restatement in
tests/window_frame_oracle.py (itself checked against SQLite in tests/test_window_frames.py).  Bit-exact except float SUM and AVG,
which are held to the header's bar over each frame's own rows."""
import ctypes as C
import math
import os

import numpy as np
import pytest

import window_frame_oracle as F
from helpers import pool_used
from test_window_gpu import DTYPES, _check, _chunks, _one, _values

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
AGGS = ("sum", "count", "min", "max", "avg")


def _run(rdf, ctx, part, order, calls, lens):
    """part: [(values, mask)]; order: [((values, mask), desc)]; calls: [(fn, (values, mask), arg)] with arg the frame of an aggregate
    or (frame, n, ignore_nulls) of a value function.  Uploads chunked by lens, compares with the oracle, returns the GPU columns."""
    up = {}

    def chunks(vm):
        if id(vm) not in up:
            ch = _chunks(rdf, vm[0], vm[1], lens)
            up[id(vm)] = (ch, rdf.Column.upload(ch, ctx=ctx))
        return up[id(vm)]

    pc = [chunks(p) for p in part]
    oc = [(chunks(o), d) for o, d in order]
    gpu_calls, ora_calls = [], []
    for fn, x, arg in calls:
        if fn in F.VALUES:
            frame, nth, ign = arg
            gpu_calls.append((fn, chunks(x)[1]) + ((nth,) if fn == "nth_value" else ()) + (frame, ign))
        else:
            gpu_calls.append((fn, chunks(x)[1], arg))
        ora_calls.append((fn, chunks(x)[0], arg))
    got = rdf.window([c[1] for c in pc], [(c[1], d) for c, d in oc], gpu_calls)
    want = F.window([c[0] for c in pc], [(c[0], d) for c, d in oc], ora_calls, n=sum(lens))
    _check(got, want, ora_calls)
    return got, (pc, oc, gpu_calls)


def _calls(x, dt, frame):
    out = [(fn, x, frame) for fn in AGGS if not (fn == "avg" and np.dtype(dt).itemsize == 8 and np.dtype(dt).kind != "f")]
    return out + [("first_value", x, (frame, None, False)), ("last_value", x, (frame, None, True)), ("nth_value", x, (frame, 3, False)),
                  ("nth_value", x, (frame, 2, True))]


def _same_bits(a, b):
    (p, pm), (q, qm) = _one(a), _one(b)
    u = np.dtype(f"u{p.dtype.itemsize}")
    return np.array_equal(pm, qm) and np.array_equal(p.view(u), q.view(u))


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
def test_every_value_dtype_and_frame(rdf, ctx, dt):
    rng = np.random.default_rng(DTYPES.index(dt) + 40)
    lens = [3000, 1, 0, 4097, 64]
    n = sum(lens)
    k = _values(rng, n, "int32", 0.05, card=20)
    o = _values(rng, n, "float64", 0.05, card=60)
    x = _values(rng, n, dt, 0.15)
    for frame in (("rows", -3, 2), ("rows", None, -1), ("rows", 1, None), ("rows", -3, -1), ("range", -2.5, 1.0), ("range", 0.5, None),
                  "rows", "range", "partition"):
        _run(rdf, ctx, [k], [(o, dt in ("int8", "float32"))], _calls(x, dt, frame), lens)


@pytest.mark.gpu
@pytest.mark.parametrize("kt", ["int8", "uint16", "int64", "uint64", "float32"])
@pytest.mark.parametrize("desc", [False, True])
def test_range_keys(rdf, ctx, kt, desc):
    rng = np.random.default_rng(7 + desc)
    lens = [2500, 3333, 17]
    n = sum(lens)
    o = _values(rng, n, kt, 0.05, card=40)
    x = _values(rng, n, "float64", 0.1)
    xi = _values(rng, n, "int32", 0.1)
    offs = [(-3, 0), (None, -2), (1, 5), (-2 ** 63 + 1, 2), (-5, 2 ** 63 - 2)] if kt != "float32" else [(-3.0, 0.5), (None, -2.0), (1.0, 5.0)]
    for s, e in offs:
        frame = ("range", s, e)
        _run(rdf, ctx, [_values(rng, n, "uint8", 0.0, card=3)], [(o, desc)], _calls(x, "float64", frame) + _calls(xi, "int32", frame), lens)


@pytest.mark.gpu
def test_frame_widths_across_levels(rdf, ctx):
    """Widths that cross the hierarchy's block edges (32, 1024, 32768 rows), on chunks with empty, one-row and sliced pieces."""
    rng = np.random.default_rng(3)
    n = 120_000
    xs = (rng.integers(-2 ** 20, 2 ** 20, n) / 1024.0, rng.random(n) > 0.1)   # exact oracle sums
    xi = _values(rng, n, "int16", 0.1)
    lens = [40_000, 0, 1, 50_000, 29_999]
    for w in (1, 2, 31, 32, 33, 1023, 1024, 1025, 5000, 100_000):
        calls = [(fn, xs, ("rows", -(w - 1), 0)) for fn in AGGS] + [("max", xi, ("rows", -(w // 2), w - 1 - w // 2)),
                                                                     ("sum", xi, ("rows", 1, w))]
        _run(rdf, ctx, [], [], calls, lens)


@pytest.mark.gpu
def test_one_partition_wide_frame_and_determinism(rdf, ctx):
    rng = np.random.default_rng(11)
    n = 1_500_000
    x = (rng.integers(-2 ** 20, 2 ** 20, n) / 1024.0, rng.random(n) > 0.05)
    xf = _values(rng, n, "float32", 0.05)
    o = _values(rng, n, "int64", 0.01, card=400_000)
    frame = ("rows", -100_000, 0)
    calls = [("sum", x, frame), ("avg", x, frame), ("max", x, frame), ("count", x, ("range", -20_000, 20_000)),
             ("last_value", x, (("rows", None, 0), None, True))]
    got, (pc, oc, gcalls) = _run(rdf, ctx, [], [(o, False)], calls, [700_000, 800_000])
    again = rdf.window([c[1] for c in pc], [(c[1], d) for c, d in oc], gcalls)
    assert all(_same_bits(a, b) for a, b in zip(got, again))
    # a second chunking of the same rows: the same bits
    lens2 = [1, 299_999, 0, 1_200_000]
    up2 = lambda vm: rdf.Column.upload(_chunks(rdf, vm[0], vm[1], lens2), ctx=ctx)
    x2, o2, xf2 = up2(x), up2(o), up2(xf)
    calls2 = [("sum", x2, frame), ("avg", x2, frame), ("max", x2, frame), ("count", x2, ("range", -20_000, 20_000)),
              ("last_value", x2, ("rows", None, 0), True)]
    other = rdf.window([], [(o2, False)], calls2)
    assert all(_same_bits(a, b) for a, b in zip(got, other))
    s1 = rdf.window([], [], [("sum", x2, ("rows", -5000, 5000)), ("sum", xf2, ("rows", -5000, 5000))])
    s2 = rdf.window([], [], [("sum", up2(x), ("rows", -5000, 5000)), ("sum", up2(xf), ("rows", -5000, 5000))])
    assert all(_same_bits(a, b) for a, b in zip(s1, s2))


@pytest.mark.gpu
def test_equivalent_specifications_give_the_existing_bits(rdf, ctx):
    rng = np.random.default_rng(21)
    n = 40_000
    k = rdf.Column.upload(_chunks(rdf, *_values(rng, n, "int16", 0.05, card=30), [n]), ctx=ctx)
    for kt in ("int32", "float64"):
        o = rdf.Column.upload(_chunks(rdf, *_values(rng, n, kt, 0.05, card=200), [17_000, 23_000]), ctx=ctx)
        x = rdf.Column.upload(_chunks(rdf, *_values(rng, n, "float64", 0.1), [17_000, 23_000]), ctx=ctx)
        for a, b in ((("rows", None, 0), "rows"), (("rows", None, None), "partition"), (("range", None, 0), "range"),
                     (("range", None, None), "partition")):
            got = rdf.window([k], [(o, True)], [(fn, x, a) for fn in AGGS] + [(fn, x, b) for fn in AGGS])
            assert all(_same_bits(got[i], got[i + 5]) for i in range(5)), (kt, a, b)


@pytest.mark.gpu
def test_device_generated_2_pow_24_rows(rdf, ctx):
    n = 2 ** 24 + 5
    lens = [2 ** 23, 2 ** 23 + 5]
    k = rdf.Column.generate(rdf.I8, lens, kind=2, col_id=1, ctx=ctx)
    x = rdf.Column.generate(rdf.I32, lens, kind=2, col_id=3, null_mod=13, ctx=ctx)
    calls = [("sum", x, ("rows", -99, 0)), ("max", x, ("rows", -99, 0)), ("avg", x, ("rows", -2, 2)), ("last_value", x, ("rows", None, 0), True)]
    got = rdf.window([k], [], calls)
    kch, xch = k.download(), x.download()
    ora = [("sum", xch, ("rows", -99, 0)), ("max", xch, ("rows", -99, 0)), ("avg", xch, ("rows", -2, 2)), ("last_value", xch, (("rows", None, 0), None, True))]
    _check(got, F.window([kch], [], ora, n=n), ora)


@pytest.mark.gpu
def test_pool_and_errors(rdf, ctx):
    N = rdf.native
    P = rdf.PrimitiveArray
    a = rdf.Column.upload([P.from_numpy(np.arange(100, dtype=np.int32))], ctx=ctx)
    f = rdf.Column.upload([P.from_numpy(np.arange(100, dtype=np.float64))], ctx=ctx)
    ctx.synchronize()
    before = pool_used(ctx)
    res = rdf.window([a], [(f, True)], [("sum", a, ("rows", -3, 3)), ("avg", a, ("range", -2.5, 0.0)), ("first_value", a, ("rows", 1, 4), True),
                                         ("nth_value", f, 2, ("range", None, 1.0))])
    for r in res:
        r.free()
    ctx.synchronize()
    assert pool_used(ctx) == before
    I64_MIN, I64_MAX = -2 ** 63, 2 ** 63 - 1

    def call(order, fn, col, frame, **kw):
        ok = (N.SortKeyC * 1)()
        if order is not None:
            ok[0].column, ok[0].descending = order.handle.value, 0
        arr = (N.WindowCall * 1)()
        arr[0].function, arr[0].frame, arr[0].column = fn, frame, col.handle.value
        for name, v in kw.items():
            setattr(arr[0], name, v)
        out = (C.c_void_p * 1)()
        st = N.lib().bdf_window_dev(ctx.handle, 0, None, 1 if order is not None else 0, ok if order is not None else None, 1, arr, out)
        assert out[0] is None
        return st

    RB, GB = N.FRAME_ROWS_BETWEEN, N.FRAME_RANGE_BETWEEN
    assert call(a, N.WIN_SUM, a, RB, start=2, end=1) == N.INVALID                          # start > end
    assert call(a, N.WIN_SUM, a, RB, start=I64_MAX, end=I64_MAX) == N.INVALID              # starts at UNBOUNDED FOLLOWING
    assert call(a, N.WIN_SUM, a, RB, start=I64_MIN, end=I64_MIN) == N.INVALID              # ends at UNBOUNDED PRECEDING
    assert call(f, N.WIN_SUM, a, GB, start_f=math.nan, end_f=0.0) == N.INVALID             # NaN offset
    assert call(f, N.WIN_SUM, a, GB, start_f=1.0, end_f=0.0) == N.INVALID
    assert call(f, N.WIN_SUM, a, GB, start_f=math.inf, end_f=math.inf) == N.INVALID
    assert call(None, N.WIN_SUM, a, GB, start=-1, end=0) == N.INVALID                      # RANGE without an order column
    assert call(a, N.WIN_NTH_VALUE, a, RB, start=-1, end=0, offset=0) == N.INVALID         # n < 1
    assert call(a, N.WIN_SUM, a, RB, start=-1, end=0, ignore_nulls=1) == N.INVALID         # IGNORE NULLS on an aggregate
    assert call(a, N.WIN_LAG, a, 0, offset=1, ignore_nulls=1) == N.INVALID
    assert call(a, 99, a, 0) == N.UNSUPPORTED
    assert call(a, N.WIN_SUM, a, 7) == N.UNSUPPORTED
    assert call(a, 15, a, 0) == N.UNSUPPORTED
    with pytest.raises(rdf.UnsupportedType):
        rdf.window([a], [], [("ntile", a)])
    with pytest.raises(rdf.UnsupportedType):
        rdf.window([a], [], [("sum", a, "groups")])
    ctx.synchronize()
    assert pool_used(ctx) == before


@pytest.mark.gpu
def test_multi_gpu_context_is_refused(rdf):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU: no multi-GPU context")
    fleet = rdf.Context.multi(0)
    try:
        fk = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.arange(10, dtype=np.int64))], ctx=fleet)
        with pytest.raises(rdf.UnsupportedType):
            rdf.window([], [], [("sum", fk, ("rows", -1, 1))])
    finally:
        fleet.close()


@pytest.mark.gpu
def test_device_frame_moving_average(rdf, ctx):
    from rust_dataframe_b200.frame import select, window

    path = os.path.join(ROOT, "tests", "golden", "uk_cities_with_headers.csv")
    frame = rdf.DeviceFrame.from_csv(path, ctx=ctx)
    host = {n: c.download() for n, c in frame.columns.items()}
    out = frame.window([], [("lng", False)], [("ma", "avg", "lat", ("rows", -2, 2)), ("lo", "first_value", "lat", ("range", -0.5, 0.5))])
    assert list(out.schema)[-2:] == ["ma", "lo"]
    ora = [("avg", host["lat"], ("rows", -2, 2)), ("first_value", host["lat"], (("range", -0.5, 0.5), None, False))]
    _check([out.column("ma"), out.column("lo")], F.window([], [(host["lng"], False)], ora), ora)
    ev = frame.evaluate([window([], [], [("ma", "avg", "lat", ("rows", -9, 0))]), select(["ma"])])
    lat = np.concatenate([a.value_slice() for a in host["lat"]])
    c = np.concatenate([[0.0], np.cumsum(lat)])
    i = np.arange(lat.shape[0])
    want = (c[i + 1] - c[np.maximum(i - 9, 0)]) / np.minimum(i + 1, 10)
    got, gm = _one(ev.column("ma"))
    assert gm.all() and np.allclose(got, want, rtol=1e-12, atol=0)
