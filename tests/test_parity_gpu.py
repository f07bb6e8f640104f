"""GPU parity: every operator of the hot path, called through the C ABI (ctypes -> libb200df.so), against
the CPU oracle on the same seeded inputs.

Bars (BASELINE.json north_star):
  * integer arithmetic, cast (values AND which slots become NULL), count, min/max, wrapping sums,
    IEEE add/sub/mul/div on f32/f64: BIT-EXACT;
  * f64 sin/cos/tan vs glibc: <= 3 ulp; f32: <= 5 ulp (CUDA documents 2/2/2 and 2/2/4 ulp, glibc < 1 ulp);
    other float unaries (N1 row): <= 4 ulp f64 / <= 6 ulp f32, exact for ceil/floor/round/sqrt/abs;
  * float sum: |gpu - exact| <= 16*log2(n)*eps*sum|x|, and the reference's own sequential fold is within
    n*eps*sum|x| of the same exact value (SURVEY 8(a) row A9).
"""
import json
import os

import numpy as np
import pytest

from helpers import assert_same_array, pool_used, random_mask, ulp_distance

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ALL_TYPES = ["I8", "I16", "I32", "I64", "U8", "U16", "U32", "U64", "F32", "F64"]
INT_TYPES = ALL_TYPES[:8]
RAGGED = [0, 1, 5, 31, 32, 33, 255, 2047, 2048, 2049, 4096, 10007, 70001]


def rand_values(rng, npdt, n, nonzero=False):
    npdt = np.dtype(npdt)
    if npdt.kind == "f":
        v = rng.uniform(-1e3, 1e3, n).astype(npdt)
        if nonzero:
            v[v == 0] = 1
        return v
    info = np.iinfo(npdt)
    v = rng.integers(info.min, info.max, n, dtype=npdt, endpoint=True)
    if nonzero:
        v[v == 0] = 1
        if info.min < 0:
            v[v == -1] = 3  # iN::MIN / -1 is unspecified in the reference
    return v


def make_column(rdf, rng, dtype, lens, null_frac=0.0, sliced=False, nonzero=False):
    """A column as ragged chunks; sliced=True gives every chunk a non-zero, non-byte-aligned offset."""
    chunks = []
    for k, n in enumerate(lens):
        pad = (3 + 5 * k) % 29 if sliced else 0
        v = rand_values(rng, rdf.NP_DTYPES[dtype], n + pad + 2, nonzero)
        if null_frac > 0:
            arr = rdf.PrimitiveArray.from_numpy(v, random_mask(rng, n + pad + 2, null_frac))
        else:
            arr = rdf.PrimitiveArray.from_numpy(v)
        arr.null_count = -1 if arr.validity is not None else 0
        chunks.append(arr.slice(pad, n) if sliced else arr.slice(0, n))
    return chunks


# ---------------------------------------------------------------------------------------------------------
# K1 binary arithmetic

@pytest.mark.parametrize("tname", ALL_TYPES)
def test_binary_ops_bit_exact(rdf, ctx, oracle, tname):
    dtype = getattr(rdf, tname)
    rng = np.random.default_rng(100 + dtype)
    SF = rdf.ScalarFunctions
    for null_a, null_b, sliced in [(0, 0, False), (0.1, 0, False), (0.1, 0.3, True), (0, 0.05, True)]:
        a = make_column(rdf, rng, dtype, RAGGED, null_a, sliced)
        b = make_column(rdf, rng, dtype, RAGGED, null_b, sliced, nonzero=True)
        for name, op, fn in [("add", oracle.ADD, SF.add), ("subtract", oracle.SUB, SF.subtract),
                             ("multiply", oracle.MUL, SF.multiply), ("par_multiply", oracle.MUL, SF.par_multiply),
                             ("divide", oracle.DIV, SF.divide)]:
            got = fn(a, b)
            st, want = oracle.col_binary(op, dtype, a, b)
            assert st == oracle.OK and len(got) == len(want)
            for i, (g, w) in enumerate(zip(got, want)):
                assert_same_array(g, w, what=f"{name}<{tname}> chunk {i} nulls=({null_a},{null_b}) sliced={sliced}")
                if null_a == 0 and null_b == 0:
                    assert g.validity is None  # neither input has a bitmap -> none on the output


def test_binary_float_special_values(rdf, ctx, oracle):
    sp = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-310, -1e-310, 1.7976931348623157e308, 5e-324, 1.0, -1.0, 3.0])
    a = np.repeat(sp, len(sp))
    b = np.tile(sp, len(sp))
    for dtype, npdt in ((rdf.F64, np.float64), (rdf.F32, np.float32)):
        with np.errstate(all="ignore"):
            A, B = rdf.PrimitiveArray.from_numpy(a.astype(npdt)), rdf.PrimitiveArray.from_numpy(b.astype(npdt))
        for op, fn in [(oracle.ADD, rdf.ScalarFunctions.add), (oracle.SUB, rdf.ScalarFunctions.subtract),
                       (oracle.MUL, rdf.ScalarFunctions.multiply)]:
            st, want = oracle.col_binary(op, dtype, [A], [B])
            assert_same_array(fn([A], [B])[0], want[0], what=f"special values op {op}")
        # divide: mask out zero divisors (they raise), keep subnormals / inf / nan
        nz = b.astype(npdt) != 0
        A2, B2 = rdf.PrimitiveArray.from_numpy(a.astype(npdt)[nz]), rdf.PrimitiveArray.from_numpy(b.astype(npdt)[nz])
        st, want = oracle.col_binary(oracle.DIV, dtype, [A2], [B2])
        assert st == oracle.OK
        assert_same_array(rdf.ScalarFunctions.divide([A2], [B2])[0], want[0], what="special values divide")


def test_divide_by_zero_and_errors(rdf, ctx, oracle):
    P = rdf.PrimitiveArray
    for dtype, zero in ((rdf.I32, 0), (rdf.F64, 0.0), (rdf.F64, -0.0), (rdf.U8, 0), (rdf.I64, 0), (rdf.F32, 0.0)):
        a = P.from_pylist(dtype, [6, 8, 10])
        with pytest.raises(rdf.DivideByZero):
            rdf.ScalarFunctions.divide([a], [P.from_pylist(dtype, [2, zero, 5])])
        npdt = rdf.NP_DTYPES[dtype]
        b = P.from_numpy(np.array([2, zero, 5], dtype=npdt), np.array([True, False, True]))
        assert rdf.ScalarFunctions.divide([a], [b])[0].to_pylist() == [3, None, 2]
        a2 = P.from_numpy(np.array([6, 8, 10], dtype=npdt), np.array([True, False, True]))
        assert rdf.ScalarFunctions.divide([a2], [P.from_pylist(dtype, [2, zero, 5])])[0].to_pylist() == [3, None, 2]
    # zero divisor far inside a large later chunk
    big = np.ones(300001, dtype=np.int64)
    big[299999] = 0
    ok = P.from_numpy(np.ones(5, dtype=np.int64))
    with pytest.raises(rdf.DivideByZero):
        rdf.ScalarFunctions.divide([ok, P.from_numpy(big)], [ok, P.from_numpy(big)])
    # on device columns DivideByZero comes after the output column (and the fused aggregate's future) was made: nothing leaks
    ca = rdf.Column.upload([P.from_pylist(rdf.F64, [6.0, 8.0, 10.0])], ctx=ctx)
    cz = rdf.Column.upload([P.from_pylist(rdf.F64, [2.0, 0.0, 5.0])], ctx=ctx)
    ca.divide(ca).free()
    ca.binary_agg(rdf.native.DIV, ca)[0].free()
    ctx.synchronize()
    before = pool_used(ctx)
    with pytest.raises(rdf.DivideByZero):
        ca.divide(cz)
    with pytest.raises(rdf.DivideByZero):
        ca.binary_agg(rdf.native.DIV, cz)
    ctx.synchronize()
    assert pool_used(ctx) == before
    # length mismatch: same message as the reference (src/functions/scalar.rs:508-511)
    with pytest.raises(rdf.ComputeError, match="Cannot perform math operation on arrays of different length"):
        rdf.ScalarFunctions.add([P.from_pylist(rdf.I64, [1, 2, 3])], [P.from_pylist(rdf.I64, [1, 2])])
    # zip() truncates to the shorter Vec
    x = P.from_pylist(rdf.I64, [1, 2, 3])
    assert len(rdf.ScalarFunctions.add([x, x, x], [x])) == 1
    assert rdf.ScalarFunctions.add([], []) == []
    # MIN / -1 wraps, truncation toward zero
    a = P.from_pylist(rdf.I32, [7, -7, 7, -7, -2 ** 31])
    b = P.from_pylist(rdf.I32, [2, 2, -2, -2, -1])
    assert rdf.ScalarFunctions.divide([a], [b])[0].to_pylist() == [3, -3, -3, 3, -2 ** 31]
    # trait bounds of the reference
    with pytest.raises(rdf.UnsupportedType):
        rdf.ScalarFunctions.sin([P.from_pylist(rdf.I32, [1])])
    with pytest.raises(rdf.UnsupportedType):
        rdf.ScalarFunctions.abs([P.from_pylist(rdf.U32, [1])])
    with pytest.raises(rdf.UnsupportedType):
        rdf.AggregateFunctions.max([P.from_pylist(rdf.F64, [1.0])])


def test_upload_many_bad_view_leaks_nothing(rdf, ctx):
    """A bad view in the second column is found after the first column's arenas were allocated."""
    import ctypes as C
    N = rdf.native
    good = [rdf.PrimitiveArray.from_numpy(np.arange(1000, dtype=np.int64))]
    for col in rdf.Column.upload_many([good, good], ctx=ctx):
        col.free()
    views = [N.make_views(good), N.make_views(good)]
    views[1][0].values = None   # 1000 rows without a values buffer
    dtypes, counts = (C.c_int32 * 2)(rdf.I64, rdf.I64), (C.c_int64 * 2)(1, 1)
    ptrs = (C.POINTER(N.View) * 2)(*[C.cast(v, C.POINTER(N.View)) for v in views])
    outs = (C.c_void_p * 2)()
    ctx.synchronize()
    before = pool_used(ctx)
    assert N.lib().bdf_upload_many(ctx.handle, 2, dtypes, counts, ptrs, 0, outs) == N.INVALID
    assert N.lib().bdf_last_error() == b"bad view 0"
    assert outs[0] is None and outs[1] is None
    ctx.synchronize()
    assert pool_used(ctx) == before


def test_reference_goldens_on_gpu(rdf, ctx, oracle):
    """The reference's own test vectors, evaluated by the CUDA path (SURVEY 8(c))."""
    P, SF, AF = rdf.PrimitiveArray, rdf.ScalarFunctions, rdf.AggregateFunctions
    assert SF.abs([P.from_pylist(rdf.I32, [-5, -6, 7, -8, -0])])[0].to_pylist() == [5, 6, 7, 8, 0]     # scalar.rs:576-584
    c = SF.abs([P.from_pylist(rdf.F64, [-5.2, -6.1, 7.3, -8.6, -0.0])])[0].to_pylist()                 # scalar.rs:565-573
    assert c == [5.2, 6.1, 7.3, 8.6, 0.0]
    x = P.from_pylist(rdf.F64, [-0.2, 0.25, 0.75])                                                      # scalar.rs:587-602
    for got, want in zip(SF.acos([x])[0].to_pylist(), [1.7721542475852274, 1.318116071652818, 0.7227342478134157]):
        assert want - got < np.finfo(np.float64).eps and abs(want - got) <= 4 * np.spacing(want)
    for got, want in zip(SF.cos([x])[0].to_pylist(), [0.9800665778412416, 0.9689124217106447, 0.7316888688738209]):
        assert want - got < np.finfo(np.float64).eps and abs(want - got) <= 3 * np.spacing(want)
    assert AF.count([P.from_pylist(rdf.I32, [5, 6, 7, 8, 9])]) == 5                                     # aggregate.rs:123-127
    a, b = P.from_pylist(rdf.I32, [0, 1, 2, 3, 4]), P.from_pylist(rdf.I32, [5, 6, 7, 8, 9])
    assert AF.avg([a, b]) == 4.5                                                                        # aggregate.rs:130-146
    assert AF.avg([P.from_pylist(rdf.I32, [0, None, 1, None, 2, 3, 4]), b]) == 4.5
    m = P.from_pylist(rdf.I32, [None, 200, None, -256, None])                                           # scalar.rs:621-671
    out = SF.par_multiply([m] * 380, [m] * 380)
    assert len(out) == 380 and all(o.to_pylist() == [None, 40000, None, 65536, None] and o.null_count == 3 for o in out)
    with open(os.path.join(HERE, "golden", "uk_cities.json")) as f:
        cities = json.load(f)
    lat, lng = P.from_numpy(np.array(cities["lat"])), P.from_numpy(np.array(cities["lng"]))
    s = SF.add([lat], [lng])[0]
    assert abs(cities["reference_asserts"]["lat_plus_lng_row0"] - s.value(0)) < 1e-4                   # dataframe.rs:803-808
    assert [float(v).hex() for v in s.value_slice()] == cities["derived"]["lat_plus_lng_hex"]
    assert abs(cities["reference_asserts"]["abs_lng_row0"] - SF.abs([lng])[0].value(0)) < np.finfo(np.float64).eps
    want_sum = float.fromhex(cities["derived"]["sum_lat_hex"])
    assert abs(AF.sum([lat]) - want_sum) <= 37 * np.spacing(want_sum)
    sin_want = np.array([float.fromhex(h) for h in cities["derived"]["sin_lat_hex"]])
    assert ulp_distance(SF.sin([lat])[0].value_slice().copy(), sin_want).max() <= 3


# ---------------------------------------------------------------------------------------------------------
# K2 unary

TRIG_TOL = {"F64": 3, "F32": 5}
N1_TOL = {"F64": 4, "F32": 6}
EXACT_UNARIES = {"abs", "ceil", "floor", "round", "sqrt", "degrees", "radians"}


def unary_inputs(rng, npdt, name, n):
    if name in ("acos", "asin"):
        v = rng.uniform(-1, 1, n)
    elif name in ("log10", "log2", "sqrt"):
        v = rng.uniform(1e-3, 1e6, n)
    elif name in ("exp", "expm1", "cosh", "sinh"):
        v = rng.uniform(-20, 20, n)
    else:
        v = np.concatenate([rng.uniform(-2e6, 2e6, n // 2), rng.uniform(-10, 10, n - n // 2)])
    return v.astype(npdt)


@pytest.mark.parametrize("tname", ["F64", "F32"])
def test_unary_float_functions(rdf, ctx, oracle, tname):
    dtype = getattr(rdf, tname)
    npdt = rdf.NP_DTYPES[dtype]
    rng = np.random.default_rng(7)
    names = ["abs", "sin", "cos", "tan", "acos", "asin", "atan", "cbrt", "ceil", "cosh", "degrees", "exp", "expm1",
             "floor", "log10", "log2", "radians", "round", "sinh", "sqrt", "tanh"]
    for name in names:
        op = getattr(oracle, name.upper())
        lens = [0, 3, 2049, 50021]
        chunks = []
        for k, n in enumerate(lens):
            v = unary_inputs(rng, npdt, name, n + 11)
            arr = rdf.PrimitiveArray.from_numpy(v, random_mask(rng, n + 11, 0.1) if k % 2 else None)
            arr.null_count = -1 if arr.validity is not None else 0
            chunks.append(arr.slice(5, n))
        got = getattr(rdf.ScalarFunctions, name)(chunks)
        st, want = oracle.col_unary(op, dtype, chunks)
        assert st == oracle.OK
        tol = 0 if name in EXACT_UNARIES else (TRIG_TOL[tname] if name in ("sin", "cos", "tan") else N1_TOL[tname])
        for i, (g, w) in enumerate(zip(got, want)):
            assert_same_array(g, w, what=f"{name}<{tname}> chunk {i}", exact=(tol == 0), max_ulp=tol, check_payload=False)
            assert np.all(g.value_slice()[~g.valid_mask()] == 0)  # null payload 0, like the builder


def test_trig_special_values_and_large_arguments(rdf, ctx, oracle):
    x = np.array([0.0, -0.0, 1e-300, 0.5, -2.5, 1e6, 1e15, 1e22, 1.7e308, np.inf, -np.inf, np.nan, np.pi, np.pi / 2])
    arr = rdf.PrimitiveArray.from_numpy(x)
    for name in ("sin", "cos", "tan"):
        got = getattr(rdf.ScalarFunctions, name)([arr])[0].value_slice()
        st, want = oracle.col_unary(getattr(oracle, name.upper()), oracle.F64, [arr])
        assert ulp_distance(got.copy(), want[0].values).max() <= 3, name   # NaN <-> NaN, +-inf -> NaN
    s = rdf.ScalarFunctions.sin([arr])[0].value_slice()
    assert np.signbit(s[1]) and s[1] == 0  # sin(-0.0) = -0.0
    big = np.random.default_rng(1).uniform(-1e12, 1e12, 20000)   # Payne-Hanek slow path
    arrb = rdf.PrimitiveArray.from_numpy(big)
    for name in ("sin", "cos"):
        st, want = oracle.col_unary(getattr(oracle, name.upper()), oracle.F64, [arrb])
        assert ulp_distance(getattr(rdf.ScalarFunctions, name)([arrb])[0].value_slice().copy(), want[0].values).max() <= 3


@pytest.mark.parametrize("tname", ["I8", "I16", "I32", "I64"])
def test_abs_signed_ints_wrap(rdf, ctx, oracle, tname):
    dtype = getattr(rdf, tname)
    rng = np.random.default_rng(3)
    cols = make_column(rdf, rng, dtype, [7, 4099], 0.2, True)
    info = np.iinfo(rdf.NP_DTYPES[dtype])
    cols.append(rdf.PrimitiveArray.from_numpy(np.array([info.min, info.max, -1, 0], dtype=rdf.NP_DTYPES[dtype])))
    got = rdf.ScalarFunctions.abs(cols)
    st, want = oracle.col_unary(oracle.ABS, dtype, cols)
    for g, w in zip(got, want):
        assert_same_array(g, w, what=f"abs<{tname}>")
    assert got[-1].value(0) == info.min  # num::abs wraps at MIN in release builds


def test_math_op_binaries(rdf, ctx, oracle):
    rng = np.random.default_rng(9)
    for dtype, npdt, tol in ((rdf.F64, np.float64, 4), (rdf.F32, np.float32, 6)):
        a = rdf.PrimitiveArray.from_numpy(rng.uniform(0.1, 100, 5001).astype(npdt), random_mask(rng, 5001, 0.1))
        b = rdf.PrimitiveArray.from_numpy(rng.uniform(1.5, 100, 5001).astype(npdt), random_mask(rng, 5001, 0.1))
        for name, op in (("atan2", oracle.ATAN2), ("hypot", oracle.HYPOT), ("log", oracle.LOG)):
            got = getattr(rdf.ScalarFunctions, name)(a, b)
            st, want = oracle.col_binary(op, dtype, [a], [b])
            assert_same_array(got, want[0], what=name, exact=False, max_ulp=tol, check_payload=False)


# ---------------------------------------------------------------------------------------------------------
# K3 cast

def cast_inputs(rdf, rng, f, n):
    npdt = np.dtype(rdf.NP_DTYPES[f])
    if npdt.kind == "f":
        edges = [0.0, -0.0, 0.5, -0.5, -0.9999, -1.0, 1.9, -1.9, 127.0, 127.9, 128.0, -128.0, -128.9, -129.0, 255.0, 255.9,
                 256.0, 32767.9, 32768.0, -32768.9, -32769.0, 65535.9, 65536.0, 2147483647.0, 2147483648.0, -2147483648.0,
                 -2147483649.0, 4294967295.0, 4294967296.0, 9.223372036854775e18, 9.223372036854776e18,
                 -9.223372036854776e18, -9.223372036854778e18, 1.8446744073709552e19, 1.844674407370955e19, 3e10, -3e10,
                 1e300, -1e300, 3.4028235e38, 3.5e38, np.inf, -np.inf, np.nan, 1e-320, 16777217.0, 9007199254740993.0]
        with np.errstate(all="ignore"):
            base = np.array(edges, dtype=np.float64).astype(npdt)
            body = np.concatenate([rng.uniform(-300, 300, n // 2), rng.uniform(-7e4, 7e4, n // 4),
                                   rng.uniform(-1e19, 1e19, n - n // 2 - n // 4)]).astype(npdt)
        return np.concatenate([base, body])
    info = np.iinfo(npdt)
    edges = [0, 1, -1, 127, 128, -128, -129, 255, 256, 32767, 32768, -32768, -32769, 65535, 65536, 2 ** 31 - 1, 2 ** 31,
             -2 ** 31, -2 ** 31 - 1, 2 ** 32 - 1, 2 ** 32, 2 ** 53 + 1, 2 ** 53 + 3, 2 ** 63 - 1, -2 ** 63, 2 ** 64 - 1, 16777217]
    base = np.array([e for e in edges if info.min <= e <= info.max], dtype=npdt)
    return np.concatenate([base, rng.integers(info.min, info.max, n, dtype=npdt, endpoint=True),
                           rng.integers(max(info.min, -300), min(info.max, 300), n, dtype=npdt, endpoint=True)])


@pytest.mark.parametrize("fname", ALL_TYPES)
def test_cast_matrix_bit_exact(rdf, ctx, oracle, fname):
    f = getattr(rdf, fname)
    rng = np.random.default_rng(50 + f)
    v = cast_inputs(rdf, rng, f, 6000)
    plain = rdf.PrimitiveArray.from_numpy(v)
    nullable = rdf.PrimitiveArray.from_numpy(v, random_mask(rng, len(v), 0.1))
    nullable.null_count = -1
    sl = nullable.slice(3, len(v) - 9)
    empty = plain.slice(0, 0)
    for tname in ALL_TYPES:
        t = getattr(rdf, tname)
        for chunks in ([plain], [sl, empty, plain]):
            got = rdf.cast(chunks, t)
            st, want = oracle.col_cast(f, t, chunks)
            assert st == oracle.OK
            for i, (g, w) in enumerate(zip(got, want)):
                assert g.dtype == t
                assert_same_array(g, w, what=f"cast {fname}->{tname} chunk {i}")


def test_cast_parity_cases_from_survey(rdf, ctx):
    """SURVEY 8(d) config 4 'extra parity-only cases'."""
    P = rdf.PrimitiveArray
    f = P.from_pylist(rdf.F64, [float("nan"), float("inf"), float("-inf"), 3e10, -3e10, -1.9])
    assert rdf.cast([f], rdf.I32)[0].to_pylist() == [None, None, None, None, None, -1]
    assert rdf.cast([P.from_pylist(rdf.I64, [2 ** 31, -2 ** 31 - 1, 7])], rdf.I32)[0].to_pylist() == [None, None, 7]
    assert rdf.cast([P.from_pylist(rdf.I32, [-1, 5])], rdf.U64)[0].to_pylist() == [None, 5]
    assert rdf.cast([P.from_pylist(rdf.I64, [2 ** 53 + 1, 2 ** 53 + 3])], rdf.F64)[0].to_pylist() == [float(2 ** 53), float(2 ** 53 + 4)]
    out = rdf.cast([P.from_pylist(rdf.I32, [1, None, -3])], rdf.F64)[0]
    assert out.to_pylist() == [1.0, None, -3.0] and out.null_count == 1


# ---------------------------------------------------------------------------------------------------------
# K4 aggregates

@pytest.mark.parametrize("tname", INT_TYPES)
def test_int_aggregates_exact(rdf, ctx, oracle, tname):
    dtype = getattr(rdf, tname)
    rng = np.random.default_rng(200 + dtype)
    AF = rdf.AggregateFunctions
    lens = [n for n in RAGGED if n > 0]
    for null_frac, sliced in ((0, False), (0.1, True), (0.9, True)):
        col = make_column(rdf, rng, dtype, lens, null_frac, sliced)
        if null_frac:  # make sure no chunk is entirely null (that is the panic case, tested below)
            col = [c for c in col if c.valid_mask().any()]
        for name, op in (("sum", oracle.SUM), ("min", oracle.MIN), ("max", oracle.MAX), ("count", oracle.COUNT)):
            st, want = oracle.aggregate(op, dtype, col)
            assert st == oracle.OK
            got = getattr(AF, name)(col)
            assert int(got) == int(want), f"{name}<{tname}> nulls={null_frac}: {got} != {want}"
        allr = AF.all(col)
        for key, op in (("sum", oracle.SUM), ("min", oracle.MIN), ("max", oracle.MAX), ("count", oracle.COUNT)):
            assert int(allr[key]) == int(oracle.aggregate(op, dtype, col)[1])
        assert AF.min_as_written(col) == oracle.aggregate(oracle.MIN_AS_WRITTEN, dtype, col)[1]


def test_aggregate_option_and_panic_rules(rdf, ctx, oracle):
    P, AF = rdf.PrimitiveArray, rdf.AggregateFunctions
    allnull = P.from_numpy(np.array([1, 2], dtype=np.int64), np.array([False, False]))
    some = P.from_pylist(rdf.I64, [5, None, -7])
    empty = P.from_numpy(np.zeros(0, dtype=np.int64))
    assert AF.sum([allnull, some]) == -2
    assert AF.sum([], dtype=rdf.I64) == 0 and AF.sum([empty, allnull]) == 0
    assert AF.max([], dtype=rdf.I64) is None and AF.min([], dtype=rdf.I64) is None
    for bad in ([some, allnull], [empty, some]):
        with pytest.raises(rdf.ReferencePanic):
            AF.max(bad)
        with pytest.raises(rdf.ReferencePanic):
            AF.min(bad)
    assert AF.max([some]) == 5 and AF.min([some]) == -7 and AF.min_as_written([some]) == 5
    assert AF.count([allnull, some, empty]) == 2
    r = AF.all([allnull, some])
    assert r["would_panic"] and r["sum"] == -2 and r["count"] == 2 and r["min"] == -7 and r["max"] == 5
    r = AF.all([allnull])
    assert r["min"] is None and r["max"] is None and r["count"] == 0


@pytest.mark.parametrize("tname", ["F64", "F32"])
def test_float_sum_tolerance_and_determinism(rdf, ctx, oracle, tname):
    dtype = getattr(rdf, tname)
    npdt = rdf.NP_DTYPES[dtype]
    eps = 2.0 ** -53 if tname == "F64" else 2.0 ** -24
    rng = np.random.default_rng(17)
    lens = [1000003, 5, 2048, 777777]
    for null_frac in (0, 0.1):
        col = []
        for n in lens:
            v = rng.uniform(-1e3, 1e3, n).astype(npdt)
            col.append(rdf.PrimitiveArray.from_numpy(v, random_mask(rng, n, null_frac) if null_frac else None))
        got = rdf.AggregateFunctions.sum(col)
        again = rdf.AggregateFunctions.sum(col)
        assert got == again, "float sum must be run-to-run deterministic"
        exact, sum_abs = oracle.sum_exact(dtype, col)
        n = sum(lens)
        assert abs(np.longdouble(got) - exact) <= 16 * np.log2(n) * eps * sum_abs
        st, ref = oracle.aggregate(oracle.SUM, dtype, col)
        assert abs(np.longdouble(ref) - exact) <= n * eps * sum_abs   # the reference's own fold error bound
        assert rdf.AggregateFunctions.count(col) == oracle.aggregate(oracle.COUNT, dtype, col)[1]
    # NaN / inf propagate
    v = np.ones(5000, dtype=npdt)
    v[4000] = np.nan
    assert np.isnan(rdf.AggregateFunctions.sum([rdf.PrimitiveArray.from_numpy(v)]))
    v[4000] = np.inf
    assert np.isposinf(rdf.AggregateFunctions.sum([rdf.PrimitiveArray.from_numpy(v)]))
    # NaN under a null does not leak
    v[4000] = np.nan
    m = np.ones(5000, dtype=bool)
    m[4000] = False
    assert rdf.AggregateFunctions.sum([rdf.PrimitiveArray.from_numpy(v, m)]) == 4999


def test_avg_matches_reference_formula(rdf, ctx, oracle):
    rng = np.random.default_rng(23)
    for tname in ("I8", "I32", "U16", "F32", "F64"):
        dtype = getattr(rdf, tname)
        col = make_column(rdf, rng, dtype, [1000, 1, 30001, 17], 0.2, True)
        got = rdf.AggregateFunctions.avg(col)
        st, want = oracle.avg(dtype, col)
        assert st == oracle.OK
        import math
        vals = np.concatenate([c.value_slice()[c.valid_mask()] for c in col]).astype(np.float64)
        exact = math.fsum(vals) / len(vals)
        scale = float(np.abs(vals).max()) + 1.0
        assert abs(got - exact) <= 1e-12 * scale, (tname, got, exact)          # GPU: exact/double sums
        assert abs(want - exact) <= 1e-9 * scale, (tname, want, exact)         # reference: running mean drift
    with pytest.raises(rdf.UnsupportedType):
        rdf.AggregateFunctions.avg([rdf.PrimitiveArray.from_pylist(rdf.I64, [1])])
    assert rdf.AggregateFunctions.avg([rdf.PrimitiveArray.from_numpy(np.zeros(3, np.int32), np.zeros(3, bool))]) is None


# ---------------------------------------------------------------------------------------------------------
# device-resident chains, generator, pipelined uploads

def test_generator_matches_oracle(rdf, ctx, oracle):
    lens = [5, 4096, 0, 100003]
    cases = [(rdf.F64, 0, -1e3, 1e3, 10), (rdf.F64, 1, 0, 0, 0), (rdf.I64, 3, 0, 0, 20), (rdf.I64, 2, 0, 0, 0),
             (rdf.I32, 2, 0, 0, 10), (rdf.F32, 0, -5.0, 5.0, 3), (rdf.U8, 2, 0, 0, 2), (rdf.I16, 3, 0, 0, 0)]
    for dtype, kind, lo, hi, null_mod in cases:
        col = rdf.Column.generate(dtype, lens, kind=kind, lo=lo, hi=hi, seed=20260924, col_id=5, row0=1000, null_mod=null_mod)
        got = col.download()
        row = 1000
        for g, n in zip(got, lens):
            want = oracle.generate(dtype, kind, lo, hi, 20260924, 5, row, n, null_mod)
            assert_same_array(g, want, what=f"generate dtype={dtype} kind={kind}")
            row += n


def test_device_chain_config2_shape(rdf, ctx, oracle):
    """e=a+b; f=e*c; g=f/d; h=sin(g) without leaving HBM (SURVEY config 2, small), nulls on b and d."""
    lens = [4001, 1, 65536, 333]
    C = rdf.Column
    a = C.generate(rdf.F64, lens, 0, -1e3, 1e3, col_id=0)
    b = C.generate(rdf.F64, lens, 0, -1e3, 1e3, col_id=1, null_mod=10)
    c = C.generate(rdf.F64, lens, 0, -1e3, 1e3, col_id=2)
    d = C.generate(rdf.F64, lens, 1, col_id=3, null_mod=10)
    e = a.add(b); f = e.multiply(c); g = f.divide(d); h = g.sin()
    row, oa, ob, oc, od = 0, [], [], [], []
    for n in lens:
        oa.append(oracle.generate(oracle.F64, 0, -1e3, 1e3, 20260924, 0, row, n))
        ob.append(oracle.generate(oracle.F64, 0, -1e3, 1e3, 20260924, 1, row, n, 10))
        oc.append(oracle.generate(oracle.F64, 0, -1e3, 1e3, 20260924, 2, row, n))
        od.append(oracle.generate(oracle.F64, 1, 0, 0, 20260924, 3, row, n, 10))
        row += n
    _, oe = oracle.col_binary(oracle.ADD, oracle.F64, oa, ob)
    _, of = oracle.col_binary(oracle.MUL, oracle.F64, oe, oc)
    _, og = oracle.col_binary(oracle.DIV, oracle.F64, of, od)
    _, oh = oracle.col_unary(oracle.SIN, oracle.F64, og)
    for name, colx, want in (("e", e, oe), ("f", f, of), ("g", g, og)):
        for i, (gg, ww) in enumerate(zip(colx.download(), want)):
            assert_same_array(gg, ww, what=f"chain {name} chunk {i}")
    for i, (gg, ww) in enumerate(zip(h.download(), oh)):
        assert_same_array(gg, ww, what=f"chain h chunk {i}", exact=False, max_ulp=3, check_payload=False)
    assert h.count() == oracle.aggregate(oracle.COUNT, oracle.F64, oh)[1]
    info = h.chunk_info(2)
    assert info["len"] == 65536 and info["null_count"] == oh[2].null_count and info["has_validity"]


def test_pipelined_upload_groups(rdf, oracle):
    """Small BDF_PIPELINE_BYTES => many upload groups => operators run group by group while later chunks
    are still in flight; results must not depend on the grouping."""
    os.environ["BDF_PIPELINE_BYTES"] = "65536"
    try:
        c2 = rdf.Context(0)
    finally:
        del os.environ["BDF_PIPELINE_BYTES"]
    rng = np.random.default_rng(31)
    lens = [9000, 100, 20000, 1, 0, 50000, 8191, 30000]
    a = make_column(rdf, rng, rdf.I64, lens, 0.1, True)
    b = make_column(rdf, rng, rdf.I64, lens, 0.0, False)
    got = rdf.ScalarFunctions.add(a, b, ctx=c2)
    st, want = oracle.col_binary(oracle.ADD, oracle.I64, a, b)
    for i, (g, w) in enumerate(zip(got, want)):
        assert_same_array(g, w, what=f"pipelined add chunk {i}")
    ca = rdf.Column.upload(a, ctx=c2, asynchronous=True)
    cb = rdf.Column.upload(b, ctx=c2, asynchronous=True)
    s = ca.add(cb)
    f = s.cast(rdf.F64)
    assert int(s.sum()) == int(oracle.aggregate(oracle.SUM, oracle.I64, want)[1])
    _, wf = oracle.col_cast(oracle.I64, oracle.F64, want)
    for g, w in zip(f.download(pinned=True), wf):
        assert_same_array(g, w, what="pipelined cast")
    # a sliced column downloaded as-is gets its bitmap re-aligned to offset 0
    for g, src in zip(ca.download(), a):
        assert np.array_equal(g.valid_mask(), src.valid_mask()) and np.array_equal(g.value_slice(), src.value_slice())
    for col in (ca, cb, s, f):
        col.free()
    c2.close()


def test_pinned_host_buffers(rdf, ctx, oracle):
    rng = np.random.default_rng(41)
    v = rng.uniform(-1, 1, 100000)
    m = rng.random(100000) > 0.5
    a = ctx.pinned_array(rdf.F64, v, m)
    b = ctx.pinned_array(rdf.F64, v)
    got = rdf.ScalarFunctions.multiply([a], [b], pinned_out=True)[0]
    st, want = oracle.col_binary(oracle.MUL, oracle.F64, [a], [b])
    assert_same_array(got, want[0], what="pinned multiply")


# ---------------------------------------------------------------------------------------------------------
# full-size properties (BASELINE.json sizes): 1e8 rows, device-generated

def test_full_size_f64_add_sum_1e8(rdf, ctx, oracle):
    """The headline workload: 1e8-row f64 a+b then sum, 25 chunks x 4e6.  Bit-exact add on sampled chunks
    (regenerated by the oracle), sum within tolerance of the exact sum of the regenerated data."""
    lens = [4_000_000] * 25
    a = rdf.Column.generate(rdf.F64, lens, 0, -1e3, 1e3, col_id=0)
    b = rdf.Column.generate(rdf.F64, lens, 0, -1e3, 1e3, col_id=1)
    c = a.add(b)
    s = c.sum()
    assert c.count() == 100_000_000
    exact, sum_abs = np.longdouble(0), np.longdouble(0)
    sample = {0, 12, 24}
    row = 0
    got_chunks = None
    for i, n in enumerate(lens):
        oa = oracle.generate(oracle.F64, 0, -1e3, 1e3, 20260924, 0, row, n)
        ob = oracle.generate(oracle.F64, 0, -1e3, 1e3, 20260924, 1, row, n)
        _, oc = oracle.col_binary(oracle.ADD, oracle.F64, [oa], [ob])
        e, sa = oracle.sum_exact(oracle.F64, oc)
        exact += e
        sum_abs += sa
        if i in sample:
            if got_chunks is None:
                got_chunks = c.download()
            assert np.array_equal(got_chunks[i].value_slice().view(np.uint64), oc[0].values.view(np.uint64)), f"chunk {i}"
        row += n
    assert abs(np.longdouble(s) - exact) <= 16 * np.log2(1e8) * 2.0 ** -53 * sum_abs
    for col in (a, b, c):
        col.free()


def test_full_size_int64_linearity_1e8(rdf, ctx, oracle):
    """Size-independent properties at 1e8 rows with 10% nulls: wrapping linearity
    sum(a+b) == sum(a|valid both) + sum(b|valid both) is checked through count/sum identities:
    count(a+b) == rows - nulls(a or b);  sum over no-null columns: sum(a+b) == sum(a) + sum(b) (mod 2^64)."""
    lens = [4_000_000] * 25
    a = rdf.Column.generate(rdf.I64, lens, 2, col_id=7)           # full-range: proves wrapping parity
    b = rdf.Column.generate(rdf.I64, lens, 3, col_id=8)
    c = a.add(b)
    mask = (1 << 64) - 1
    assert (int(c.sum()) & mask) == ((int(a.sum()) + int(b.sum())) & mask)
    d = c.subtract(b)
    assert int(d.sum()) == int(a.sum()) and int(d.min()) == int(a.min()) and int(d.max()) == int(a.max())
    an = rdf.Column.generate(rdf.I64, lens, 3, col_id=9, null_mod=10)
    r = an.aggregate_all()
    assert r["rows"] == 100_000_000 and 0.099 < 1 - r["count"] / r["rows"] < 0.101
    assert -2 ** 40 <= int(r["min"]) < -2 ** 40 + 2 ** 20 and 2 ** 40 - 2 ** 20 < int(r["max"]) < 2 ** 40
    cn = an.add(b)
    assert cn.count() == r["count"]            # validity AND with a no-null column keeps the bitmap
    f = an.cast(rdf.F64)
    assert f.count() == r["count"] and abs(float(f.sum()) - float(int(r["sum"]))) <= 1e-6 * 2 ** 40
    # oracle spot check of one chunk of the nullable column (values, validity, aggregates)
    got = an.download()[3]
    want = oracle.generate(oracle.I64, 3, 0, 0, 20260924, 9, 3 * 4_000_000, 4_000_000, 10)
    assert_same_array(got, want, what="nullable i64 chunk 3")
    for col in (a, b, c, d, an, cn, f):
        col.free()


# ---------------------------------------------------------------------------------------------------------
# K5 fused operator + aggregate, async aggregates, split downloads

@pytest.mark.parametrize("tname", ALL_TYPES)
def test_fused_binary_aggregate_matches_two_pass(rdf, ctx, oracle, tname):
    dtype = getattr(rdf, tname)
    rng = np.random.default_rng(300 + dtype)
    lens = [n for n in RAGGED if n > 0]
    for null_a, null_b, sliced in [(0, 0, False), (0.1, 0.3, True)]:
        a = make_column(rdf, rng, dtype, lens, null_a, sliced)
        b = make_column(rdf, rng, dtype, lens, null_b, sliced, nonzero=True)
        ca, cb = rdf.Column.upload(a), rdf.Column.upload(b)
        for op, oop in ((rdf.native.ADD, oracle.ADD), (rdf.native.SUB, oracle.SUB), (rdf.native.MUL, oracle.MUL), (rdf.native.DIV, oracle.DIV)):
            col, agg = ca.binary_agg(op, cb)
            st, want = oracle.col_binary(oop, dtype, a, b)
            for i, (g, w) in enumerate(zip(col.download(), want)):
                assert_same_array(g, w, what=f"fused op {op} <{tname}> chunk {i}")
            two_pass = col.aggregate_all()
            st, cnt = oracle.aggregate(oracle.COUNT, dtype, want)
            assert agg["count"] == two_pass["count"] == cnt and agg["rows"] == sum(lens)
            if tname in INT_TYPES:
                for key, aop in (("sum", oracle.SUM), ("min", oracle.MIN), ("max", oracle.MAX)):
                    has_valid = [w for w in want if w.valid_mask().any()]
                    exp = oracle.aggregate(aop, dtype, has_valid)[1]
                    assert int(agg[key]) == int(two_pass[key]) == int(exp), (tname, op, key)
            else:
                exact, sum_abs = oracle.sum_exact(dtype, want)
                eps = 2.0 ** -53 if tname == "F64" else 2.0 ** -24
                assert abs(np.longdouble(agg["sum"]) - exact) <= 16 * np.log2(sum(lens)) * eps * sum_abs
            col.free()
        fut_col, fut = ca.binary_agg_async(rdf.native.ADD, cb)
        again = fut_col.aggregate_all_async()
        r1, r2 = fut.result(), again.result()
        assert r1["count"] == r2["count"] and (tname not in INT_TYPES or int(r1["sum"]) == int(r2["sum"]))
        for col in (ca, cb, fut_col):
            col.free()


def test_fused_aggregate_is_deterministic_and_rejects_math_ops(rdf, ctx):
    lens = [1_000_003, 17, 2_000_000]
    a = rdf.Column.generate(rdf.F64, lens, 0, -1e3, 1e3, col_id=0)
    b = rdf.Column.generate(rdf.F64, lens, 0, -1e3, 1e3, col_id=1, null_mod=7)
    sums = set()
    for _ in range(3):
        col, agg = a.add_agg(b)
        sums.add(float(agg["sum"]).hex())
        col.free()
    assert len(sums) == 1
    ctx.synchronize()
    before = pool_used(ctx)
    for op in (rdf.native.ATAN2, rdf.native.HYPOT, rdf.native.LOG):   # refused after the output column was made
        with pytest.raises(rdf.UnsupportedType):
            a.binary_agg(op, b)
    ctx.synchronize()
    assert pool_used(ctx) == before


def test_split_download_overlaps_and_matches(rdf, ctx, oracle):
    rng = np.random.default_rng(77)
    lens = [300_000, 5, 0, 123_457]
    a = make_column(rdf, rng, rdf.F64, lens, 0.1, True)
    b = make_column(rdf, rng, rdf.F64, lens, 0.0, False)
    ca = rdf.Column.upload(a, asynchronous=True)
    cb = rdf.Column.upload(b, asynchronous=True)
    cc, fut = ca.binary_agg_async(rdf.native.MUL, cb)
    into = rdf.native.alloc_outputs(rdf.F64, lens, ctx, pinned=True)
    cc.download_begin(into)
    agg = fut.result()
    got = cc.download_end(into)
    st, want = oracle.col_binary(oracle.MUL, oracle.F64, a, b)
    for g, w in zip(got, want):
        assert_same_array(g, w, what="split download")
    assert agg["count"] == oracle.aggregate(oracle.COUNT, oracle.F64, want)[1]
    # sliced column straight back to the host through the split path (bitmap re-aligned on the device)
    into2 = rdf.native.alloc_outputs(rdf.F64, lens, ctx)
    ca.download_begin(into2)
    for g, src in zip(ca.download_end(into2), a):
        assert np.array_equal(g.valid_mask(), src.valid_mask()) and np.array_equal(g.value_slice(), src.value_slice())


def test_concurrent_host_threads_share_one_context(rdf, ctx, oracle):
    """The reference calls arrive from rayon workers / user threads; one bdf_ctx must serialise them safely."""
    from concurrent.futures import ThreadPoolExecutor

    rng = np.random.default_rng(88)
    cols = [(make_column(rdf, rng, rdf.I64, [5000, 33, 20000], 0.1, True), make_column(rdf, rng, rdf.I64, [5000, 33, 20000], 0.2, False))
            for _ in range(8)]
    want = [oracle.col_binary(oracle.ADD, oracle.I64, a, b)[1] for a, b in cols]
    wsum = [int(oracle.aggregate(oracle.SUM, oracle.I64, w)[1]) for w in want]

    def work(k):
        a, b = cols[k % len(cols)]
        out = rdf.ScalarFunctions.add(a, b)
        s = rdf.AggregateFunctions.sum(out)
        return k % len(cols), out, int(s)

    with ThreadPoolExecutor(8) as ex:
        results = list(ex.map(work, range(64)))
    for k, out, s in results:
        assert s == wsum[k]
        for g, w in zip(out, want[k]):
            assert_same_array(g, w, what=f"threaded add {k}")


def test_c_abi_argument_validation(rdf, ctx):
    """Bad arguments come back as status codes with a message -- nothing aborts, nothing is silently computed."""
    import ctypes as C

    N = rdf.native
    L = N.lib()
    a = rdf.PrimitiveArray.from_numpy(np.arange(100, dtype=np.int32), np.arange(100) % 3 != 0)
    views = N.make_views([a])
    outs, bufs = N.alloc_outputs(rdf.I32, [100], ctx)
    assert L.bdf_binary(ctx.handle, N.ADD, 99, 1, views, 1, views, outs) == N.INVALID and b"dtype" in L.bdf_last_error()
    assert L.bdf_binary(ctx.handle, 99, rdf.I32, 1, views, 1, views, outs) == N.INVALID
    assert L.bdf_binary(None, N.ADD, rdf.I32, 1, views, 1, views, outs) == N.INVALID
    outs[0].len = 50                                         # capacity does not match the result length
    assert L.bdf_binary(ctx.handle, N.ADD, rdf.I32, 1, views, 1, views, outs) == N.INVALID and b"capacity" in L.bdf_last_error()
    outs[0].len = 100
    keep = outs[0].validity
    outs[0].validity = None                                  # the result has nulls but nowhere to put the bitmap
    assert L.bdf_binary(ctx.handle, N.ADD, rdf.I32, 1, views, 1, views, outs) == N.INVALID and b"validity" in L.bdf_last_error()
    outs[0].validity = keep
    assert L.bdf_binary(ctx.handle, N.ADD, rdf.I32, 1, views, 1, views, outs) == N.OK and outs[0].null_count == 34
    h = C.c_void_p()
    assert L.bdf_upload(ctx.handle, rdf.I32, -1, views, 0, C.byref(h)) == N.INVALID
    assert L.bdf_cast(ctx.handle, rdf.I32, 42, 1, views, outs) == N.INVALID
    some, out = C.c_int32(0), np.zeros(1, np.int64)
    assert L.bdf_aggregate(ctx.handle, 9, rdf.I32, 1, views, out.ctypes.data, C.byref(some)) == N.INVALID
    assert L.bdf_aggregate(ctx.handle, N.SUM, rdf.I32, 1, views, None, C.byref(some)) == N.INVALID
    # the context still works after all of that
    assert rdf.AggregateFunctions.count([a]) == 66
