"""N3 (SURVEY 8(f)): a chain of Calculations evaluated in one pass (bdf_eval_expr_dev) against the SAME chain run
node by node -- through the oracle (the reference's materialising evaluator, src/evaluation.rs:66-96) and through
the unfused CUDA calls.  Arithmetic chains are bit-exact; chains through libm carry the unary tolerance (<= 3 ulp
for sin vs glibc) and are bit-identical to the unfused CUDA chain, which runs the same device functions."""
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from helpers import assert_same_array, pool_used, random_mask

pytestmark = pytest.mark.gpu

RAGGED = [0, 1, 31, 33, 1023, 1024, 1025, 4099, 70001]


def make_col(rdf, rng, lens, null_frac, sliced, lo=-100.0, hi=100.0, zeros=False):
    out = []
    for k, n in enumerate(lens):
        pad = (3 + 7 * k) % 29 if sliced else 0
        v = rng.uniform(lo, hi, n + pad + 2)
        if zeros:
            v[::53] = 0.0
        a = rdf.PrimitiveArray.from_numpy(v, random_mask(rng, n + pad + 2, null_frac) if null_frac else None)
        a.null_count = -1 if a.validity is not None else 0
        out.append(a.slice(pad, n))
    return out


def oracle_chain(oracle, inputs, nodes):
    """Run the program one materialised Calculation at a time.  Returns (status, final chunks)."""
    slots = list(inputs)
    for nd in nodes:
        if len(nd) == 2:
            st, r = oracle.col_unary(getattr(oracle, nd[0].upper()), oracle.F64, slots[nd[1]])
        else:
            st, r = oracle.col_binary(nd[0], oracle.F64, slots[nd[1]], slots[nd[2]])
        if st != oracle.OK:
            return st, None
        slots.append(r)
    return oracle.OK, slots[-1]


def gpu_chain(cols, nodes):
    slots = list(cols)
    for nd in nodes:
        if len(nd) == 2:
            slots.append(getattr(slots[nd[1]], nd[0])())
        else:
            name = ["add", "subtract", "multiply", "divide"][nd[0]]
            slots.append(getattr(slots[nd[1]], name)(slots[nd[2]]))
    return slots[-1], slots[len(cols):-1]


@pytest.mark.parametrize("nulls", [(0, 0, 0, 0), (0.2, 0, 0, 0.1), (0.1, 0.3, 0.2, 0.1)])
def test_arithmetic_chain_bit_exact(rdf, ctx, oracle, nulls):
    rng = np.random.default_rng(int(sum(nulls) * 100))
    N = rdf.native
    host = [make_col(rdf, rng, RAGGED, nulls[i], sliced=bool(sum(nulls)), lo=(1.0 if i == 3 else -100.0)) for i in range(4)]
    cols = [rdf.Column.upload(h) for h in host]
    programs = [
        [(N.ADD, 0, 1)],
        [(N.ADD, 0, 1), (N.MUL, 4, 2), (N.DIV, 5, 3)],
        [(N.SUB, 0, 1), (N.MUL, 4, 4), (N.ADD, 5, 2), (N.DIV, 6, 3), (N.SUB, 7, 0), ("abs", 8)],
        [("abs", 2), ("sqrt", 4), ("floor", 5), (N.MUL, 6, 3)],
        # both operands intermediate at two levels -> both temporaries: ((a+b)*(c-d)) / ((a-b)+(c*d)) ... - a
        [(N.ADD, 0, 1), (N.SUB, 2, 3), (N.MUL, 4, 5), (N.SUB, 0, 1), (N.MUL, 2, 3), (N.ADD, 7, 8), (N.SUB, 6, 9), (N.SUB, 10, 0)],
        # a shared sub-expression used three times, once reversed (x - s), once with itself
        [(N.ADD, 0, 1), (N.MUL, 4, 4), (N.SUB, 2, 4), (N.ADD, 5, 6), (N.MUL, 7, 4), (N.DIV, 8, 3)],
    ]
    for prog in programs:
        got = rdf.eval_expr(cols, prog).download()
        st, want = oracle_chain(oracle, host, prog)
        assert st == oracle.OK
        for i, (g, w) in enumerate(zip(got, want)):
            assert_same_array(g, w, what=f"expr {prog} chunk {i} nulls={nulls}", check_payload=False)
            if g.validity is not None:   # null slots of a fused result carry payload 0
                assert not g.value_slice()[~g.valid_mask()].any()
    for c in cols:
        c.free()


def test_trig_chain_matches_unfused_gpu_and_oracle(rdf, ctx, oracle):
    rng = np.random.default_rng(11)
    N = rdf.native
    host = [make_col(rdf, rng, RAGGED, nf, sliced=True, lo=lo) for nf, lo in ((0, -100.0), (0.2, -100.0), (0, -100.0), (0.1, 1.0))]
    cols = [rdf.Column.upload(h) for h in host]
    prog = [(N.ADD, 0, 1), (N.MUL, 4, 2), (N.DIV, 5, 3), ("sin", 6)]
    fused = rdf.eval_expr(cols, prog)
    unfused, tmp = gpu_chain(cols, prog)
    st, want = oracle_chain(oracle, host, prog)
    gf, gu = fused.download(), unfused.download()
    for i in range(len(RAGGED)):
        assert_same_array(gf[i], want[i], what=f"sin chain chunk {i}", exact=False, max_ulp=3, check_payload=False)
        m = gf[i].valid_mask()
        assert np.array_equal(m, gu[i].valid_mask())
        assert np.array_equal(gf[i].value_slice()[m].view(np.uint64), gu[i].value_slice()[m].view(np.uint64))
    assert fused.count() == unfused.count()
    for prog2, tol in (([("cos", 0), ("tan", 2), (N.ATAN2, 4, 5), (N.HYPOT, 6, 3)], 6), ([("exp", 3), ("log2", 4), ("tanh", 5), ("cbrt", 6)], 6)):
        got = rdf.eval_expr(cols, prog2).download()
        slots = list(host)
        for nd in prog2:   # atan2/hypot live in col_binary like the arithmetic ops
            if len(nd) == 2:
                _, r = oracle.col_unary(getattr(oracle, nd[0].upper()), oracle.F64, slots[nd[1]])
            else:
                _, r = oracle.col_binary(nd[0], oracle.F64, slots[nd[1]], slots[nd[2]])
            slots.append(r)
        for i, (g, w) in enumerate(zip(got, slots[-1])):
            # each libm node is within its own 2-4 ulp of glibc, but an error entering tan/exp is amplified by the
            # function's condition number: compare the VALIDITY exactly and the values with a relative bound.
            assert np.array_equal(g.valid_mask(), w.valid_mask())
            m = g.valid_mask()
            gv, wv = g.value_slice()[m], w.values[w.offset:w.offset + w.length][m]
            ok = np.isclose(gv, wv, rtol=1e-9, atol=0, equal_nan=True)
            assert ok.all(), f"{prog2} chunk {i}: {gv[~ok][:4]} vs {wv[~ok][:4]}"


def test_divide_by_zero_follows_the_materialised_chain(rdf, ctx, oracle):
    rng = np.random.default_rng(3)
    N = rdf.native
    lens = [5000, 33]
    a = make_col(rdf, rng, lens, 0, False)
    z = make_col(rdf, rng, lens, 0, False, zeros=True)
    # z null exactly where it is zero -> no error; a zero divisor under a NULL numerator slot -> no error either
    zmask = [rdf.PrimitiveArray.from_numpy(c.value_slice().copy(), c.value_slice() != 0.0) for c in z]
    anull = [rdf.PrimitiveArray.from_numpy(c.value_slice().copy(), zc.value_slice() != 0.0) for c, zc in zip(a, z)]
    ca, cz, czm, can = (rdf.Column.upload(x) for x in (a, z, zmask, anull))
    with pytest.raises(rdf.DivideByZero):
        rdf.eval_expr([ca, cz], [(N.ADD, 0, 0), (N.DIV, 2, 1)])
    assert oracle_chain(oracle, [a, z], [(N.ADD, 0, 0), (N.DIV, 2, 1)])[0] == oracle.DIVIDE_BY_ZERO
    for ins, hs in (([ca, czm], [a, zmask]), ([can, cz], [anull, z])):
        prog = [(N.ADD, 0, 0), (N.DIV, 2, 1), (N.MUL, 3, 0)]
        got = rdf.eval_expr(ins, prog).download()
        st, want = oracle_chain(oracle, hs, prog)
        assert st == oracle.OK
        for g, w in zip(got, want):
            assert_same_array(g, w, what="masked zero divisors", check_payload=False)
    # a zero that only appears in an INTERMEDIATE (a - a) is found too; the refused calls drop their output columns
    ctx.synchronize()
    before = pool_used(ctx)
    with pytest.raises(rdf.DivideByZero):
        rdf.eval_expr([ca], [(N.SUB, 0, 0), (N.DIV, 0, 1)])
    with pytest.raises(rdf.DivideByZero):
        rdf.eval_expr([ca, cz], [(N.ADD, 0, 0), (N.DIV, 2, 1)])
    ctx.synchronize()
    assert pool_used(ctx) == before


def test_argument_validation(rdf, ctx):
    N = rdf.native
    a = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.arange(10.0))])
    b = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.arange(11.0))])
    i = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.arange(10, dtype=np.int64))])
    with pytest.raises(rdf.ComputeError):
        rdf.eval_expr([a, b], [(N.ADD, 0, 1)])
    assert np.array_equal(rdf.eval_expr([a, i], [(N.ADD, 0, 1)]).download()[0].value_slice(), 2 * np.arange(10.0))   # Int64 input read `as f64`
    with pytest.raises(rdf.UnsupportedType):
        rdf.eval_expr([a, a.gt(3.0)], [(N.ADD, 0, 1)])            # a boolean column is not numeric
    for bad in ([(N.ADD, 0, 2)], [(N.ADD, 0, 1), (N.MUL, 3, 0)], [(99, 0, 0)], [(N.EXPR_UNARY + 50, 0)], [(N.ADD, 0, 0)] * 13):
        with pytest.raises(rdf.ArrowError):
            rdf.eval_expr([a, a], bad)
    with pytest.raises(rdf.ArrowError):
        rdf.eval_expr([a] * 7, [(N.ADD, 0, 1)])
    with pytest.raises(rdf.ArrowError):          # a dead node: the materialised chain would still evaluate it
        rdf.eval_expr([a, a], [(N.DIV, 0, 1), (N.ADD, 0, 1)])
    with pytest.raises(rdf.UnsupportedType):     # three shared intermediates alive at once: more than the two temporaries
        rdf.eval_expr([a, a], [(N.ADD, 0, 1), (N.SUB, 0, 1), (N.MUL, 0, 1), (N.MUL, 2, 3), (N.MUL, 5, 4), (N.ADD, 6, 2), (N.ADD, 7, 3),
                               (N.ADD, 8, 4)])
    out = rdf.eval_expr([a, a], [(N.ADD, 0, 1), (N.MUL, 2, 2)]).download()[0]
    assert np.array_equal(out.value_slice(), (2 * np.arange(10.0)) ** 2)


def test_trailing_aggregate_matches_two_pass(rdf, ctx, oracle):
    """sum/count of the chain's last column folded into the same pass: equal to aggregating the materialised column
    (same per-tile fold order is not required -- the tolerance is the float-sum bound of the aggregate tests), the
    column bit-identical to eval_expr's, deterministic run to run, and the column is optional."""
    rng = np.random.default_rng(21)
    N = rdf.native
    lens = [0, 5, 2047, 2048, 2049, 300_001]
    host = [make_col(rdf, rng, lens, nf, sliced=True, lo=lo) for nf, lo in ((0, -100.0), (0.2, -100.0), (0.1, 1.0))]
    cols = [rdf.Column.upload(h) for h in host]
    prog = [(N.ADD, 0, 1), (N.DIV, 3, 2), ("cos", 4)]
    plain = rdf.eval_expr(cols, prog)
    col, agg = rdf.eval_expr_agg(cols, prog)
    none, agg2 = rdf.eval_expr_agg(cols, prog, materialise=False)
    _, fut = rdf.eval_expr_agg(cols, prog, materialise=False, asynchronous=True)
    assert none is None
    want_chunks = plain.download()
    for g, w in zip(col.download(), want_chunks):
        assert np.array_equal(g.valid_mask(), w.valid_mask())
        assert np.array_equal(g.value_slice().view(np.uint64), w.value_slice().view(np.uint64))
    valid = np.concatenate([w.value_slice()[w.valid_mask()] for w in want_chunks])
    exact = np.sum(valid.astype(np.longdouble))
    bound = 16 * np.log2(valid.size) * 2.0 ** -53 * np.sum(np.abs(valid).astype(np.longdouble))
    assert agg["count"] == valid.size == plain.count() and agg["rows"] == sum(lens)
    assert abs(np.longdouble(agg["sum"]) - exact) <= bound
    assert agg["min"] is None and agg["max"] is None
    assert agg2 == agg and fut.result() == agg                     # same tiles, same fold: bit-identical sums
    assert abs(agg["sum"] - plain.sum()) <= 2 * float(bound)
    # DivideByZero wins over the aggregate; an all-null result has count 0 and sum 0
    z = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.zeros(n)) for n in lens])
    with pytest.raises(rdf.DivideByZero):
        rdf.eval_expr_agg([cols[0], z], [(N.DIV, 0, 1)], materialise=False)
    nulls = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.ones(n), np.zeros(n, bool)) for n in lens])
    _, a0 = rdf.eval_expr_agg([cols[0], nulls], [(N.MUL, 0, 1)], materialise=False)
    assert a0["count"] == 0 and a0["sum"] == 0.0


@pytest.mark.parametrize("tname", ["I8", "I16", "I32", "I64", "U8", "U16", "U32", "U64", "F32"])
def test_non_float64_inputs_are_cast_on_load(rdf, ctx, oracle, tname):
    """An input column of another numeric type = Function::Cast to Float64 (`as f64`, infallible, validity kept)
    followed by the chain: compared with the oracle's cast + materialised chain, bit for bit."""
    dtype = getattr(rdf, tname)
    npdt = np.dtype(rdf.NP_DTYPES[dtype])
    rng = np.random.default_rng(50 + dtype)
    N = rdf.native
    typed, other = [], []
    for k, n in enumerate(RAGGED):
        pad = (5 + 3 * k) % 17
        if npdt.kind == "f":
            v = rng.normal(0, 1e3, n + pad + 2).astype(npdt)
        else:
            info = np.iinfo(npdt)
            v = rng.integers(info.min, info.max, n + pad + 2, dtype=npdt, endpoint=True)
        a = rdf.PrimitiveArray.from_numpy(v, random_mask(rng, n + pad + 2, 0.2))
        a.null_count = -1
        typed.append(a.slice(pad, n))
        other.append(rdf.PrimitiveArray.from_numpy(rng.uniform(1.0, 9.0, n)))
    ct, co = rdf.Column.upload(typed), rdf.Column.upload(other)
    prog = [(N.MUL, 0, 1), (N.SUB, 2, 0), (N.DIV, 3, 1), ("abs", 4)]
    got = rdf.eval_expr([ct, co], prog).download()
    st, as_f64 = oracle.col_cast(dtype, oracle.F64, typed)
    assert st == oracle.OK
    st, want = oracle_chain(oracle, [as_f64, other], prog)
    assert st == oracle.OK
    for i, (g, w) in enumerate(zip(got, want)):
        assert_same_array(g, w, what=f"expr over {tname} chunk {i}", check_payload=False)
    # and against the unfused device path: cast_dev, then the chain
    unfused, _ = gpu_chain([ct.cast(rdf.F64), co], prog)
    for g, u in zip(got, unfused.download()):
        m = g.valid_mask()
        assert np.array_equal(m, u.valid_mask()) and np.array_equal(g.value_slice()[m].view(np.uint64), u.value_slice()[m].view(np.uint64))


def test_config2_chain_fused_1e8(rdf, ctx, oracle):
    """BASELINE config 2 at full size in ONE pass: h = sin(((a+b)*c)/d), 10% nulls on b and d."""
    CH, NCH = 4_000_000, 25
    lens = [CH] * NCH
    C, N = rdf.Column, rdf.native
    a = C.generate(rdf.F64, lens, 0, -1e3, 1e3, col_id=20)
    b = C.generate(rdf.F64, lens, 0, -1e3, 1e3, col_id=21, null_mod=10)
    c = C.generate(rdf.F64, lens, 0, -1e3, 1e3, col_id=22)
    d = C.generate(rdf.F64, lens, 1, col_id=23, null_mod=10)
    prog = [(N.ADD, 0, 1), (N.MUL, 4, 2), (N.DIV, 5, 3), ("sin", 6)]
    h, agg = rdf.eval_expr_agg([a, b, c, d], prog)
    _, agg_only = rdf.eval_expr_agg([a, b, c, d], prog, materialise=False)
    got = h.download()
    hcount = h.count()

    def ref(i):
        g = lambda col, kind=0, lo=-1e3, hi=1e3, nm=0: oracle.generate(oracle.F64, kind, lo, hi, 20260924, col, i * CH, CH, nm)
        oa, ob, oc, od = g(20), g(21, nm=10), g(22), g(23, 1, 0, 0, 10)
        st, w = oracle_chain(oracle, [[oa], [ob], [oc], [od]], [(oracle.ADD, 0, 1), (oracle.MUL, 4, 2), (oracle.DIV, 5, 3), ("sin", 6)])
        assert st == oracle.OK
        return w[0]

    with ThreadPoolExecutor(16) as ex:
        refs = list(ex.map(ref, range(NCH)))
    count, exact, sum_abs = 0, np.longdouble(0), np.longdouble(0)
    for i, w in enumerate(refs):
        assert_same_array(got[i], w, what=f"fused cfg2 chunk {i}", exact=False, max_ulp=3, check_payload=False)
        count += w.length - w.null_count
        e, sa = oracle.sum_exact(oracle.F64, [w])
        exact += e; sum_abs += sa
    assert hcount == count == agg["count"] and agg_only == agg
    # sum(h): 3 ulp of |sin| <= 1 per element on top of the float-sum bound
    assert abs(np.longdouble(agg["sum"]) - exact) <= 16 * np.log2(1e8) * 2.0 ** -53 * sum_abs + 3 * 2.0 ** -53 * count
