"""The float function library on the GPU at the edges of every domain, against the oracle (glibc) AND the correctly
rounded reference of tests/math_reference.py.

Inputs: the edge set, the uniform values and the bit-pattern sweep of each function and width, laid out so that
every edge runs through both paths of the streaming kernels -- once inside a chunk longer than a tile (the vector
path of a full tile) and once at the end of a chunk (the scalar tail path) -- in sliced chunks with about 10% nulls.
An edge that is null in the long chunk is valid in the tail chunks.

Bars (the existing ones of test_parity_gpu.py, not loosened):
  * results fixed by IEEE 754 / Annex F, and results whose true value is a float that glibc returns (log2(2^k),
    log10(10^k), cbrt of a cube, exp(0), ceil / floor / round / sqrt / abs, ...): bit-exact, sign of zero included;
  * every other value: within TRIG_TOL / N1_TOL of the true value, and within the same bar of glibc wherever glibc
    itself is within 1 ulp of the true value (test_math_reference.py pins where it is not);
  * the fused kernel (eval_expr, Float64): bit-identical to the unfused kernels for all 21 unaries and atan2 / hypot /
    log, alone and inside two-node chains, and eval_expr_agg counts what the unfused column counts;
  * cast: int -> float ties, f64 -> f32 ties and the float -> int window bounds bit-exact against the oracle and an
    exact int / Fraction reference.
"""
import numpy as np
import pytest

import math_reference as R
from helpers import assert_same_array
from test_parity_gpu import N1_TOL, TRIG_TOL

pytestmark = pytest.mark.gpu

TILE = {"F64": 2048, "F32": 4096}          # rows of one k_unary / k_binary tile (16 KiB of the widest array)
EXPR_TILE = 2048                           # rows of one k_expr tile
EXACT_UNARIES = {"abs", "ceil", "floor", "round", "sqrt", "degrees", "radians"}
BINARY_TOL = {"F64": 4, "F32": 6}          # the bar of test_math_op_binaries


def unary_tol(name, tname):
    if name in EXACT_UNARIES:
        return 0
    return TRIG_TOL[tname] if name in ("sin", "cos", "tan") else N1_TOL[tname]


@pytest.fixture(scope="module")
def unary_refs():
    return {(n, t): R.unary_case(n, t) for t in ("F64", "F32") for n in R.UNARIES}


@pytest.fixture(scope="module")
def binary_refs():
    return {(n, t): R.binary_case(n, t) for t in ("F64", "F32") for n in R.BINARIES}


def layout(n_points, n_edges, tile, seed):
    """Row indices (into the point array, whose first n_edges points are the edges) of each chunk, and which rows
    are valid.  Chunk 0 holds every point with the edges in its body, well inside full tiles; every following chunk
    ends with a piece of the edges, in the partial last tile."""
    rng = np.random.default_rng(seed)
    rest = np.arange(n_edges, n_points)
    head = rest[: tile // 2]
    idx = [np.concatenate([head, np.arange(n_edges), rest[tile // 2:]])]
    assert n_edges + len(head) <= (len(idx[0]) // tile) * tile, "the edges must lie in full tiles of chunk 0"
    piece = tile // 4
    for k, s in enumerate(range(0, n_edges, piece)):
        edges = np.arange(s, min(s + piece, n_edges))
        filler = rng.choice(rest, (tile + 3 + 7 * k) if k % 2 else (5 + k), replace=True)
        idx.append(np.concatenate([filler, edges]))
    valid0 = rng.random(len(idx[0])) >= 0.1
    null_in_0 = np.zeros(n_points, bool)
    null_in_0[idx[0][~valid0]] = True
    masks = [valid0] + [(rng.random(len(i)) >= 0.1) | null_in_0[i] for i in idx[1:]]
    return idx, masks


def make_chunks(rdf, x, idx, masks):
    """Sliced PrimitiveArrays with the given rows and validity (non-zero, non-byte-aligned offsets)."""
    out = []
    for k, (i, m) in enumerate(zip(idx, masks)):
        pad = (3 + 5 * k) % 29
        filler = np.resize(x, pad + 2)
        v = np.concatenate([filler[:pad], x[i], filler[pad:]])
        mm = np.concatenate([np.ones(pad, bool), m, np.ones(2, bool)])
        arr = rdf.PrimitiveArray.from_numpy(v, mm)
        arr.null_count = -1
        out.append(arr.slice(pad, len(i)))
    return out


def check_values(what, got, orc, ref_vals, exact, tol):
    """got / orc: values of the valid rows; ref_vals: the correctly rounded values; exact: rows held bit-exact."""
    bad = np.nonzero(exact & ~(R.same_bits(got, orc) & R.same_bits(got, ref_vals)))[0]
    assert bad.size == 0, f"{what}: {bad.size} exact results differ, first got {got[bad[:4]].tolist()}, glibc {orc[bad[:4]].tolist()}, true {ref_vals[bad[:4]].tolist()}"
    d_true = R.ulps(got, ref_vals)
    bad = np.nonzero(~exact & (d_true > tol))[0]
    assert bad.size == 0, f"{what}: {int(d_true[bad].max())} ulp from the true value > {tol}: got {got[bad[:4]].tolist()}, true {ref_vals[bad[:4]].tolist()}"
    glibc_close = R.ulps(orc, ref_vals) <= 1
    d_orc = R.ulps(got, orc)
    bad = np.nonzero(~exact & glibc_close & (d_orc > tol))[0]
    assert bad.size == 0, f"{what}: {int(d_orc[bad].max())} ulp from glibc > {tol}: got {got[bad[:4]].tolist()}, glibc {orc[bad[:4]].tolist()}"
    return int(d_true.max()) if d_true.size else 0


# ---- a. every unary x {F32, F64} through ScalarFunctions ----------------------------------------------------------

@pytest.mark.parametrize("tname", ["F64", "F32"])
@pytest.mark.parametrize("name", R.UNARIES)
def test_unary_edges(rdf, ctx, oracle, unary_refs, name, tname):
    ref = unary_refs[(name, tname)]
    x = ref.x[0]
    n_edges = len(R.unary_points(name, tname)[0])
    idx, masks = layout(len(x), n_edges, TILE[tname], seed=R.UNARIES.index(name))
    chunks = make_chunks(rdf, x, idx, masks)
    dtype = getattr(rdf, tname)
    got = getattr(rdf.ScalarFunctions, name)(chunks)
    st, want = oracle.col_unary(getattr(oracle, name.upper()), dtype, chunks)
    assert st == oracle.OK
    glibc_exact = ref.ieee | (ref.representable & R.same_bits(
        oracle.col_unary(getattr(oracle, name.upper()), dtype, [rdf.PrimitiveArray.from_numpy(x)])[1][0].values, ref.values))
    tol = unary_tol(name, tname)
    seen = np.zeros(n_edges, bool)
    for k, (g, w, i) in enumerate(zip(got, want, idx)):
        m = g.valid_mask()
        assert np.array_equal(m, w.valid_mask()), f"{name}<{tname}> chunk {k}: validity"
        assert not g.value_slice()[~m].any(), f"{name}<{tname}> chunk {k}: null payload must be 0"
        iv = i[m]
        check_values(f"{name}<{tname}> chunk {k}", g.value_slice()[m], w.values[m], ref.values[iv],
                     np.ones(iv.size, bool) if tol == 0 else glibc_exact[iv], tol)
        seen[iv[iv < n_edges]] = True
    assert seen.all(), "every edge must be valid somewhere"


# ---- b. the fused path (Float64) --------------------------------------------------------------------------------

def same_column(what, a, b):
    """Two downloaded device columns: same validity, same bits in every valid slot, payload 0 in the null slots."""
    for k, (x, y) in enumerate(zip(a, b)):
        m = x.valid_mask()
        assert np.array_equal(m, y.valid_mask()), f"{what} chunk {k}: validity"
        bad = np.nonzero(~R.same_bits(x.value_slice()[m], y.value_slice()[m]))[0]
        assert bad.size == 0, f"{what} chunk {k}: {bad.size} values differ, fused {x.value_slice()[m][bad[:4]].tolist()} vs unfused {y.value_slice()[m][bad[:4]].tolist()}"
        assert not x.value_slice()[~m].any()


def factor_chunks(rdf, idx, seed):
    """A second input of the same shape: 1, 0.5 or 2 (exact scalings) with its own 10% nulls."""
    rng = np.random.default_rng(seed)
    return make_chunks(rdf, rng.choice(np.array([1.0, 0.5, 2.0]), max(len(i) for i in idx) + 64),
                       [np.arange(len(i)) for i in idx], [rng.random(len(i)) >= 0.1 for i in idx])


@pytest.mark.parametrize("name", R.UNARIES)
def test_fused_unary_matches_unfused(rdf, ctx, unary_refs, name):
    N = rdf.native
    op = getattr(N, name.upper())
    x = unary_refs[(name, "F64")].x[0]
    idx, masks = layout(len(x), len(R.unary_points(name, "F64")[0]), EXPR_TILE, seed=100 + op)
    a = rdf.Column.upload(make_chunks(rdf, x, idx, masks), ctx=ctx)
    f = rdf.Column.upload(factor_chunks(rdf, idx, 200 + op), ctx=ctx)
    cases = [([a], [(name, 0)], lambda: a.unary(op)),
             ([a, f], [(N.MUL, 0, 1), (name, 2)], lambda: a.multiply(f).unary(op)),
             ([a, f], [(name, 0), (N.ADD, 2, 1)], lambda: a.unary(op).add(f))]
    for inputs, prog, unfused in cases:
        fused_col, u = rdf.eval_expr(inputs, prog), unfused()
        same_column(f"{prog}", fused_col.download(), u.download())
        _, agg = rdf.eval_expr_agg(inputs, prog, materialise=False)
        assert agg["count"] == u.count() == fused_col.count(), prog
        fused_col.free()
        u.free()
    a.free()
    f.free()


@pytest.mark.parametrize("name", R.BINARIES)
def test_fused_binary_matches_unfused(rdf, ctx, binary_refs, name):
    N = rdf.native
    op = getattr(N, name.upper())
    ref = binary_refs[(name, "F64")]
    n_edges = len(R.binary_specials("F64")) ** 2
    idx, masks = layout(len(ref.x[0]), n_edges, EXPR_TILE, seed=300 + op)
    a = rdf.Column.upload(make_chunks(rdf, ref.x[0], idx, masks), ctx=ctx)
    b = rdf.Column.upload(make_chunks(rdf, ref.x[1], idx, [np.roll(m, 1) | m for m in masks]), ctx=ctx)
    col_op = lambda l, r: getattr(l, name)(r)          # Column.atan2 / hypot / log
    for prog, unfused in (([(op, 0, 1)], lambda: col_op(a, b)),
                          ([(op, 0, 1), (N.MUL, 2, 1)], lambda: col_op(a, b).multiply(b)),
                          ([(N.ADD, 0, 0), (op, 2, 1)], lambda: col_op(a.add(a), b))):
        fused_col, u = rdf.eval_expr([a, b], prog), unfused()
        same_column(f"{prog}", fused_col.download(), u.download())
        _, agg = rdf.eval_expr_agg([a, b], prog, materialise=False)
        assert agg["count"] == u.count(), prog
        fused_col.free()
        u.free()
    a.free()
    b.free()


# ---- c. the math binaries, both widths --------------------------------------------------------------------------

@pytest.mark.parametrize("tname", ["F64", "F32"])
@pytest.mark.parametrize("name", R.BINARIES)
def test_math_binary_edges(rdf, ctx, oracle, binary_refs, name, tname):
    """The cross product of the specials and the sweep: Annex F / formula results and representable results
    bit-exact (sign of zero included), every other value within the bar of test_math_op_binaries."""
    ref = binary_refs[(name, tname)]
    a, b = ref.x
    dtype = getattr(rdf, tname)
    rng = np.random.default_rng(400 + R.BINARIES.index(name))
    pad = 13
    ma = np.concatenate([np.ones(pad, bool), rng.random(len(a)) >= 0.1])
    A = rdf.PrimitiveArray.from_numpy(np.concatenate([a[:pad], a]), ma).slice(pad, len(a))
    B = rdf.PrimitiveArray.from_numpy(np.concatenate([b[:pad], b]), None).slice(pad, len(b))
    A.null_count = -1
    got = getattr(rdf.ScalarFunctions, name)(A, B)
    st, want = oracle.col_binary(getattr(oracle, name.upper()), dtype, [A], [B])
    assert st == oracle.OK
    m = got.valid_mask()
    assert np.array_equal(m, want[0].valid_mask()) and not got.value_slice()[~m].any()
    full = oracle.col_binary(getattr(oracle, name.upper()), dtype, [rdf.PrimitiveArray.from_numpy(a)], [rdf.PrimitiveArray.from_numpy(b)])[1][0].values
    exact = ref.ieee | (ref.representable & R.same_bits(full, ref.values))
    n_sp = len(R.binary_specials(tname)) ** 2
    assert m[:n_sp].mean() > 0.8
    check_values(f"{name}<{tname}>", got.value_slice()[m], want[0].values[m], ref.values[m], exact[m], BINARY_TOL[tname])
    # the nulls hid ~10% of the cross product: run it once more without any
    sp = rdf.ScalarFunctions
    g2 = getattr(sp, name)(rdf.PrimitiveArray.from_numpy(a[:n_sp]), rdf.PrimitiveArray.from_numpy(b[:n_sp])).value_slice()
    check_values(f"{name}<{tname}> specials", g2, full[:n_sp], ref.values[:n_sp], exact[:n_sp], BINARY_TOL[tname])


# ---- d. cast ties and window bounds -------------------------------------------------------------------------------

INT_NAMES = ["I8", "I16", "I32", "I64", "U8", "U16", "U32", "U64"]


def cast_chunks(rdf, x, tile, seed):
    """Every value in full tiles of chunk 0 (10% nulls), and again, always valid, at the end of a chunk whose last
    tile is partial."""
    rng = np.random.default_rng(seed)
    reps = -(-(len(x) + tile) // len(x))
    idx = [np.arange(len(x) * reps) % len(x)]
    masks = [rng.random(len(idx[0])) >= 0.1]
    piece = tile // 4
    for k, s in enumerate(range(0, len(x), piece)):
        vals = np.arange(s, min(s + piece, len(x)))
        filler = rng.integers(0, len(x), (tile + 3 + 7 * k) if k % 2 else (5 + k))
        idx.append(np.concatenate([filler, vals]))
        masks.append(np.concatenate([rng.random(len(filler)) >= 0.1, np.ones(len(vals), bool)]))
    return make_chunks(rdf, x, idx, masks), idx


def check_cast(rdf, oracle, from_name, to_name, x, exact_fn):
    f, t = getattr(rdf, from_name), getattr(rdf, to_name)
    w = max(np.dtype(rdf.NP_DTYPES[f]).itemsize, np.dtype(rdf.NP_DTYPES[t]).itemsize)
    chunks, idx = cast_chunks(rdf, x, 16384 // w, seed=f * 16 + t)
    got = rdf.cast(chunks, t)
    st, want = oracle.col_cast(f, t, chunks)
    assert st == oracle.OK
    exact = [exact_fn(v) for v in x.tolist()]
    for k, (g, o, i) in enumerate(zip(got, want, idx)):
        assert_same_array(g, o, what=f"cast {from_name}->{to_name} chunk {k}")
        m = g.valid_mask()
        in_valid = chunks[k].valid_mask()
        assert np.array_equal(m, in_valid & np.array([exact[j] is not None for j in i])), f"cast {from_name}->{to_name} chunk {k}: validity"
        vals = g.value_slice()
        npdt = np.dtype(rdf.NP_DTYPES[t])
        ref = np.array([0 if exact[j] is None else exact[j] for j in i], dtype=npdt)
        if npdt.kind == "f":
            bad = np.nonzero(m & ~R.same_bits(vals, ref))[0]
        else:
            bad = np.nonzero(m & (vals != ref))[0]
        assert bad.size == 0, f"cast {from_name}->{to_name} chunk {k}: got {vals[bad[:4]].tolist()} for {x[i[bad[:4]]].tolist()}, exact {ref[bad[:4]].tolist()}"


@pytest.mark.parametrize("iname", ["I32", "I64", "U32", "U64"])
def test_cast_int_to_float_ties(rdf, ctx, oracle, iname):
    for tname in ("F32", "F64"):
        vals = R.int_to_float_ties(iname, tname)
        if not vals:
            continue
        x = np.array(vals, rdf.NP_DTYPES[getattr(rdf, iname)])
        check_cast(rdf, oracle, iname, tname, x, lambda v, t=tname: R.exact_int_to_float(int(v), t))


def test_cast_f64_to_f32_ties(rdf, ctx, oracle):
    check_cast(rdf, oracle, "F64", "F32", R.float_to_float_ties(), R.exact_f64_to_f32)


@pytest.mark.parametrize("fname", ["F32", "F64"])
def test_cast_float_to_int_window_bounds(rdf, ctx, oracle, fname):
    for iname in INT_NAMES:
        check_cast(rdf, oracle, fname, iname, R.float_to_int_bounds(fname, iname),
                   lambda v, i=iname: R.exact_float_to_int(float(v), i))
