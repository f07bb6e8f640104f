"""The streaming kernels where their geometry changes, against the CPU oracle and exact aggregates.

Every streaming kernel picks its tile from the dtype and has a full-tile fast path whose code differs from its tail path; the
reductions add packed 8/16-bit lanes, K tiles per CTA and a fold of partials whose grid is capped by the SM count; the element-wise
operators run chunk group by chunk group while uploads are in flight.  The tests here put chunk ends, bit offsets, planted extremes
and partial counts exactly where those paths meet:

  * TILE: the tile of every kernel and dtype, restated from csrc/ (a non-GPU test re-reads the constants, so a retuned kernel
    fails loudly here instead of silently testing the wrong edges);
  * tile edges: chunks of 1, T-1, T, T+1, 2T-1, 2T+1 rows (and K*T-1, K*T, K*T+1 for the reduction), without a bitmap, with
    ~10 % nulls, and sliced at every bit offset 0..7 -- bit-exact, null counts per chunk included;
  * planted extremes: one valid minimum and one valid maximum in a narrow body, the type's MIN and MAX under nulls around them,
    swept over every slot of a 16-byte vector, lanes, warps, unroll steps, the K tiles of a reduce CTA and the tail;
  * aggregate_all_many on one GPU over interleaved dtypes and odd chunkings; fold grids past their SM cap; pipelined groups.
"""
import math
import os
import re

import numpy as np
import pytest

from helpers import assert_same_array, random_mask
import temporal_oracle as TO

gpu = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "rust-dataframe_b200", "csrc")

ALL_TYPES = ["I8", "I16", "I32", "I64", "U8", "U16", "U32", "U64", "F32", "F64"]
INT_TYPES = ALL_TYPES[:8]
WIDTH = {"I8": 1, "U8": 1, "I16": 2, "U16": 2, "I32": 4, "U32": 4, "F32": 4, "I64": 8, "U64": 8, "F64": 8}

# ---------------------------------------------------------------------------------------------------------
# tile geometry, in elements (rows); test_tile_table_matches_csrc re-reads every constant below from the sources

THREADS = 256                              # common.cuh kThreads
UNROLL = 4                                 # common.cuh kUnroll
TILE_BYTES = THREADS * UNROLL * 16         # common.cuh kTileBytes = 16 KiB of the widest array
BOOL_TILE = THREADS * UNROLL * 32          # k_filter.cu kBoolTile: boolean slots per tile
EXPR_UNROLL = 4                            # k_expr.cu kExprUnroll: 2 Float64 rows per 16-byte vector
REDUCE_K = {"int": 8, "float": 2}          # k_reduce.cu kReduceTilesInt / kReduceTilesFloat: tiles per reduce CTA
CMP_INT_TILES = 4                          # k_filter.cu kCmpIntTiles: compare tiles per CTA of the integer-scalar fast path


def temporal_unroll(e):                    # k_temporal.cu temporal_unroll
    return 2 if e >= 4 else UNROLL


def _build_tile_table():
    t = {}
    for a in ALL_TYPES:
        w = WIDTH[a]
        t[("binary", a)] = TILE_BYTES // w             # k_binary.cu elems_per_tile_binary, op <= OP_DIV
        if a in ("F32", "F64"):
            t[("binary_libm", a)] = THREADS * 2 * 16 // w   # op > OP_DIV (atan2/hypot/log): UnrollOf = 2
        t[("unary", a)] = TILE_BYTES // w              # k_unary.cu elems_per_tile_unary
        t[("reduce", a)] = TILE_BYTES // w             # common.cuh elems_per_tile (k_binary.cu), used by k_reduce
        t[("filter", a)] = TILE_BYTES // w             # runtime.cu filter: elems_per_tile(dtype); k_filter_scatter TILE
        for b in ALL_TYPES:
            t[("cast", a, b)] = TILE_BYTES // max(w, WIDTH[b])   # k_cast.cu elems_per_tile_cast: the wider of the two
    t[("compare",)] = THREADS * UNROLL * 2     # k_filter.cu compare_tile_elems (k_compare_int walks the same tiles)
    t[("boolean",)] = BOOL_TILE                # k_filter.cu bool_tile_elems
    t[("expr",)] = THREADS * EXPR_UNROLL * 2   # k_expr.cu expr_tile_elems
    for i in ("I32", "I64"):
        for o in ("I32", "I64"):
            w = max(WIDTH[i], WIDTH[o])
            t[("temporal", i, o)] = THREADS * temporal_unroll(16 // w) * (16 // w)   # k_temporal.cu elems_per_tile_temporal
            for b in ("I32", "I64"):
                t[("temporal2", i, b, o)] = TILE_BYTES // max(w, WIDTH[b])         # elems_per_tile_temporal2
    return t


TILE = _build_tile_table()


def reduce_k(tname):
    return REDUCE_K["float" if tname in ("F32", "F64") else "int"]


def edge_lens(T, K=None):
    lens = [1, T - 1, T, T + 1, 2 * T - 1, 2 * T + 1]
    if K:
        lens += [K * T - 1, K * T, K * T + 1]
    return lens


def _read(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def test_tile_table_matches_csrc():
    """The constants TILE is built from, read back from the kernel sources."""
    common, binary, filt = _read("common.cuh"), _read("k_binary.cu"), _read("k_filter.cu")
    expr, temporal, red = _read("k_expr.cu"), _read("k_temporal.cu"), _read("k_reduce.cu")
    unary, cast, runtime = _read("k_unary.cu"), _read("k_cast.cu"), _read("runtime.cu")

    def num(src, pat):
        m = re.search(pat, src)
        assert m, f"pattern {pat!r} not found"
        return int(m.group(1))

    assert num(common, r"constexpr int kThreads = (\d+);") == THREADS
    assert num(common, r"constexpr int kUnroll = (\d+);") == UNROLL
    assert re.search(r"constexpr int kTileBytes = kThreads \* kUnroll \* 16;", common)
    assert re.search(r"constexpr int kBoolTile = kThreads \* kUnroll \* 32;", filt) and BOOL_TILE == THREADS * UNROLL * 32
    assert num(expr, r"constexpr int kExprUnroll = (\d+);") == EXPR_UNROLL
    assert re.search(r"int expr_tile_elems\(\) \{ return kThreads \* kExprUnroll \* 2; \}", expr)
    assert num(red, r"constexpr int kReduceTilesInt = (\d+)") == REDUCE_K["int"]
    assert num(red, r"kReduceTilesFloat = (\d+);") == REDUCE_K["float"]
    assert num(filt, r"constexpr int kCmpIntTiles = (\d+);") == CMP_INT_TILES
    assert re.search(r"int compare_tile_elems\(\) \{ return kThreads \* kUnroll \* 2; \}", filt)
    # temporal: U = 2 for 4-byte-or-narrower lanes (E >= 4), else kUnroll
    m = re.search(r"constexpr int temporal_unroll\(int e\) \{ return e >= (\d+) \? (\d+) : kUnroll; \}", temporal)
    assert m and all(temporal_unroll(e) == (int(m.group(2)) if e >= int(m.group(1)) else UNROLL) for e in (1, 2, 4, 8, 16))
    assert re.search(r"return kThreads \* temporal_unroll\(16 / w\) \* \(16 / w\);", temporal)
    assert re.search(r"w = w > dtype_width\(out_dtype\) \? w : dtype_width\(out_dtype\);\s*return kTileBytes / w;", temporal)
    # binary: the op > OP_DIV rule, in both the host tile and the kernel's unroll
    assert re.search(r"OP_ADD = 0, OP_SUB, OP_MUL, OP_DIV, OP_ATAN2, OP_HYPOT, OP_LOG", binary)
    assert re.search(r"return \(op > OP_DIV \? kThreads \* 2 \* 16 : kTileBytes\) / dtype_width\(dtype\);", binary)
    assert re.search(r"UnrollOf \{ static constexpr int value = \(OP > OP_DIV\) \? 2 : kUnroll; \}", binary)
    assert re.search(r"int elems_per_tile\(int dtype\) \{ return kTileBytes / dtype_width\(dtype\); \}", binary)
    assert re.search(r"int elems_per_tile_unary\(int op, int dtype\) \{ return kTileBytes / dtype_width\(dtype\); \}", unary)
    assert re.search(r"dtype_width\(from\) > dtype_width\(to\) \? dtype_width\(from\) : dtype_width\(to\);\s*return kTileBytes / w;", cast)
    # the operators number their tiles with these functions
    for pat in (r"const int tile = elems_per_tile_binary\(op, dtype\);", r"elems_per_tile_cast\(from, to\) : elems_per_tile_unary\(op_or_to, from\)",
                r"const int tile = elems_per_tile\(dtype\);", r"const int tile = expr_tile_elems\(\);",
                r"const int tile = elems_per_tile_temporal\(pl.in_dtype, pl.out_dtype\);", r"compare_tile_elems\(\), sizeof\(BinDesc\)",
                r"bool_tile_elems\(\), bool_desc_size\(\)"):
        assert re.search(pat, runtime), pat
    # the fold grids whose caps the fold tests drive past
    assert re.search(r"int64_t grid = \(n_parts \+ 4 \* kThreads - 1\) / \(4 \* kThreads\);\s*if \(grid > sm_count\) grid = sm_count;", binary)
    assert re.search(r"sm_count / \(n < 4 \? 1 : 4\)", binary)
    assert TILE[("binary", "I8")] == 16384 and TILE[("binary", "F64")] == 2048 and TILE[("binary_libm", "F32")] == 2048
    assert TILE[("cast", "I8", "F64")] == 2048 and TILE[("temporal", "I32", "I32")] == 2048 and TILE[("temporal2", "I32", "I32", "I32")] == 4096
    assert reduce_k("I8") * TILE[("reduce", "I8")] == 131072


# ---------------------------------------------------------------------------------------------------------
# inputs

def np_dtype(tname):
    return np.dtype({"I8": np.int8, "I16": np.int16, "I32": np.int32, "I64": np.int64, "U8": np.uint8, "U16": np.uint16,
                     "U32": np.uint32, "U64": np.uint64, "F32": np.float32, "F64": np.float64}[tname])


def rand_values(rng, tname, n, nonzero=False, lo=-1e3, hi=1e3):
    npdt = np_dtype(tname)
    if npdt.kind == "f":
        v = rng.uniform(lo, hi, n).astype(npdt)
        if nonzero:
            v[v == 0] = 1
        return v
    info = np.iinfo(npdt)
    v = rng.integers(info.min, info.max, n, dtype=npdt, endpoint=True)
    if nonzero:
        v[v == 0] = 1
        if info.min < 0:
            v[v == -1] = 3
    return v


MODES = ("plain", "nulls", "sliced")


def make_chunks(rdf, rng, tname, lens, mode, gen=None, reps=None):
    """One multi-chunk column: no bitmap ("plain"), ~10 % nulls ("nulls"), or every length at every bit offset 0..7 ("sliced").
    reps: chunks per length (8 pairs a column with a sliced one)."""
    gen = gen or (lambda n: rand_values(rng, tname, n))
    reps = reps or (8 if mode == "sliced" else 1)
    out = []
    for n in lens:
        for off in (range(8) if mode == "sliced" else [0] * reps):
            v = gen(n + off)
            if mode == "plain":
                a = rdf.PrimitiveArray.from_numpy(v)
                a.null_count = 0
            else:
                a = rdf.PrimitiveArray.from_numpy(v, random_mask(rng, n + off, 0.1))
                a.null_count = -1
            out.append(a.slice(off, n))
    return out


def make_bools(rdf, rng, lens, mode, p_true=0.5):
    out = []
    for n in lens:
        for off in (range(8) if mode == "sliced" else [0]):
            m = None if mode == "plain" else rng.random(n + off) >= 0.1
            out.append(rdf.BooleanArray.from_numpy(rng.random(n + off) < p_true, m).slice(off, n))
    return out


def check_all(got, want, what, **kw):
    assert len(got) == len(want), what
    for i, (g, w) in enumerate(zip(got, want)):
        assert_same_array(g, w, what=f"{what} chunk {i} (len {w.length})", **kw)


def check_bool(got, want, what):
    assert got.length == want.length, what
    gm, wm = got.valid_mask(), want.valid_mask()
    assert np.array_equal(gm, wm), f"{what}: validity differs at {np.nonzero(gm != wm)[0][:8]}"
    gv, wv = got.value_bits(), want.value_bits()
    assert np.array_equal(gv, wv), f"{what}: values differ at {np.nonzero(gv != wv)[0][:8]}"
    assert (got.null_count if got.validity is not None else 0) == int((~wm).sum()), f"{what}: null_count"


# ---------------------------------------------------------------------------------------------------------
# tile edges: K1 binary, K2 unary, K3 cast

@gpu
@pytest.mark.parametrize("tname", ALL_TYPES)
def test_binary_tile_edges(rdf, ctx, oracle, tname):
    dtype = getattr(rdf, tname)
    rng = np.random.default_rng(1000 + dtype)
    SF = rdf.ScalarFunctions
    lens = edge_lens(TILE[("binary", tname)])
    divisor = lambda n: rand_values(rng, tname, n, nonzero=True)
    for mode in MODES:
        a = make_chunks(rdf, rng, tname, lens, mode)
        rhs_modes = ["plain"] + ([mode] if mode != "plain" else [])
        for rmode in rhs_modes:
            rhs = make_chunks(rdf, rng, tname, lens, rmode, divisor, reps=len(a) // len(lens))
            for name, op, fn in (("add", oracle.ADD, SF.add), ("subtract", oracle.SUB, SF.subtract), ("multiply", oracle.MUL, SF.multiply),
                                 ("par_multiply", oracle.MUL, SF.par_multiply), ("divide", oracle.DIV, SF.divide)):
                st, want = oracle.col_binary(op, dtype, a, rhs)
                assert st == oracle.OK
                check_all(fn(a, rhs), want, f"{name}<{tname}> {mode} rhs={rmode}")


@gpu
@pytest.mark.parametrize("tname", ["F32", "F64"])
def test_libm_binary_tile_edges(rdf, ctx, oracle, tname):
    dtype = getattr(rdf, tname)
    rng = np.random.default_rng(1100 + dtype)
    lens = edge_lens(TILE[("binary_libm", tname)])
    tol = 4 if tname == "F64" else 6
    for mode in MODES:
        a = make_chunks(rdf, rng, tname, lens, mode, lambda n: rand_values(rng, tname, n, lo=0.1, hi=100))
        b = make_chunks(rdf, rng, tname, lens, mode, lambda n: rand_values(rng, tname, n, lo=1.5, hi=100))
        ca, cb = rdf.Column.upload(a), rdf.Column.upload(b)
        for name, op in (("atan2", oracle.ATAN2), ("hypot", oracle.HYPOT), ("log", oracle.LOG)):
            st, want = oracle.col_binary(op, dtype, a, b)
            got = getattr(ca, name)(cb)
            check_all(got.download(), want, f"{name}<{tname}> {mode}", exact=False, max_ulp=tol, check_payload=False)
            got.free()
        ca.free(); cb.free()


@gpu
@pytest.mark.parametrize("tname", ["I8", "I16", "I32", "I64", "F32", "F64"])
def test_unary_tile_edges(rdf, ctx, oracle, tname):
    dtype = getattr(rdf, tname)
    rng = np.random.default_rng(1200 + dtype)
    lens = edge_lens(TILE[("unary", tname)])
    names = [("abs", 0)] if tname[0] == "I" else [("abs", 0), ("sqrt", 0), ("sin", 3 if tname == "F64" else 5)]
    for mode in MODES:
        gen = (lambda n: rand_values(rng, tname, n, lo=1e-3, hi=1e4)) if tname[0] == "F" else None
        a = make_chunks(rdf, rng, tname, lens, mode, gen)
        if tname[0] == "I":   # MIN wraps: put it in a full tile and at the chunk ends
            info = np.iinfo(a[0].values.dtype)
            for c in a:
                if c.length > 3:
                    c.values[c.offset] = info.min
                    c.values[c.offset + c.length - 1] = info.min
        for name, tol in names:
            st, want = oracle.col_unary(getattr(oracle, name.upper()), dtype, a)
            assert st == oracle.OK
            check_all(getattr(rdf.ScalarFunctions, name)(a), want, f"{name}<{tname}> {mode}", exact=(tol == 0), max_ulp=tol,
                      check_payload=(tol == 0))


CAST_EDGES_INT = [0, 1, -1, 127, 128, -128, -129, 255, 256, 32767, 32768, -32768, -32769, 65535, 65536, 2 ** 31 - 1, 2 ** 31, -2 ** 31,
                  -2 ** 31 - 1, 2 ** 32 - 1, 2 ** 32, 2 ** 63 - 1, -2 ** 63, 2 ** 64 - 1]
CAST_EDGES_FLOAT = [0.0, -0.0, 0.5, -0.9999, -1.0, 127.9, 128.0, -128.9, -129.0, 255.9, 256.0, 65535.9, 65536.0, 2147483648.0, -2147483649.0,
                    4294967296.0, 9.223372036854776e18, 1.8446744073709552e19, 3e10, -3e10, 1e300, np.inf, -np.inf, np.nan]


def cast_gen(rng, tname):
    npdt = np_dtype(tname)
    if npdt.kind == "f":
        with np.errstate(all="ignore"):
            edges = np.array(CAST_EDGES_FLOAT).astype(npdt)

        def gen(n):
            with np.errstate(all="ignore"):
                v = np.concatenate([rng.uniform(-300, 300, n // 2), rng.uniform(-1e19, 1e19, n - n // 2)]).astype(npdt)
            k = min(n, len(edges))
            v[rng.integers(0, n, k)] = edges[:k]
            return v
        return gen
    info = np.iinfo(npdt)
    edges = np.array([e for e in CAST_EDGES_INT if info.min <= e <= info.max], dtype=npdt)

    def gen(n):
        v = np.where(rng.random(n) < 0.5, rand_values(rng, tname, n),
                     rng.integers(max(info.min, -300), min(info.max, 300), n, endpoint=True).astype(npdt))
        k = min(n, len(edges))
        v[rng.integers(0, n, k)] = edges[:k]
        return v
    return gen


@gpu
@pytest.mark.parametrize("fname", ALL_TYPES)
def test_cast_tile_edges(rdf, ctx, oracle, fname):
    """One column per source type holds the edges of every target's tile (the tile is set by the wider of the pair)."""
    f = getattr(rdf, fname)
    rng = np.random.default_rng(1300 + f)
    tiles = sorted({TILE[("cast", fname, t)] for t in ALL_TYPES})
    lens = [n for T in tiles for n in edge_lens(T)]
    for mode in MODES:
        chunks = make_chunks(rdf, rng, fname, lens, mode, cast_gen(rng, fname))
        for tname in ALL_TYPES:
            t = getattr(rdf, tname)
            st, want = oracle.col_cast(f, t, chunks)
            assert st == oracle.OK
            check_all(rdf.cast(chunks, t), want, f"cast {fname}->{tname} {mode}")


# ---------------------------------------------------------------------------------------------------------
# tile edges: compare, and/or/not, filter, fused expressions, temporal

@gpu
@pytest.mark.parametrize("tname", ALL_TYPES)
def test_compare_tile_edges(rdf, ctx, oracle, tname):
    dtype = getattr(rdf, tname)
    rng = np.random.default_rng(1400 + dtype)
    T = TILE[("compare",)]
    lens = edge_lens(T, CMP_INT_TILES)   # the integer-scalar path walks CMP_INT_TILES tiles per CTA
    gen = lambda n: (rand_values(rng, tname, n, lo=-50, hi=50) if tname[0] == "F" else
                     rng.integers(0 if tname[0] == "U" else -50, 50, n).astype(np_dtype(tname)))
    for mode in MODES:
        a = make_chunks(rdf, rng, tname, lens, mode, gen)
        b = make_chunks(rdf, rng, tname, lens, "nulls" if mode == "plain" else mode, gen)
        ca, cb = rdf.Column.upload(a), rdf.Column.upload(b)
        for op in range(6):
            got = ca.compare(op, cb)
            for i, g in enumerate(got.download()):
                st, want = oracle.compare(op, a[i], b[i])
                assert st == oracle.OK
                check_bool(g, want, f"compare op{op} <{tname}> {mode} chunk {i} (len {a[i].length})")
            got.free()
            for s in (3.0, 2.5):
                got = ca.compare(op, s)
                for i, g in enumerate(got.download()):
                    st, want = oracle.compare(op, a[i], None, scalar=s)
                    assert st == oracle.OK
                    check_bool(g, want, f"compare op{op} <{tname}> scalar {s} {mode} chunk {i} (len {a[i].length})")
                got.free()
        ca.free(); cb.free()


@gpu
def test_boolean_tile_edges(rdf, ctx, oracle):
    rng = np.random.default_rng(1500)
    lens = edge_lens(TILE[("boolean",)])
    for mode in MODES:
        A = make_bools(rdf, rng, lens, mode)
        B = make_bools(rdf, rng, lens, "nulls" if mode == "plain" else mode, 0.3)
        ca, cb = rdf.Column.upload(A), rdf.Column.upload(B)
        for name, col, oop in (("and", ca.logical_and(cb), oracle.AND), ("or", ca.logical_or(cb), oracle.OR), ("not", ca.logical_not(), oracle.NOT)):
            for i, g in enumerate(col.download()):
                st, want = oracle.boolean(oop, A[i], None if oop == oracle.NOT else B[i])
                assert st == oracle.OK
                check_bool(g, want, f"{name} {mode} chunk {i} (len {A[i].length})")
            col.free()
        ca.free(); cb.free()


@gpu
@pytest.mark.parametrize("tname", ALL_TYPES)
def test_filter_tile_edges(rdf, ctx, oracle, tname):
    dtype = getattr(rdf, tname)
    rng = np.random.default_rng(1600 + dtype)
    lens = edge_lens(TILE[("filter", tname)])
    for mode in MODES:
        vals = make_chunks(rdf, rng, tname, lens, mode)
        masks = make_bools(rdf, rng, lens, mode)
        cv, cm = rdf.Column.upload(vals), rdf.Column.upload(masks)
        out = cv.filter(cm)
        got = out.download()
        assert len(got) == len(vals)
        for i, g in enumerate(got):
            st, want = oracle.filter_chunk(vals[i], masks[i])
            assert st == oracle.OK
            assert_same_array(g, want, what=f"filter<{tname}> {mode} chunk {i} (len {vals[i].length})")
        for col in (cv, cm, out):
            col.free()


def oracle_chain(oracle, inputs, nodes):
    slots = list(inputs)
    for nd in nodes:
        if len(nd) == 2:
            st, r = oracle.col_unary(getattr(oracle, nd[0].upper()), oracle.F64, slots[nd[1]])
        else:
            st, r = oracle.col_binary(nd[0], oracle.F64, slots[nd[1]], slots[nd[2]])
        assert st == oracle.OK
        slots.append(r)
    return slots[-1]


@gpu
def test_expr_tile_edges(rdf, ctx, oracle):
    rng = np.random.default_rng(1700)
    N = rdf.native
    T = TILE[("expr",)]
    lens = edge_lens(T) + [T // 2 - 1, T // 2, T // 2 + 1]   # the bulk path stages half tiles
    prog = [(N.ADD, 0, 1), (N.MUL, 3, 2), (N.SUB, 4, 0), ("abs", 5), (N.DIV, 6, 2)]
    for mode in MODES:
        reps = 8 if mode == "sliced" else 1
        host = [make_chunks(rdf, rng, "F64", lens, m, (lambda n: rand_values(rng, "F64", n, lo=1.0, hi=100.0)) if k == 2 else None, reps)
                for k, m in enumerate((mode, "plain" if mode == "plain" else "nulls", mode))]
        cols = [rdf.Column.upload(h) for h in host]
        want = oracle_chain(oracle, host, prog)
        got = rdf.eval_expr(cols, prog)
        check_all(got.download(), want, f"expr {mode}", check_payload=False)
        fused, agg = rdf.eval_expr_agg(cols, prog)
        check_all(fused.download(), want, f"expr+agg {mode}", check_payload=False)
        _, agg_only = rdf.eval_expr_agg(cols, prog, materialise=False)
        exact, sum_abs = oracle.sum_exact(oracle.F64, want)
        count = sum(w.length - (w.null_count if w.validity is not None else 0) for w in want)
        n = sum(w.length for w in want)
        for a in (agg, agg_only):
            assert a["count"] == count
            assert abs(np.longdouble(a["sum"]) - exact) <= 16 * np.log2(n) * 2.0 ** -53 * sum_abs
        assert float(agg["sum"]).hex() == float(agg_only["sum"]).hex()
        for c in cols + [got, fused]:
            c.free()


def temporal_chunks(rdf, rng, t, lens, mode):
    upd, _ = TO.per_day(t.kind, t.unit)
    npdt = np.int32 if t.dtype == rdf.I32 else np.int64

    def gen(n):
        days = rng.integers(-200000, 200000, n)
        v = days * upd + (rng.integers(0, upd, n) if upd > 1 else 0)
        v[rng.random(n) < 0.02] = TO.MAX_DAY * upd + upd   # out of chrono's range: NULL
        return v.astype(npdt)
    chunks = make_chunks(rdf, rng, "I32" if npdt == np.int32 else "I64", lens, mode, gen)
    for c in chunks:
        c.temporal = t
    vals = np.concatenate([c.value_slice() for c in chunks]).astype(np.int64)
    mask = np.concatenate([c.valid_mask() for c in chunks])
    return chunks, vals, mask


def check_temporal(got, lens_chunks, want_v, want_ok, what):
    assert [g.length for g in got] == [c.length for c in lens_chunks], what
    gv = np.concatenate([g.value_slice() for g in got])
    gm = np.concatenate([g.valid_mask() for g in got])
    bad = np.nonzero(gm != want_ok)[0]
    assert bad.size == 0, f"{what}: validity differs at {bad[:8]}"
    bad = np.nonzero(gv.view(f"u{gv.dtype.itemsize}") != want_v.view(f"u{want_v.dtype.itemsize}"))[0]
    assert bad.size == 0, f"{what}: values differ at {bad[:8]}"
    for i, g in enumerate(got):
        assert g.null_count == g.length - int(g.valid_mask().sum()), f"{what}: null_count of chunk {i}"


@gpu
def test_temporal_tile_edges(rdf, ctx):
    T = rdf.TemporalType
    rng = np.random.default_rng(1800)
    for t in (T.date32(), T.timestamp("us")):
        lens = edge_lens(TILE[("temporal", "I32" if t.dtype == rdf.I32 else "I64", "I32")])
        for mode in MODES:
            chunks, v, m = temporal_chunks(rdf, rng, t, lens, mode)
            col = rdf.Column.upload(chunks, ctx, dtype=t.dtype).with_temporal(t)
            out = col.year()
            want_v, want_ok = TO.unary("year", t.kind, t.unit, t.tz, v, m)
            check_temporal(out.download(), chunks, want_v, want_ok, f"year {t!r} {mode}")
            col.free(); out.free()
    for ta, tb in ((T.date32(), T.date32()), (T.timestamp("us"), T.date32())):
        key = ("temporal2", "I32" if ta.dtype == rdf.I32 else "I64", "I32" if tb.dtype == rdf.I32 else "I64", "I32")
        lens = edge_lens(TILE[key])
        for mode in MODES:
            ca, va, ma = temporal_chunks(rdf, rng, ta, lens, mode)
            cb, vb, mb = temporal_chunks(rdf, rng, tb, lens, "nulls" if mode == "plain" else mode)
            A = rdf.Column.upload(ca, ctx, dtype=ta.dtype).with_temporal(ta)
            B = rdf.Column.upload(cb, ctx, dtype=tb.dtype).with_temporal(tb)
            out = A.date_diff(B)
            want_v, want_ok = TO.binary("date_diff", (ta.kind, ta.unit, ta.tz), va, ma, (tb.kind, tb.unit, tb.tz), vb, mb)
            check_temporal(out.download(), ca, want_v, want_ok, f"date_diff({ta!r}, {tb!r}) {mode}")
            for c in (A, B, out):
                c.free()


# ---------------------------------------------------------------------------------------------------------
# planted extremes: min / max / sum / count of K4 and K5

def planted_positions(tname):
    """(chunk length, [positions]): every slot of a 16-byte vector, lanes 0/1/15/31, each warp, each unroll step, each of the K tiles of a
    reduce CTA, the last slot of the last full tile, the first slot of the tail tile and the last row."""
    E = 16 // WIDTH[tname]
    T = TILE[("reduce", tname)]
    K = reduce_k(tname)
    L = (K + 1) * T + 38          # K full tiles in CTA 0, one full tile and a 38-row tail in CTA 1

    def at(k, j, tid, e):
        return k * T + (j * THREADS + tid) * E + e
    ps = [at(0, 0, 0, e) for e in range(E)]
    ps += [at(0, 1, lane, E - 1) for lane in (0, 1, 15, 31)]
    ps += [at(0, 2, 32 * w + 3, 0) for w in range(THREADS // 32)]
    ps += [at(0, j, 37, 1) for j in range(UNROLL)]
    ps += [at(k, 3, 200, E // 2) for k in range(K)]
    ps += [(K + 1) * T - 1, (K + 1) * T, L - 1]
    assert len(ps) <= 64 and max(ps) < L
    return L, ps


def wrap(tname, s):
    bits = 8 * WIDTH[tname]
    s %= 1 << bits
    if tname[0] == "I" and s >= 1 << (bits - 1):
        s -= 1 << bits
    return s


def planted_int(rng, tname, L, p, nulls):
    """Values from a narrow band, the valid maximum at p and the valid minimum at p ^ 1 (the other parity, same vector), both outside the
    band and of opposite signs for signed types.  With nulls: the rest of that vector and ~10 % elsewhere are null and hold MIN / MAX."""
    npdt = np_dtype(tname)
    info = np.iinfo(npdt)
    if tname[0] == "I":
        v = rng.integers(-20, 21, L).astype(npdt)
        vmin, vmax = int(info.min) + 2, int(info.max) - 3
    else:
        v = rng.integers(100, 121, L).astype(npdt)
        vmin, vmax = 3, int(info.max) - 3
    q = p ^ 1
    v[p], v[q] = vmax, vmin
    if not nulls:
        return v, None, vmin, vmax
    mask = rng.random(L) >= 0.1
    E = 16 // WIDTH[tname]
    v0 = p - p % E
    mask[v0:v0 + E] = False
    mask[max(p - 3, 0):p + 4] = False
    mask[p] = mask[q] = True
    idx = np.nonzero(~mask)[0]
    v[idx] = np.where(idx % 2 == 0, info.min, info.max).astype(npdt)
    return v, mask, vmin, vmax


def expect_int(tname, v, mask):
    sel = v if mask is None else v[mask]
    return {"sum": wrap(tname, int(sel.astype(object).sum()) if sel.size else 0), "min": int(sel.min()), "max": int(sel.max()),
            "count": int(sel.size)}


def check_agg(got, want, what):
    for key in ("sum", "min", "max", "count"):
        assert got[key] is not None and int(got[key]) == want[key], f"{what}: {key} {got[key]} != {want[key]}"


@gpu
@pytest.mark.parametrize("nulls", [True, False], ids=["bitmap", "all_valid"])
@pytest.mark.parametrize("tname", INT_TYPES)
def test_planted_int_extremes(rdf, ctx, tname, nulls):
    dtype = getattr(rdf, tname)
    rng = np.random.default_rng(2000 + 2 * dtype + nulls)
    AF = rdf.AggregateFunctions
    L, ps = planted_positions(tname)
    cols, wants, hosts = [], [], []
    for p in ps:
        v, mask, vmin, vmax = planted_int(rng, tname, L, p, nulls)
        want = expect_int(tname, v, mask)
        assert want["min"] == vmin and want["max"] == vmax
        arr = rdf.PrimitiveArray.from_numpy(v, mask)
        what = f"{tname} bitmap={nulls} max at {p}, min at {p ^ 1}"
        # AggregateFunctions (host chunks in, one launch of k_reduce over them)
        got = {"sum": AF.sum([arr]), "min": AF.min([arr]), "max": AF.max([arr]), "count": AF.count([arr])}
        check_agg(got, want, "AggregateFunctions " + what)
        col = rdf.Column.upload([arr])
        check_agg(col.aggregate_all(), want, "Column.aggregate_all " + what)
        # K5: a + 0 with the nulls on a, or on the zero column (the sum of a's planted payload under b's nulls must not count)
        zero_m = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.zeros(L, v.dtype), mask)])
        zero = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.zeros(L, v.dtype))])
        raw = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(v)])
        for x, y, side in ((col, zero, "a"), (raw, zero_m, "b")):
            out, agg = x.binary_agg(rdf.native.ADD, y)
            check_agg(agg, want, f"binary_agg (nulls on {side}) " + what)
            assert out.chunk_info(0)["null_count"] == L - want["count"]
            out.free()
        for c in (zero_m, zero, raw):
            c.free()
        cols.append(col); wants.append(want); hosts.append(what)
    for got, want, what in zip(rdf.Column.aggregate_all_many(cols), wants, hosts):
        check_agg(got, want, "aggregate_all_many " + what)
        assert got["rows"] == L and not got["would_panic"]
    for c in cols:
        c.free()


@gpu
def test_identity_valued_columns(rdf, ctx):
    """Columns whose extremes are the identities of the min / max folds."""
    rng = np.random.default_rng(2100)
    AF = rdf.AggregateFunctions
    L = 3 * TILE[("reduce", "I8")] + 5
    cases = []
    v = rng.integers(-127, 128, L).astype(np.int8)
    m = np.zeros(L, bool)
    m[L // 2 + 1] = True
    v[L // 2 + 1] = -128
    cases.append(("I8", v, m, -128, -128))                                  # the only valid value is -128: max is -128
    cases.append(("I8", np.full(L, 127, np.int8), None, 127, 127))         # all 127: min is 127
    cases.append(("I8", np.full(L, -128, np.int8), None, -128, -128))
    cases.append(("U8", np.full(L, 255, np.uint8), None, 255, 255))
    cases.append(("U8", np.zeros(L, np.uint8), None, 0, 0))
    u = np.where(rng.random(L) < 0.5, 0, 2 ** 64 - 1).astype(np.uint64)
    cases.append(("U64", u, None, 0, 2 ** 64 - 1))
    um = rng.random(L) < 0.5
    cases.append(("U64", np.where(um, 2 ** 64 - 1, 5).astype(np.uint64), um, 2 ** 64 - 1, 2 ** 64 - 1))
    i16 = np.full(L, -32768, np.int16)
    cases.append(("I16", i16, None, -32768, -32768))
    for tname, v, m, vmin, vmax in cases:
        want = expect_int(tname, v, m)
        assert (want["min"], want["max"]) == (vmin, vmax)
        arr = rdf.PrimitiveArray.from_numpy(v, m)
        what = f"identity {tname} min={vmin} max={vmax} bitmap={m is not None}"
        check_agg(AF.all([arr]), want, "AggregateFunctions.all " + what)
        assert int(AF.min([arr])) == vmin and int(AF.max([arr])) == vmax
        col = rdf.Column.upload([arr])
        check_agg(col.aggregate_all(), want, "aggregate_all " + what)
        zero = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.zeros(L, v.dtype))])
        out, agg = col.binary_agg(rdf.native.ADD, zero)
        check_agg(agg, want, "binary_agg " + what)
        for c in (col, zero, out):
            c.free()


@gpu
@pytest.mark.parametrize("nulls", [True, False], ids=["bitmap", "all_valid"])
@pytest.mark.parametrize("tname", ["F32", "F64"])
def test_planted_float_sums(rdf, ctx, oracle, tname, nulls):
    """The same placements for floats: NaN and +-inf under nulls must not reach the sum; sums within 16 log2(n) eps sum|x|."""
    dtype = getattr(rdf, tname)
    npdt = np_dtype(tname)
    eps = 2.0 ** -53 if tname == "F64" else 2.0 ** -24
    rng = np.random.default_rng(2200 + 2 * dtype + nulls)
    L, ps = planted_positions(tname)
    cols, wants = [], []
    for p in ps:
        v = rng.uniform(-1.0, 1.0, L).astype(npdt)
        v[p], v[p ^ 1] = 1e4, -3e4
        mask = None
        if nulls:
            mask = rng.random(L) >= 0.1
            mask[max(p - 3, 0):p + 4] = False
            mask[p] = mask[p ^ 1] = True
            idx = np.nonzero(~mask)[0]
            v[idx] = np.array([np.nan, np.inf, -np.inf])[idx % 3].astype(npdt)
        arr = rdf.PrimitiveArray.from_numpy(v, mask)
        sel = v if mask is None else v[mask]
        exact = math.fsum(sel.astype(np.float64).tolist())
        bound = 16 * np.log2(L) * eps * float(np.abs(sel.astype(np.float64)).sum())
        if tname == "F32":   # the Float32 result is the double sum rounded once more
            bound += abs(exact) * 2.0 ** -24
        want = (exact, bound, int(sel.size))
        what = f"{tname} bitmap={nulls} planted at {p}"
        s = rdf.AggregateFunctions.sum([arr])
        assert abs(float(s) - exact) <= bound, f"AggregateFunctions.sum {what}: {s} vs {exact}"
        assert rdf.AggregateFunctions.count([arr]) == want[2]
        col = rdf.Column.upload([arr])
        r = col.aggregate_all()
        assert r["count"] == want[2] and abs(float(r["sum"]) - exact) <= bound, f"aggregate_all {what}: {r}"
        zero = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(np.zeros(L, npdt))])
        out, agg = col.binary_agg(rdf.native.ADD, zero)
        assert agg["count"] == want[2] and abs(float(agg["sum"]) - exact) <= bound, f"binary_agg {what}: {agg}"
        for c in (zero, out):
            c.free()
        cols.append(col); wants.append(want)
    for got, (exact, bound, count) in zip(rdf.Column.aggregate_all_many(cols), wants):
        assert got["count"] == count and abs(float(got["sum"]) - exact) <= bound
    for c in cols:
        c.free()


# ---------------------------------------------------------------------------------------------------------
# batched reduce on one GPU

def expect_cols(tname, chunks):
    """Per-column expectation from the host chunks: exact sum (wrapped / fsum), min, max, count, would_panic."""
    vals = [c.value_slice()[c.valid_mask()] for c in chunks]
    v = np.concatenate(vals) if vals else np.zeros(0, np_dtype(tname))
    r = {"count": int(v.size), "rows": sum(c.length for c in chunks), "n_chunks": len(chunks),
         "would_panic": any(c.length == 0 or not c.valid_mask().any() for c in chunks)}
    if tname[0] == "F":
        r["sum"] = math.fsum(v.astype(np.float64).tolist())
        r["sum_abs"] = float(np.abs(v.astype(np.float64)).sum())
        r["min"] = r["max"] = None
    else:
        r["sum"] = wrap(tname, int(v.astype(object).sum()) if v.size else 0)
        r["min"] = int(v.min()) if v.size else None
        r["max"] = int(v.max()) if v.size else None
    return r


def check_many(got, want, tname, what, panic_rule=True):
    """panic_rule: the blocking forms evaluate the would-panic rule; the asynchronous ones do not wait for null counts."""
    for key in ("count", "rows", "n_chunks") + (("would_panic",) if panic_rule else ()):
        assert got[key] == want[key], f"{what}: {key} {got[key]} != {want[key]}"
    if tname[0] == "F":
        eps = 2.0 ** -53 if tname == "F64" else 2.0 ** -24
        bound = 16 * np.log2(max(want["rows"], 2)) * eps * want["sum_abs"]
        if tname == "F32":   # the Float32 result is the double sum rounded once more
            bound += abs(want["sum"]) * 2.0 ** -24
        assert abs(float(got["sum"]) - want["sum"]) <= bound, f"{what}: sum {got['sum']} vs {want['sum']}"
        assert got["min"] is None and got["max"] is None
    else:
        assert int(got["sum"]) == want["sum"], f"{what}: sum"
        for key in ("min", "max"):
            assert (None if got[key] is None else int(got[key])) == want[key], f"{what}: {key} {got[key]} != {want[key]}"


def batch_columns(rdf, rng, n_cols):
    """Interleaved dtypes (so that grouping by dtype reorders them) and chunkings: zero chunks, only empty chunks, an all-null
    column, one-row chunks, chunks across CTA boundaries, planted extremes with MIN / MAX under nulls."""
    order = ["I64", "F64", "I8", "I64", "U16", "F64", "I8", "U32", "F32", "I16", "U8", "U64", "I32"]
    shapes = ["ragged", "zero_chunks", "ones", "empty_only", "all_null", "cta"]
    out = []
    for k in range(n_cols):
        tname = order[k % len(order)]
        shape = shapes[(k // len(order) + k) % len(shapes)] if n_cols > 4 else ("ragged", "cta", "ones", "all_null")[k % 4]
        T, K = TILE[("reduce", tname)], reduce_k(tname)
        lens = {"ragged": [5, 0, T + 3, 1, 2 * T - 1], "zero_chunks": [], "ones": [1] * 37, "empty_only": [0, 0, 0],
                "all_null": [T + 1, 7], "cta": [K * T - 1, K * T + 1, 3]}[shape]
        chunks = []
        for n in lens:
            v = rand_values(rng, tname, n + 3, lo=-10, hi=10)
            if tname[0] != "F":
                info = np.iinfo(v.dtype)
                v = (v % 50).astype(v.dtype) if tname[0] == "U" else (v % 50 - 25).astype(v.dtype)
            m = rng.random(n + 3) >= 0.1
            if shape == "all_null":
                m[:] = False
            if tname[0] != "F":
                idx = np.nonzero(~m)[0]
                v[idx] = np.where(idx % 2 == 0, info.min, info.max).astype(v.dtype)
                if n > 2 and shape != "all_null":
                    j = 3 + int(rng.integers(0, n))
                    v[j], m[j] = (info.min + 1 if tname[0] == "I" else 1), True
            a = rdf.PrimitiveArray.from_numpy(v, m if (shape != "ones" or k % 2) else None)
            a.null_count = -1 if a.validity is not None else 0
            chunks.append(a.slice(3, n))
        out.append((tname, shape, chunks))
    return out


@gpu
@pytest.mark.parametrize("n_cols", [1, 3, 4, 64])
def test_aggregate_all_many_matches_per_column(rdf, ctx, n_cols):
    rng = np.random.default_rng(2300 + n_cols)
    specs = batch_columns(rdf, rng, n_cols)
    cols = [rdf.Column.upload(ch, dtype=getattr(rdf, tname)) for tname, _, ch in specs]
    wants = [expect_cols(tname, ch) for tname, _, ch in specs]
    blocking = rdf.Column.aggregate_all_many(cols)
    fut = rdf.Column.aggregate_all_many(cols, asynchronous=True)
    asynchronous = fut.result()
    for k, (tname, shape, _) in enumerate(specs):
        what = f"column {k} of {n_cols} ({tname}, {shape})"
        check_many(blocking[k], wants[k], tname, "blocking " + what)
        check_many(asynchronous[k], wants[k], tname, "async " + what, panic_rule=False)
        if shape == "all_null":
            assert blocking[k]["count"] == 0 and blocking[k]["min"] is None and blocking[k]["max"] is None
        one = cols[k].aggregate_all()
        assert one["count"] == blocking[k]["count"] and one["rows"] == blocking[k]["rows"]
    for c in cols:
        c.free()


# ---------------------------------------------------------------------------------------------------------
# fold grids past their SM cap, thousands of chunks

def gen_ref(oracle, dtype, kind, lo, hi, col_id, n, null_mod=0):
    """Column.generate is a function of the row number: one oracle chunk over all rows equals the concatenated chunks."""
    return oracle.generate(dtype, kind, lo, hi, 20260924, col_id, 0, n, null_mod)


@gpu
def test_fused_fold_past_the_grid_cap(rdf, ctx, oracle):
    sm = ctx.device_info()["sm_count"]
    rng = np.random.default_rng(2400)
    lens = rng.integers(1, 4, 140000).tolist()
    n = sum(lens)
    tiles = len(lens)   # every chunk is shorter than a tile: one K5 partial per chunk
    assert tiles > sm * 4 * THREADS, "the fold grid would not reach its cap"
    a = rdf.Column.generate(rdf.F64, lens, 0, -1e3, 1e3, col_id=40)
    b = rdf.Column.generate(rdf.F64, lens, 0, -1e3, 1e3, col_id=41, null_mod=7)
    c, agg = a.binary_agg(rdf.native.ADD, b)
    oa = gen_ref(oracle, oracle.F64, 0, -1e3, 1e3, 40, n)
    ob = gen_ref(oracle, oracle.F64, 0, -1e3, 1e3, 41, n, 7)
    _, oc = oracle.col_binary(oracle.ADD, oracle.F64, [oa], [ob])
    exact, sum_abs = oracle.sum_exact(oracle.F64, oc)
    wm = oc[0].valid_mask()
    assert agg["count"] == int(wm.sum()) and agg["rows"] == n
    assert abs(np.longdouble(agg["sum"]) - exact) <= 16 * np.log2(n) * 2.0 ** -53 * sum_abs
    again = c.aggregate_all()
    assert again["count"] == agg["count"] and abs(np.longdouble(again["sum"]) - exact) <= 16 * np.log2(n) * 2.0 ** -53 * sum_abs
    got = c.download()
    gv = np.concatenate([g.value_slice() for g in got])
    gm = np.concatenate([g.valid_mask() for g in got])
    assert np.array_equal(gm, wm)
    assert np.array_equal(gv.view(np.uint64)[wm], oc[0].values.view(np.uint64)[wm])
    starts = np.cumsum([0] + lens[:-1])
    want_nulls = np.add.reduceat((~wm).astype(np.int64), starts)
    got_nulls = np.array([g.null_count if g.validity is not None else 0 for g in got])
    assert np.array_equal(got_nulls, want_nulls), f"per-chunk null counts differ at {np.nonzero(got_nulls != want_nulls)[0][:8]}"
    for col in (a, b, c):
        col.free()


@gpu
def test_reduce_fold_past_the_grid_cap(rdf, ctx, oracle):
    sm = ctx.device_info()["sm_count"]
    n = 300000
    lens = [1] * n
    # I8: K = 8 one-row tiles per CTA walk across 8 chunks; F64: K = 2 and more partials than the capped grid takes in one sweep
    for tname, kind, lo, hi, null_mod in (("I8", 2, 0, 0, 10), ("F64", 0, -1e3, 1e3, 10)):
        dtype = getattr(rdf, tname)
        parts = -(-n // reduce_k(tname))
        if tname == "F64":
            assert parts > sm * 4 * THREADS, "the fold grid would not reach its cap"
        col = rdf.Column.generate(dtype, lens, kind, lo, hi, col_id=50 + dtype, null_mod=null_mod)
        ref = gen_ref(oracle, dtype, kind, lo, hi, 50 + dtype, n, null_mod)
        want = expect_cols(tname, [rdf.PrimitiveArray.from_numpy(ref.values, ref.valid_mask())])
        want["n_chunks"], want["would_panic"] = n, True   # one-row chunks: the null rows are all-null chunks
        check_many(col.aggregate_all(), want, tname, f"aggregate_all {tname} over {n} one-row chunks")
        col.free()
    # four columns folded by one k_finish_many: its grid is capped at sm_count / 4
    m = 70000
    assert -(-m // reduce_k("F64")) > (sm // 4) * 4 * THREADS, "the batched fold grid would not reach its cap"
    cols = [rdf.Column.generate(rdf.F64, [1] * m, 0, -1e3, 1e3, col_id=60 + k, null_mod=5 if k % 2 else 0) for k in range(4)]
    got = rdf.Column.aggregate_all_many(cols)
    for k in range(4):
        ref = gen_ref(oracle, oracle.F64, 0, -1e3, 1e3, 60 + k, m, 5 if k % 2 else 0)
        want = expect_cols("F64", [rdf.PrimitiveArray.from_numpy(ref.values, ref.valid_mask())])
        want["n_chunks"], want["would_panic"] = m, bool(k % 2)
        check_many(got[k], want, "F64", f"aggregate_all_many column {k}")
        cols[k].free()


# ---------------------------------------------------------------------------------------------------------
# pipelined groups: operators that run group by group over asynchronously uploaded inputs

def assert_identical(got, want, what):
    assert len(got) == len(want), what
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.length == w.length, f"{what} chunk {i}"
        assert np.array_equal(g.valid_mask(), w.valid_mask()), f"{what} chunk {i}: validity"
        gn = g.null_count if g.validity is not None else 0
        wn = w.null_count if w.validity is not None else 0
        assert gn == wn, f"{what} chunk {i}: null_count {gn} != {wn}"
        if hasattr(g, "value_bits"):
            assert np.array_equal(g.value_bits(), w.value_bits()), f"{what} chunk {i}: values"
        else:
            gv, wv = g.value_slice(), w.value_slice()
            assert np.array_equal(gv.view(f"u{gv.itemsize}"), wv.view(f"u{wv.itemsize}")), f"{what} chunk {i}: values"


def upload_group_ends(lens, width, group_bytes):
    """runtime.cu upload: a group closes once it holds group_bytes of values, and at the last chunk."""
    ends, pending = [], 0
    for i, n in enumerate(lens):
        pending += n * width
        if pending >= group_bytes or i == len(lens) - 1:
            ends.append(i + 1)
            pending = 0
    return ends


@gpu
def test_pipelined_groups_match_resident_columns(rdf, oracle, ctx):
    """BDF_PIPELINE_SPLIT makes the operators of this context launch once per input upload group even when the copies have already
    landed, so the grouped launches -- tile numbering across groups, K5 partials at each group's tile_base, the divide flag read after
    the last group -- run on every call; the inputs are uploaded asynchronously, so groups may also still be in flight."""
    group_bytes = 65536
    env = {"BDF_PIPELINE_BYTES": str(group_bytes), "BDF_PIPELINE_SPLIT": "1"}
    os.environ.update(env)
    try:
        c2 = rdf.Context(0)
    finally:
        for k in env:
            del os.environ[k]
    live = []   # every column of the test, freed however it ends (they hold about 1.5 GB of device memory)
    try:
        _pipelined_body(rdf, ctx, c2, group_bytes, live)
    finally:
        for c in live:
            c.free()
        c2.close()


def _pipelined_body(rdf, ctx, c2, group_bytes, live):
    rng = np.random.default_rng(2500)
    lens = [4_000_000, 1, 3_000_001, 2048, 5_000_000, 0, 4_000_003]
    lens.append(32_000_000 - sum(lens))   # 8 chunks, 32M rows: 256 MB per Float64 column
    T = rdf.TemporalType

    def f64(mask_frac, nonzero=False):
        out = []
        for n in lens:
            v = rng.uniform(-1e3, 1e3, n)
            if nonzero:
                v[v == 0] = 1.0
            a = rdf.PrimitiveArray.from_numpy(v, random_mask(rng, n, mask_frac) if mask_frac else None)
            a.null_count = -1 if a.validity is not None else 0
            out.append(a)
        return out

    def dates():
        out = []
        for n in lens:
            a = rdf.PrimitiveArray.from_numpy(rng.integers(-200000, 200000, n).astype(np.int32), random_mask(rng, n, 0.1))
            a.null_count = -1
            a.temporal = T.date32()
            out.append(a)
        return out

    A, B, D1, D2 = f64(0.1), f64(0.0, nonzero=True), dates(), dates()
    I = []
    for n in lens:
        a = rdf.PrimitiveArray.from_numpy(rng.integers(-2 ** 40, 2 ** 40, n), random_mask(rng, n, 0.1))
        a.null_count = -1
        I.append(a)
    src = {"a": (A, rdf.F64, 8), "b": (B, rdf.F64, 8), "d1": (D1, rdf.I32, 4), "d2": (D2, rdf.I32, 4), "i": (I, rdf.I64, 8)}
    resident = {}
    for name, (h, dt, _) in src.items():
        resident[name] = rdf.Column.upload(h, ctx=ctx, dtype=dt)
        live.append(resident[name])
    resident["d1"].with_temporal(T.date32()); resident["d2"].with_temporal(T.date32())

    def fresh(*names):
        """Asynchronous uploads on the pipelined context."""
        cols = [rdf.Column.upload(src[n][0], ctx=c2, asynchronous=True, dtype=src[n][1]) for n in names]
        live.extend(cols)
        for n, c in zip(names, cols):
            if n in ("d1", "d2"):
                c.with_temporal(T.date32())
        return cols

    def groups(*names):   # the operator's groups: the union of its inputs' group ends (none of them holds only empty chunks)
        return len(set().union(*[upload_group_ends(lens, src[n][2], group_bytes) for n in names]))

    # (name, inputs, call, launches: one per group, + the k_finish of K5; compare always runs as one launch)
    calls = [
        ("add", ("a", "b"), lambda x, y: x.add(y), groups("a", "b")),
        ("divide", ("a", "b"), lambda x, y: x.divide(y), groups("a", "b")),
        ("binary_agg", ("a", "b"), lambda x, y: x.binary_agg(rdf.native.ADD, y), groups("a", "b") + 1),
        ("sin", ("a",), lambda x: x.sin(), groups("a")),
        ("cast I64->I32", ("i",), lambda x: x.cast(rdf.I32), groups("i")),
        ("year", ("d1",), lambda x: x.year(), groups("d1")),
        ("date_diff", ("d1", "d2"), lambda x, y: x.date_diff(y), groups("d1", "d2")),
        ("compare", ("a", "b"), lambda x, y: x.gt(y), 1),
    ]
    assert groups("a", "b") == 5 and groups("d1") == 5
    for name, inputs, fn, launches in calls:
        cols = fresh(*inputs)
        before = c2.launch_count()
        got = fn(*cols)
        delta = c2.launch_count() - before
        want = fn(*[resident[n] for n in inputs])
        if name == "binary_agg":
            (got, gagg), (want, wagg) = got, want
        live.extend([got, want])
        if name == "binary_agg":
            assert float(gagg["sum"]).hex() == float(wagg["sum"]).hex() and gagg["count"] == wagg["count"], (name, gagg, wagg)
        assert_identical(got.download(), want.download(), f"pipelined {name}")
        assert delta == launches, f"pipelined {name}: {delta} launches, {launches} expected"
        for c in cols + [got, want]:
            c.free()
