"""The fused expression path on the device over every program shape: a stratified few hundred programs of the random corpus of
tests/expr_reference.py (every binop as BIN and as RBIN, all 21 unaries, 0, 1 and 2 temporaries), run by eval_expr and by the unfused
device chain, bit for bit; exact programs also against the oracle.  Then DivideByZero placements, the trailing aggregate, the bulk-copy
kernel (BDF_EXPR_BULK=1, in a child process) and a differential of DeviceFrame.evaluate with and without the planner's fusion.

Bit for bit means every valid slot, with any NaN equal to any other NaN (IEEE 754 leaves a produced NaN's payload open; see
math_reference.same_bits).  Null slots: the fused kernel documents payload 0 and is checked for it; the unfused kernels document no
null payload, so their values are compared under the valid slots only."""
import hashlib
import json
import os
import subprocess
import sys
from collections import Counter, OrderedDict

import numpy as np
import pytest

import expr_reference as er
from helpers import assert_same_array
from math_reference import same_bits
from rust_dataframe_b200.arrays import BooleanArray
from test_expr_programs import harness  # noqa: F401  (the session fixture)

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
TILE = er.C["tile"]
# more than 2 x SMs x TILE rows (H100 SXM: 132 SMs): the bulk kernel's CTAs walk several tiles
BIG = 2 * 144 * TILE + 4097
LENS = [0, 1, TILE // 2 - 1, TILE // 2, TILE // 2 + 1, TILE - 1, TILE, TILE + 1, 2 * TILE + 1, BIG]
BIN_NAMES = ["add", "subtract", "multiply", "divide", "atan2", "hypot", "log"]
SPECIALS = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 5e-324, -5e-324, 1e-310, -2.2250738585072014e-308, 1.0, -1.0])
N_PROGRAMS = 240


# ---- programs -------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def programs(harness):  # noqa: F811
    dags = er.random_dags(30_000, 777)
    accepted = []
    for d, (c, p) in zip(dags, harness.compile(dags)):
        if c == 0:
            accepted.append((d, p, er.interpret(d, p)))
    pick = er.stratified(accepted, N_PROGRAMS, seed=5)
    return pick


def test_programs_cover_every_form(programs):
    runs = [r for _, _, r in programs]
    assert set().union(*(r.bin for r in runs)) == set(range(er.N_BINOPS))
    assert set().union(*(r.rbin for r in runs)) == set(range(er.N_BINOPS))
    assert set().union(*(r.unops for r in runs)) == set(range(er.N_UNOPS))
    assert {r.n_temps for r in runs} == {0, 1, 2} and any(r.both_live for r in runs) and any(r.second_reuse for r in runs)


# ---- data -----------------------------------------------------------------------------------------------------------------------

def float_chunks(rdf, seed, k, zeros: bool, lens=LENS, plant=True):
    """Input k: values in [-4, 4] with planted specials (unless not `plant`); inputs 0 and 3 have no bitmap, the others 15 % nulls
    and start at a different validity bit offset in every chunk."""
    rng = np.random.default_rng(seed * 100 + k)
    out = []
    for j, n in enumerate(lens):
        pad = 0 if k % 3 == 0 else (5 * k + 3 * j) % 37
        v = rng.uniform(-4.0, 4.0, n + pad)
        sp = SPECIALS if zeros else SPECIALS[2:]
        hit = rng.random(n + pad) < (0.03 if plant else 0.0)
        v[hit] = rng.choice(sp, int(hit.sum()))
        if n and plant:
            v[pad + rng.integers(0, n, 3)] = rng.choice(sp, 3)
        mask = None if k % 3 == 0 else rng.random(n + pad) >= 0.15
        a = rdf.PrimitiveArray.from_numpy(v, mask)
        a.null_count = -1 if mask is not None else 0
        out.append(a.slice(pad, n) if pad else a)
    return out


@pytest.fixture(scope="module")
def pools(rdf, ctx):
    """Two sets of six inputs: with planted ±0 (divides often raise) and without (divides mostly compute)."""
    out = {}
    for zeros in (True, False):
        host = [float_chunks(rdf, 1 + zeros, k, zeros) for k in range(er.C["kExprMaxInputs"])]
        out[zeros] = (host, [rdf.Column.upload(h) for h in host])
    yield out
    for _, cols in out.values():
        for c in cols:
            c.free()


def unfused_chain(rdf, cols, nodes):
    """The program one device call per node (the materialised chain)."""
    N = rdf.native
    slots, made = list(cols), []
    try:
        for nd in nodes:
            if len(nd) == 2:
                r = slots[nd[1]].unary(getattr(N, nd[0].upper()))
            else:
                r = getattr(slots[nd[1]], BIN_NAMES[nd[0]])(slots[nd[2]])
            slots.append(r); made.append(r)
        return slots[-1], made[:-1]
    except BaseException:
        for c in made:
            c.free()
        raise


def run_both(rdf, cols, nodes):
    """(fused chunks or the exception class, unfused chunks or the exception class)."""
    try:
        fc = rdf.eval_expr(cols, nodes)
        f = fc.download(); fc.free()
    except rdf.DivideByZero as e:
        f = type(e)
    try:
        uc, tmp = unfused_chain(rdf, cols, nodes)
        u = uc.download()
        for c in tmp + [uc]:
            c.free()
    except rdf.DivideByZero as e:
        u = type(e)
    return f, u


def same_chunks(what, got, want, fused_payload=True):
    assert len(got) == len(want), what
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.length == w.length, f"{what} chunk {i}"
        m = g.valid_mask()
        assert np.array_equal(m, w.valid_mask()), f"{what} chunk {i}: validity"
        assert int((~m).sum()) == int((~w.valid_mask()).sum())
        if g.null_count >= 0 and w.null_count >= 0:
            assert g.null_count == w.null_count, f"{what} chunk {i}: null count"
        bad = np.flatnonzero(~same_bits(g.value_slice()[m], w.value_slice()[m]))
        assert bad.size == 0, f"{what} chunk {i}: {bad.size} values differ, first {g.value_slice()[m][bad[:3]]} vs {w.value_slice()[m][bad[:3]]}"
        if fused_payload and g.validity is not None:
            assert not g.value_slice()[~m].view(np.uint64).any(), f"{what} chunk {i}: a null slot of the fused result is not +0.0"


def _inputs_for(d, seed):
    """Which pool columns feed the DAG's inputs: a rotation, so every input position sees every bitmap layout."""
    return [(seed + i) % er.C["kExprMaxInputs"] for i in range(d[0])]


def test_fused_programs_match_the_unfused_chain(rdf, ctx, oracle, programs, pools):
    raised = computed = exact = 0
    for zeros in (True, False):
        host, cols = pools[zeros]
        for n, (d, _, _) in enumerate(programs):
            nodes = er.eval_nodes(d)
            sel = _inputs_for(d, n)
            f, u = run_both(rdf, [cols[i] for i in sel], nodes)
            what = f"program {n} {d} zeros={zeros}"
            if isinstance(f, type) or isinstance(u, type):
                assert f is u is rdf.DivideByZero, what
                raised += 1
            else:
                same_chunks(what, f, u)
                computed += 1
    # the same shapes with exact operators only (binop mod 4; abs, ceil, floor, round, sqrt): also against the oracle
    host, cols = pools[False]
    exact_un = sorted(er.EXACT_UNOPS)
    for n, (d, _, _) in enumerate(programs[::3]):
        d = (d[0], tuple((er.UNARY_BASE + exact_un[op % 5], a, b) if er.is_unary(op) else (op % 4, a, b) for op, a, b in d[1]))
        nodes = er.eval_nodes(d)
        sel = _inputs_for(d, n)
        f, u = run_both(rdf, [cols[i] for i in sel], nodes)
        st, want = oracle_chain(oracle, [host[i] for i in sel], nodes)
        what = f"exact program {n} {d}"
        assert (f is rdf.DivideByZero) == (u is rdf.DivideByZero) == (st == oracle.DIVIDE_BY_ZERO), what
        if st == oracle.OK:
            same_chunks(what, f, u)
            for i, (g, w) in enumerate(zip(f, want)):
                assert_same_array(g, w, what=f"{what} chunk {i} vs oracle", check_payload=False)
            exact += 1
    assert computed > N_PROGRAMS and raised > 20 and exact > 20, (computed, raised, exact)


def oracle_chain(oracle, inputs, nodes):
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


# ---- typed inputs ---------------------------------------------------------------------------------------------------------------

TYPED = ["I8", "I16", "I32", "I64", "U8", "U16", "U32", "U64", "F32", "F64"]


def typed_chunks(rdf, tname, seed, lens=LENS):
    dtype = getattr(rdf, tname)
    npdt = np.dtype(rdf.NP_DTYPES[dtype])
    rng = np.random.default_rng(seed)
    if npdt.kind == "f" and npdt.itemsize == 4:
        plant = np.array([0x7fc00001, 0xffc12345, 0x7fa00000, 0x00000001, 0x807fffff, 0x00400000, 0x7f7fffff, 0xff800000, 0x80000000],
                         np.uint32).view(np.float32)            # NaN payloads (quiet and signalling), subnormals, max, -inf, -0
    elif npdt.kind == "f":
        plant = SPECIALS[2:]
    else:
        info = np.iinfo(npdt)
        extra = []
        if npdt.itemsize == 8:   # values that round to even on `as f64`
            extra = [2 ** 53 + 1, 2 ** 53 + 3, 2 ** 63 - 1, 2 ** 62 + 2 ** 9 + 1] + ([2 ** 64 - 1, 2 ** 63 + 2 ** 10 + 1] if npdt.kind == "u" else
                                                                                     [-(2 ** 53) - 1, -(2 ** 63) + 1])
        plant = np.array([info.min, info.max, info.min + 1, info.max - 1] + extra, dtype=npdt)
    out = []
    for j, n in enumerate(lens):
        pad = (3 * j + 1) % 29
        if npdt.kind == "f":
            v = rng.normal(0, 100, n + pad).astype(npdt)
        else:
            info = np.iinfo(npdt)
            v = rng.integers(info.min, info.max, n + pad, dtype=npdt, endpoint=True)
        hit = rng.random(n + pad) < 0.05
        v[hit] = rng.choice(plant, int(hit.sum()))
        if n >= TILE:            # every planted value inside a full tile too (the width-specific staging path)
            v[pad:pad + len(plant)] = plant
        mask = rng.random(n + pad) >= 0.1
        a = rdf.PrimitiveArray.from_numpy(v, mask)
        a.null_count = -1
        out.append(a.slice(pad, n))
    return out


@pytest.mark.parametrize("tname", TYPED)
def test_typed_inputs_in_programs_with_temporaries(rdf, ctx, programs, pools, tname):
    """A typed column read `as f64` on load, in programs with 0, 1 and 2 temporaries: the same bits as cast to Float64 then the
    unfused chain."""
    dtype = getattr(rdf, tname)
    typed = rdf.Column.upload(typed_chunks(rdf, tname, 300 + dtype))
    cast = typed.cast(rdf.F64) if dtype != rdf.F64 else typed
    host, cols = pools[False]
    chosen = {t: [p for p in programs if p[2].n_temps == t and p[0][0] >= 2][:6] for t in range(3)}
    assert all(chosen.values())
    for t, plist in chosen.items():
        for n, (d, _, _) in enumerate(plist):
            nodes = er.eval_nodes(d)
            for pos in {0, d[0] - 1}:     # the typed column as the first input and as the last
                fused_in = [typed if i == pos else cols[(n + i) % 6] for i in range(d[0])]
                plain_in = [cast if i == pos else c for i, c in enumerate(fused_in)]
                try:
                    fc = rdf.eval_expr(fused_in, nodes); f = fc.download(); fc.free()
                except rdf.DivideByZero:
                    f = rdf.DivideByZero
                try:
                    uc, tmp = unfused_chain(rdf, plain_in, nodes); u = uc.download()
                    for c in tmp + [uc]:
                        c.free()
                except rdf.DivideByZero:
                    u = rdf.DivideByZero
                what = f"{tname} at input {pos} of {d}"
                if f is rdf.DivideByZero or u is rdf.DivideByZero:
                    assert f is u, what
                else:
                    same_chunks(what, f, u)
    # and the conversion alone, every element: abs of the value read `as f64` on load is abs of the cast kernel's value in every
    # bit, NaNs included (both convert with the same instruction; abs clears only the sign, so a widened payload is compared too)
    f = rdf.eval_expr([typed], [("abs", 0)]).download()
    u = cast.unary(rdf.native.ABS).download()
    same_chunks(f"abs({tname})", f, u)
    for i, (g, w) in enumerate(zip(f, u)):
        m = g.valid_mask()
        gv, wv = g.value_slice()[m].view(np.uint64), w.value_slice()[m].view(np.uint64)
        bad = np.flatnonzero(gv != wv)
        assert bad.size == 0, f"abs({tname}) chunk {i}: bits {[hex(x) for x in gv[bad[:3]]]} vs {[hex(x) for x in wv[bad[:3]]]}"
    if cast is not typed:
        cast.free()
    typed.free()


# ---- DivideByZero ---------------------------------------------------------------------------------------------------------------

def test_divide_by_zero_placements(rdf, ctx):
    """Inputs a (numerator side), b (divisor side: each divisor below is zero exactly where b is) and m (read by a later node).
    A zero divisor raises when both operands of the divide are valid, also when a later node masks the slot, and not when only the
    divisor is valid or the divisor is null.  BIN, RBIN, a divisor held in a temporary and a divide of two intermediates."""
    N = rdf.native
    progs = [[(N.DIV, 0, 1), (N.ADD, 3, 2)],                                  # BIN, the divisor a column
             [(N.ADD, 1, 1), (N.DIV, 0, 3), (N.MUL, 4, 2)],                   # RBIN: a / (b + b)
             [("abs", 1), (N.DIV, 0, 3), (N.MUL, 4, 3), (N.ADD, 5, 2)],       # |b| shared: held in a temporary
             [(N.ADD, 0, 0), (N.ADD, 1, 1), (N.DIV, 3, 4), (N.SUB, 5, 2)]]    # both operands intermediate
    lens = [TILE + 7, 3 * TILE, 37]
    for row in (5, TILE + 3, 2 * TILE + 100, 3 * TILE + TILE + 7 + 20):       # in full tiles and in tails, in several chunks
        for case, (a_ok, b_ok, m_ok, raises) in {"both valid": (1, 1, 1, True), "numerator null": (0, 1, 1, False),
                                                  "masked later": (1, 1, 0, True), "divisor null": (1, 0, 1, False)}.items():
            cols_host = []
            for k, ok in enumerate((a_ok, b_ok, m_ok)):
                v = np.linspace(1.0, 2.0, sum(lens))
                mask = np.ones(sum(lens), bool)
                if k == 1:
                    v[row] = 0.0
                mask[row] = bool(ok)
                starts = np.cumsum([0] + lens)
                cols_host.append(rdf.Column.upload([rdf.PrimitiveArray.from_numpy(v[s:e].copy(), mask[s:e].copy()) for s, e in zip(starts, starts[1:])]))
            for p in progs:
                f, u = run_both(rdf, cols_host, p)
                got = (f is rdf.DivideByZero, u is rdf.DivideByZero)
                assert got == (raises, raises), (case, row, p, got)
            for c in cols_host:
                c.free()


# ---- trailing aggregate ---------------------------------------------------------------------------------------------------------

def test_trailing_aggregate_over_programs(rdf, ctx, programs):
    """eval_expr_agg, materialised or not and asynchronous: the column eval_expr makes, and count and sum within the float-sum bound
    of the exact sum of that column (inputs without planted specials, so that most sums are finite)."""
    cols = [rdf.Column.upload(float_chunks(rdf, 3, k, False, plant=False)) for k in range(er.C["kExprMaxInputs"])]
    checked = 0
    for n, (d, _, r) in enumerate(programs[::6]):
        nodes = er.eval_nodes(d)
        ins = [cols[i] for i in _inputs_for(d, n)]
        try:
            plain = rdf.eval_expr(ins, nodes)
        except rdf.DivideByZero:
            with pytest.raises(rdf.DivideByZero):
                rdf.eval_expr_agg(ins, nodes, materialise=False)
            continue
        col, agg = rdf.eval_expr_agg(ins, nodes)
        none, agg2 = rdf.eval_expr_agg(ins, nodes, materialise=False)
        _, fut = rdf.eval_expr_agg(ins, nodes, materialise=False, asynchronous=True)
        assert none is None
        want = plain.download()
        same_chunks(f"agg column {d}", col.download(), want)
        valid = np.concatenate([w.value_slice()[w.valid_mask()] for w in want])
        assert agg["count"] == valid.size == plain.count() and agg["rows"] == sum(LENS)
        for other in (agg2, fut.result()):      # the same tiles and the same fold: equal counts, and sums equal in every bit
            assert set(other) == set(agg) and other["count"] == agg["count"] and other["rows"] == agg["rows"], d
            assert other["min"] == agg["min"] and other["max"] == agg["max"], d
            assert np.float64(other["sum"]).view(np.uint64) == np.float64(agg["sum"]).view(np.uint64), d
        if np.isfinite(valid).all() and np.abs(valid).max(initial=0) < 1e290:
            exact = np.sum(valid.astype(np.longdouble))
            bound = 16 * np.log2(max(valid.size, 2)) * 2.0 ** -53 * np.sum(np.abs(valid).astype(np.longdouble))
            assert abs(np.longdouble(agg["sum"]) - exact) <= bound, d
            checked += 1
        elif np.isnan(valid).any():
            assert np.isnan(agg["sum"]), d
        for c in (plain, col):
            c.free()
    for c in cols:
        c.free()
    assert checked > 5


# ---- the bulk-copy kernel -------------------------------------------------------------------------------------------------------

def digests(rdf, programs, pools):
    """sha256 of every untyped program's result (values bit for bit, validity, null counts, lengths) or its error: both kernels run
    the same node code on the same inputs, so even NaN payloads must agree."""
    host, cols = pools[False]
    out = []
    for n, (d, _, _) in enumerate(programs):
        nodes = er.eval_nodes(d)
        try:
            c = rdf.eval_expr([cols[i] for i in _inputs_for(d, n)], nodes)
        except rdf.DivideByZero:
            out.append("DivideByZero"); continue
        h = hashlib.sha256()
        for a in c.download():
            m = a.valid_mask()
            h.update(np.int64([a.length, int((~m).sum())]).tobytes())
            h.update(np.ascontiguousarray(a.value_slice()).view(np.uint8).tobytes())   # raw bits, NaN payloads included
            h.update(np.packbits(m).tobytes())
        c.free()
        out.append(h.hexdigest())
    return out


CHILD = """
import json, sys
sys.path[:0] = [{root!r}, {here!r}]
import expr_reference as er
import test_expr_programs_gpu as t
import rust_dataframe_b200 as rdf
prog = [tuple(x) for x in json.load(open({dags!r}))]
progs = [((ni, tuple(tuple(n) for n in nodes)), None, None) for ni, nodes in prog]
host = [t.float_chunks(rdf, 1, k, False) for k in range(er.C["kExprMaxInputs"])]
pools = {{False: (host, [rdf.Column.upload(h) for h in host])}}
json.dump(t.digests(rdf, progs, pools), open({out!r}, "w"))
"""


def test_bulk_kernel_is_bit_identical(rdf, ctx, programs, pools, tmp_path):
    """k_expr_bulk (BDF_EXPR_BULK=1, read once per process: so in a child process) gives the default kernel's bits."""
    dags = [d for d, _, _ in programs]
    (tmp_path / "dags.json").write_text(json.dumps(dags))
    out = tmp_path / "bulk.json"
    root = os.path.dirname(HERE)
    code = CHILD.format(root=root, here=HERE, dags=str(tmp_path / "dags.json"), out=str(out))
    env = dict(os.environ, BDF_EXPR_BULK="1")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    bulk = json.loads(out.read_text())
    want = digests(rdf, programs, pools)
    diff = [(i, dags[i]) for i in range(len(dags)) if bulk[i] != want[i]]
    assert diff[:5] == [], f"{len(diff)} programs differ under the bulk kernel"
    assert sum(x != "DivideByZero" for x in want) > N_PROGRAMS // 2


# ---- the planner ----------------------------------------------------------------------------------------------------------------

def _frame(rdf, seed):
    from rust_dataframe_b200.arrays import TemporalType
    rng = np.random.default_rng(seed)
    lens = [0, 1, 700, TILE + 1, 5000]
    def f64(lo, hi, nf):
        return [rdf.PrimitiveArray.from_numpy(rng.uniform(lo, hi, n), (rng.random(n) >= nf) if nf else None) for n in lens]
    cols = OrderedDict([("a", f64(-3, 3, 0)), ("b", f64(-3, 3, 0.15)), ("c", f64(0.5, 4, 0.05)), ("d", f64(-1, 1, 0.1))])
    cols["x"] = [rdf.PrimitiveArray.from_numpy(rng.normal(0, 3, n).astype(np.float32), rng.random(n) >= 0.1) for n in lens]
    cols["i"] = [rdf.PrimitiveArray.from_numpy(rng.integers(-5, 6, n).astype(np.int32), rng.random(n) >= 0.1) for n in lens]
    cols["k"] = [rdf.PrimitiveArray.from_numpy(rng.integers(0, 4, n).astype(np.int64)) for n in lens]
    cols["flag"] = [rdf.BooleanArray.from_numpy(rng.random(n) < 0.5, rng.random(n) >= 0.1) for n in lens]
    frame = rdf.DeviceFrame.from_host(cols)
    day = rdf.Column.upload([rdf.PrimitiveArray.from_numpy(rng.integers(0, 20000, n).astype(np.int32)) for n in lens], dtype=rdf.I32)
    frame = frame.with_column("day", day.with_temporal(TemporalType.date32()))
    other = rdf.DeviceFrame.from_host(OrderedDict([("k", [rdf.PrimitiveArray.from_numpy(np.arange(4, dtype=np.int64))]),
                                                   ("w", [rdf.PrimitiveArray.from_numpy(np.array([0.5, -1.5, 2.0, 3.25]))])]))
    return frame, other


def random_pipeline(rdf, rng, schema, other):
    F = rdf.frame
    names = OrderedDict(schema)
    steps, fresh = [], [0]

    def new():
        fresh[0] += 1
        return f"t{fresh[0]}"
    for _ in range(int(rng.integers(3, 14))):
        floats = [k for k, t in names.items() if t == rdf.F64]
        r = rng.random()
        if r < 0.55 and floats:
            recent = [n for n in floats if n.startswith("t")][-3:]
            pick = lambda: str(rng.choice(recent)) if recent and rng.random() < 0.6 else str(rng.choice(floats))
            u = rng.random()
            out = new() if u < 0.75 else (pick() if u < 0.9 else str(rng.choice(list(names))))   # overwrites, of a run's own input too
            if rng.random() < 0.7:
                steps.append(F.calculate(str(rng.choice(["add", "subtract", "multiply", "divide"])), [pick(), pick()], out))
            else:
                steps.append(F.calculate(str(rng.choice(["sine", "cosine", "tangent"])), [pick()], out))
            names.pop(out, None); names[out] = rdf.F64
        elif r < 0.63 and len(floats) >= 2:
            # three intermediates shared by the Calculations after them (test_frame.py's three-shared shape, ops and operands
            # drawn): more than the compiler's two temporaries, so it refuses the whole run and the planner must shorten it
            x, y = (str(v) for v in rng.choice(floats, 2, replace=False))
            ops = ["add", "subtract", "multiply"]
            s1, s2, s3, t, u, v, w, z = (new() for _ in range(8))
            block = [(s1, [x, y]), (s2, [x, y]), (s3, [x, y]), (t, [s1, s2]), (u, [t, s3]), (v, [u, s1]), (w, [v, s2]), (z, [w, s3])]
            for out, ins in block:
                steps.append(F.calculate(str(rng.choice(ops)), ins, out)); names[out] = rdf.F64
        elif r < 0.70:
            numeric = [n for n, t in names.items() if t != rdf.F64 and 0 <= t < 10 and n != "day"]   # not Boolean, not Date32
            src = str(rng.choice(numeric if numeric and rng.random() < 0.9 else list(names)))      # sometimes one that is refused
            to = rdf.F64 if rng.random() < 0.75 else int(rng.choice([rdf.F32, rdf.I64, rdf.I32]))
            out = new()
            steps.append(F.calculate("cast", [src], out, to)); names[out] = to
            if to == rdf.F64 and floats and rng.random() < 0.6:            # read at once: a cast the planner can fold into the load
                out2 = new()
                steps.append(F.calculate(str(rng.choice(["add", "multiply", "subtract"])), [out, str(rng.choice(floats))], out2))
                names[out2] = rdf.F64
        elif r < 0.74 and len(names) > 2:
            victims = [str(v) for v in rng.choice(list(names), int(rng.integers(1, 3)), replace=False)]
            steps.append(F.drop(victims))
            for v in victims:
                names.pop(v)
        elif r < 0.78 and len(names) > 3:
            keep = [str(v) for v in rng.choice(list(names), int(rng.integers(2, len(names))), replace=False)]
            steps.append(F.select(keep)); names = OrderedDict((k, t) for k, t in names.items() if k in keep)
        elif r < 0.83 and floats:
            if names.get("flag") == rdf.native.BOOL and rng.random() < 0.9:   # a filter refuses to carry a Boolean column
                steps.append(F.drop(["flag"])); names.pop("flag")
            steps.append(F.filter_(("gt", F.col(str(rng.choice(floats))), F.lit(float(rng.normal())))))
        elif r < 0.87 and floats:
            steps.append(F.sort([(str(rng.choice(floats)), bool(rng.random() < 0.5))]))
        elif r < 0.90:
            steps.append(F.limit(int(rng.integers(0, 3000))))
        elif r < 0.93 and names.get("k") == rdf.I64:
            steps.append(F.join(other, [("k", "k")], str(rng.choice(["inner", "left"]))))
            names = OrderedDict(F.plan_join(names, other.schema, [("k", "k")], "inner"))
        elif r < 0.96 and floats and names.get("k") == rdf.I64:
            out = new()
            steps.append(F.window(["k"], [(str(rng.choice(floats)), False)], [(out, "row_number")]))
            names[out] = rdf.U32
        elif len(names) > 1:
            old = str(rng.choice(list(names)))
            out = f"r{new()}"
            steps.append(F.calculate("rename", [old], out)); names = OrderedDict(((out if k == old else k), t) for k, t in names.items())
    if rng.random() < 0.7 and len(names) > 1:     # the usual end of a lazy pipeline: a few columns, intermediates dead
        keep = [str(v) for v in rng.choice(list(names), int(rng.integers(1, 3)), replace=False)]
        last = [n for n in names if n.startswith("t")]
        steps.append(F.select(keep + last[-1:]))
    return steps


def evaluate(frame, steps, **kw):
    try:
        return frame.evaluate(steps, **kw)
    except Exception as e:   # the same error class on every path is part of the claim
        return type(e)


def frames_equal(x, y, what):
    if isinstance(x, type) or isinstance(y, type):
        assert x is y, what
        return
    assert list(x.columns) == list(y.columns), what
    hx, hy = x.to_host(), y.to_host()
    for name in hx:
        assert len(hx[name]) == len(hy[name]), (what, name)
        for cx, cy in zip(hx[name], hy[name]):
            assert cx.length == cy.length, (what, name)
            m = cx.valid_mask()
            assert np.array_equal(m, cy.valid_mask()), (what, name)
            if isinstance(cx, BooleanArray):
                assert isinstance(cy, BooleanArray), (what, name)
                assert np.array_equal(cx.value_bits()[m], cy.value_bits()[m]), (what, name)
            else:
                vx, vy = cx.value_slice()[m], cy.value_slice()[m]
                assert np.array_equal(vx.view(f"u{vx.dtype.itemsize}"), vy.view(f"u{vy.dtype.itemsize}")), (what, name)


class CheckRecorder:
    """Stands in for the library while plan_fusion runs and records the verdict of every bdf_expr_check call the planner makes."""

    def __init__(self, lib, refused_status):
        self.lib, self.refused_status, self.calls, self.refused = lib, refused_status, 0, 0

    def __getattr__(self, name):
        return getattr(self.lib, name)

    def bdf_expr_check(self, *args):
        st = self.lib.bdf_expr_check(*args)
        self.calls += 1
        self.refused += st == self.refused_status
        return st


def plan_with_refusals(rdf, monkeypatch, schema, steps):
    """(plan, how many runs the compiler refused while the planner made it)."""
    rec = CheckRecorder(rdf.native.lib(), rdf.native.UNSUPPORTED)
    with monkeypatch.context() as m:
        m.setattr(rdf.frame.N, "lib", lambda: rec)
        plan = rdf.frame.plan_fusion(schema, steps)
    return plan, rec.refused


def test_planner_differential(rdf, ctx, monkeypatch):
    """Seeded random pipelines: evaluate(fuse=True), evaluate(fuse=True, fuse_casts=False) and evaluate(fuse=False) give equal
    frames or raise the same error class.  Some pipelines carry runs the compiler refuses (three shared intermediates): the
    planner shortens those runs, and the shortened plans must evaluate to the unfused frame too."""
    frame, other = _frame(rdf, 9)
    rng = np.random.default_rng(2026)
    n, fused, refused, refused_fused, cast_fused, errors = 240, 0, 0, 0, 0, Counter()
    for trial in range(n):
        steps = random_pipeline(rdf, rng, frame.schema, other)
        plan, n_refused = plan_with_refusals(rdf, monkeypatch, frame.schema, steps)
        kinds = [k for k, _ in plan]
        fused += "fused" in kinds
        cast_fused += any(k == "fused" and any(c.function == "cast" for c in a.replaced) for k, a in plan)
        want = evaluate(frame, steps, fuse=False)
        if isinstance(want, type):
            errors[want.__name__] += 1
        elif n_refused:
            refused += 1
            refused_fused += "fused" in kinds       # refused, shortened, and still fused in part
        frames_equal(evaluate(frame, steps), want, (trial, steps))
        frames_equal(evaluate(frame, steps, fuse_casts=False), want, (trial, steps, "fuse_casts=False"))
    print(f"{fused} of {n} pipelines fused, {cast_fused} with a cast, {refused} evaluated with a run the compiler refused "
          f"({refused_fused} of them still fused in part), raised: {dict(errors)}")
    assert fused >= n // 4 and cast_fused >= 5 and refused >= 8 and refused_fused >= 5 and sum(errors.values()) < n // 4
