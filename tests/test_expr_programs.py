"""The fused expression path's host compiler (expr_compile in csrc/k_expr.cu) over every small DAG and 200 k random ones, checked by the
symbolic accumulator machine of tests/expr_reference.py.  No GPU: tests/expr_harness.cu includes k_expr.cu and is compiled by nvcc as a
host program.  BDF_EXPR_CSRC points the build at another copy of csrc/.

Corpus: every DAG of at most 4 nodes over 1, 2 and 3 inputs, every DAG of at most 5 nodes over 2 inputs (up to the operator: the
compiler only tells unary from binary), and 200 k seeded random DAGs of 6 to 12 nodes over 1 to 6 inputs, biased towards shared
nodes, x == y and binary nodes whose operands are both intermediate."""
import ctypes as C
import os
import shutil
import subprocess
from collections import Counter

import pytest

import expr_reference as er

HERE = os.path.dirname(os.path.abspath(__file__))
EXHAUSTIVE = [(1, 4), (2, 4), (3, 4), (2, 5)]     # (inputs, at most this many nodes)
N_RANDOM, RANDOM_SEED = 200_000, 20261018

# Code-2 refusals ("more than two intermediates alive at once") of the exhaustive sets.  Any change to the compiler's rule must edit
# these.  Some of them a better evaluation order would avoid (x == y holds x in a temporary it does not need); that is not a bug.
PINNED = {
    (1, 4): {0: 674, 1: 2364, 2: 0},
    (2, 4): {0: 5730, 1: 38988, 2: 0},
    (3, 4): {0: 24780, 1: 285072, 2: 0},
    (2, 5): {0: 110850, 1: 1744812, 2: 3456},
}


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and os.path.exists(cand):
            return cand
    return None


class Harness:
    def __init__(self, exe):
        self.exe = exe

    def compile(self, dags):
        """(code, Prog or None) of every DAG."""
        text = "".join(er.dag_line(d) + "\n" for d in dags)
        out = subprocess.run([self.exe], input=text, capture_output=True, text=True, check=True).stdout.splitlines()
        assert len(out) == len(dags)
        return [er.parse_result(line) for line in out]

    def constants(self):
        out = subprocess.run([self.exe, "constants"], capture_output=True, text=True, check=True).stdout.split()
        return {k: int(v) for k, v in zip(out[::2], out[1::2])}


_BUILT = {}   # csrc directory -> Harness: one build per session, also when another test module imports this fixture


@pytest.fixture(scope="session")
def harness(tmp_path_factory):
    """nvcc over tests/expr_harness.cu and the k_expr.cu of BDF_EXPR_CSRC (default: the package's csrc/).  PTX only: the kernels are
    compiled but never run."""
    if er.CSRC in _BUILT:
        return _BUILT[er.CSRC]
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc is not installed: the expression compiler cannot be built for the host")
    exe = str(tmp_path_factory.mktemp("expr_harness") / "expr_harness")
    subprocess.run([nvcc, "-std=c++17", "-O2", "-w", "-gencode", "arch=compute_90a,code=compute_90a", "-I", er.CSRC,
                    os.path.join(HERE, "expr_harness.cu"), "-o", exe], check=True)
    _BUILT[er.CSRC] = Harness(exe)
    return _BUILT[er.CSRC]


@pytest.fixture(scope="session")
def exhaustive(harness):
    """{(inputs, max nodes): [(dag, code, prog)]}"""
    out = {}
    for ni, nn in EXHAUSTIVE:
        dags = list(er.enumerate_dags(ni, nn))
        assert len(dags) == er.count_dags(ni, nn)
        out[(ni, nn)] = [(d, c, p) for d, (c, p) in zip(dags, harness.compile(dags))]
    return out


@pytest.fixture(scope="session")
def random_corpus(harness):
    dags = er.random_dags(N_RANDOM, RANDOM_SEED)
    return [(d, c, p) for d, (c, p) in zip(dags, harness.compile(dags))]


def _all(exhaustive, random_corpus):
    for rows in exhaustive.values():
        yield from rows
    yield from random_corpus


def test_constants_read_from_the_source_are_the_compiled_ones(harness):
    got = harness.constants()
    for name in ("kExprMaxInputs", "kExprMaxNodes", "kExprMaxIns", "kExprMaxTemps", "kExprUnroll", "kBulkU", "kThreads", "XI_BIN",
                 "XI_RBIN", "XI_LOAD", "XI_STORE", "XI_UN", "kOperandAcc"):
        assert got[name] == er.C[name], name
    assert got["expr_tile_elems"] == er.C["tile"]
    assert er.C["kExprMaxTemps"] == 2 and er.C["kExprUnaryBase"] == er.UNARY_BASE


def test_random_corpus_has_the_shapes_it_promises(random_corpus):
    assert len(random_corpus) >= 200_000
    sizes = Counter(len(d[1]) for d, _, _ in random_corpus)
    inputs = Counter(d[0] for d, _, _ in random_corpus)
    assert set(sizes) == set(range(6, 13)) and set(inputs) == set(range(1, 7))
    codes = Counter(c for _, c, _ in random_corpus)
    assert codes[0] >= 50_000 and codes[1] >= 20_000 and codes[2] >= 20_000, codes


def test_every_accepted_program_computes_its_dag(exhaustive, random_corpus):
    """The symbolic machine: the result is the DAG's last node, its validity the inputs that node reaches, every node computed
    exactly once, no temporary read before it is written, no slot beyond n_slots <= n_inputs + 2; no program longer than kExprMaxIns."""
    bad, n, max_ins = [], 0, 0
    for dag, code, prog in _all(exhaustive, random_corpus):
        assert code in (0, 1, 2), (dag, code)          # code 3 (too long) is unreachable with 12 nodes: at most 3 instructions each
        if code:
            continue
        n += 1
        max_ins = max(max_ins, prog.n_ins)
        run = er.interpret(dag, prog)
        if run.errors and len(bad) < 8:
            bad.append((dag, prog.ins, run.errors))
    assert bad == []
    assert n > 200_000
    assert max_ins <= er.C["kExprMaxIns"]
    print(f"{n} accepted programs, at most {max_ins} instructions")


def test_code_1_exactly_when_a_node_is_unused(exhaustive, random_corpus):
    wrong = [(d, c) for d, c, _ in _all(exhaustive, random_corpus) if (c == 1) != er.has_dead_node(d)]
    assert wrong[:8] == []


def test_trees_with_a_leaf_operand_are_always_accepted(exhaustive, random_corpus):
    """No shared node and a column operand on every binary node, like BASELINE config 2's chain: never refused."""
    n, refused = 0, []
    for d, c, _ in _all(exhaustive, random_corpus):
        if er.tree_with_leaf_operands(d):
            n += 1
            if c != 0:
                refused.append((d, c))
    assert refused[:8] == [] and n > 10_000


def test_refusal_counts_are_pinned(exhaustive):
    got = {k: dict(sorted(Counter(c for _, c, _ in rows).items())) for k, rows in exhaustive.items()}
    for k in got:
        got[k] = {code: got[k].get(code, 0) for code in (0, 1, 2)}
    assert got == PINNED


def test_corpus_reaches_every_branch_of_the_compiler(exhaustive, random_corpus):
    """RBIN with each binop (a leaf left operand), BIN with each, every unary, x == y (the accumulator as operand), 0, 1 and 2
    temporaries, a temporary re-taken after it was freed (the second one too), and both temporaries live at once."""
    rbin, binops, unops, temps = Counter(), Counter(), Counter(), Counter()
    reuse = second = both = acc_operand = 0
    for d, c, p in random_corpus:
        if c:
            continue
        run = er.interpret(d, p)
        rbin.update(run.rbin); binops.update(run.bin); unops.update(run.unops); temps[run.n_temps] += 1
        reuse += run.temp_reuse; second += run.second_reuse; both += run.both_live
        acc_operand += any(src == er.ACC for _, src in p.ins)
    assert set(rbin) == set(binops) == set(range(er.N_BINOPS)) and min(rbin.values()) > 100
    assert set(unops) == set(range(er.N_UNOPS))
    assert set(temps) == {0, 1, 2} and temps[1] > 100 and temps[2] > 100   # most 0-temporary programs are in the exhaustive sets
    assert reuse > 100 and second > 100 and both > 100 and acc_operand > 100
    # and the exhaustive sets reach RBIN, x == y and both temporaries too
    runs = [er.interpret(d, p) for d, c, p in exhaustive[(2, 5)] if c == 0]
    assert any(r.rbin for r in runs) and any(r.both_live for r in runs) and any(r.second_reuse for r in runs)


def test_library_compiler_is_the_harness_compiler(rdf, exhaustive, random_corpus):
    """bdf_expr_check (the shipped library, no GPU) gives the same verdict, instruction count and temporaries for every corpus DAG:
    the harness compiles the code the library runs."""
    N = rdf.native
    check = N.lib().bdf_expr_check
    Node = N.ExprNode
    want_status = {0: N.OK, 1: N.INVALID, 2: N.UNSUPPORTED}
    ni_, nt_ = C.c_int32(), C.c_int32()
    bad = []
    for d, c, p in _all(exhaustive, random_corpus):
        nodes = d[1]
        arr = (Node * len(nodes))(*[Node(o, a, b) for o, a, b in nodes])
        ni_.value = nt_.value = -1
        st = check(d[0], None, len(nodes), arr, C.byref(ni_), C.byref(nt_))
        if st != want_status[c] or (c == 0 and (ni_.value, nt_.value) != (p.n_ins, p.n_slots - d[0])):
            bad.append((d, c, st, ni_.value, nt_.value))
            if len(bad) >= 8:
                break
    assert bad == []


def test_the_interpreter_rejects_wrong_programs(harness):
    """The reference itself: swapped RBIN operands, a lost STORE, a temporary read before it is written, a node computed twice, a
    slot beyond n_slots and a wrong validity are each reported."""
    dag = (2, ((er.SUB, 0, 1), (er.MUL, 2, 2), (er.DIV, 0, 3), (er.ADD, 4, 2)))
    (code, prog), = harness.compile([dag])
    assert code == 0 and er.interpret(dag, prog).errors == []
    ops = [o for o, _ in prog.ins]
    assert er.XI_RBIN + er.DIV in ops and er.XI_STORE in ops

    def broken(f):
        ins = [list(x) for x in prog.ins]
        f(ins)
        return er.interpret(dag, er.Prog(len(ins), prog.n_slots, [tuple(x) for x in ins])).errors
    k_rbin = ops.index(er.XI_RBIN + er.DIV)
    k_store = ops.index(er.XI_STORE)

    def swap(ins):
        ins[k_rbin][0] = er.XI_BIN + er.DIV
    assert broken(swap)
    assert broken(lambda ins: ins.pop(k_store))
    assert broken(lambda ins: ins.__setitem__(k_store, [er.XI_LOAD, 0]))
    assert broken(lambda ins: ins.insert(1, list(ins[1])))
    assert broken(lambda ins: ins.__setitem__(k_store, [er.XI_STORE, prog.n_slots]))
    assert broken(lambda ins: ins.__setitem__(0, [er.XI_LOAD, 1]))
