"""A reference for the fused expression path's host compiler (expr_compile in csrc/k_expr.cu): a corpus of straight-line DAGs, a
symbolic interpreter of the accumulator machine the kernels run, and the compiler's acceptance rules.  Standard library only; no GPU.

A DAG is (n_inputs, nodes).  Slot s < n_inputs is input s, slot n_inputs + k is node k, and a node is (op, a, b) in the C ABI's
numbering: op 0..6 is a binary operator (ADD SUB MUL DIV ATAN2 HYPOT LOG), op 100 + u the unary function u with b == a.

The interpreter restates the node loop of k_expr / k_expr_bulk over expressions instead of numbers.  Each slot and the accumulator hold
an interned expression (op and ordered operands) and the set of inputs its validity depends on, so a program is checked exactly: it
must compute the DAG's last node, compute every node exactly once (so each divide can raise exactly when the materialised chain's
would), never read a temporary it has not written, and stay inside the slots it declares."""
from __future__ import annotations

import os
import random
import re
from collections import Counter
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.environ.get("BDF_EXPR_CSRC", os.path.join(os.path.dirname(HERE), "rust-dataframe_b200", "csrc"))

UNARY_BASE = 100
N_BINOPS, N_UNOPS = 7, 21
ADD, SUB, MUL, DIV, ATAN2, HYPOT, LOG = range(7)


def constants() -> Dict[str, int]:
    """The compiler's limits, the opcodes and the tile sizes, read from the sources the harness compiles."""
    src = open(os.path.join(CSRC, "k_expr.cu")).read()
    common = open(os.path.join(CSRC, "common.cuh")).read()
    out = {}
    for name in ("kExprMaxInputs", "kExprMaxNodes", "kExprMaxIns", "kExprUnroll", "kExprMaxTemps", "kBulkU", "kOperandAcc",
                 "kExprUnaryBase"):
        out[name] = int(re.search(rf"constexpr int {name} = (\d+);", src).group(1))
    for name in ("XI_BIN", "XI_RBIN", "XI_LOAD", "XI_STORE", "XI_UN"):
        out[name] = int(re.search(rf"\b{name} = (\d+)", src).group(1))
    out["kThreads"] = int(re.search(r"constexpr int kThreads = (\d+);", common).group(1))
    out["tile"] = out["kThreads"] * out["kExprUnroll"] * 2
    out["half_tile"] = out["kThreads"] * out["kBulkU"] * 2
    return out


C = constants()
XI_BIN, XI_RBIN, XI_LOAD, XI_STORE, XI_UN, ACC = C["XI_BIN"], C["XI_RBIN"], C["XI_LOAD"], C["XI_STORE"], C["XI_UN"], C["kOperandAcc"]


def is_unary(op: int) -> bool:
    return op >= UNARY_BASE


# ---- the corpus ------------------------------------------------------------------------------------------------------------------

def enumerate_dags(n_inputs: int, max_nodes: int, binop: int = ADD, unop: int = UNARY_BASE):
    """Every DAG of 1..max_nodes nodes over n_inputs inputs, up to the operator: the compiler only tells unary from binary, so each
    node is one unary (one operand) or one binary (an ordered pair of operands) over the slots before it."""
    def grow(nodes):
        yield (n_inputs, tuple(nodes))
        if len(nodes) == max_nodes:
            return
        s = n_inputs + len(nodes)
        for x in range(s):
            yield from grow(nodes + [(unop, x, x)])
        for x in range(s):
            for y in range(s):
                yield from grow(nodes + [(binop, x, y)])
    for first in grow([]):
        if first[1]:
            yield first


def count_dags(n_inputs: int, max_nodes: int) -> int:
    total, prod = 0, 1
    for k in range(max_nodes):
        s = n_inputs + k
        prod *= s + s * s
        total += prod
    return total


def random_dags(n: int, seed: int, min_nodes: int = 6, max_nodes: int = 12, max_inputs: int = 6) -> List[tuple]:
    """Seeded random DAGs, biased towards what makes the compiler work: operands taken from the last few nodes, nodes not used yet,
    x == y, and binary nodes whose two operands are both intermediate.  Operators are drawn from all 7 binaries and 21 unaries."""
    rng = random.Random(seed)
    out = []
    for _ in range(n):
        ni = rng.randint(1, max_inputs)
        nn = rng.randint(min_nodes, max_nodes)
        nodes, unused = [], []
        for k in range(nn):
            s = ni + k

            def pick():
                r = rng.random()
                if unused and r < 0.35:                                         # a node not used yet
                    return rng.choice(unused)
                if k and r < 0.7:
                    return ni + k - 1 - min(int(rng.expovariate(0.8)), k - 1)   # recent nodes
                return rng.randrange(s)
            if len(unused) >= 2 and nn - k <= len(unused) and rng.random() < 0.9:
                x, y = rng.sample(unused, 2)                                     # use up the unused nodes: most DAGs stay live
                nodes.append((rng.randrange(N_BINOPS), x, y))
            elif rng.random() < 0.28:
                x = pick()
                nodes.append((UNARY_BASE + rng.randrange(N_UNOPS), x, x))
            else:
                x = pick()
                r = rng.random()
                if r < 0.12:
                    y = x
                elif r < 0.45 and k >= 2:
                    y = rng.randrange(ni, s)                                     # both operands intermediate (often)
                    x = x if x >= ni else rng.randrange(ni, s)
                else:
                    y = pick()
                if rng.random() < 0.5:
                    x, y = y, x
                nodes.append((rng.randrange(N_BINOPS), x, y))
            for v in set(nodes[-1][1:]):
                if v in unused:
                    unused.remove(v)
            unused.append(s)
        out.append((ni, tuple(nodes)))
    return out


# ---- DAG properties ----------------------------------------------------------------------------------------------------------

def uses(dag) -> List[int]:
    """References to every slot, with one for the result column (the compiler's count)."""
    ni, nodes = dag
    u = [0] * (ni + len(nodes))
    u[-1] = 1
    for op, a, b in nodes:
        u[a] += 1
        if not is_unary(op):
            u[b] += 1
    return u


def has_dead_node(dag) -> bool:
    ni, nodes = dag
    return any(c == 0 for c in uses(dag)[ni:])


def tree_with_leaf_operands(dag) -> bool:
    """No node is used more than once, and every binary node has an input column for an operand (like BASELINE config 2's chain):
    the compiler must accept every such DAG."""
    ni, nodes = dag
    if any(c != 1 for c in uses(dag)[ni:]):
        return False
    return all(is_unary(op) or a < ni or b < ni for op, a, b in nodes)


class Interner:
    def __init__(self):
        self.ids: Dict[tuple, int] = {}

    def __call__(self, key: tuple) -> int:
        i = self.ids.get(key)
        if i is None:
            i = self.ids[key] = len(self.ids)
        return i


def node_exprs(dag, intern: Interner) -> Tuple[List[int], List[frozenset]]:
    """The interned expression and the input set of every node."""
    ni, nodes = dag
    ex = [intern(("in", i)) for i in range(ni)]
    dep = [frozenset([i]) for i in range(ni)]
    for op, a, b in nodes:
        if is_unary(op):
            ex.append(intern((op, ex[a]))); dep.append(dep[a])
        else:
            ex.append(intern((op, ex[a], ex[b]))); dep.append(dep[a] | dep[b])
    return ex[ni:], dep[ni:]


# ---- the accumulator machine, symbolically --------------------------------------------------------------------------------------

@dataclass
class Prog:
    n_ins: int
    n_slots: int
    ins: List[Tuple[int, int]]          # (op, src)


@dataclass
class Run:
    """What one program did, for the coverage counts."""
    errors: List[str] = field(default_factory=list)
    rbin: set = field(default_factory=set)          # binops used in RBIN form
    bin: set = field(default_factory=set)           # binops used in BIN form
    unops: set = field(default_factory=set)
    n_temps: int = 0
    temp_reuse: bool = False                        # a temporary stored again after its value was read (freed and re-taken)
    second_reuse: bool = False                      # ... temporary 1 in particular (taken only while temporary 0 was busy)
    both_live: bool = False                         # both temporaries hold a value that is still to be read


def interpret(dag, prog: Prog) -> Run:
    """Run `prog` over expressions and check it against `dag`."""
    ni, nodes = dag
    run = Run()
    err = run.errors.append
    intern = Interner()
    want, wdep = node_exprs(dag, intern)
    want_count = Counter(want)
    if prog.n_slots > ni + C["kExprMaxTemps"] or prog.n_slots < ni:
        err(f"n_slots {prog.n_slots} for {ni} inputs")
    if prog.n_ins != len(prog.ins) or prog.n_ins > C["kExprMaxIns"]:
        err(f"n_ins {prog.n_ins}")
    slot_ex: List[Optional[int]] = [intern(("in", i)) for i in range(ni)] + [None] * C["kExprMaxTemps"]
    slot_dep: List[Optional[frozenset]] = [frozenset([i]) for i in range(ni)] + [None] * C["kExprMaxTemps"]
    acc, adep = None, None
    computed = Counter()
    stores = [0] * C["kExprMaxTemps"]
    pending = [False] * C["kExprMaxTemps"]          # stored and not read since
    read_since = [False] * C["kExprMaxTemps"]

    def operand(src):
        if src == ACC:
            if acc is None:
                err("reads the accumulator before it is loaded")
            return acc, adep
        if src < 0 or src >= prog.n_slots:
            err(f"operand slot {src} outside n_slots {prog.n_slots}")
            return None, None
        if src >= ni:
            t = src - ni
            if slot_ex[src] is None:
                err(f"reads temporary {t} before writing it")
            pending[t] = False; read_since[t] = True
        return slot_ex[src], slot_dep[src]

    for op, src in prog.ins:
        if run.errors:
            break
        if op >= XI_UN:
            u = op - XI_UN
            if acc is None or u >= N_UNOPS:
                err(f"unary {u} on an empty accumulator or out of range"); break
            acc = intern((UNARY_BASE + u, acc)); computed[acc] += 1; run.unops.add(u)
        elif op == XI_STORE:
            if acc is None or src < ni or src >= prog.n_slots:
                err(f"store to slot {src}"); break
            t = src - ni
            if stores[t] and read_since[t]:
                run.temp_reuse = True
                run.second_reuse = run.second_reuse or t == 1
            stores[t] += 1
            slot_ex[src], slot_dep[src] = acc, adep
            pending[t] = True; read_since[t] = False
            if all(pending):
                run.both_live = True
            run.n_temps = max(run.n_temps, t + 1)
        elif op == XI_LOAD:
            if src == ACC:
                err("LOAD of the accumulator"); break
            acc, adep = operand(src)
        elif XI_BIN <= op < XI_BIN + N_BINOPS or XI_RBIN <= op < XI_RBIN + N_BINOPS:
            o, odep = operand(src)
            if acc is None or o is None:
                err("binary on an empty operand"); break
            if op >= XI_RBIN:
                b = op - XI_RBIN; acc = intern((b, o, acc)); run.rbin.add(b)
            else:
                b = op - XI_BIN; acc = intern((b, acc, o)); run.bin.add(b)
            adep = adep | odep
            computed[acc] += 1
        else:
            err(f"unknown opcode {op}")
    if not run.errors:
        if acc != want[-1]:
            err("the result is not the DAG's last node")
        elif adep != wdep[-1]:
            err(f"validity depends on {sorted(adep)}, the last node on {sorted(wdep[-1])}")
        if computed != want_count:
            err("some node is computed a different number of times than the DAG has it")
    return run


# ---- the harness's output -------------------------------------------------------------------------------------------------------

def dag_line(dag) -> str:
    ni, nodes = dag
    return f"{ni} {len(nodes)} " + " ".join(f"{o} {a} {b}" for o, a, b in nodes)


def parse_result(line: str) -> Tuple[int, Optional[Prog]]:
    v = list(map(int, line.split()))
    if v[0] != 0:
        return v[0], None
    n_ins, n_slots = v[1], v[2]
    return 0, Prog(n_ins, n_slots, [(v[3 + 2 * k], v[4 + 2 * k]) for k in range(n_ins)])


# ---- node tuples for rdf.eval_expr / the unfused chain ----------------------------------------------------------------------

UNARY_NAMES = ["abs", "sin", "cos", "tan", "acos", "asin", "atan", "cbrt", "ceil", "cosh", "degrees", "exp", "expm1", "floor",
               "log10", "log2", "radians", "round", "sinh", "sqrt", "tanh"]
EXACT_UNOPS = {0, 8, 13, 17, 19}                 # abs, ceil, floor, round, sqrt: correctly rounded everywhere
EXACT_BINOPS = {ADD, SUB, MUL, DIV}


def eval_nodes(dag) -> List[tuple]:
    """The DAG as eval_expr's node list: (binop, a, b) or (unop name, a)."""
    return [(UNARY_NAMES[op - UNARY_BASE], a) if is_unary(op) else (op, a, b) for op, a, b in dag[1]]


def exact_only(dag) -> bool:
    return all((op - UNARY_BASE in EXACT_UNOPS) if is_unary(op) else op in EXACT_BINOPS for op, _, _ in dag[1])


def stratified(dags_progs: Sequence[Tuple[tuple, Prog, Run]], n: int, seed: int) -> List[Tuple[tuple, Prog, Run]]:
    """A few hundred accepted programs that together use every binop as BIN and as RBIN, every unary, 0, 1 and 2 temporaries, and
    temporaries re-taken after a free; the rest drawn at random."""
    rng = random.Random(seed)
    pool = list(dags_progs)
    rng.shuffle(pool)
    want = {("bin", b) for b in range(N_BINOPS)} | {("rbin", b) for b in range(N_BINOPS)} | {("un", u) for u in range(N_UNOPS)}
    want |= {("temps", t) for t in range(3)} | {("reuse", True), ("both", True), ("second", True)}
    pick, seen = [], set()

    def feats(r: Run):
        f = {("bin", b) for b in r.bin} | {("rbin", b) for b in r.rbin} | {("un", u) for u in r.unops} | {("temps", r.n_temps)}
        return f | {("reuse", r.temp_reuse), ("both", r.both_live), ("second", r.second_reuse)}
    for item in pool:
        f = feats(item[2]) & want
        if f - seen:
            pick.append(item); seen |= f
    missing = want - seen
    assert not missing, f"the corpus lacks {sorted(missing)}"
    rest = [it for it in pool if it not in pick]
    # an even share of 0, 1 and 2 temporaries in the remainder
    by_t = {t: [it for it in rest if it[2].n_temps == t] for t in range(3)}
    while len(pick) < n and any(by_t.values()):
        for t in range(3):
            if by_t[t] and len(pick) < n:
                pick.append(by_t[t].pop())
    return pick
