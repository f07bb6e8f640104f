"""Device-resident mirror of the reference's lazy evaluator for the transformations on the path.

``Evaluate::evaluate`` (src/evaluation.rs:66-96) walks a list of Transformations and rebuilds the DataFrame after each
one; ``Evaluate::calculate`` (:97-323) dispatches a Calculation to ScalarFunctions / cast and appends the result with
``with_column``.  ``DeviceFrame`` does the same with columns that live in HBM (one ``Column`` per name, one chunk per
RecordBatch), so a pipeline of Calculations, filters and a sort never crosses PCIe between steps:

    frame = DeviceFrame.from_arrow("in.arrow")                        # DataFrame::from_arrow
    frame = frame.evaluate([calculate("add", ["a", "b"], "e"), ..., select(["h"])])
    frame.to_arrow("out.arrow")                                       # DataFrame::to_arrow

``plan_fusion`` is the optimiser pass SURVEY 8(f) N3 asks for (the natural neighbour of src/optimiser.rs): a run of
consecutive Float64 Calculations (and casts TO Float64 that feed them) whose intermediate columns are removed by a
later Select/Drop before anything else reads them is replaced by ONE fused step (``bdf_eval_expr_dev``); what the caller can observe does not change.
The planner is plain host logic (tested without a GPU); everything that touches data goes through the C ABI.

Kept as the reference has it: select/drop keep frame order (:258-330), with_column replaces an existing name by
drop + append (:97-113), arithmetic Calculations exist for the 8 types of calculate's match (Int8/UInt8 panic with
"Unsupported operation"), trig for floats only, GroupAggregate panics.  Different on purpose: ``limit`` gathers the
first rows into one chunk (the reference slices chunks zero-copy).  Join (``DeviceFrame.join``, the ``("join", (other,
criteria, how))`` step) plans the schema ``Dataset::try_join`` plans and takes every column by the index pairs of
``bdf_join_indices_dev``, whose order is defined where the reference's is not (src/functions/join.rs emits its pairs in
HashMap iteration order): left rows in row order, each one's partners in right row order; a null key matches nothing, and
FULL is the SQL full outer join (include/b200df.h lists the five departures).  Window functions (``DeviceFrame.window``, the
``("window", (partition_by, order_by, calls))`` step) add one column per call in the frame's row order, as ``with_column`` does; the
reference declares WindowSpec and WindowFunctions without bodies (src/window.rs:8-22, src/functions/window.rs:1-11).
"""
from __future__ import annotations

import json
from collections import OrderedDict
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np

from . import _native as N
from .arrays import F32, F64, I8, I64, NP_DTYPES, U8, U32, U64, PrimitiveArray, is_float
from .functions import Column, ListColumn, _expr_nodes, eval_expr, sort_indices, top_k_indices, window as _window
from .csv_reader import CsvFile, write_csv
from .json_reader import JsonFile, write_json
from .parquet_reader import ParquetFile, write_parquet
from .ipc import BOOL, IpcFile, write_ipc

ARITH = {"add": N.ADD, "subtract": N.SUB, "multiply": N.MUL, "divide": N.DIV}
TRIG = {"sine": "sin", "cosine": "cos", "tangent": "tan"}
CMP = {"gt": N.GT, "ge": N.GE, "eq": N.EQ, "ne": N.NE, "lt": N.LT, "le": N.LE}
FLIP = {"gt": "lt", "ge": "le", "lt": "gt", "le": "ge", "eq": "eq", "ne": "ne"}


@dataclass
class Calculation:
    """expression.rs:410-416: inputs by name, one output column, a Function."""
    function: str                      # add | subtract | multiply | divide | sine | cosine | tangent | cast | rename
    inputs: List[str]
    output: str
    dtype: Optional[int] = None        # output type (cast: the target; others: the inputs' type)


@dataclass
class Fused:
    """A run of Calculations the planner merged: slots 0..len(inputs)-1 are input columns, node k is slot len(inputs)+k."""
    inputs: List[str]
    nodes: List[tuple]
    output: str
    replaced: List[Calculation] = field(default_factory=list)


def calculate(function: str, inputs: Sequence[str], output: str, dtype: Optional[int] = None):
    return ("calculate", Calculation(function, list(inputs), output, dtype))


def select(names: Sequence[str]):
    return ("select", list(names))


def drop(names: Sequence[str]):
    return ("drop", list(names))


def filter_(condition):
    return ("filter", condition)


def limit(n: int):
    return ("limit", int(n))


def sort(criteria: Sequence[Tuple[str, bool]]):
    """criteria: [(column, descending)] -- SortCriteria::nulls_first is ignored by the reference (dataframe.rs:205-208)."""
    return ("sort", [(c, bool(d)) for c, d in criteria])


# AggregateFunction (expression.rs:696-710) by the name used in output columns; None = planned but refused by try_aggregate
AGGREGATE_FUNCTIONS = {"sum": "sum", "max": "max", "min": "min", "avg": "avg", "count": "count", "countdistinct": "count_distinct",
                       "first": "first", "last": "last", "kurtosis": None, "skewness": None, "stddev": None, "sumdistinct": None,
                       "variance": None}


def _aggregate_function(name: str) -> Optional[str]:
    key = str(name).replace("_", "").lower()
    if key not in AGGREGATE_FUNCTIONS:
        raise N.UnsupportedType(f"unknown aggregate function {name!r}")
    return AGGREGATE_FUNCTIONS[key]


def plan_aggregate(schema: Dict[str, int], groups: Sequence[str], aggregations: Sequence[Tuple[str, Sequence[str]]]) -> List[Tuple[str, int]]:
    """The output schema `Dataset::try_aggregate` (expression.rs:114-221) plans for `GroupAggregate(groups, aggr)`, as
    [(name, dtype)]: the group columns, then `fn(x)` for every column of every Aggregation (``(function, [columns])``, the shape
    of `Aggregation { function, columns }`).  Its checks in its order: a missing group column, then per aggregation and column a
    missing column ("... does not exist") or kurtosis / skewness / stddev / sum_distinct / variance ("Aggregation not yet
    supported") -- ComputeError.  Then what the device path adds: non-numeric columns and avg of Int64 / UInt64 are
    UnsupportedType.  Departures from the reference's types, on purpose: avg(x) is Float64 (try_aggregate types it as x).
    count(x) / count_distinct(x) are UInt32 as planned."""
    out: List[Tuple[str, int]] = []
    for g in groups:
        if g not in schema:
            raise N.ComputeError(f"Grouping column {json.dumps(g)} does not exist")
        out.append((g, schema[g]))
    planned = []
    for function, columns in aggregations:
        fn = _aggregate_function(function)
        for x in columns:
            if x not in schema:
                raise N.ComputeError(f"Aggregating column {json.dumps(x)} does not exist")
            if fn is None:
                raise N.ComputeError("Aggregation not yet supported")
            planned.append((fn, x))
    for name in list(groups) + [x for _, x in planned]:
        if schema[name] == BOOL or not 0 <= schema[name] <= F64:
            raise N.UnsupportedType(f"column {name!r} is not numeric: group-by keys and aggregated columns must be")
    for fn, x in planned:
        if fn == "avg" and schema[x] in (I64, U64):
            raise N.UnsupportedType("avg needs f64: From<T::Native>")
        out.append((f"{fn}({x})", U32 if fn in ("count", "count_distinct") else F64 if fn == "avg" else schema[x]))
    return out


def join(other: "DeviceFrame", criteria: Sequence[Tuple[str, str]], how: str):
    """Transformation::Join against `other`: criteria [(column of this frame, column of other)], how in left | right | inner | full |
    left_semi | left_anti."""
    return ("join", (other, [(a, b) for a, b in criteria], how))


def join_asof(other: "DeviceFrame", left_on: str, right_on: Optional[str] = None, by: Sequence[Tuple[str, str]] = (), direction: str = "backward",
              allow_exact_matches: bool = True, tolerance=None):
    """An as-of join against `other` (DeviceFrame.join_asof): `by` is [(column of this frame, column of other)]."""
    return ("join_asof", (other, left_on, left_on if right_on is None else right_on, [(a, b) for a, b in by], direction, allow_exact_matches,
                          tolerance))


EXISTENCE_JOINS = ("left_semi", "left_anti")


def distinct(subset: Optional[Sequence[str]] = None, keep="first"):
    """DeviceFrame.drop_duplicates(subset, keep) as a step; distinct() is drop_duplicates() over every column."""
    return ("distinct", (None if subset is None else list(subset), keep))


SET_OPS = ("union", "union_by_name", "intersect", "intersect_all", "subtract", "except_all")


def set_op(other: "DeviceFrame", op: str):
    """One of SET_OPS against `other` as a step (the DeviceFrame method of that name)."""
    return ("set_op", (other, op))


def plan_set_op(schema_a: Dict[str, int], schema_b: Dict[str, int], op: str) -> List[Tuple[str, int]]:
    """The schema of a union / set operation: a's names and types.  The columns pair up by position (by name for union_by_name,
    whose name sets must be equal) and each pair must have one dtype: else UnsupportedType with Spark's text.  Every operation but
    the unions compares all the columns, so a list column there, or more than 16 columns (the limit of group-by and join), is
    UnsupportedType too."""
    if op not in SET_OPS:
        raise N.UnsupportedType(f"set operation {op!r} is not one of {list(SET_OPS)}")
    if len(schema_a) != len(schema_b) or (op == "union_by_name" and set(schema_a) != set(schema_b)):
        raise N.UnsupportedType("Union can only be performed on tables with compatible column types")
    pairs = [(t, schema_b[n]) for n, t in schema_a.items()] if op == "union_by_name" else list(zip(schema_a.values(), schema_b.values()))
    if any(a != b for a, b in pairs):
        raise N.UnsupportedType("Union can only be performed on tables with compatible column types")
    if op not in ("union", "union_by_name"):
        _check_compared(schema_a, list(schema_a), op)
    return list(schema_a.items())


def _check_compared(schema: Dict[str, int], names: Sequence[str], what: str) -> None:
    if not 1 <= len(names) <= 16:
        raise N.UnsupportedType(f"{what} compares 1..16 columns (the limit of group-by and join), not {len(names)}")
    for n in names:
        if n not in schema:
            raise N.ReferencePanic(f"column {n!r} not found (column_by_name panics)")
        if schema[n] >= N.LIST_BASE:
            raise N.UnsupportedType(f"column {n!r} is a list column: {what} compares numeric, Boolean and temporal columns only")


def plan_join(schema_a: Dict[str, int], schema_b: Dict[str, int], criteria: Sequence[Tuple[str, str]], how: Optional[str] = None) -> List[Tuple[str, int]]:
    """The joined schema `Dataset::try_join` (expression.rs:223-287) plans for `criteria` ([(column of a, column of b)]), as
    [(name, dtype)]: a's columns, then b's; a name present on both sides becomes `a.<name>` / `b.<name>`.  Its checks in its
    order, per criterion: both missing, a missing, b missing, different types -- ComputeError with its texts.  Then what the
    device path adds: non-numeric keys are UnsupportedType, and zero criteria (a cross join in the reference) are refused.
    how = "left_semi" | "left_anti": the same checks, and a's columns only, names unchanged."""
    for a, b in criteria:
        if a not in schema_a and b not in schema_b:
            raise N.ComputeError("Join columns do not exist in tables")
        if a not in schema_a:
            raise N.ComputeError("Join column does not exist in table A")
        if b not in schema_b:
            raise N.ComputeError("Join column does not exist in table B")
        if schema_a[a] != schema_b[b]:
            raise N.ComputeError("Join columns must have compatible types")
    for a, _ in criteria:
        if schema_a[a] == BOOL or not 0 <= schema_a[a] <= F64:
            raise N.UnsupportedType(f"join column {a!r} is not numeric: join keys must be")
    if not criteria:
        raise N.ComputeError("Join criteria cannot be empty")
    if how in EXISTENCE_JOINS:
        return list(schema_a.items())
    out = [(f"a.{n}" if n in schema_b else n, t) for n, t in schema_a.items()]
    return out + [(f"b.{n}" if n in schema_a else n, t) for n, t in schema_b.items()]


def window(partition_by: Sequence[str], order_by: Sequence[Tuple[str, bool]], calls: Sequence[tuple]):
    """Window functions over one WindowSpec: ``calls`` are ``(output, function, *arguments)`` with column arguments by name, e.g.
    ``("r", "rank")``, ``("prev", "lag", "x", 1, 0.0)``, ``("s", "sum", "x", "range")``, a moving average ``("ma", "avg", "x", ("rows", -99, 0))``
    or a forward fill ``("x", "last_value", "x", ("rows", None, 0), True)`` (see functions.window)."""
    return ("window", (list(partition_by), [(c, bool(d)) for c, d in order_by], [tuple(c) for c in calls]))


WINDOW_RANKING = {"row_number": U32, "rank": U32, "dense_rank": U32, "percent_rank": F64, "cume_dist": F64}


def _window_columns(partition_by, order_by, calls) -> List[str]:
    return list(partition_by) + [c for c, _ in order_by] + [c[2] for c in calls if c[1] not in WINDOW_RANKING and len(c) > 2]


def plan_window(schema: Dict[str, int], partition_by: Sequence[str], order_by: Sequence[Tuple[str, bool]], calls: Sequence[tuple]) -> List[Tuple[str, int]]:
    """The frame after a window step, as [(name, dtype)]: the frame's columns, then every call's output in call order; an output
    whose name exists replaces that column in place of the old one at the end, as with_column does.  A missing column is a
    ComputeError; an unknown function, a non-numeric column and avg of Int64 / UInt64 are UnsupportedType.  Output types: UInt32
    for row_number / rank / dense_rank, Float64 for percent_rank / cume_dist / avg, Int64 for count, the column's type otherwise
    (lag / lead, sum / min / max, first_value / last_value / nth_value)."""
    for name in _window_columns(partition_by, order_by, calls):
        if name not in schema:
            raise N.ComputeError(f"Window column {json.dumps(name)} does not exist")
    out = OrderedDict(schema)
    for call in calls:
        fn = call[1]
        if fn not in N.WINDOW_FNS:
            raise N.UnsupportedType(f"window function {fn!r} is not one of {sorted(N.WINDOW_FNS)}")
        if fn not in WINDOW_RANKING and len(call) < 3:
            raise N.ComputeError(f"{fn} needs a column")
    for name in _window_columns(partition_by, order_by, calls):
        if schema[name] == BOOL or not 0 <= schema[name] <= F64:
            raise N.UnsupportedType(f"column {name!r} is not numeric: window keys and values must be")
    for call in calls:
        fn = call[1]
        if fn == "avg" and schema[call[2]] in (I64, U64):
            raise N.UnsupportedType("avg needs f64: From<T::Native>")
        t = WINDOW_RANKING.get(fn, F64 if fn == "avg" else I64 if fn == "count" else schema[call[2]] if len(call) > 2 else None)
        out.pop(call[0], None)
        out[call[0]] = t
    return list(out.items())


# ---- BooleanFilter (expression.rs:752-763) as nested tuples: ("col", name) | ("scalar", v) | ("not", x) | ("and", a, b) | ("gt", a, b) ...
def col(name: str):
    return ("col", name)


def lit(v: float):
    return ("scalar", float(v))


# null tests as condition nodes: ("is_null", x) | ("is_not_null", x) | ("is_nan", x), x a ("col", name) node
NULL_TESTS = {"is_null": N.IS_NULL, "is_not_null": N.IS_NOT_NULL, "is_nan": N.IS_NAN}


def is_null(x):
    return ("is_null", col(x) if isinstance(x, str) else x)


def is_not_null(x):
    return ("is_not_null", col(x) if isinstance(x, str) else x)


def is_nan(x):
    return ("is_nan", col(x) if isinstance(x, str) else x)


def _filter_columns(cond) -> set:
    if cond[0] == "col":
        return {cond[1]}
    if cond[0] == "scalar":
        return set()
    out = set()
    for x in cond[1:]:
        out |= _filter_columns(x)
    return out


# ---------------------------------------------------------------------------------------------------------
# the optimiser pass: which Calculations can be evaluated in one fused step

def _columns_read(t, schema: Optional[Dict[str, int]] = None) -> set:
    """The columns step t reads; `schema` (the frame's before the step) names them for the steps that read every column."""
    kind, arg = t
    if kind == "calculate":
        return set(arg.inputs)
    if kind == "fused":
        return set(arg.inputs)
    if kind == "filter":
        return _filter_columns(arg)
    if kind == "sort":
        return {c for c, _ in arg}
    if kind == "window":
        return set(_window_columns(*arg))
    if kind == "join_asof":
        return {arg[1]} | {a for a, _ in arg[3]}
    if kind == "distinct":   # the compared columns: the subset, or every column of the frame
        return set(schema or ()) if arg[0] is None else set(arg[0])
    if kind == "set_op":     # the left frame's columns are compared (or, for the unions, carried) by position
        return set(schema or ())
    return set()


def _needed_after(transformations: Sequence[tuple], final_columns: Sequence[str], schemas: Optional[Sequence[Dict[str, int]]] = None) -> List[set]:
    """needed[i] = names whose VALUES can still be observed after step i (read by a later step or present at the end).  schemas[i]:
    the schema before step i (_schema_walk), for the steps that read every column."""
    needed = [set() for _ in transformations]
    live = set(final_columns)
    for i in range(len(transformations) - 1, -1, -1):
        needed[i] = set(live)
        kind, arg = transformations[i]
        if kind == "select":
            live = set(live) if "*" in arg else {n for n in live if n in arg}
        elif kind == "drop":
            live = set(live)            # a dropped name is not in `live` here unless a later step re-creates it
        elif kind == "calculate":
            if arg.function == "rename":
                live = (live - {arg.output}) | {arg.inputs[0]}
            else:
                live = (live - {arg.output}) | set(arg.inputs)   # a Calculation is kept even when its output is dead:
        elif kind == "window":                                  # its DivideByZero panic is observable
            live = (live - {c[0] for c in arg[2]}) | _columns_read(transformations[i])   # the outputs are new columns
        else:
            live = live | _columns_read(transformations[i], schemas[i] if schemas else None)
    return needed


def _schema_walk(schema: "OrderedDict[str, int]", transformations: Sequence[tuple]) -> List["OrderedDict[str, int]"]:
    """Schema BEFORE each step (and after the last one as the final element)."""
    out = []
    cur = OrderedDict(schema)
    for kind, arg in transformations:
        out.append(OrderedDict(cur))
        if kind == "select":
            cur = OrderedDict((n, t) for n, t in cur.items() if "*" in arg or n in arg)
        elif kind == "drop":
            cur = OrderedDict((n, t) for n, t in cur.items() if n not in arg)
        elif kind == "calculate":
            if arg.function == "rename":
                cur = OrderedDict(((arg.output if n == arg.inputs[0] else n), t) for n, t in cur.items())
            else:
                t = arg.dtype if arg.function == "cast" else cur.get(arg.inputs[0], F64)
                cur.pop(arg.output, None)
                cur[arg.output] = t
        elif kind in ("join", "join_asof"):
            try:
                if kind == "join":
                    cur = OrderedDict(plan_join(cur, arg[0].schema, arg[1], arg[2]))
                else:
                    cur = OrderedDict(plan_join(cur, arg[0].schema, list(arg[3]) + [(arg[1], arg[2])]))
            except N.ArrowError:       # the step itself raises when it is evaluated; nothing after it is fused
                cur = OrderedDict()
        elif kind == "window":
            try:
                cur = OrderedDict(plan_window(cur, *arg))
            except N.ArrowError:
                cur = OrderedDict()
        elif kind == "set_op":
            try:
                cur = OrderedDict(plan_set_op(cur, arg[0].schema, arg[1]))
            except N.ArrowError:
                cur = OrderedDict()
        elif kind == "distinct":   # the rows change, the schema does not
            try:
                _check_compared(cur, list(cur) if arg[0] is None else arg[0], "drop_duplicates")
            except N.ArrowError:
                cur = OrderedDict()
    out.append(cur)
    return out


def _fusable(calc: Calculation, schema, fuse_casts: bool = True) -> bool:
    if calc.function == "cast":      # a numeric column read as Float64: the fused kernel converts on load (`as f64`, never fails)
        return fuse_casts and calc.dtype == F64 and schema.get(calc.inputs[0], -1) in range(0, 10)
    if calc.function not in ARITH and calc.function not in TRIG:
        return False
    return all(schema.get(n) == F64 for n in calc.inputs)   # integer columns add/multiply as integers (wrapping): not this kernel


def plan_fusion(schema: "OrderedDict[str, int]", transformations: Sequence[tuple], max_inputs: int = 6, max_nodes: int = 12,
                fuse_casts: bool = True) -> List[tuple]:
    """Rewrite ``transformations``: runs of fusable Calculations whose intermediates nobody can observe become one
    ("fused", Fused) step.  The result evaluates to the same frame (same columns, same order, same values).
    ``fuse_casts`` also folds a cast TO Float64 into the fused load (one pass instead of a cast launch plus the chain).
    A sort followed by a limit becomes one ("top_k", (criteria, n)) step (_plan_top_k)."""
    steps = list(transformations)
    schemas = _schema_walk(schema, steps)
    needed = _needed_after(steps, list(schemas[-1].keys()), schemas)
    for i, (kind, _) in enumerate(steps):
        if kind in ("join", "join_asof", "set_op") or (kind == "distinct" and steps[i][1][0] is None):
            # every column of the frame reaches the joined frame (perhaps renamed), or is compared: all are observable
            for j in range(i):
                needed[j] |= set(schemas[i])
    out: List[tuple] = []
    i = 0
    while i < len(steps):
        kind, arg = steps[i]
        if kind != "calculate" or not _fusable(arg, schemas[i], fuse_casts):
            out.append(steps[i]); i += 1
            continue
        j = i
        while j + 1 < len(steps) and steps[j + 1][0] == "calculate" and _fusable(steps[j + 1][1], schemas[j + 1], fuse_casts):
            j += 1
        fused = None
        while j > i and fused is None:
            fused = _try_fuse([s[1] for s in steps[i:j + 1]], needed[j], max_inputs, max_nodes)
            if fused is None:
                j -= 1
        if fused is None:
            out.append(steps[i]); i += 1
        else:
            out.append(("fused", fused)); i = j + 1
    return _plan_top_k(out)


def _plan_top_k(steps: List[tuple]) -> List[tuple]:
    """A sort followed by a limit, with only select / drop steps (which keep the rows) between them, becomes one
    ("top_k", (criteria, n)) step at the sort's place; the limit moves up."""
    out: List[tuple] = []
    i = 0
    while i < len(steps):
        if steps[i][0] == "sort":
            j = i + 1
            while j < len(steps) and steps[j][0] in ("select", "drop"):
                j += 1
            if j < len(steps) and steps[j][0] == "limit":
                out.append(("top_k", (steps[i][1], steps[j][1])))
                out.extend(steps[i + 1:j])
                i = j + 1
                continue
        out.append(steps[i]); i += 1
    return out


def _try_fuse(run: List[Calculation], needed_after_run: set, max_inputs: int, max_nodes: int) -> Optional[Fused]:
    outputs = [c.output for c in run]
    final = run[-1].output
    if run[-1].function == "cast" or len(set(outputs)) != len(outputs):
        return None                                   # a cast produces no node of its own; a name produced twice: do not fuse
    inputs: List[str] = []
    produced: Dict[str, tuple] = {}                   # name -> ("in", k) | ("node", k)
    nodes: List[tuple] = []
    used = set()
    for c in run:
        ops = []
        for name in c.inputs:
            if name in produced:
                ops.append(produced[name]); used.add(name)
            else:
                if name not in inputs:
                    inputs.append(name)
                ops.append(("in", inputs.index(name)))
        if c.function == "cast":
            produced[c.output] = ops[0]               # the same slot, read as Float64
        else:
            nodes.append((c.function, ops))
            produced[c.output] = ("node", len(nodes) - 1)
    if len(inputs) > max_inputs or len(nodes) > max_nodes or len(nodes) < 1 or len(run) < 2:
        return None
    for name in outputs[:-1]:
        if name in needed_after_run or name not in used or name in inputs:
            return None                               # observable later, dead inside the run, or shadows an input
    if final in inputs:
        return None
    ni = len(inputs)
    slot = lambda o: o[1] if o[0] == "in" else ni + o[1]
    prog = []
    for fn, ops in nodes:
        if fn in ARITH:
            prog.append((ARITH[fn], slot(ops[0]), slot(ops[1])))
        else:
            prog.append((TRIG[fn], slot(ops[0])))
    if N.lib().bdf_expr_check(ni, None, len(prog), _expr_nodes(prog), None, None) != N.OK:
        return None                                   # e.g. more than two intermediates alive at once: the caller tries a shorter run
    return Fused(inputs, prog, final, list(run))


# ---------------------------------------------------------------------------------------------------------

def fill_value_fits(dtype: int, value) -> bool:
    """Can a column of `dtype` hold `value` exactly?  A bool only a Boolean column; an int an integer column whose range holds it
    or a float column that represents it exactly; a float a float column that represents it exactly (NaN and the infinities
    included)."""
    if isinstance(value, (bool, np.bool_)):
        return dtype == BOOL
    if dtype == BOOL or not 0 <= dtype < len(NP_DTYPES):
        return False
    npt = NP_DTYPES[dtype]
    if isinstance(value, (int, np.integer)):
        if is_float(dtype):
            x = npt.type(value)
            return bool(np.isfinite(x)) and int(x) == int(value)
        info = np.iinfo(npt)
        return info.min <= int(value) <= info.max
    if isinstance(value, (float, np.floating)):
        if not is_float(dtype):
            return False
        x = npt.type(value)
        return float(x) == float(value) or (x != x and value != value)
    return False


class DeviceFrame:
    """Ordered name -> Column or ListColumn; every column has the same chunk lengths (the frame's RecordBatches).  A ListColumn is
    carried through filter, sort, limit, join, select, drop, with_column and window; it is reported in the schema as
    ``BDF_LIST_BASE + T``, so the planners refuse it as a key or an aggregated column, and it cannot be computed on, compared or
    sorted by."""

    def __init__(self, columns: "OrderedDict[str, Column]"):
        self.columns: "OrderedDict[str, Column]" = OrderedDict(columns)

    # -- construction / export --
    @classmethod
    def from_arrow(cls, path: str, columns: Optional[Sequence[str]] = None, ctx: Optional[N.Context] = None) -> "DeviceFrame":
        with IpcFile(path) as f:
            # Date / Time / Timestamp columns come in tagged when they are named; with no names the frame is what it always was
            names = [n for n, dt, _ in f.schema if (dt >= 0 or (columns is not None and n in f.temporal_columns)) and (columns is None or n in columns)]
            cols = f.read(names, ctx=ctx)
        return cls(OrderedDict((n, cols[n]) for n in names))

    @classmethod
    def from_csv(cls, path: str, has_header: bool = True, delimiter: str = ",", max_records: Optional[int] = None, batch_size: int = 1024,
                 schema: Optional[Sequence[int]] = None, columns: Optional[Sequence[str]] = None,
                 ctx: Optional[N.Context] = None) -> "DeviceFrame":
        """DataFrame::from_csv(path, None) with the defaults: a header, ',' and a schema inferred from every record, 1024 rows per
        RecordBatch.  Utf8 columns are not on the device path and are left out (read them on the CPU)."""
        with CsvFile(path, has_header=has_header, delimiter=delimiter, max_records=max_records, batch_size=batch_size, schema=schema,
                     ctx=ctx) as f:
            names = [n for n, dt, _ in f.schema if dt >= 0 and (columns is None or n in columns)]
            cols = f.read(names)
        return cls(OrderedDict((n, cols[n]) for n in names))

    @classmethod
    def from_json(cls, path: str, schema: Optional[Sequence[Tuple[str, int]]] = None, max_records: Optional[int] = None, batch_size: int = 1024,
                  ctx: Optional[N.Context] = None) -> "DeviceFrame":
        """DataFrame::from_json over a line-delimited file: one object per line, the schema inferred from every record (or the given
        (name, dtype) pairs), 1024 rows per RecordBatch.  The numeric and Boolean columns are taken; List columns (read them with
        JsonFile.read_list and add them with with_column) and columns off the device path are left out."""
        with JsonFile(path, schema=schema, max_records=max_records, batch_size=batch_size, ctx=ctx) as f:
            names = [n for n, dt, _ in f.schema if 0 <= dt <= N.BOOL]
            cols = f.read(names)
        return cls(OrderedDict((n, cols[n]) for n in names))

    @classmethod
    def from_parquet(cls, path: str, columns: Optional[Sequence[str]] = None, batch_size: int = 1024,
                     ctx: Optional[N.Context] = None) -> "DeviceFrame":
        """DataFrame::from_parquet over a file or a directory of files: the columns on the device path (numeric, Boolean and
        temporal, the last tagged), or the named ones, one chunk per RecordBatch of batch_size rows.  String, nested and other
        columns are left out."""
        with ParquetFile(path, batch_size=batch_size) as f:
            names = [n for n, dt, _ in f.schema if dt >= 0 and (columns is None or n in columns)]
            cols = f.read(names, ctx=ctx)
        return cls(OrderedDict((n, cols[n]) for n in names))

    @classmethod
    def from_host(cls, columns: Dict[str, list], ctx: Optional[N.Context] = None) -> "DeviceFrame":
        names = list(columns)
        cols = Column.upload_many([columns[n] for n in names], ctx=ctx)
        return cls(OrderedDict(zip(names, cols)))

    def to_arrow(self, path: str) -> None:
        write_ipc(path, dict(self.columns))

    def _refuse_lists(self, what: str) -> None:
        for n, c in self.columns.items():
            if isinstance(c, ListColumn):
                raise N.UnsupportedType(f"column {n!r} is a list column: {what} does not write lists (to_arrow does)")

    def to_csv(self, path: str, has_header: bool = True, delimiter: str = ",") -> None:
        """DataFrame::to_csv: the frame's text is formatted on the device and streamed to the file (write_csv).  A frame with a
        temporal or a list column is refused: its raw Int32 / Int64 values are not the text a reader would expect."""
        self._refuse_lists("the CSV writer")
        for n, c in self.columns.items():
            if getattr(c, "temporal", None) is not None:
                raise N.UnsupportedType(f"column {n!r} is {c.temporal!r}: temporal text is not written by the CSV writer")
        write_csv(path, self.columns, has_header=has_header, delimiter=delimiter)

    def to_json(self, path: str, explicit_nulls: bool = False) -> None:
        """DataFrame::to_json as line-delimited JSON: one object per row, formatted on the device and streamed to the file
        (write_json).  Every column a device frame holds is written: numeric and Boolean values, temporal columns as date / time /
        timestamp strings, list columns as arrays.  NULL members are left out unless ``explicit_nulls``."""
        write_json(path, self.columns, explicit_nulls=explicit_nulls)

    def to_parquet(self, path: str, compression: str = "none", dictionary: bool = True, row_group_rows: int = 0) -> None:
        """DataFrame::to_parquet: the frame's pages are encoded (and compressed) on the device and streamed to the file
        (write_parquet); temporal columns are written as Date / Time / Timestamp columns.  A frame with a list column is refused."""
        self._refuse_lists("the Parquet writer")
        write_parquet(path, self.columns, compression=compression, dictionary=dictionary, row_group_rows=row_group_rows)

    def to_host(self) -> Dict[str, list]:
        return {n: c.download() for n, c in self.columns.items()}

    @property
    def schema(self) -> "OrderedDict[str, int]":
        return OrderedDict((n, N.LIST_BASE + c.dtype if isinstance(c, ListColumn) else c.dtype) for n, c in self.columns.items())

    def column(self, name: str) -> Column:
        if name not in self.columns:
            raise N.ReferencePanic(f"column {name!r} not found (column_by_name panics)")
        return self.columns[name]

    def _numeric(self, name: str, what: str) -> Column:
        c = self.column(name)
        if isinstance(c, ListColumn):
            raise N.UnsupportedType(f"column {name!r} is a list column: {what} needs a numeric column")
        return c

    # -- DataFrame methods --
    def with_column(self, name: str, column: Column) -> "DeviceFrame":
        cols = OrderedDict((n, c) for n, c in self.columns.items() if n != name)
        cols[name] = column
        return DeviceFrame(cols)

    def select(self, names: Sequence[str]) -> "DeviceFrame":
        return DeviceFrame(OrderedDict((n, c) for n, c in self.columns.items() if "*" in names or n in names))

    def drop(self, names: Sequence[str]) -> "DeviceFrame":
        return DeviceFrame(OrderedDict((n, c) for n, c in self.columns.items() if n not in names))

    def filter(self, cond) -> "DeviceFrame":
        for name in _filter_columns(cond):
            if name in self.columns:
                self._numeric(name, "a filter condition")
        mask = self._boolean(cond)
        return DeviceFrame(OrderedDict((n, c.filter(mask)) for n, c in self.columns.items()))

    def fill_null(self, value, subset: Optional[Sequence[str]] = None) -> "DeviceFrame":
        """pandas' fillna / Spark's na.fill: the NULL slots of columns replaced by coalesce(column, value).  `value` is a scalar or a
        {column: value} dict.  With a scalar and no subset, every column that can hold the value exactly is filled: an int fills the
        integer columns whose range holds it and the float columns that hold it exactly, a float fills the float columns that hold
        it, a bool fills the Boolean columns; temporal and list columns are never filled by default.  A named column that cannot
        hold its value raises UnsupportedType before any device work."""
        if isinstance(value, dict):
            plan = dict(value)
        elif subset is None:
            plan = {n: value for n, c in self.columns.items()
                    if not isinstance(c, ListColumn) and getattr(c, "temporal", None) is None and fill_value_fits(c.dtype, value)}
        else:
            plan = {n: value for n in subset}
        for n, v in plan.items():
            c = self._numeric(n, "fill_null")
            if not fill_value_fits(c.dtype, v):
                raise N.UnsupportedType(f"column {n!r} (dtype {c.dtype}) cannot hold {v!r} exactly")
        return DeviceFrame(OrderedDict((n, c.fill_null(plan[n]) if n in plan else c) for n, c in self.columns.items()))

    def drop_nulls(self, subset: Optional[Sequence[str]] = None, how: str = "any") -> "DeviceFrame":
        """pandas' dropna / Spark's na.drop: the rows where any (how="any") or every (how="all") column of `subset` (default: all)
        is NULL are removed -- the AND / OR of is_not_null masks, then the frame's filter."""
        if how not in ("any", "all"):
            raise N.ComputeError(f"how must be 'any' or 'all', not {how!r}")
        names = list(self.columns) if subset is None else list(subset)
        if not names:
            return self
        masks = [self._numeric(n, "drop_nulls").is_not_null() for n in names]
        mask = masks[0]
        for m in masks[1:]:
            mask = mask.logical_and(m) if how == "any" else mask.logical_or(m)
        return DeviceFrame(OrderedDict((n, c.filter(mask)) for n, c in self.columns.items()))

    def sort(self, criteria: Sequence[Tuple[str, bool]]) -> "DeviceFrame":
        if not criteria:
            raise N.ComputeError("Sort criteria cannot be empty")
        idx = sort_indices([(self._numeric(c, "a sort key"), d) for c, d in criteria])
        return DeviceFrame(OrderedDict((n, c.take(idx)) for n, c in self.columns.items()))

    def top_k(self, criteria: Sequence[Tuple[str, bool]], k: int) -> "DeviceFrame":
        """self.sort(criteria).limit(k) without sorting every row: the k rows are chosen by a radix select of the sort keys, then
        only they are sorted and every column is taken at them.  A negative k gives no rows, as limit does."""
        if not criteria:
            raise N.ComputeError("Sort criteria cannot be empty")
        idx = top_k_indices([(self._numeric(c, "a sort key"), d) for c, d in criteria], max(int(k), 0))
        return DeviceFrame(OrderedDict((n, c.take(idx)) for n, c in self.columns.items()))

    def group_aggregate(self, groups, aggregates: Sequence[Tuple[str, str]]) -> "DeviceFrame":
        """What `Transformation::GroupAggregate` is meant to do (the reference's evaluator panics on it, src/evaluation.rs:73, and
        `evaluate` below mirrors that): group by ONE key column (`groups`: its name, or a one-element list like the reference's
        `&[&str]`), fold `(column, "sum" | "count" | "min" | "max")` per group.  The result frame has the schema
        `Dataset::try_aggregate` plans (src/expression.rs:114-221): the group column, then one column per aggregate named
        `sum(x)` / `min(x)` / `max(x)` (type of x) or `count(x)` (UInt32); groups in ascending key order, the null key last
        (bdf_group_aggregate_dev).  A missing column is the ComputeError of :121-126,140-145; the aggregates the plan lists but this
        path does not compute (avg, first, last, count_distinct, ...) are UnsupportedType."""
        from .functions import group_aggregate

        if not isinstance(groups, str):
            groups = list(groups)
            if len(groups) != 1:
                raise N.UnsupportedType("group-by over one key column is on the path; got %d grouping columns" % len(groups))
            groups = groups[0]
        if groups not in self.columns:
            raise N.ComputeError(f"Grouping column {groups!r} does not exist")
        self._numeric(groups, "a group key")
        for cname, fn in aggregates:
            if cname not in self.columns:
                raise N.ComputeError(f"Aggregating column {cname!r} does not exist")
            if fn not in ("sum", "count", "min", "max"):
                raise N.UnsupportedType(f"aggregate {fn!r} is not on the path")
            self._numeric(cname, "an aggregate")
            if fn == "sum" and getattr(self.columns[cname], "temporal", None) is not None:
                raise N.UnsupportedType(f"sum of {cname!r} ({self.columns[cname].temporal!r}): temporal values are not summed")
        names = list(OrderedDict.fromkeys(c for c, _ in aggregates))
        keys, res = group_aggregate(self.column(groups), [self.column(c) for c in names])
        out: "OrderedDict[str, Column]" = OrderedDict([(groups, keys)])
        used = set()
        try:
            for cname, fn in aggregates:
                r = res[names.index(cname)]
                if f"{fn}({cname})" in out:
                    continue
                if r[fn] is None:
                    raise N.UnsupportedType("min/max need T::Native: Ord (integers only)")
                # count(x) is planned as UInt32 (:169-173); a group never has 2^32 rows (row numbers are UInt32), so the cast cannot fail
                out[f"{fn}({cname})"] = r[fn].cast(U32) if fn == "count" else r[fn]
                if fn != "count":
                    used.add(id(r[fn]))
        finally:
            for r in res:   # aggregates nobody asked for, and the Int64 counts behind count(x)
                for c in r.values():
                    if c is not None and id(c) not in used:
                        c.free()
        return DeviceFrame(out)

    def aggregate(self, groups: Sequence[str], aggregations: Sequence[Tuple[str, Sequence[str]]]) -> "DeviceFrame":
        """`LazyFrame::aggregate` / `Transformation::GroupAggregate(groups, aggr)` over any number of key columns
        (bdf_group_by_dev): the frame has the columns and types of `plan_aggregate`; groups in the order DataFrame::sort gives the
        group columns (ascending, nulls last).  An output name planned twice is computed once."""
        from .functions import group_by

        if isinstance(groups, str):
            groups = [groups]
        plan = plan_aggregate(self.schema, groups, aggregations)
        pairs = [(fn, x) for function, columns in aggregations for x in columns for fn in [_aggregate_function(function)]]
        wanted = list(OrderedDict.fromkeys(pairs))
        key_names = list(OrderedDict.fromkeys(groups))
        keys, res = group_by([self.column(g) for g in key_names], [(self.column(x), fn) for fn, x in wanted])
        cols: Dict[str, Column] = dict(zip(key_names, keys))
        for (fn, x), r in zip(wanted, res):
            if fn in ("count", "count_distinct"):   # planned as UInt32; a group never has 2^32 rows (row numbers are UInt32)
                cols[f"{fn}({x})"] = r.cast(U32)
                r.free()
            else:
                cols[f"{fn}({x})"] = r
        return DeviceFrame(OrderedDict((name, cols[name]) for name, _ in plan))

    def join(self, other: "DeviceFrame", criteria: Sequence[Tuple[str, str]], how: str) -> "DeviceFrame":
        """DataFrame::join (src/dataframe.rs:626-719): the schema of `plan_join`, every column of both sides taken by the index
        pairs of `join_indices` (one chunk each; a NULL index gives a NULL slot)."""
        from .functions import join_indices

        plan = plan_join(self.schema, other.schema, criteria, how)
        li, ri = join_indices([self.column(a) for a, _ in criteria], [other.column(b) for _, b in criteria], how)
        if how in EXISTENCE_JOINS:   # the left rows that have (lack) a partner, in left order: this frame's columns only
            try:
                return DeviceFrame(OrderedDict((name, c.take(li)) for name, c in self.columns.items()))
            finally:
                li.free()
        try:
            cols = [c.take(li) for c in self.columns.values()] + [c.take(ri) for c in other.columns.values()]
        finally:
            li.free()
            ri.free()
        return DeviceFrame(OrderedDict((name, c) for (name, _), c in zip(plan, cols)))

    def join_asof(self, other: "DeviceFrame", left_on: str, right_on: Optional[str] = None, by: Sequence[Tuple[str, str]] = (),
                  direction: str = "backward", allow_exact_matches: bool = True, tolerance=None) -> "DeviceFrame":
        """pandas' merge_asof (join_asof_indices): every row of this frame, in its order, with the columns of the `other` row whose
        `right_on` key is the last at or before its `left_on` key ("backward"), the first at or after it ("forward") or the nearer
        ("nearest"), among the rows whose `by` pairs [(column of this frame, column of other)] are equal.  The schema is plan_join's
        (this frame's columns, then other's, `a.` / `b.` on a name clash); other's columns are NULL where there is no partner.  The
        two `on` columns must have the same temporal type; for a Date / Timestamp / Time key `tolerance` may be a datetime.timedelta,
        which must be a whole number of the key's unit."""
        from .functions import join_asof_indices

        right_on = left_on if right_on is None else right_on
        plan = plan_join(self.schema, other.schema, list(by) + [(left_on, right_on)])
        lon, ron = self.column(left_on), other.column(right_on)
        if lon.temporal != ron.temporal:
            raise N.UnsupportedType(f"as-of keys {left_on!r} ({lon.temporal!r}) and {right_on!r} ({ron.temporal!r}) have different temporal types")
        ri = join_asof_indices(lon, ron, [self.column(a) for a, _ in by], [other.column(b) for _, b in by], direction, allow_exact_matches,
                               tolerance)
        try:
            cols = list(self.columns.values()) + [c.take(ri) for c in other.columns.values()]
        finally:
            ri.free()
        return DeviceFrame(OrderedDict((name, c) for (name, _), c in zip(plan, cols)))

    # -- distinct rows and set operations (include/b200df.h "distinct rows and set operations") --
    def _compared(self, subset: Optional[Sequence[str]], what: str) -> List[Column]:
        names = list(self.columns) if subset is None else list(subset)
        _check_compared(self.schema, names, what)
        return [self.columns[n] for n in names]

    def duplicated(self, subset: Optional[Sequence[str]] = None, keep="first") -> Column:
        """pandas' duplicated: a Boolean Column without nulls, true for the rows that repeat an earlier row of `subset` (default:
        every column) with keep="first", a later one with "last", or any other one with False.  Nulls equal each other, all NaNs
        are one value and -0.0 == 0.0.  At most 16 compared columns (the limit of group-by and join); no list columns."""
        from .functions import duplicated

        return duplicated(self._compared(subset, "duplicated"), keep)

    def drop_duplicates(self, subset: Optional[Sequence[str]] = None, keep="first") -> "DeviceFrame":
        """pandas' drop_duplicates / Spark's dropDuplicates: the rows duplicated() does not mark, every column (list, Boolean and
        temporal columns included) filtered, in row order."""
        from .functions import duplicated

        mask = duplicated(self._compared(subset, "drop_duplicates"), keep)
        return self._keep(mask, invert=True)

    def distinct(self) -> "DeviceFrame":
        """Spark's distinct: drop_duplicates() over every column (at most 16, none of them a list column)."""
        return self.drop_duplicates()

    def _keep(self, mask: Column, invert: bool = False) -> "DeviceFrame":
        from .functions import filter_any

        out: "OrderedDict[str, Column]" = OrderedDict()
        try:
            m = mask.logical_not() if invert else mask
            try:
                for n, c in self.columns.items():
                    out[n] = filter_any(c, m)
            finally:
                if invert:
                    m.free()
        except BaseException:
            for c in out.values():   # the columns filtered before the failure
                c.free()
            raise
        finally:
            mask.free()
        return DeviceFrame(out)

    def _check_temporal(self, other: "DeviceFrame", pairs: Sequence[Tuple[str, str]]) -> None:
        for a, b in pairs:
            ta, tb = getattr(self.columns[a], "temporal", None), getattr(other.columns[b], "temporal", None)
            if ta != tb:
                raise N.UnsupportedType(f"Union can only be performed on tables with compatible column types ({a!r}: {ta!r}, {b!r}: {tb!r})")

    def _pairs(self, other: "DeviceFrame", op: str) -> List[Tuple[str, str]]:
        plan_set_op(self.schema, other.schema, op)
        pairs = [(n, n) for n in self.columns] if op == "union_by_name" else list(zip(self.columns, other.columns))
        self._check_temporal(other, pairs)
        return pairs

    def union(self, other: "DeviceFrame") -> "DeviceFrame":
        """Spark's union (UNION ALL): this frame's chunks, then other's, column by column by position (bdf_concat_dev); the names
        are this frame's.  The types at every position must be equal (no widening), temporal types included."""
        return self._union(other, "union")

    def union_by_name(self, other: "DeviceFrame") -> "DeviceFrame":
        """Spark's unionByName: union with other's columns matched by name (both frames must have the same names)."""
        return self._union(other, "union_by_name")

    def _union(self, other: "DeviceFrame", op: str) -> "DeviceFrame":
        from .functions import concat

        pairs = self._pairs(other, op)
        return DeviceFrame(OrderedDict((a, concat([self.columns[a], other.columns[b]])) for a, b in pairs))

    def _set_op(self, other: "DeviceFrame", op: str, native: str) -> "DeviceFrame":
        from .functions import set_op_mask

        pairs = self._pairs(other, op)
        mask = set_op_mask([self.columns[a] for a, _ in pairs], [other.columns[b] for _, b in pairs], native)
        return self._keep(mask)

    def intersect(self, other: "DeviceFrame") -> "DeviceFrame":
        """Spark's intersect: the distinct rows of this frame that other also has (the first copy of each, in row order).  The
        columns are compared by position; nulls equal each other, all NaNs are one value and -0.0 == 0.0.  At most 16 columns."""
        return self._set_op(other, "intersect", "intersect")

    def intersect_all(self, other: "DeviceFrame") -> "DeviceFrame":
        """Spark's intersectAll: of every row value present l times here and r times in other, the first min(l, r) copies."""
        return self._set_op(other, "intersect_all", "intersect_all")

    def subtract(self, other: "DeviceFrame") -> "DeviceFrame":
        """Spark's subtract (EXCEPT DISTINCT): the distinct rows of this frame that other does not have, the first copy of each."""
        return self._set_op(other, "subtract", "except")

    def except_all(self, other: "DeviceFrame") -> "DeviceFrame":
        """Spark's exceptAll: of every row value present l times here and r times in other, the first max(l - r, 0) copies."""
        return self._set_op(other, "except_all", "except_all")

    def window(self, partition_by: Sequence[str], order_by: Sequence[Tuple[str, bool]], calls: Sequence[tuple]) -> "DeviceFrame":
        """Window functions over one specification (bdf_window_dev, one sort for all calls): every call ``(output, function,
        *arguments)`` adds its column as with_column does (an existing name is replaced); the other columns are untouched."""
        plan_window(self.schema, partition_by, order_by, calls)
        args = []
        for call in calls:
            rest = list(call[2:])
            if call[1] not in WINDOW_RANKING:
                rest[0] = self.column(rest[0])
            args.append((call[1], *rest))
        res = _window([self.column(p) for p in partition_by], [(self.column(c), d) for c, d in order_by], args)
        frame = self
        for call, r in zip(calls, res):
            frame = frame.with_column(call[0], r)
        return frame

    def limit(self, count: int) -> "DeviceFrame":
        if not self.columns:
            return self
        first = next(iter(self.columns.values()))
        n = min(int(count), len(first))
        idx = Column.upload([PrimitiveArray.from_numpy(np.arange(n, dtype=np.uint32))], ctx=first.ctx)
        return DeviceFrame(OrderedDict((name, c.take(idx)) for name, c in self.columns.items()))

    def _boolean(self, cond) -> Column:
        kind = cond[0]
        if kind == "col":
            c = self.column(cond[1])
            if c.dtype != BOOL:
                raise N.UnsupportedType("a BooleanFilter input column must be Boolean unless it is compared")
            return c
        if kind == "not":
            return self._boolean(cond[1]).logical_not()
        if kind in ("and", "or"):
            a, b = self._boolean(cond[1]), self._boolean(cond[2])
            return a.logical_and(b) if kind == "and" else a.logical_or(b)
        if kind in NULL_TESTS:
            if cond[1][0] != "col":
                raise N.UnsupportedType(f"{kind} needs a column operand")
            return self._numeric(cond[1][1], f"{kind}")._null_test(NULL_TESTS[kind])
        if kind in CMP:
            l, r = cond[1], cond[2]
            if l[0] == "scalar" and r[0] == "col":
                kind, l, r = FLIP[kind], r, l
            if l[0] != "col":
                raise N.UnsupportedType("comparison needs a column on one side")
            left = self.column(l[1])
            if r[0] == "col":
                return left.compare(CMP[kind], self.column(r[1]))
            if r[0] == "scalar":
                return left.compare(CMP[kind], r[1])
        raise N.UnsupportedType(f"BooleanFilter node {kind!r} is not on the path")

    def calculate(self, calc: Calculation) -> "DeviceFrame":
        fn = calc.function
        if fn == "rename":
            return DeviceFrame(OrderedDict(((calc.output if n == calc.inputs[0] else n), c) for n, c in self.columns.items()))
        cols = [self._numeric(n, "a Calculation") for n in calc.inputs]
        if fn in ARITH:
            if cols[0].dtype in (I8, U8) or cols[0].dtype == BOOL:
                raise N.ReferencePanic("Unsupported operation")          # evaluation.rs:116-244 has no Int8/UInt8 arm
            out = cols[0]._bin(ARITH[fn], cols[1])
        elif fn in TRIG:
            if not is_float(cols[0].dtype):
                raise N.ReferencePanic(f"Expecting float datatype for operation, found {cols[0].dtype}")
            out = getattr(cols[0], TRIG[fn])()
        elif fn == "cast":
            out = cols[0].cast(calc.dtype)
        else:
            raise N.ReferencePanic(f"Function {fn!r} not supported")
        return self.with_column(calc.output, out)

    def evaluate(self, transformations: Sequence[tuple], fuse: bool = True, fuse_casts: bool = True) -> "DeviceFrame":
        steps = plan_fusion(self.schema, transformations, fuse_casts=fuse_casts) if fuse else list(transformations)
        frame = self
        for kind, arg in steps:
            if kind == "calculate":
                frame = frame.calculate(arg)
            elif kind == "fused":
                try:
                    frame = frame.with_column(arg.output, eval_expr([frame._numeric(n, "a Calculation") for n in arg.inputs], arg.nodes))
                except N.UnsupportedType:      # e.g. more than two live intermediates: run the Calculations one by one
                    for calc in arg.replaced:
                        frame = frame.calculate(calc)
            elif kind == "select":
                frame = frame.select(arg)
            elif kind == "drop":
                frame = frame.drop(arg)
            elif kind == "filter":
                frame = frame.filter(arg)
            elif kind == "limit":
                frame = frame.limit(arg)
            elif kind == "sort":
                frame = frame.sort(arg)
            elif kind == "top_k":
                frame = frame.top_k(*arg)
            elif kind == "join":
                frame = frame.join(*arg)
            elif kind == "join_asof":
                frame = frame.join_asof(*arg)
            elif kind == "window":
                frame = frame.window(*arg)
            elif kind == "distinct":
                frame = frame.drop_duplicates(*arg)
            elif kind == "set_op":
                frame = getattr(frame, arg[1])(arg[0])
            elif kind == "group_aggregate":
                raise N.ReferencePanic("aggregations not supported")       # evaluation.rs:73
            else:
                raise N.UnsupportedType(f"transformation {kind!r} is not on the path")
        return frame
