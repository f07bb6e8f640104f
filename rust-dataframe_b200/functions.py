"""Python mirror of the reference's operator interface for the hot path, over the C ABI.

Same names, argument meaning and error behaviour as the reference (nevi-me/rust-dataframe @ a8310afd):

* ``ScalarFunctions``     src/functions/scalar.rs:14-497   (add, subtract, multiply, par_multiply, divide,
                          abs, sin, cos, tan, acos, ...; each takes the column as a list of chunks)
* ``AggregateFunctions``  src/functions/aggregate.rs:9-103 (sum, min, max, count, avg)
* ``cast``                the arrow::compute::cast call of Function::Cast, src/evaluation.rs:296-315

Every function makes exactly one call into libb200df.so (CUDA); nothing here computes on the CPU.
``Column`` is the device-resident handle used to chain operators without leaving HBM.
"""
from __future__ import annotations

import ctypes as C
import datetime
import math
from typing import List, Optional, Sequence

import numpy as np

from . import _native as N
from .arrays import DATE32, DATE64, F32, F64, I64, NP_DTYPES, TIMESTAMP, PrimitiveArray, TemporalType, is_float, width_of

Chunks = Sequence[PrimitiveArray]


def _dtype_of(chunks: Chunks, other: Optional[Chunks] = None) -> int:
    for c in list(chunks) + list(other or []):
        return c.dtype
    raise ValueError("empty column: the element type cannot be inferred; pass at least one chunk")


def _check_same_type(chunks: Chunks, dtype: int) -> None:
    for c in chunks:
        if c.dtype != dtype:
            # col_to_prim_arrays::<T> downcast .unwrap() panics on a type mismatch (src/table.rs:120)
            raise N.ReferencePanic("chunk type does not match the column type (downcast_ref::<PrimitiveArray<T>>().unwrap())")


def _binary(op: int, left: Chunks, right: Chunks, ctx: Optional[N.Context], pinned_out: bool) -> List[PrimitiveArray]:
    ctx = ctx or N.default_context()
    n = min(len(left), len(right))  # zip()
    if n == 0:
        return []
    dtype = _dtype_of(left, right)
    _check_same_type(left[:n], dtype)
    _check_same_type(right[:n], dtype)
    outs, bufs = N.alloc_outputs(dtype, [left[i].length for i in range(n)], ctx, pinned_out)
    st = N.lib().bdf_binary(ctx.handle, op, dtype, len(left), N.make_views(left), len(right), N.make_views(right), outs)
    N.raise_for_status(st)
    return N.collect_outputs(dtype, outs, bufs)


def _unary(op: int, array: Chunks, ctx: Optional[N.Context], pinned_out: bool) -> List[PrimitiveArray]:
    ctx = ctx or N.default_context()
    if len(array) == 0:
        return []
    dtype = _dtype_of(array)
    _check_same_type(array, dtype)
    outs, bufs = N.alloc_outputs(dtype, [c.length for c in array], ctx, pinned_out)
    N.raise_for_status(N.lib().bdf_unary(ctx.handle, op, dtype, len(array), N.make_views(array), outs))
    return N.collect_outputs(dtype, outs, bufs)


class ScalarFunctions:
    """src/functions/scalar.rs: static functions over ``Vec<&PrimitiveArray<T>>`` (one entry per chunk)."""

    # -- binary arithmetic: arrow::compute::{add,subtract,multiply,divide} per chunk (scalar.rs:16-103) --
    @staticmethod
    def add(left: Chunks, right: Chunks, ctx=None, pinned_out=False) -> List[PrimitiveArray]:
        return _binary(N.ADD, left, right, ctx, pinned_out)

    @staticmethod
    def subtract(left: Chunks, right: Chunks, ctx=None, pinned_out=False) -> List[PrimitiveArray]:
        return _binary(N.SUB, left, right, ctx, pinned_out)

    @staticmethod
    def multiply(left: Chunks, right: Chunks, ctx=None, pinned_out=False) -> List[PrimitiveArray]:
        return _binary(N.MUL, left, right, ctx, pinned_out)

    @staticmethod
    def par_multiply(left: Chunks, right: Chunks, ctx=None, pinned_out=False) -> List[PrimitiveArray]:
        # the reference's rayon variant (scalar.rs:87-103); on the GPU every chunk is already in one launch
        return _binary(N.MUL, left, right, ctx, pinned_out)

    @staticmethod
    def divide(left: Chunks, right: Chunks, ctx=None, pinned_out=False) -> List[PrimitiveArray]:
        return _binary(N.DIV, left, right, ctx, pinned_out)

    # -- math_op binaries on single arrays (scalar.rs:148,274,291) --
    @staticmethod
    def atan2(a: PrimitiveArray, b: PrimitiveArray, ctx=None) -> PrimitiveArray:
        return _binary(N.ATAN2, [a], [b], ctx, False)[0]

    @staticmethod
    def hypot(a: PrimitiveArray, b: PrimitiveArray, ctx=None) -> PrimitiveArray:
        return _binary(N.HYPOT, [a], [b], ctx, False)[0]

    @staticmethod
    def log(a: PrimitiveArray, b: PrimitiveArray, ctx=None) -> PrimitiveArray:
        return _binary(N.LOG, [a], [b], ctx, False)[0]


def _add_unary(name: str, op: int) -> None:
    def fn(array: Chunks, ctx=None, pinned_out=False) -> List[PrimitiveArray]:
        return _unary(op, array, ctx, pinned_out)

    fn.__name__ = name
    fn.__doc__ = f"ScalarFunctions::{name}: scalar_op over every chunk (src/functions/scalar.rs:525-540)."
    setattr(ScalarFunctions, name, staticmethod(fn))


for _name, _op in [("abs", N.ABS), ("sin", N.SIN), ("cos", N.COS), ("tan", N.TAN), ("acos", N.ACOS), ("asin", N.ASIN),
                   ("atan", N.ATAN), ("cbrt", N.CBRT), ("ceil", N.CEIL), ("cosh", N.COSH), ("degrees", N.DEGREES),
                   ("exp", N.EXP), ("expm1", N.EXPM1), ("floor", N.FLOOR), ("log10", N.LOG10), ("log2", N.LOG2),
                   ("radians", N.RADIANS), ("round", N.ROUND), ("sinh", N.SINH), ("sqrt", N.SQRT), ("tanh", N.TANH)]:
    _add_unary(_name, _op)


def cast(arrays: Chunks, to_dtype: int, ctx=None, pinned_out=False) -> List[PrimitiveArray]:
    """arrow::compute::cast over every chunk of a column, as Function::Cast does (src/evaluation.rs:296-315)."""
    ctx = ctx or N.default_context()
    if len(arrays) == 0:
        return []
    from_dtype = _dtype_of(arrays)
    _check_same_type(arrays, from_dtype)
    outs, bufs = N.alloc_outputs(to_dtype, [c.length for c in arrays], ctx, pinned_out)
    N.raise_for_status(N.lib().bdf_cast(ctx.handle, from_dtype, to_dtype, len(arrays), N.make_views(arrays), outs))
    return N.collect_outputs(to_dtype, outs, bufs)


# ---------------------------------------------------------------------------------------------------------
# dates and timestamps (include/b200df.h "dates and timestamps")


def _temporal_c(t: TemporalType) -> "N.TemporalTypeC":
    return N.TemporalTypeC(t.kind, t.unit, t.tz.encode() if t.tz is not None else None)


def temporal_result(fn, temporal: TemporalType, arg: int = 0):
    """bdf_temporal_result: ``(result dtype, result TemporalType or None)`` of a temporal function (a name of ``native.TEMPORAL_FNS`` or
    its number) on a column of type ``temporal``; raises exactly what the function itself would for (fn, type, arg).  No GPU needed."""
    fn = N.TEMPORAL_FNS[fn] if isinstance(fn, str) else int(fn)
    tc, dt, ot = _temporal_c(temporal), C.c_int32(0), N.TemporalTypeC()
    N.raise_for_status(N.lib().bdf_temporal_result(fn, C.byref(tc), int(arg), C.byref(dt), C.byref(ot)))
    out = None
    if ot.kind:
        tz = None if not ot.tz else ot.tz.decode()
        out = TemporalType(ot.kind, ot.unit, tz)
    return dt.value, out


_WEEKDAYS = {"su": 1, "mo": 2, "tu": 3, "we": 4, "th": 5, "fr": 6, "sa": 7}


def _temporal_arg(fn: int, arg) -> int:
    """Names accepted for the argument: date_trunc units ("day", "month" ...), time units ("s" .. "ns"), weekdays ("tuesday", "tue")."""
    if isinstance(arg, str):
        a = arg.lower()
        if fn == N.T_DATE_TRUNC:
            return N.TRUNC_UNITS[{"yyyy": "year", "yy": "year", "mm": "month", "mon": "month", "dd": "day"}.get(a, a)]
        if fn == N.T_TO_TIMESTAMP:
            return N.TIME_UNITS[a]
        if fn == N.T_NEXT_DAY and len(a) >= 2 and a[:2] in _WEEKDAYS:
            return _WEEKDAYS[a[:2]]
        raise N.ComputeError(f"argument {arg!r} is not understood by temporal function {fn}")
    return int(arg)


def _temporal_of(arrays: Chunks, temporal: Optional[TemporalType]) -> TemporalType:
    if temporal is None:
        for c in arrays:
            temporal = getattr(c, "temporal", None)
            break
    if temporal is None:
        raise N.UnsupportedType("a temporal function needs the column's temporal type (pass temporal=TemporalType...)")
    return temporal


def _temporal_host(fn: int, arrays: Chunks, temporal: Optional[TemporalType], arg, ctx, pinned_out: bool) -> List[PrimitiveArray]:
    ctx = ctx or N.default_context()
    t = _temporal_of(arrays, temporal)
    a = _temporal_arg(fn, arg)
    out_dtype, out_t = temporal_result(fn, t, a)
    if len(arrays) == 0:
        return []
    _check_same_type(arrays, t.dtype)
    outs, bufs = N.alloc_outputs(out_dtype, [c.length for c in arrays], ctx, pinned_out)
    tc = _temporal_c(t)
    N.raise_for_status(N.lib().bdf_temporal(ctx.handle, fn, C.byref(tc), a, len(arrays), N.make_views(arrays), outs))
    res = N.collect_outputs(out_dtype, outs, bufs)
    for r in res:
        r.temporal = out_t
    return res


def _add_temporal(name: str, fn: int, has_arg: bool) -> None:
    if has_arg:
        def f(arrays: Chunks, arg, temporal: Optional[TemporalType] = None, ctx=None, pinned_out=False) -> List[PrimitiveArray]:
            return _temporal_host(fn, arrays, temporal, arg, ctx, pinned_out)
    else:
        def f(arrays: Chunks, temporal: Optional[TemporalType] = None, ctx=None, pinned_out=False) -> List[PrimitiveArray]:
            return _temporal_host(fn, arrays, temporal, 0, ctx, pinned_out)
    f.__name__ = name
    f.__doc__ = (f"ScalarFunctions::{name} over every chunk of a Date32 / Date64 / Timestamp{' / Time' if fn in (N.T_HOUR, N.T_MINUTE, N.T_SECOND) else ''}"
                 " column (one bdf_temporal call); the chunks' .temporal tag or `temporal` gives the type.")
    setattr(ScalarFunctions, name, staticmethod(f))


for _name, _fn in N.TEMPORAL_FNS.items():
    _add_temporal(_name, _fn, _fn in (N.T_DATE_ADD, N.T_DATE_SUB, N.T_ADD_MONTHS, N.T_NEXT_DAY, N.T_DATE_TRUNC, N.T_TO_TIMESTAMP))


def _temporal_binary_host(fn: int, a: Chunks, b: Chunks, ta, tb, ctx) -> List[PrimitiveArray]:
    ctx = ctx or N.default_context()
    ta, tb = _temporal_of(a, ta), _temporal_of(b, tb)
    ca = Column.upload(a, ctx, dtype=ta.dtype).with_temporal(ta)
    cb = Column.upload(b, ctx, dtype=tb.dtype).with_temporal(tb)
    return ca._temporal_binary(fn, cb).download()


def _date_diff_host(end: Chunks, start: Chunks, temporal_end=None, temporal_start=None, ctx=None) -> List[PrimitiveArray]:
    """Spark's datediff(end, start): days(to_date(end)) - days(to_date(start)) as Int32, chunk by chunk."""
    return _temporal_binary_host(N.T_DATE_DIFF, end, start, temporal_end, temporal_start, ctx)


def _months_between_host(a: Chunks, b: Chunks, temporal_a=None, temporal_b=None, ctx=None) -> List[PrimitiveArray]:
    """Spark 2.4's months_between(a, b) with roundOff = true, Float64, chunk by chunk."""
    return _temporal_binary_host(N.T_MONTHS_BETWEEN, a, b, temporal_a, temporal_b, ctx)


ScalarFunctions.date_diff = staticmethod(_date_diff_host)
ScalarFunctions.months_between = staticmethod(_months_between_host)


def _refuse_temporal(what: str, *cols) -> None:
    """Operations that would treat dates as numbers (arithmetic, sums, float comparison) refuse tagged columns before any device call."""
    for c in cols:
        t = getattr(c, "temporal", None)
        if t is not None:
            raise N.UnsupportedType(f"{what} of a {t!r} column: only numeric types are summed or computed on (temporal values are not)")


def _scalar_from_bits(dtype: int, bits: int):
    return np.array([bits], dtype=np.uint64).view(NP_DTYPES[dtype])[0]


class AggregateFunctions:
    """src/functions/aggregate.rs.  ``None`` mirrors Rust's ``Option::None``.

    ``min`` returns the true minimum (what arrow's compute::min does).  The reference's ``min`` body is a
    copy of ``max`` (aggregate.rs:22-31); ``min_as_written`` reproduces that behaviour for completeness."""

    @staticmethod
    def _agg(op: int, arrays: Chunks, dtype: Optional[int], ctx):
        ctx = ctx or N.default_context()
        if dtype is None:
            dtype = _dtype_of(arrays) if len(arrays) else N_I64_FALLBACK
        _check_same_type(arrays, dtype)
        out = np.zeros(1, dtype=np.int64 if op == N.COUNT else NP_DTYPES[dtype])
        some = C.c_int32(0)
        st = N.lib().bdf_aggregate(ctx.handle, op, dtype, len(arrays), N.make_views(arrays), out.ctypes.data, C.byref(some))
        N.raise_for_status(st)
        return out[0] if some.value else None

    @staticmethod
    def sum(arrays: Chunks, dtype: Optional[int] = None, ctx=None):
        return AggregateFunctions._agg(N.SUM, arrays, dtype, ctx)

    @staticmethod
    def max(arrays: Chunks, dtype: Optional[int] = None, ctx=None):
        return AggregateFunctions._agg(N.MAX, arrays, dtype, ctx)

    @staticmethod
    def min(arrays: Chunks, dtype: Optional[int] = None, ctx=None):
        return AggregateFunctions._agg(N.MIN, arrays, dtype, ctx)

    @staticmethod
    def min_as_written(arrays: Chunks, dtype: Optional[int] = None, ctx=None):
        return AggregateFunctions._agg(N.MAX, arrays, dtype, ctx)

    @staticmethod
    def count(arrays: Chunks, dtype: Optional[int] = None, ctx=None):
        v = AggregateFunctions._agg(N.COUNT, arrays, dtype, ctx)
        return None if v is None else int(v)

    @staticmethod
    def avg(arrays: Chunks, dtype: Optional[int] = None, ctx=None):
        ctx = ctx or N.default_context()
        if dtype is None:
            dtype = _dtype_of(arrays) if len(arrays) else N_I64_FALLBACK
        out, some = C.c_double(0), C.c_int32(0)
        st = N.lib().bdf_avg(ctx.handle, dtype, len(arrays), N.make_views(arrays), C.byref(out), C.byref(some))
        N.raise_for_status(st)
        return out.value if some.value else None

    @staticmethod
    def all(arrays: Chunks, dtype: Optional[int] = None, ctx=None) -> dict:
        """sum, min, max and count from ONE pass over the data (fused 4-in-1 reduction)."""
        ctx = ctx or N.default_context()
        if dtype is None:
            dtype = _dtype_of(arrays)
        a = N.Agg4()
        N.raise_for_status(N.lib().bdf_aggregate_all(ctx.handle, dtype, len(arrays), N.make_views(arrays), C.byref(a)))
        return _agg4_to_dict(dtype, a)

    # -- statistical aggregates (include/b200df.h "statistical aggregates"): the stubs of aggregate.rs:81,94-102 --
    @staticmethod
    def moments(arrays: Chunks, dtype: Optional[int] = None, ctx=None) -> dict:
        """The moment record {count, mean, m2, m3, m4} of the valid values, every numeric type read ``as f64``."""
        ctx = ctx or N.default_context()
        if dtype is None:
            dtype = _dtype_of(arrays) if len(arrays) else N_I64_FALLBACK
        r = N.MomentRec()
        N.raise_for_status(N.lib().bdf_moments(ctx.handle, dtype, len(arrays), N.make_views(arrays), C.byref(r)))
        return _moments_to_dict(r)

    @staticmethod
    def variance(arrays: Chunks, dtype: Optional[int] = None, ctx=None) -> Optional[float]:
        """Sample variance m2 / (n - 1), as Spark's variance."""
        return moments_stat(AggregateFunctions.moments(arrays, dtype, ctx), "variance")

    @staticmethod
    def variance_pop(arrays: Chunks, dtype: Optional[int] = None, ctx=None) -> Optional[float]:
        return moments_stat(AggregateFunctions.moments(arrays, dtype, ctx), "var_pop")

    @staticmethod
    def stddev(arrays: Chunks, dtype: Optional[int] = None, ctx=None) -> Optional[float]:
        """Sample standard deviation sqrt(m2 / (n - 1)), as Spark's stddev."""
        return moments_stat(AggregateFunctions.moments(arrays, dtype, ctx), "stddev")

    @staticmethod
    def stddev_pop(arrays: Chunks, dtype: Optional[int] = None, ctx=None) -> Optional[float]:
        return moments_stat(AggregateFunctions.moments(arrays, dtype, ctx), "stddev_pop")

    @staticmethod
    def skewness(arrays: Chunks, dtype: Optional[int] = None, ctx=None) -> Optional[float]:
        return moments_stat(AggregateFunctions.moments(arrays, dtype, ctx), "skewness")

    @staticmethod
    def kurtosis(arrays: Chunks, dtype: Optional[int] = None, ctx=None) -> Optional[float]:
        """Excess kurtosis n m4 / m2^2 - 3."""
        return moments_stat(AggregateFunctions.moments(arrays, dtype, ctx), "kurtosis")

    @staticmethod
    def _distinct(arrays: Chunks, dtype: Optional[int], ctx):
        ctx = ctx or N.default_context()
        if dtype is None:
            dtype = _dtype_of(arrays) if len(arrays) else N_I64_FALLBACK
        r = N.DistinctRec()
        N.raise_for_status(N.lib().bdf_distinct(ctx.handle, dtype, len(arrays), N.make_views(arrays), C.byref(r)))
        return dtype, r

    @staticmethod
    def count_distinct(arrays: Chunks, dtype: Optional[int] = None, ctx=None) -> int:
        """The number of distinct valid values (all NaNs are one value, -0.0 == 0.0)."""
        return int(AggregateFunctions._distinct(arrays, dtype, ctx)[1].count)

    @staticmethod
    def sum_distinct(arrays: Chunks, dtype: Optional[int] = None, ctx=None):
        """The sum of the distinct valid values in the dtype of the column (0 when there is none, like ``sum``)."""
        dtype, r = AggregateFunctions._distinct(arrays, dtype, ctx)
        return _scalar_from_bits(dtype, r.sum)

    # -- distributions (include/b200df.h "distributions") --
    @staticmethod
    def percentile(arrays: Chunks, p, dtype: Optional[int] = None, ctx=None):
        """Spark's exact percentile of the valid values at p in [0, 1] (a float, or a sequence of up to 1024 of them): a float, or
        ``None`` without a valid value; a list for a sequence."""
        ctx = ctx or N.default_context()
        if dtype is None:
            dtype = _dtype_of(arrays) if len(arrays) else N_I64_FALLBACK
        ps, out, some = _percentile_args(p)
        N.raise_for_status(N.lib().bdf_percentile(ctx.handle, dtype, len(arrays), N.make_views(arrays), len(np.atleast_1d(p)), ps, out, some))
        return _percentile_result(p, out, some)

    @staticmethod
    def median(arrays: Chunks, dtype: Optional[int] = None, ctx=None) -> Optional[float]:
        return AggregateFunctions.percentile(arrays, 0.5, dtype, ctx)

    @staticmethod
    def mode(arrays: Chunks, dtype: Optional[int] = None, ctx=None):
        """The most frequent valid value (ties: the smallest), in the dtype of the column; ``None`` without a valid value."""
        ctx = ctx or N.default_context()
        if dtype is None:
            dtype = _dtype_of(arrays) if len(arrays) else N_I64_FALLBACK
        bits, freq, some = C.c_uint64(0), C.c_int64(0), C.c_int32(0)
        N.raise_for_status(N.lib().bdf_mode(ctx.handle, dtype, len(arrays), N.make_views(arrays), C.byref(bits), C.byref(freq), C.byref(some)))
        return _scalar_from_bits(dtype, bits.value) if some.value else None


N_I64_FALLBACK = 3  # Int64: only used to type an empty Vec (results do not depend on it)


def _percentile_args(p):
    ps = np.ascontiguousarray(np.atleast_1d(np.asarray(p, dtype=np.float64)))
    n = len(ps)
    return ps.ctypes.data_as(C.POINTER(C.c_double)), (C.c_double * max(n, 1))(), (C.c_int32 * max(n, 1))()


def _percentile_result(p, out, some):
    vals = [out[i] if some[i] else None for i in range(len(np.atleast_1d(p)))]
    return vals if np.ndim(p) else vals[0]


def hist_density(edges, counts) -> np.ndarray:
    """bdf_hist_density: numpy's ``density=True`` from the edges and counts of a histogram (no context and no GPU needed)."""
    e = np.ascontiguousarray(edges, dtype=np.float64)
    c = np.ascontiguousarray(counts, dtype=np.int64)
    out = np.zeros(len(c), dtype=np.float64)
    N.raise_for_status(N.lib().bdf_hist_density(len(c), e.ctypes.data_as(C.POINTER(C.c_double)), c.ctypes.data_as(C.POINTER(C.c_int64)),
                                                out.ctypes.data_as(C.POINTER(C.c_double))))
    return out


def _moments_to_dict(r: "N.MomentRec") -> dict:
    return {"count": int(r.count), "mean": float(r.mean), "m2": float(r.m2), "m3": float(r.m3), "m4": float(r.m4)}


def moments_stat(rec: dict, stat: str) -> Optional[float]:
    """bdf_moments_stat: one of "variance", "var_pop", "stddev", "stddev_pop", "skewness", "kurtosis" from a moment record (no
    context and no GPU needed); ``None`` is Rust's None."""
    if stat not in N.STATS:
        raise N.ComputeError(f"unknown statistic {stat!r}")
    r = N.MomentRec(rec["count"], rec["mean"], rec["m2"], rec["m3"], rec["m4"])
    out, some = C.c_double(0), C.c_int32(0)
    N.raise_for_status(N.lib().bdf_moments_stat(C.byref(r), N.STATS[stat], C.byref(out), C.byref(some)))
    return out.value if some.value else None


def moments_merge(a: dict, b: dict) -> dict:
    """bdf_moments_merge: the record of the union of two sets of values (the merge the library uses across GPUs)."""
    ra = N.MomentRec(a["count"], a["mean"], a["m2"], a["m3"], a["m4"])
    rb = N.MomentRec(b["count"], b["mean"], b["m2"], b["m3"], b["m4"])
    out = N.MomentRec()
    N.raise_for_status(N.lib().bdf_moments_merge(C.byref(ra), C.byref(rb), C.byref(out)))
    return _moments_to_dict(out)


def _agg4_to_dict(dtype: int, a: "N.Agg4") -> dict:
    res = {"sum": _scalar_from_bits(dtype, a.sum), "count": int(a.count), "rows": int(a.rows),
           "would_panic": bool(a.would_panic), "n_chunks": int(a.n_chunks), "min": None, "max": None}
    if not is_float(dtype) and a.any_valid:
        res["min"] = _scalar_from_bits(dtype, a.min)
        res["max"] = _scalar_from_bits(dtype, a.max)
    return res


# ---------------------------------------------------------------------------------------------------------
# device-resident columns


class Column:
    """A column living in HBM (list of Arrow chunks).  Operators return new Columns; nothing crosses PCIe
    until ``download``.  Mirrors how Evaluate::calculate (src/evaluation.rs:97-323) materialises every
    Calculation as a new column of the frame."""

    def __init__(self, ctx: N.Context, handle: C.c_void_p, temporal: Optional[TemporalType] = None):
        self.ctx = ctx
        self.handle = handle
        self.temporal = temporal   # a TemporalType when the Int32 / Int64 values are dates, times or timestamps

    def with_temporal(self, t: Optional[TemporalType]) -> "Column":
        """Tag the column with a temporal type (None removes the tag); the values are not touched.  The tag is set IN PLACE and the
        column itself is returned: a Column taken from a DeviceFrame is the frame's own object, so the frame's column is retagged too."""
        if t is not None and t.dtype != self.dtype:
            raise N.ComputeError(f"a column of dtype {self.dtype} cannot hold {t!r} (physical dtype {t.dtype})")
        self.temporal = t
        return self

    # -- construction --
    @classmethod
    def upload(cls, arrays: Chunks, ctx: Optional[N.Context] = None, asynchronous: bool = False,
               dtype: Optional[int] = None) -> "Column":
        ctx = ctx or N.default_context()
        if dtype is None:
            dtype = _dtype_of(arrays)
        _check_same_type(arrays, dtype)
        h = C.c_void_p()
        st = N.lib().bdf_upload(ctx.handle, dtype, len(arrays), N.make_views(arrays), N.ASYNC if asynchronous else 0, C.byref(h))
        N.raise_for_status(st)
        tags = {getattr(a, "temporal", None) for a in arrays}
        col = cls(ctx, h, tags.pop() if len(tags) == 1 else None)   # chunks that all carry one temporal type tag the column
        col._hold = arrays if asynchronous else None  # keep host buffers alive while copies are in flight
        return col

    @classmethod
    def upload_many(cls, columns: Sequence[Chunks], ctx: Optional[N.Context] = None, asynchronous: bool = False) -> List["Column"]:
        """Upload several columns with their chunks interleaved (a0,b0,a1,b1,...) -- one Vec<RecordBatch>."""
        ctx = ctx or N.default_context()
        k = len(columns)
        dtypes = (C.c_int32 * k)(*[_dtype_of(col) for col in columns])
        counts = (C.c_int64 * k)(*[len(col) for col in columns])
        views = [N.make_views(col) for col in columns]
        ptrs = (C.POINTER(N.View) * k)(*[C.cast(v, C.POINTER(N.View)) for v in views])
        outs = (C.c_void_p * k)()
        st = N.lib().bdf_upload_many(ctx.handle, k, dtypes, counts, ptrs, N.ASYNC if asynchronous else 0, outs)
        N.raise_for_status(st)
        cols = []
        for i in range(k):
            col = cls(ctx, C.c_void_p(outs[i]))
            col._hold = (columns[i], views) if asynchronous else None
            cols.append(col)
        return cols

    @classmethod
    def generate(cls, dtype: int, chunk_lens: Sequence[int], kind: int = 0, lo: float = 0.0, hi: float = 1.0,
                 seed: int = 20260924, col_id: int = 0, row0: int = 0, null_mod: int = 0,
                 ctx: Optional[N.Context] = None) -> "Column":
        ctx = ctx or N.default_context()
        lens = (C.c_int64 * max(len(chunk_lens), 1))(*chunk_lens)
        h = C.c_void_p()
        st = N.lib().bdf_generate(ctx.handle, dtype, kind, lo, hi, seed, col_id, len(chunk_lens), lens, row0, null_mod, C.byref(h))
        N.raise_for_status(st)
        return cls(ctx, h)

    # -- metadata --
    def describe(self):
        dt, n, total = C.c_int32(), C.c_int64(), C.c_int64()
        N.raise_for_status(N.lib().bdf_col_describe(self.handle, C.byref(dt), C.byref(n), C.byref(total)))
        return dt.value, n.value, total.value

    @property
    def dtype(self) -> int:
        return self.describe()[0]

    @property
    def n_chunks(self) -> int:
        return self.describe()[1]

    def __len__(self) -> int:
        return self.describe()[2]

    def chunk_info(self, i: int):
        ln, nc, hv = C.c_int64(), C.c_int64(), C.c_int32()
        N.raise_for_status(N.lib().bdf_col_chunk_info(self.ctx.handle, self.handle, i, C.byref(ln), C.byref(nc), C.byref(hv)))
        return {"len": ln.value, "null_count": nc.value, "has_validity": bool(hv.value)}

    def wait(self):
        N.raise_for_status(N.lib().bdf_col_wait(self.ctx.handle, self.handle))

    # -- operators --
    def _bin(self, op: int, other: "Column") -> "Column":
        _refuse_temporal("arithmetic", self, other)
        h = C.c_void_p()
        N.raise_for_status(N.lib().bdf_binary_dev(self.ctx.handle, op, self.handle, other.handle, C.byref(h)))
        return Column(self.ctx, h)

    def add(self, o): return self._bin(N.ADD, o)
    def subtract(self, o): return self._bin(N.SUB, o)
    def multiply(self, o): return self._bin(N.MUL, o)
    def divide(self, o): return self._bin(N.DIV, o)
    def atan2(self, o): return self._bin(N.ATAN2, o)
    def hypot(self, o): return self._bin(N.HYPOT, o)
    def log(self, o): return self._bin(N.LOG, o)

    # -- fused operator + aggregate of the result (one pass; SURVEY K5) --
    def binary_agg(self, op: int, other: "Column"):
        """(self op other) materialised as a Column AND sum/min/max/count of it, from one kernel pass."""
        _refuse_temporal("arithmetic", self, other)
        h, a = C.c_void_p(), N.Agg4()
        N.raise_for_status(N.lib().bdf_binary_agg_dev(self.ctx.handle, op, self.handle, other.handle, C.byref(h), C.byref(a)))
        return Column(self.ctx, h), _agg4_to_dict(self.dtype, a)

    def add_agg(self, o): return self.binary_agg(N.ADD, o)

    def binary_agg_async(self, op: int, other: "Column"):
        """Like binary_agg but returns (Column, AggFuture) without waiting for the GPU."""
        _refuse_temporal("arithmetic", self, other)
        h, f = C.c_void_p(), C.c_void_p()
        N.raise_for_status(N.lib().bdf_binary_agg_dev_async(self.ctx.handle, op, self.handle, other.handle, C.byref(h), C.byref(f)))
        return Column(self.ctx, h), AggFuture(self.ctx, f, self.dtype)

    def take(self, indices: "Column") -> "Column":
        """Column::take (src/table.rs:218-241): values at the UInt32 row numbers, as ONE chunk; null index -> null slot."""
        h = C.c_void_p()
        N.raise_for_status(N.lib().bdf_take_dev(self.ctx.handle, self.handle, indices.handle, C.byref(h)))
        return Column(self.ctx, h, self.temporal)

    def aggregate_all_async(self) -> "AggFuture":
        _refuse_temporal("sum", self)
        f = C.c_void_p()
        N.raise_for_status(N.lib().bdf_aggregate_all_dev_async(self.ctx.handle, self.handle, C.byref(f)))
        return AggFuture(self.ctx, f, self.dtype)

    # -- N2: BooleanFilter comparisons, boolean kernels, filter (SURVEY 8(f)) --
    def compare(self, op: int, other) -> "Column":
        """BooleanFilter::{Gt,Ge,Eq,Ne,Lt,Le}: both sides cast to Float64, compared; `other` is a Column or a scalar
        (BooleanInput::Scalar).  Returns a boolean mask column.  A Date64 / Timestamp / Time64 column is refused: the Float64 comparison
        is not exact for 64-bit instants; compare to_date() (Date32, exact in f64) or unix_timestamp() instead."""
        _refuse_temporal("Float64 comparison", *[c for c in (self, other) if getattr(getattr(c, "temporal", None), "dtype", None) == I64])
        h = C.c_void_p()
        if isinstance(other, Column):
            st = N.lib().bdf_compare_dev(self.ctx.handle, op, self.handle, other.handle, 0.0, C.byref(h))
        else:
            st = N.lib().bdf_compare_dev(self.ctx.handle, op, self.handle, None, float(other), C.byref(h))
        N.raise_for_status(st)
        return Column(self.ctx, h)

    def gt(self, o): return self.compare(N.GT, o)
    def ge(self, o): return self.compare(N.GE, o)
    def eq(self, o): return self.compare(N.EQ, o)
    def ne(self, o): return self.compare(N.NE, o)
    def lt(self, o): return self.compare(N.LT, o)
    def le(self, o): return self.compare(N.LE, o)

    def _boolean(self, op: int, other: Optional["Column"]) -> "Column":
        h = C.c_void_p()
        N.raise_for_status(N.lib().bdf_boolean_dev(self.ctx.handle, op, self.handle, other.handle if other is not None else None, C.byref(h)))
        return Column(self.ctx, h)

    def logical_and(self, o): return self._boolean(N.AND, o)
    def logical_or(self, o): return self._boolean(N.OR, o)
    def logical_not(self): return self._boolean(N.NOT, None)

    def filter(self, mask: "Column") -> "Column":
        """ChunkedArray::filter: keep the slots where the boolean mask column is valid and true."""
        h = C.c_void_p()
        N.raise_for_status(N.lib().bdf_filter_dev(self.ctx.handle, self.handle, mask.handle, C.byref(h)))
        return Column(self.ctx, h, self.temporal)

    # -- null handling and conditional selection (include/b200df.h "null handling and conditional selection") --
    def _null_test(self, fn: int) -> "Column":
        h = C.c_void_p()
        N.raise_for_status(N.lib().bdf_null_test_dev(self.ctx.handle, fn, self.handle, C.byref(h)))
        return Column(self.ctx, h)

    def is_null(self) -> "Column": return self._null_test(N.IS_NULL)
    def is_not_null(self) -> "Column": return self._null_test(N.IS_NOT_NULL)
    def is_nan(self) -> "Column": return self._null_test(N.IS_NAN)

    def fill_null(self, value) -> "Column":
        """coalesce(self, value): the NULL slots replaced by a scalar (or by the slots of another column)."""
        return coalesce(self, value)

    def nanvl(self, other) -> "Column":
        """Spark's nanvl: self where it is not NaN, `other` where it is NaN, NULL where self is NULL (Float32 / Float64)."""
        return _rowwise(N.ROW_NANVL, (self, other))

    def unary(self, op: int) -> "Column":
        _refuse_temporal("a math function", self)
        h = C.c_void_p()
        N.raise_for_status(N.lib().bdf_unary_dev(self.ctx.handle, op, self.handle, C.byref(h)))
        return Column(self.ctx, h)

    def sin(self): return self.unary(N.SIN)
    def cos(self): return self.unary(N.COS)
    def tan(self): return self.unary(N.TAN)
    def abs(self): return self.unary(N.ABS)

    def cast(self, to_dtype: int) -> "Column":
        _refuse_temporal("cast", self)
        h = C.c_void_p()
        N.raise_for_status(N.lib().bdf_cast_dev(self.ctx.handle, to_dtype, self.handle, C.byref(h)))
        return Column(self.ctx, h)

    def aggregate(self, op: int):
        if op == N.SUM:
            _refuse_temporal("sum", self)
        dtype = self.dtype
        out = np.zeros(1, dtype=np.int64 if (op == N.COUNT or dtype == N.BOOL) else NP_DTYPES[dtype])
        some = C.c_int32(0)
        N.raise_for_status(N.lib().bdf_aggregate_dev(self.ctx.handle, op, self.handle, out.ctypes.data, C.byref(some)))
        return out[0] if some.value else None

    def sum(self): return self.aggregate(N.SUM)
    def min(self): return self.aggregate(N.MIN)
    def max(self): return self.aggregate(N.MAX)
    def count(self): return int(self.aggregate(N.COUNT))

    def aggregate_all(self) -> dict:
        _refuse_temporal("sum", self)
        a = N.Agg4()
        N.raise_for_status(N.lib().bdf_aggregate_all_dev(self.ctx.handle, self.handle, C.byref(a)))
        return _agg4_to_dict(self.dtype, a)

    def avg(self):
        _refuse_temporal("avg", self)
        out, some = C.c_double(0), C.c_int32(0)
        N.raise_for_status(N.lib().bdf_avg_dev(self.ctx.handle, self.handle, C.byref(out), C.byref(some)))
        return out.value if some.value else None

    def moments(self) -> dict:
        _refuse_temporal("a statistic", self)
        r = N.MomentRec()
        N.raise_for_status(N.lib().bdf_moments_dev(self.ctx.handle, self.handle, C.byref(r)))
        return _moments_to_dict(r)

    def variance(self): return moments_stat(self.moments(), "variance")
    def variance_pop(self): return moments_stat(self.moments(), "var_pop")
    def stddev(self): return moments_stat(self.moments(), "stddev")
    def stddev_pop(self): return moments_stat(self.moments(), "stddev_pop")
    def skewness(self): return moments_stat(self.moments(), "skewness")
    def kurtosis(self): return moments_stat(self.moments(), "kurtosis")

    def _distinct(self):
        r = N.DistinctRec()
        N.raise_for_status(N.lib().bdf_distinct_dev(self.ctx.handle, self.handle, C.byref(r)))
        return r

    def count_distinct(self) -> int: return int(self._distinct().count)
    def sum_distinct(self):
        _refuse_temporal("sum_distinct", self)
        return _scalar_from_bits(self.dtype, self._distinct().sum)

    # -- distributions (include/b200df.h "distributions"): Column::hist and Column::uniques of src/table.rs, Spark's percentile and mode --
    def percentile(self, p):
        """Spark's exact percentile at p (a float, or a sequence of up to 1024): a float or None, or a list of them."""
        _refuse_temporal("a percentile", self)
        ps, out, some = _percentile_args(p)
        N.raise_for_status(N.lib().bdf_percentile_dev(self.ctx.handle, self.handle, len(np.atleast_1d(p)), ps, out, some))
        return _percentile_result(p, out, some)

    def median(self) -> Optional[float]: return self.percentile(0.5)

    def _mode(self):
        bits, freq, some = C.c_uint64(0), C.c_int64(0), C.c_int32(0)
        N.raise_for_status(N.lib().bdf_mode_dev(self.ctx.handle, self.handle, C.byref(bits), C.byref(freq), C.byref(some)))
        return (_scalar_from_bits(self.dtype, bits.value), int(freq.value)) if some.value else (None, 0)

    def mode(self):
        """The most frequent valid value (ties: the smallest in key order), or None."""
        return self._mode()[0]

    def uniques(self) -> "Column":
        """The distinct valid values, ascending, as a one-chunk column (all NaNs are one value, -0.0 == 0.0)."""
        h = C.c_void_p()
        N.raise_for_status(N.lib().bdf_uniques_dev(self.ctx.handle, self.handle, C.byref(h), None))
        return Column(self.ctx, h, self.temporal)

    def value_counts(self):
        """``(values, counts)``: the distinct valid values ascending (as ``uniques``) and the Int64 number of rows of each."""
        h, hc = C.c_void_p(), C.c_void_p()
        N.raise_for_status(N.lib().bdf_uniques_dev(self.ctx.handle, self.handle, C.byref(h), C.byref(hc)))
        return Column(self.ctx, h, self.temporal), Column(self.ctx, hc)

    def hist(self, nbins: int, density: bool = False, range=None):
        """numpy.histogram's equal-width bins: ``(edges, counts)`` as numpy arrays (Float64 densities when ``density``); NaN is skipped."""
        _refuse_temporal("a histogram", self)
        edges = np.zeros(max(int(nbins), 0) + 1, dtype=np.float64)
        counts = np.zeros(max(int(nbins), 0), dtype=np.int64)
        rng = None if range is None else (C.c_double * 2)(float(range[0]), float(range[1]))
        N.raise_for_status(N.lib().bdf_hist_dev(self.ctx.handle, self.handle, int(nbins), rng, edges.ctypes.data_as(C.POINTER(C.c_double)),
                                                counts.ctypes.data_as(C.POINTER(C.c_int64))))
        return edges, (hist_density(edges, counts) if density else counts)

    # -- dates and timestamps (include/b200df.h "dates and timestamps"); the column must carry a temporal tag --
    def _temporal_fn(self, fn: int, arg=0) -> "Column":
        t = _temporal_of([self], None) if self.temporal is None else self.temporal
        a = _temporal_arg(fn, arg)
        _, out_t = temporal_result(fn, t, a)
        tc = _temporal_c(t)
        h = C.c_void_p()
        N.raise_for_status(N.lib().bdf_temporal_dev(self.ctx.handle, fn, C.byref(tc), a, self.handle, C.byref(h)))
        return Column(self.ctx, h, out_t)

    def _temporal_binary(self, fn: int, other: "Column") -> "Column":
        ta, tb = _temporal_of([self], self.temporal), _temporal_of([other], other.temporal)
        ca, cb = _temporal_c(ta), _temporal_c(tb)
        h = C.c_void_p()
        N.raise_for_status(N.lib().bdf_temporal_binary_dev(self.ctx.handle, fn, C.byref(ca), self.handle, C.byref(cb), other.handle, C.byref(h)))
        return Column(self.ctx, h)

    def year(self): return self._temporal_fn(N.T_YEAR)
    def quarter(self): return self._temporal_fn(N.T_QUARTER)
    def month(self): return self._temporal_fn(N.T_MONTH)
    def day_of_month(self): return self._temporal_fn(N.T_DAY_OF_MONTH)
    def day_of_year(self): return self._temporal_fn(N.T_DAY_OF_YEAR)
    def day_of_week(self): return self._temporal_fn(N.T_DAY_OF_WEEK)
    def hour(self): return self._temporal_fn(N.T_HOUR)
    def minute(self): return self._temporal_fn(N.T_MINUTE)
    def second(self): return self._temporal_fn(N.T_SECOND)
    def to_date(self): return self._temporal_fn(N.T_TO_DATE)
    def date_add(self, days: int): return self._temporal_fn(N.T_DATE_ADD, days)
    def date_sub(self, days: int): return self._temporal_fn(N.T_DATE_SUB, days)
    def add_months(self, months: int): return self._temporal_fn(N.T_ADD_MONTHS, months)
    def last_day(self): return self._temporal_fn(N.T_LAST_DAY)
    def next_day(self, day_of_week): return self._temporal_fn(N.T_NEXT_DAY, day_of_week)
    def date_trunc(self, unit): return self._temporal_fn(N.T_DATE_TRUNC, unit)
    def unix_timestamp(self): return self._temporal_fn(N.T_UNIX_TIMESTAMP)
    def to_timestamp(self, unit="us"): return self._temporal_fn(N.T_TO_TIMESTAMP, unit)
    def date_diff(self, start: "Column"): return self._temporal_binary(N.T_DATE_DIFF, start)
    def months_between(self, other: "Column"): return self._temporal_binary(N.T_MONTHS_BETWEEN, other)

    @staticmethod
    def aggregate_all_many(columns: Sequence["Column"], asynchronous: bool = False):
        """sum/min/max/count of several columns in ONE call: one reduction per column, one host wait and (on a rank of
        a communicator) one grouped collective for all of them.  Returns a list of dicts (or an AggFuture of one)."""
        ctx = columns[0].ctx
        k = len(columns)
        cols = (C.c_void_p * k)(*[c.handle for c in columns])
        _refuse_temporal("sum", *columns)
        dtypes = [c.dtype for c in columns]
        if asynchronous:
            f = C.c_void_p()
            N.raise_for_status(N.lib().bdf_aggregate_all_many_dev_async(ctx.handle, k, cols, C.byref(f)))
            return AggFuture(ctx, f, dtypes)
        out = (N.Agg4 * k)()
        N.raise_for_status(N.lib().bdf_aggregate_all_many_dev(ctx.handle, k, cols, out))
        return [_agg4_to_dict(dtypes[i], out[i]) for i in range(k)]

    # -- back to the host --
    def download(self, pinned: bool = False, into=None) -> List[PrimitiveArray]:
        dtype, n, _ = self.describe()
        if into is not None:
            outs, bufs = into
        else:
            lens = [self.chunk_len(i) for i in range(n)]
            outs, bufs = N.alloc_outputs(dtype, lens, self.ctx, pinned)
        if dtype != N.BOOL:
            for i in range(n):
                outs[i].len = bufs[i][0].shape[0]
        N.raise_for_status(N.lib().bdf_download(self.ctx.handle, self.handle, outs))
        res = N.collect_outputs(dtype, outs, bufs)
        if self.temporal is not None:
            for r in res:
                r.temporal = self.temporal
        return res

    def download_begin(self, into):
        """Enqueue the device->host copies into `into` = alloc_outputs(...); pair with download_end(into)."""
        outs, bufs = into
        for i in range(len(bufs)):
            outs[i].len = bufs[i][0].shape[0]
        N.raise_for_status(N.lib().bdf_download_begin(self.ctx.handle, self.handle, outs))

    def download_end(self, into) -> List[PrimitiveArray]:
        outs, bufs = into
        N.raise_for_status(N.lib().bdf_download_end(self.ctx.handle, self.handle, outs))
        return N.collect_outputs(self.dtype, outs, bufs)

    def chunk_len(self, i: int) -> int:
        ln = C.c_int64()
        N.raise_for_status(N.lib().bdf_col_chunk_info(self.ctx.handle, self.handle, i, C.byref(ln), None, None))
        return ln.value

    def free(self):
        if self.handle is not None and self.ctx.handle:
            N.lib().bdf_col_free(self.ctx.handle, self.handle)
        self.handle = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


# ---- null handling and conditional selection ---------------------------------------------------------------------------
def _scalar_bits(dtype: int, v) -> int:
    """T::Native bits of the Python scalar v in a column of `dtype` (the column arguments type the scalars); a value the type
    cannot hold exactly is refused, as the casts the caller would otherwise write."""
    if dtype == N.BOOL:
        if not isinstance(v, (bool, np.bool_)):
            raise N.UnsupportedType(f"{v!r} is not a Boolean scalar")
        return int(bool(v))
    if isinstance(v, (bool, np.bool_)):
        raise N.UnsupportedType(f"a Boolean scalar in a {dtype} argument list")
    npt = NP_DTYPES[dtype]
    if is_float(dtype):
        x = npt.type(v)
        if not (float(x) == float(v) or (x != x and v != v)):
            raise N.UnsupportedType(f"{v!r} is not exactly a {npt} value")
    else:
        if isinstance(v, (float, np.floating)):
            if not float(v).is_integer():
                raise N.UnsupportedType(f"{v!r} is not an integer")
            v = int(v)
        info = np.iinfo(npt)
        if not info.min <= int(v) <= info.max:
            raise N.UnsupportedType(f"{v!r} is out of range for {npt}")
        x = npt.type(int(v))
    return int(np.array([x], dtype=npt).view(np.dtype(f"u{npt.itemsize}"))[0])


def _args_type(columns, what: str):
    """(dtype, temporal tag) of the column arguments; mismatched temporal types are refused here, before any device work."""
    if not columns:
        raise N.ComputeError(f"{what} needs at least one column argument: the columns give the result type")
    tags = {repr(getattr(c, "temporal", None)) for c in columns}
    if len(tags) > 1:
        raise N.UnsupportedType(f"{what} of columns of different temporal types ({', '.join(sorted(tags))}): cast them first")
    for c in columns:
        if isinstance(c, ListColumn):
            raise N.UnsupportedType(f"{what} of a list column")
    return columns[0].dtype, getattr(columns[0], "temporal", None)


def _make_args(values, dtype: int):
    args = (N.Arg * max(len(values), 1))()
    for i, v in enumerate(values):
        if isinstance(v, Column):
            args[i].column, args[i].valid = v.handle, 1
        elif v is None:
            args[i].column, args[i].valid = None, 0
        else:
            args[i].column, args[i].bits, args[i].valid = None, _scalar_bits(dtype, v), 1
    return args


def _rowwise(fn: int, values, what: str = "a row-wise function") -> "Column":
    cols = [v for v in values if isinstance(v, (Column, ListColumn))]
    dtype, tag = _args_type(cols, what)
    args = _make_args(values, dtype)
    h = C.c_void_p()
    N.raise_for_status(N.lib().bdf_rowwise_dev(cols[0].ctx.handle, fn, len(values), args, C.byref(h)))
    return Column(cols[0].ctx, h, tag)


def coalesce(*args) -> "Column":
    """Spark's coalesce: per row the first argument valid there, NULL where every argument is NULL (1..64 arguments, Columns or
    scalars of the columns' type; None is a NULL literal)."""
    return _rowwise(N.ROW_COALESCE, args, "coalesce")


def greatest(*args) -> "Column":
    """Spark's greatest: the largest valid argument per row in DataFrame::sort's order (NaN above +inf); NULL only where every
    argument is NULL; among equal values the earliest argument's bits (2..64 arguments)."""
    return _rowwise(N.ROW_GREATEST, args, "greatest")


def least(*args) -> "Column":
    """Spark's least: greatest with the order reversed."""
    return _rowwise(N.ROW_LEAST, args, "least")


def nanvl(a, b) -> "Column":
    return _rowwise(N.ROW_NANVL, (a, b), "nanvl")


class CaseWhen:
    """``when(c1, v1).when(c2, v2).otherwise(v)``: SQL's CASE WHEN.  Each row takes the value of the first branch whose Boolean
    condition is valid and true there (a NULL condition counts as false); rows no branch takes get the ``otherwise`` value
    (None, or no ``otherwise`` call at all through ``end()``, means NULL)."""

    def __init__(self, branches):
        self.branches = list(branches)

    def when(self, cond: "Column", value) -> "CaseWhen":
        return CaseWhen(self.branches + [(cond, value)])

    def otherwise(self, value=None) -> "Column":
        conds = [c for c, _ in self.branches]
        values = [v for _, v in self.branches] + [value]
        for c in conds:
            if not isinstance(c, Column):
                raise N.UnsupportedType("a case_when condition must be a Boolean Column")
        dtype, tag = _args_type([v for v in values if isinstance(v, (Column, ListColumn))], "case_when")
        args = _make_args(values, dtype)
        ca = (C.c_void_p * len(conds))(*[c.handle for c in conds])
        h = C.c_void_p()
        N.raise_for_status(N.lib().bdf_case_when_dev(conds[0].ctx.handle, len(conds), ca, args, C.byref(h)))
        return Column(conds[0].ctx, h, tag)

    def end(self) -> "Column":
        return self.otherwise(None)


def when(cond: "Column", value) -> CaseWhen:
    return CaseWhen([(cond, value)])


def _rowwise_host(fn: int, args, ctx) -> List[PrimitiveArray]:
    """A row-wise function over host chunks: every chunk list is uploaded, the device entry runs, the result comes back."""
    ctx = ctx or N.default_context()
    cols = []
    try:
        vals = []
        for a in args:
            if a is None or not isinstance(a, (list, tuple)):
                vals.append(a)
            else:
                cols.append(Column.upload(a, ctx, dtype=_dtype_of(a) if len(a) else None))
                vals.append(cols[-1])
        out = _rowwise(fn, vals)
        try:
            return out.download()
        finally:
            out.free()
    finally:
        for c in cols:
            c.free()


def _scalar_fn(fn: int, doc: str):
    def f(*args, ctx=None) -> List[PrimitiveArray]:
        return _rowwise_host(fn, args, ctx)
    f.__doc__ = doc
    return staticmethod(f)


ScalarFunctions.coalesce = _scalar_fn(N.ROW_COALESCE, "coalesce over columns given as lists of chunks (or scalars): scalar.rs's empty stub, Spark's definition.")
ScalarFunctions.greatest = _scalar_fn(N.ROW_GREATEST, "greatest over columns given as lists of chunks (or scalars): scalar.rs's empty stub, Spark's definition.")
ScalarFunctions.least = _scalar_fn(N.ROW_LEAST, "least over columns given as lists of chunks (or scalars): scalar.rs's empty stub, Spark's definition.")
ScalarFunctions.nanvl = _scalar_fn(N.ROW_NANVL, "nanvl(a, b) over columns given as lists of chunks: scalar.rs's nanv1 stub, Spark's definition.")


def sort_indices(criteria: Sequence[tuple]) -> "Column":
    """compute::lexsort_to_indices as DataFrame::sort calls it (src/dataframe.rs:194-213).  criteria: [(Column, descending)];
    stable, nulls last.  Returns a one-chunk UInt32 Column of row numbers."""
    if not criteria:
        raise N.ComputeError("Sort criteria cannot be empty")
    ctx = criteria[0][0].ctx
    arr = (N.SortKeyC * len(criteria))()
    for i, (col, desc) in enumerate(criteria):
        arr[i].column, arr[i].descending = col.handle.value if isinstance(col.handle, C.c_void_p) else col.handle, 1 if desc else 0
    h = C.c_void_p()
    N.raise_for_status(N.lib().bdf_sort_indices_dev(ctx.handle, len(criteria), arr, C.byref(h)))
    return Column(ctx, h)


def top_k_indices(criteria: Sequence[tuple], k: int) -> "Column":
    """The first min(k, n) entries of sort_indices(criteria), chosen without sorting every row (SQL's ORDER BY ... LIMIT k).
    criteria: [(Column, descending)]; the same order and errors as sort_indices, and k < 0 is refused.  Returns a one-chunk
    UInt32 Column of row numbers."""
    if not criteria:
        raise N.ComputeError("Sort criteria cannot be empty")
    ctx = criteria[0][0].ctx
    arr = (N.SortKeyC * len(criteria))()
    for i, (col, desc) in enumerate(criteria):
        arr[i].column, arr[i].descending = col.handle.value if isinstance(col.handle, C.c_void_p) else col.handle, 1 if desc else 0
    h = C.c_void_p()
    N.raise_for_status(N.lib().bdf_top_k_indices_dev(ctx.handle, len(criteria), arr, int(k), C.byref(h)))
    return Column(ctx, h)


def sort_columns(criteria: Sequence[tuple], columns: Sequence["Column"]) -> List["Column"]:
    """DataFrame::sort: the index sort, then DataFrame::sort_by_indices (Column::take of every column, one chunk each)."""
    idx = sort_indices(criteria)
    return [c.take(idx) for c in columns]


def group_aggregate(key: "Column", values: Sequence["Column"]):
    """Group-by aggregate (`GroupAggregate`, unimplemented in the reference: src/evaluation.rs:73): returns
    ``(keys Column, [ {"sum": Column, "count": Column, "min": Column | None, "max": Column | None} per value column ])``.
    Groups in ascending key order, the null key last; see include/b200df.h bdf_group_aggregate_dev.  For a temporal value column
    "sum" is None (dates are not summed; the device's sum is freed unread) and min / max carry the column's tag."""
    ctx = key.ctx
    k = len(values)
    cols = (C.c_void_p * max(k, 1))(*[v.handle for v in values])
    outs = (N.GroupOut * max(k, 1))()
    hk, ng = C.c_void_p(), C.c_int64(0)
    N.raise_for_status(N.lib().bdf_group_aggregate_dev(ctx.handle, key.handle, k, cols, C.byref(hk), outs, C.byref(ng)))
    wrap = lambda p, t=None: Column(ctx, C.c_void_p(p), t) if p else None
    res = []
    for j, v in enumerate(values):
        t = getattr(v, "temporal", None)
        s = wrap(outs[j].sum)
        if t is not None and s is not None:
            s.free()
            s = None
        res.append({"sum": s, "count": wrap(outs[j].count), "min": wrap(outs[j].min, t), "max": wrap(outs[j].max, t)})
    return Column(ctx, hk, key.temporal), res


def group_by(keys: Sequence["Column"], aggregations: Sequence[tuple]):
    """Group-by over 1..16 key columns (bdf_group_by_dev).  ``aggregations``: ``[(Column, function)]`` with function one of
    "sum", "max", "min", "avg", "count", "count_distinct", "first", "last", "kurtosis", "skewness", "stddev", "sum_distinct",
    "variance", "stddev_pop", "var_pop", "exact_median", "mode", "collect_list", "collect_set".  Returns ``([key Column per key],
    [result per aggregation])``; groups in the order DataFrame::sort gives (ascending, nulls last per key).  Counts are Int64, avg,
    median and the statistics are Float64, collect_list / collect_set are ListColumns of one chunk (bdf_group_by_lists_dev, called
    only when one of them is asked for), everything else has the value column's type; see include/b200df.h for the NULL rules.  A
    temporal column is refused for collect: a ListColumn carries no temporal tag."""
    fns = []
    for col, fn in aggregations:
        if fn not in N.GROUP_FNS and fn not in N.COLLECT_FNS:
            raise N.UnsupportedType(f"group function {fn!r} is not on the path")
        if isinstance(col, ListColumn):
            raise N.UnsupportedType(f"{fn} of a list column: aggregated columns must be numeric")
        if fn not in _CARRY_GROUP and fn not in ("count", "count_distinct"):
            _refuse_temporal(fn, col)   # collect too: a ListColumn carries no temporal tag
        fns.append(N.GROUP_FNS.get(fn, N.COLLECT_FNS.get(fn)))
    if any(isinstance(k, ListColumn) for k in keys):
        raise N.UnsupportedType("a list column is not a group key: group-by keys must be numeric")
    ctx = keys[0].ctx if keys else (aggregations[0][0].ctx if aggregations else N.default_context())
    nk, na = len(keys), len(aggregations)
    kcols = (C.c_void_p * max(nk, 1))(*[k.handle for k in keys])
    aggs = (N.GroupAggC * max(na, 1))()
    for j, ((col, _), f) in enumerate(zip(aggregations, fns)):
        aggs[j].column, aggs[j].function = col.handle.value if isinstance(col.handle, C.c_void_p) else col.handle, f
    hk = (C.c_void_p * max(nk, 1))()
    out = (C.c_void_p * max(na, 1))()
    ng = C.c_int64(0)
    if any(fn in N.COLLECT_FNS for _, fn in aggregations):   # list outputs: the entry that can return them
        lists = (C.c_void_p * max(na, 1))()
        N.raise_for_status(N.lib().bdf_group_by_lists_dev(ctx.handle, nk, kcols, na, aggs, hk, out, lists, C.byref(ng)))
    else:
        lists = None
        N.raise_for_status(N.lib().bdf_group_by_dev(ctx.handle, nk, kcols, na, aggs, hk, out, C.byref(ng)))
    carry = lambda col, fn: getattr(col, "temporal", None) if fn in _CARRY_GROUP else None
    result = lambda j: (ListColumn(ctx, C.c_void_p(lists[j])) if lists is not None and lists[j]
                        else Column(ctx, C.c_void_p(out[j]), carry(*aggregations[j])))
    return ([Column(ctx, C.c_void_p(hk[k]), keys[k].temporal) for k in range(nk)], [result(j) for j in range(na)])


_CARRY_GROUP = ("min", "max", "first", "last", "mode")   # aggregations whose results are values of the column: a temporal tag carries


def join_indices(left_keys: Sequence["Column"], right_keys: Sequence["Column"], how: str):
    """calc_equijoin_indices (src/functions/join.rs:19-137) on the device (bdf_join_indices_dev): criterion k is
    ``(left_keys[k], right_keys[k])``; ``how`` is "left", "right", "inner", "full", "left_semi" or "left_anti".  Returns
    ``(left_idx, right_idx)``, two one-chunk UInt32 Columns of row numbers (NULL = no partner) to ``take`` each side's columns with.
    The order of the pairs is fixed (left rows in row order, each one's partners in right row order; see include/b200df.h), a null
    key matches nothing, NaN == NaN and -0.0 == 0.0.  "left_semi" / "left_anti" return ``(left_idx, None)``: the left rows that have
    (lack) a partner, each once, ascending, without nulls."""
    if how not in N.JOIN_TYPES:
        raise N.UnsupportedType(f"join type {how!r} is not one of {sorted(N.JOIN_TYPES)}")
    if len(left_keys) != len(right_keys):
        raise N.ComputeError("every join criterion needs a left and a right column")
    if not left_keys:
        raise N.ComputeError("Join criteria cannot be empty")
    ctx = left_keys[0].ctx
    n = len(left_keys)
    lk = (C.c_void_p * n)(*[k.handle for k in left_keys])
    rk = (C.c_void_p * n)(*[k.handle for k in right_keys])
    hl, hr, rows = C.c_void_p(), C.c_void_p(), C.c_int64(0)
    N.raise_for_status(N.lib().bdf_join_indices_dev(ctx.handle, N.JOIN_TYPES[how], n, lk, rk, C.byref(hl), C.byref(hr), C.byref(rows)))
    if how in ("left_semi", "left_anti"):
        return Column(ctx, hl), None
    return Column(ctx, hl), Column(ctx, hr)


_TIME_UNIT_NS = (10 ** 9, 10 ** 6, 1000, 1)   # nanoseconds per arrow TimeUnit s, ms, us, ns


def _asof_tolerance(tolerance, on: "Column"):
    """(has_tolerance, tolerance, tolerance_f) of bdf_asof_spec: a float for a Float32 / Float64 key (+inf allowed), an integer in the
    key's own units otherwise, or a datetime.timedelta for a Date / Timestamp / Time key, converted exactly to its unit."""
    if tolerance is None:
        return 0, 0, 0.0
    if isinstance(tolerance, datetime.timedelta):
        t = getattr(on, "temporal", None)
        if t is None:
            raise N.ComputeError("a timedelta tolerance needs a Date, Timestamp or Time key")
        us = (tolerance.days * 86_400 + tolerance.seconds) * 10 ** 6 + tolerance.microseconds
        per = 86_400 * 10 ** 9 if t.kind == DATE32 else 10 ** 6 if t.kind == DATE64 else _TIME_UNIT_NS[t.unit]
        if (us * 1000) % per:
            raise N.ComputeError(f"tolerance {tolerance!r} is not a whole number of the key's unit")
        tolerance = us * 1000 // per
    elif is_float(on.dtype):
        v = float(tolerance)
        if not v >= 0:
            raise N.ComputeError(f"the as-of tolerance must be >= 0, not {tolerance!r}")
        return 1, 0, v
    if isinstance(tolerance, float) and not tolerance.is_integer():
        raise N.ComputeError(f"tolerance {tolerance!r} over an integer key must be an integer")
    v = int(tolerance)
    if not 0 <= v <= _INT64_MAX:
        raise N.ComputeError(f"the as-of tolerance must be in 0..2^63-1, not {tolerance!r}")
    return 1, v, 0.0


def join_asof_indices(left_on: "Column", right_on: "Column", left_by: Sequence["Column"] = (), right_by: Sequence["Column"] = (),
                      direction: str = "backward", allow_exact_matches: bool = True, tolerance=None) -> "Column":
    """pandas' merge_asof on the device (bdf_join_asof_dev): for every left row, the right row whose ``on`` key is the last at or before
    its own ("backward"), the first at or after it ("forward") or the nearer of the two ("nearest", ties backward), among the right rows
    whose ``by`` keys equal the left row's.  Of equal keys, backward takes the last right row and forward the first.  Returns one
    one-chunk UInt32 Column with a right row number per left row (NULL = no partner) to ``take`` the right columns with; left order
    is kept.  ``allow_exact_matches=False`` makes the bounds strict; ``tolerance`` (see _asof_tolerance) nulls a pick farther away.
    Neither side needs to be sorted; null and NaN keys match nothing (include/b200df.h)."""
    if direction not in N.ASOF_DIRECTIONS:
        raise N.UnsupportedType(f"as-of direction {direction!r} is not one of {sorted(N.ASOF_DIRECTIONS)}")
    if len(left_by) != len(right_by):
        raise N.ComputeError("every as-of by key needs a left and a right column")
    if len(left_by) > 16:
        raise N.ComputeError("0..16 as-of by keys")
    cols = [left_on, right_on, *left_by, *right_by]
    if any(isinstance(c, ListColumn) for c in cols):
        raise N.UnsupportedType("a list column is not a join key: as-of keys must be numeric")
    if getattr(left_on, "temporal", None) != getattr(right_on, "temporal", None):
        raise N.UnsupportedType(f"as-of keys of different temporal types ({left_on.temporal!r}, {right_on.temporal!r}): cast them first")
    spec = N.AsofSpec(N.ASOF_DIRECTIONS[direction], 1 if allow_exact_matches else 0, *_asof_tolerance(tolerance, left_on))
    ctx = left_on.ctx
    n = len(left_by)
    lb = (C.c_void_p * max(n, 1))(*[k.handle for k in left_by])
    rb = (C.c_void_p * max(n, 1))(*[k.handle for k in right_by])
    h = C.c_void_p()
    N.raise_for_status(N.lib().bdf_join_asof_dev(ctx.handle, left_on.handle, right_on.handle, n, lb, rb, C.byref(spec), C.byref(h)))
    return Column(ctx, h)


_KEEP = {"first": N.KEEP_FIRST, "last": N.KEEP_LAST, False: N.KEEP_NONE}
MAX_SET_KEYS = 16   # the key limit of group-by and join


def _set_keys(keys: Sequence["Column"], what: str) -> None:
    if not 1 <= len(keys) <= MAX_SET_KEYS:
        raise N.UnsupportedType(f"{what} compares 1..{MAX_SET_KEYS} columns (the limit of group-by and join), not {len(keys)}")
    if any(isinstance(k, ListColumn) for k in keys):
        raise N.UnsupportedType(f"a list column cannot be compared by {what}: the compared columns must be numeric or Boolean")


def duplicated(keys: Sequence["Column"], keep="first") -> "Column":
    """pandas' duplicated over the rows of `keys` (bdf_duplicated_dev): a Boolean Column without nulls, chunked like the keys, true
    for every row of a run of equal rows except its first ("first"), except its last ("last"), or for every row of a run longer
    than one (False).  Nulls equal each other, all NaNs are one value and -0.0 == 0.0 (group-by's equality); Boolean keys are
    allowed."""
    if not (keep is False or (isinstance(keep, str) and keep in ("first", "last"))):
        raise N.UnsupportedType(f"keep must be 'first', 'last' or False, not {keep!r}")
    _set_keys(keys, "duplicated")
    ctx = keys[0].ctx
    ks = (C.c_void_p * len(keys))(*[k.handle for k in keys])
    h = C.c_void_p()
    N.raise_for_status(N.lib().bdf_duplicated_dev(ctx.handle, len(keys), ks, _KEEP[keep], C.byref(h)))
    return Column(ctx, h)


def set_op_mask(left: Sequence["Column"], right: Sequence["Column"], op: str) -> "Column":
    """The rows of `left` a set operation keeps (bdf_set_op_dev), as a Boolean Column over the left rows, chunked like left[0]:
    op is "intersect", "intersect_all", "except" (Spark's subtract) or "except_all".  In a run of equal rows with cl left and cr
    right rows, the run keeps its first min(cl, cr) ("intersect_all"), max(cl - cr, 0) ("except_all"), one if cr > 0
    ("intersect") or one if cr == 0 ("except") left rows in row order.  Equality is duplicated's."""
    if op not in N.SET_OPS:
        raise N.UnsupportedType(f"set operation {op!r} is not one of {sorted(N.SET_OPS)}")
    if len(left) != len(right):
        raise N.UnsupportedType("Union can only be performed on tables with the same number of columns")
    _set_keys(left, op)
    _set_keys(right, op)
    for a, b in zip(left, right):
        if a.dtype != b.dtype or getattr(a, "temporal", None) != getattr(b, "temporal", None):
            raise N.UnsupportedType("Union can only be performed on tables with compatible column types")
    ctx = left[0].ctx
    lk = (C.c_void_p * len(left))(*[k.handle for k in left])
    rk = (C.c_void_p * len(right))(*[k.handle for k in right])
    h = C.c_void_p()
    N.raise_for_status(N.lib().bdf_set_op_dev(ctx.handle, N.SET_OPS[op], len(left), lk, rk, C.byref(h)))
    return Column(ctx, h)


def filter_any(column, mask: "Column"):
    """column.filter(mask) for every kind of column: a Boolean column goes through the filter as UInt8 (bdf_bool_widen_dev) and comes
    back through a != 0 comparison, nulls kept; a ListColumn uses its own filter."""
    if isinstance(column, ListColumn) or column.dtype != N.BOOL:
        return column.filter(mask)
    h = C.c_void_p()
    N.raise_for_status(N.lib().bdf_bool_widen_dev(column.ctx.handle, column.handle, C.byref(h)))
    wide = Column(column.ctx, h)
    try:
        kept = wide.filter(mask)
    finally:
        wide.free()
    try:
        return kept.ne(0)
    finally:
        kept.free()


def concat(columns: Sequence) -> "Column":
    """pandas' concat of columns (bdf_concat_dev / bdf_list_concat_dev): the chunks of columns[0], then those of columns[1], and so
    on, copied on the device.  The columns must have one dtype and one temporal type; ListColumns concatenate with ListColumns."""
    columns = list(columns)
    if not columns:
        raise N.ComputeError("concat needs at least one column")
    if any(isinstance(c, ListColumn) for c in columns):
        if not all(isinstance(c, ListColumn) for c in columns):
            raise N.UnsupportedType("a list column concatenates only with list columns")
        return ListColumn.concat(columns)
    dtypes = {c.dtype for c in columns}
    tags = {getattr(c, "temporal", None) for c in columns}
    if len(dtypes) != 1 or len(tags) != 1:
        raise N.UnsupportedType("Union can only be performed on tables with compatible column types")
    ctx = columns[0].ctx
    cs = (C.c_void_p * len(columns))(*[c.handle for c in columns])
    h = C.c_void_p()
    N.raise_for_status(N.lib().bdf_concat_dev(ctx.handle, len(columns), cs, C.byref(h)))
    return Column(ctx, h, tags.pop())


_INT64_MIN, _INT64_MAX = -2 ** 63, 2 ** 63 - 1
_TIMESTAMP_UNIT_US = (10 ** 6, 1000, 1)   # microseconds per arrow TimeUnit s, ms, us (ns: x 1000)


def _frame_offset(v, key, upper: bool):
    """One bound of a ("rows" | "range", start, end) frame as the C call takes it: None is UNBOUNDED (PRECEDING for the start, FOLLOWING
    for the end).  A RANGE offset is typed by the order key: a float offset for a Float32 / Float64 key, an integer otherwise, and a
    datetime.timedelta for a Date or Timestamp key, converted to the key's unit (days for Date32, ms for Date64)."""
    is_float = key is not None and key[0] in (F32, F64)
    if v is None:
        return (math.inf if upper else -math.inf) if is_float else (_INT64_MAX if upper else _INT64_MIN)
    if isinstance(v, datetime.timedelta):
        t = key[1] if key is not None else None
        if t is None or t.kind not in (DATE32, DATE64, TIMESTAMP):
            raise N.ComputeError("a timedelta frame offset needs a Date or Timestamp order key")
        us = (v.days * 86_400 + v.seconds) * 10 ** 6 + v.microseconds
        if t.kind == TIMESTAMP and t.unit == 3:
            return us * 1000
        per = {DATE32: 86_400 * 10 ** 6, DATE64: 1000}.get(t.kind) or _TIMESTAMP_UNIT_US[t.unit]
        if us % per:
            raise N.ComputeError(f"frame offset {v!r} is not a whole number of the order key's unit")
        return us // per
    if is_float:
        return float(v)
    if isinstance(v, float) and not v.is_integer():
        raise N.ComputeError(f"frame offset {v!r} over an integer order key must be an integer")
    return int(v)


def _window_frame(k: "N.WindowCall", frame, ordered: bool, key) -> None:
    if frame is None:
        frame = "range" if ordered else "partition"
    if isinstance(frame, tuple):
        if len(frame) != 3 or frame[0] not in N.BOUNDED_FRAMES:
            raise N.UnsupportedType(f"window frame {frame!r} is not (\"rows\" | \"range\", start, end)")
        k.frame = N.BOUNDED_FRAMES[frame[0]]
        rng = frame[0] == "range"
        s, e = (_frame_offset(frame[1], key if rng else None, False), _frame_offset(frame[2], key if rng else None, True))
        if rng and key is not None and key[0] in (F32, F64):
            k.start_f, k.end_f = s, e
        else:
            for v in (s, e):
                if not _INT64_MIN <= v <= _INT64_MAX:
                    raise N.ComputeError(f"frame offset {v} does not fit Int64")
            k.start, k.end = s, e
        return
    if frame not in N.WINDOW_FRAMES:
        raise N.UnsupportedType(f"window frame {frame!r} is not one of {sorted(N.WINDOW_FRAMES)}")
    k.frame = N.WINDOW_FRAMES[frame]


_WINDOW_VALUES = ("first_value", "last_value", "nth_value")


def _window_call(call: tuple, ordered: bool, key=None) -> "N.WindowCall":
    """One call tuple -> bdf_window_call.  ``("row_number",)`` .. ``("cume_dist",)``; ``("lag" | "lead", x, offset=1, default=None)``;
    ``("sum" | "count" | "min" | "max" | "avg", x, frame=None)``; ``("first_value" | "last_value", x, frame=None, ignore_nulls=False)``
    and ``("nth_value", x, n, frame=None, ignore_nulls=False)``.  A frame is "rows", "range" or "partition" (None: SQL's default,
    "range" with an ORDER BY and "partition" without), or a bounded ``("rows" | "range", start, end)`` with signed offsets (negative =
    PRECEDING, 0 = CURRENT ROW, positive = FOLLOWING, None = UNBOUNDED).  ``key``: (dtype, TemporalType or None) of the single order
    column, which types RANGE offsets."""
    name = call[0]
    if name not in N.WINDOW_FNS:
        raise N.UnsupportedType(f"window function {name!r} is not one of {sorted(N.WINDOW_FNS)}")
    fn = N.WINDOW_FNS[name]
    k = N.WindowCall()
    k.function = fn
    if fn <= N.WIN_CUME_DIST:
        if len(call) != 1:
            raise N.ComputeError(f"{name} takes no column")
        return k
    if len(call) < 2:
        raise N.ComputeError(f"{name} needs a column")
    x = call[1]
    if name not in ("lag", "lead", "min", "max", "count") + _WINDOW_VALUES:
        _refuse_temporal(name, x)
    k.column = x.handle.value if isinstance(x.handle, C.c_void_p) else x.handle
    if fn in (N.WIN_LAG, N.WIN_LEAD):
        k.offset = int(call[2]) if len(call) > 2 else 1
        default = call[3] if len(call) > 3 else None
        if default is not None:
            raw = np.array(default, dtype=NP_DTYPES[x.dtype]).tobytes()   # T::Native in the low bytes
            k.default_bits = int.from_bytes(raw.ljust(8, b"\0"), "little")
            k.has_default = 1
        return k
    rest = list(call[2:])
    if name == "nth_value":
        if not rest:
            raise N.ComputeError("nth_value needs n")
        k.offset = int(rest.pop(0))
    _window_frame(k, rest[0] if rest else None, ordered, key)
    if name in _WINDOW_VALUES:
        k.ignore_nulls = 1 if len(rest) > 1 and rest[1] else 0
    elif len(rest) > 1:
        raise N.ComputeError(f"{name} takes a column and a frame")
    return k


def window(partition_by: Sequence["Column"], order_by: Sequence[tuple], calls: Sequence[tuple]) -> List["Column"]:
    """Window functions over one specification (bdf_window_dev): rows are partitioned by the tuple of ``partition_by`` columns
    and ordered inside a partition by ``order_by`` (``[(Column, descending)]``; nulls last in both directions, ties in row order).
    ``calls`` are tuples as ``_window_call`` describes, e.g. ``("row_number",)``, ``("lag", x, 1, 0.0)``, ``("sum", x, "range")``,
    ``("avg", x, ("rows", -99, 0))`` or ``("last_value", x, ("rows", None, 0), True)`` (forward fill).  Returns one one-chunk Column
    per call, in the caller's row order: row r of each belongs to input row r."""
    cols = list(partition_by) + [c for c, _ in order_by] + [c[1] for c in calls if len(c) > 1]
    ctx = cols[0].ctx if cols else N.default_context()
    key = (order_by[0][0].dtype, getattr(order_by[0][0], "temporal", None)) if len(order_by) == 1 else None
    arr = (N.WindowCall * max(len(calls), 1))()
    for j, call in enumerate(calls):
        arr[j] = _window_call(call, bool(order_by), key)
    handle = lambda c: c.handle.value if isinstance(c.handle, C.c_void_p) else c.handle
    pk = (C.c_void_p * max(len(partition_by), 1))(*[handle(c) for c in partition_by])
    ok = (N.SortKeyC * max(len(order_by), 1))()
    for i, (c, desc) in enumerate(order_by):
        ok[i].column, ok[i].descending = handle(c), 1 if desc else 0
    out = (C.c_void_p * max(len(calls), 1))()
    N.raise_for_status(N.lib().bdf_window_dev(ctx.handle, len(partition_by), pk, len(order_by), ok, len(calls), arr, out))
    carry = lambda c: getattr(c[1], "temporal", None) if c[0] in ("lag", "lead", "min", "max") + _WINDOW_VALUES else None
    return [Column(ctx, C.c_void_p(out[j]), carry(calls[j])) for j in range(len(calls))]


def _expr_nodes(nodes: Sequence[tuple]):
    arr = (N.ExprNode * len(nodes))()
    for k, nd in enumerate(nodes):
        if len(nd) == 2:
            op = nd[0]
            if isinstance(op, str):
                op = N.EXPR_UNARY + getattr(N, op.upper())
            arr[k].op, arr[k].a, arr[k].b = op, nd[1], nd[1]
        else:
            arr[k].op, arr[k].a, arr[k].b = nd
    return arr


def eval_expr(inputs: Sequence["Column"], nodes: Sequence[tuple]) -> "Column":
    """Evaluate a chain of Calculations in ONE pass over Float64 columns (SURVEY 8(f) N3).

    ``nodes`` is a straight-line program: slots ``0..len(inputs)-1`` are the input columns, node ``k`` writes slot
    ``len(inputs)+k``.  A node is ``(binop, a, b)`` with ``binop`` in native.ADD..LOG, or ``("sin", a)`` / ``(native.EXPR_UNARY + unop, a)``
    for a unary function.  The last node is the result column; intermediates never touch HBM."""
    _refuse_temporal("a fused expression", *inputs)
    ctx = inputs[0].ctx
    cols = (C.c_void_p * len(inputs))(*[c.handle for c in inputs])
    h = C.c_void_p()
    N.raise_for_status(N.lib().bdf_eval_expr_dev(ctx.handle, len(inputs), cols, len(nodes), _expr_nodes(nodes), C.byref(h)))
    return Column(ctx, h)


def eval_expr_agg(inputs: Sequence["Column"], nodes: Sequence[tuple], materialise: bool = True, asynchronous: bool = False):
    """eval_expr with sum/count of the result folded into the same pass.  Returns ``(Column or None, aggregate)`` where the
    aggregate is a dict (or an AggFuture when ``asynchronous``); ``materialise=False`` never writes the result column."""
    _refuse_temporal("a fused expression", *inputs)
    ctx = inputs[0].ctx
    cols = (C.c_void_p * len(inputs))(*[c.handle for c in inputs])
    h = C.c_void_p()
    hp = C.byref(h) if materialise else None
    if asynchronous:
        f = C.c_void_p()
        N.raise_for_status(N.lib().bdf_eval_expr_agg_dev_async(ctx.handle, len(inputs), cols, len(nodes), _expr_nodes(nodes), hp, C.byref(f)))
        agg = AggFuture(ctx, f, F64)
    else:
        a = N.Agg4()
        N.raise_for_status(N.lib().bdf_eval_expr_agg_dev(ctx.handle, len(inputs), cols, len(nodes), _expr_nodes(nodes), hp, C.byref(a)))
        agg = _agg4_to_dict(F64, a)
    return (Column(ctx, h) if materialise else None), agg


class AggFuture:
    """An aggregate whose kernels are enqueued; result() blocks until the value is on the host."""

    def __init__(self, ctx: N.Context, handle: C.c_void_p, dtype):
        """dtype: an int (one aggregate -> result() is a dict) or a list (multi-column call -> a list of dicts)."""
        self.ctx, self.handle, self.dtype = ctx, handle, dtype
        self._value = None

    def result(self):
        if self.handle is not None:
            many = isinstance(self.dtype, (list, tuple))
            k = len(self.dtype) if many else 1
            a = (N.Agg4 * k)()
            N.raise_for_status(N.lib().bdf_future_wait(self.ctx.handle, self.handle, a))
            self.handle = None
            self._value = [_agg4_to_dict(self.dtype[i], a[i]) for i in range(k)] if many else _agg4_to_dict(self.dtype, a[0])
        return self._value

    def __del__(self):
        try:
            if self.handle is not None and self.ctx.handle:
                N.lib().bdf_future_wait(self.ctx.handle, self.handle, None)
                self.handle = None
        except Exception:
            pass


# ---------------------------------------------------------------------------------------------------
# list columns (ArrayFunctions, src/functions/array.rs; rules in include/b200df.h "list columns")


def _value_bits(dtype: int, value) -> int:
    """T::Native of the list's element type in the low bytes of a u64 (bdf_window_call.default_bits)."""
    return int(np.array([value], dtype=NP_DTYPES[dtype]).view(f"u{width_of(dtype)}")[0])


class ListColumn:
    """A ``List<T>`` column in HBM: per chunk the list validity, rebased Int32 offsets and the elements, which are an ordinary
    ``Column`` (``values``)."""

    def __init__(self, ctx: N.Context, handle: C.c_void_p):
        self.ctx = ctx
        self.handle = handle

    @classmethod
    def upload(cls, arrays: Sequence, ctx: Optional[N.Context] = None, dtype: Optional[int] = None) -> "ListColumn":
        ctx = ctx or N.default_context()
        if dtype is None:
            if not arrays:
                raise ValueError("empty list column: the element type cannot be inferred; pass at least one chunk")
            dtype = arrays[0].dtype
        views = (N.ListView * max(len(arrays), 1))()
        for i, a in enumerate(arrays):
            if a.dtype != dtype:
                raise N.UnsupportedType("list chunks of different element types")
            views[i].offsets = a.offsets.ctypes.data
            views[i].validity = a.validity.ctypes.data if a.validity is not None else None
            views[i].len = a.length
            views[i].offset = a.offset
            views[i].null_count = a.null_count
            views[i].values = N.make_views([a.values])[0]
        h = C.c_void_p()
        N.raise_for_status(N.lib().bdf_list_upload(ctx.handle, dtype, len(arrays), views, 0, C.byref(h)))
        return cls(ctx, h)

    def describe(self):
        dt, n, total = C.c_int32(), C.c_int64(), C.c_int64()
        N.raise_for_status(N.lib().bdf_list_describe(self.handle, C.byref(dt), C.byref(n), C.byref(total)))
        return dt.value, n.value, total.value

    @property
    def dtype(self) -> int:
        return self.describe()[0]

    @property
    def n_chunks(self) -> int:
        return self.describe()[1]

    def __len__(self) -> int:
        return self.describe()[2]

    def chunk_info(self, i: int) -> dict:
        ln, nc, ne = C.c_int64(), C.c_int64(), C.c_int64()
        N.raise_for_status(N.lib().bdf_list_chunk_info(self.ctx.handle, self.handle, i, C.byref(ln), C.byref(nc), C.byref(ne)))
        return {"len": ln.value, "null_count": nc.value, "n_elements": ne.value}

    def values(self) -> "Column":
        """The elements as a Column (borrowed: valid while this list lives; freeing it does nothing)."""
        col = _BorrowedColumn(self.ctx, C.c_void_p(N.lib().bdf_list_values(self.handle)))
        col._owner = self
        return col

    def download(self) -> List:
        from .arrays import ListArray

        dtype, n, _ = self.describe()
        outs = (N.ListOut * max(n, 1))()
        keep = []
        for i in range(n):
            info = self.chunk_info(i)
            ln, ne = info["len"], info["n_elements"]
            off = np.zeros(ln + 1, dtype=np.int32)
            val = np.zeros((ln + 7) // 8 + 1, dtype=np.uint8)
            vals = np.zeros(ne, dtype=NP_DTYPES[dtype])
            vval = np.zeros((ne + 7) // 8 + 1, dtype=np.uint8)
            outs[i].offsets, outs[i].validity = off.ctypes.data, val.ctypes.data
            outs[i].values = vals.ctypes.data if ne else None
            outs[i].value_validity = vval.ctypes.data
            keep.append((off, val, vals, vval))
        N.raise_for_status(N.lib().bdf_list_download(self.ctx.handle, self.handle, outs))
        res = []
        for i, (off, val, vals, vval) in enumerate(keep):
            child = PrimitiveArray(dtype, vals, vval if outs[i].has_value_validity else None, 0, vals.shape[0],
                                   int(outs[i].value_null_count))
            res.append(ListArray(dtype, off, val if outs[i].has_validity else None, 0, off.shape[0] - 1, int(outs[i].null_count), child))
        return res

    # -- ArrayFunctions on the device --
    def _col(self, fn, *args) -> "Column":
        h = C.c_void_p()
        N.raise_for_status(fn(self.ctx.handle, *args, C.byref(h)))
        return Column(self.ctx, h)

    def _list(self, fn, *args) -> "ListColumn":
        h = C.c_void_p()
        N.raise_for_status(fn(self.ctx.handle, *args, C.byref(h)))
        return ListColumn(self.ctx, h)

    def array_contains(self, value) -> "Column":
        return self._col(N.lib().bdf_list_find_dev, N.LIST_CONTAINS, self.handle, _value_bits(self.dtype, value))

    def array_position(self, value) -> "Column":
        return self._col(N.lib().bdf_list_find_dev, N.LIST_POSITION, self.handle, _value_bits(self.dtype, value))

    def array_max(self) -> "Column":
        return self._col(N.lib().bdf_list_reduce_dev, N.LIST_MAX, self.handle)

    def array_min(self) -> "Column":
        return self._col(N.lib().bdf_list_reduce_dev, N.LIST_MIN, self.handle)

    def size(self) -> "Column":
        return self._col(N.lib().bdf_list_reduce_dev, N.LIST_SIZE, self.handle)

    def array_remove(self, value) -> "ListColumn":
        return self._list(N.lib().bdf_list_transform_dev, N.LIST_REMOVE, self.handle, _value_bits(self.dtype, value), 0)

    def array_sort(self) -> "ListColumn":
        return self._list(N.lib().bdf_list_transform_dev, N.LIST_SORT, self.handle, 0, 0)

    def array_distinct(self) -> "ListColumn":
        return self._list(N.lib().bdf_list_transform_dev, N.LIST_DISTINCT, self.handle, 0, 0)

    def array_repeat(self, count: int) -> "ListColumn":
        return self._list(N.lib().bdf_list_transform_dev, N.LIST_REPEAT, self.handle, 0, int(count))

    def array_except(self, other: "ListColumn") -> "ListColumn":
        return self._list(N.lib().bdf_list_set_dev, N.LIST_EXCEPT, self.handle, other.handle)

    def array_intersect(self, other: "ListColumn") -> "ListColumn":
        return self._list(N.lib().bdf_list_set_dev, N.LIST_INTERSECT, self.handle, other.handle)

    def array_union(self, other: "ListColumn") -> "ListColumn":
        return self._list(N.lib().bdf_list_set_dev, N.LIST_UNION, self.handle, other.handle)

    def take(self, indices: "Column") -> "ListColumn":
        """Column::take of whole lists: out[i] = self[indices[i]] (UInt32 row numbers through the chunks), one chunk; a null
        index gives a null list."""
        return self._list(N.lib().bdf_list_take_dev, self.handle, indices.handle)

    def filter(self, mask: "Column") -> "ListColumn":
        """ChunkedArray::filter of whole lists: the lists where the Boolean mask is valid and true, chunk by chunk."""
        return self._list(N.lib().bdf_list_filter_dev, self.handle, mask.handle)

    @staticmethod
    def concat(lists: Sequence["ListColumn"]) -> "ListColumn":
        """The chunks of lists[0], then those of lists[1], and so on, copied on the device (bdf_list_concat_dev); one element type."""
        lists = list(lists)
        if not lists:
            raise N.ComputeError("concat needs at least one list column")
        if len({l.dtype for l in lists}) != 1:
            raise N.UnsupportedType("Union can only be performed on tables with compatible column types")
        ctx = lists[0].ctx
        ls = (C.c_void_p * len(lists))(*[l.handle for l in lists])
        h = C.c_void_p()
        N.raise_for_status(N.lib().bdf_list_concat_dev(ctx.handle, len(lists), ls, C.byref(h)))
        return ListColumn(ctx, h)

    def explode(self):
        """(UInt32 parent row numbers, values): one row per element of every valid list; null and empty lists give none."""
        rows, vals = C.c_void_p(), C.c_void_p()
        N.raise_for_status(N.lib().bdf_list_explode_dev(self.ctx.handle, self.handle, C.byref(rows), C.byref(vals)))
        return Column(self.ctx, rows), Column(self.ctx, vals)

    def free(self):
        if self.handle is not None and self.ctx.handle:
            N.lib().bdf_list_free(self.ctx.handle, self.handle)
        self.handle = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class _BorrowedColumn(Column):
    """A Column whose memory belongs to a ListColumn."""

    def free(self):
        self.handle = None


def _as_list_column(x, ctx) -> ListColumn:
    return x if isinstance(x, ListColumn) else ListColumn.upload(list(x), ctx)


class ArrayFunctions:
    """ArrayFunctions (src/functions/array.rs) plus Spark's size / explode, one device call each.  Arguments are the column's
    ListArray chunks (or a ListColumn); list results come back as ListArray chunks, the others as PrimitiveArray /
    BooleanArray chunks."""

    @staticmethod
    def _run(arrays, ctx, fn):
        ctx = ctx or N.default_context()
        lc = _as_list_column(arrays, ctx)
        out = fn(lc)
        return out.download()

    @staticmethod
    def array_contains(arrays, value, ctx=None): return ArrayFunctions._run(arrays, ctx, lambda l: l.array_contains(value))

    @staticmethod
    def array_position(arrays, value, ctx=None): return ArrayFunctions._run(arrays, ctx, lambda l: l.array_position(value))

    @staticmethod
    def array_max(arrays, ctx=None): return ArrayFunctions._run(arrays, ctx, lambda l: l.array_max())

    @staticmethod
    def array_min(arrays, ctx=None): return ArrayFunctions._run(arrays, ctx, lambda l: l.array_min())

    @staticmethod
    def size(arrays, ctx=None): return ArrayFunctions._run(arrays, ctx, lambda l: l.size())

    @staticmethod
    def array_remove(arrays, value, ctx=None): return ArrayFunctions._run(arrays, ctx, lambda l: l.array_remove(value))

    @staticmethod
    def array_sort(arrays, ctx=None): return ArrayFunctions._run(arrays, ctx, lambda l: l.array_sort())

    @staticmethod
    def array_distinct(arrays, ctx=None): return ArrayFunctions._run(arrays, ctx, lambda l: l.array_distinct())

    @staticmethod
    def array_repeat(arrays, count: int, ctx=None): return ArrayFunctions._run(arrays, ctx, lambda l: l.array_repeat(count))

    @staticmethod
    def _set(a, b, ctx, name):
        ctx = ctx or N.default_context()
        la, lb = _as_list_column(a, ctx), _as_list_column(b, ctx)
        return getattr(la, name)(lb).download()

    @staticmethod
    def array_except(a, b, ctx=None): return ArrayFunctions._set(a, b, ctx, "array_except")

    @staticmethod
    def array_intersect(a, b, ctx=None): return ArrayFunctions._set(a, b, ctx, "array_intersect")

    @staticmethod
    def array_union(a, b, ctx=None): return ArrayFunctions._set(a, b, ctx, "array_union")

    @staticmethod
    def explode(arrays, ctx=None):
        ctx = ctx or N.default_context()
        rows, vals = _as_list_column(arrays, ctx).explode()
        return rows.download()[0], vals.download()[0]
