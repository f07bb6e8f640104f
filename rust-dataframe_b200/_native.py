"""ctypes binding of libb200df.so (include/b200df.h).  Loading fails loudly when the CUDA library has not
been built: there is no CPU or PyTorch fallback anywhere in this package."""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional, Sequence

import numpy as np

from .arrays import NP_DTYPES, PrimitiveArray, width_of

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libb200df.so")

# enums (must match include/b200df.h)
ADD, SUB, MUL, DIV, ATAN2, HYPOT, LOG = range(7)
(ABS, SIN, COS, TAN, ACOS, ASIN, ATAN, CBRT, CEIL, COSH, DEGREES, EXP, EXPM1, FLOOR, LOG10, LOG2, RADIANS, ROUND, SINH,
 SQRT, TANH) = range(21)
SUM, MIN, MAX, COUNT = range(4)
OK, LENGTH_MISMATCH, DIVIDE_BY_ZERO, UNSUPPORTED, CUDA, NCCL, OOM, WOULD_PANIC, INVALID, PARSE = range(10)
ASYNC = 1
(K_BINARY, K_UNARY, K_CAST, K_REDUCE, K_GENERATE, K_AVG, K_COMPARE, K_FILTER, K_EXPR, K_SORT, K_TAKE, K_GROUP, K_JOIN, K_CSV, K_WINDOW,
 K_MOMENTS, K_CSV_WRITE, K_LIST, K_TEMPORAL, K_JSON, K_PARQUET) = range(21)
KERNEL_NAMES = ["binary", "unary", "cast", "reduce", "generate", "avg", "compare", "filter", "expr", "sort", "take", "group", "join", "csv",
                "window", "moments", "csv_write", "list", "temporal", "json", "parquet", "parquet_write", "select", "hist"]
K_SELECT, K_HIST = 22, 23
K_JSON_WRITE = 24   # BDF_K_JSON_WRITE, the id that follows the bdf_kernel_id enum
# KERNEL_NAMES mirrors the bdf_kernel_id enum; the ids after it (include/b200df.h) extend it for the launch records
LAUNCH_KERNEL_NAMES = KERNEL_NAMES + ["json_write"]
EXPR_UNARY = 100
GT, GE, EQ, NE, LT, LE = range(6)
AND, OR, NOT = range(3)
# null handling and conditional selection (bdf_row_fn, bdf_null_test)
ROW_COALESCE, ROW_GREATEST, ROW_LEAST, ROW_NANVL = range(4)
IS_NULL, IS_NOT_NULL, IS_NAN = range(3)
BOOL = 10
UTF8 = 11   # CSV schema entry only: a string column the device skips
# bdf_group_fn (AggregateFunction order)
(GROUP_SUM, GROUP_MAX, GROUP_MIN, GROUP_AVG, GROUP_COUNT, GROUP_COUNT_DISTINCT, GROUP_FIRST, GROUP_LAST, GROUP_KURTOSIS, GROUP_SKEWNESS,
 GROUP_STDDEV, GROUP_SUM_DISTINCT, GROUP_VARIANCE, GROUP_STDDEV_POP, GROUP_VAR_POP) = range(15)
GROUP_MEDIAN, GROUP_MODE = 32, 33   # the distributions: a block of their own (not AggregateFunction members)
GROUP_FNS = {"sum": GROUP_SUM, "max": GROUP_MAX, "min": GROUP_MIN, "avg": GROUP_AVG, "count": GROUP_COUNT,
             "count_distinct": GROUP_COUNT_DISTINCT, "first": GROUP_FIRST, "last": GROUP_LAST, "kurtosis": GROUP_KURTOSIS,
             "skewness": GROUP_SKEWNESS, "stddev": GROUP_STDDEV, "sum_distinct": GROUP_SUM_DISTINCT, "variance": GROUP_VARIANCE,
             "stddev_pop": GROUP_STDDEV_POP, "var_pop": GROUP_VAR_POP, "exact_median": GROUP_MEDIAN,
             "mode": GROUP_MODE}
GROUP_COLLECT_LIST, GROUP_COLLECT_SET = 48, 49   # the list builders: bdf_group_by_lists_dev only
COLLECT_FNS = {"collect_list": GROUP_COLLECT_LIST, "collect_set": GROUP_COLLECT_SET}
# bdf_stat
STAT_VARIANCE, STAT_VAR_POP, STAT_STDDEV, STAT_STDDEV_POP, STAT_SKEWNESS, STAT_KURTOSIS = range(6)
STATS = {"variance": STAT_VARIANCE, "var_pop": STAT_VAR_POP, "stddev": STAT_STDDEV, "stddev_pop": STAT_STDDEV_POP,
         "skewness": STAT_SKEWNESS, "kurtosis": STAT_KURTOSIS}
# bdf_join_type (JoinType order)
JOIN_LEFT, JOIN_RIGHT, JOIN_INNER, JOIN_FULL, JOIN_LEFT_SEMI, JOIN_LEFT_ANTI = range(6)
JOIN_TYPES = {"left": JOIN_LEFT, "right": JOIN_RIGHT, "inner": JOIN_INNER, "full": JOIN_FULL, "left_semi": JOIN_LEFT_SEMI,
              "left_anti": JOIN_LEFT_ANTI}
# bdf_asof_direction
ASOF_BACKWARD, ASOF_FORWARD, ASOF_NEAREST = range(3)
ASOF_DIRECTIONS = {"backward": ASOF_BACKWARD, "forward": ASOF_FORWARD, "nearest": ASOF_NEAREST}
# bdf_keep / bdf_setop
KEEP_FIRST, KEEP_LAST, KEEP_NONE = range(3)
SETOP_INTERSECT, SETOP_INTERSECT_ALL, SETOP_EXCEPT, SETOP_EXCEPT_ALL = range(4)
SET_OPS = {"intersect": SETOP_INTERSECT, "intersect_all": SETOP_INTERSECT_ALL, "except": SETOP_EXCEPT, "except_all": SETOP_EXCEPT_ALL}
# bdf_window_fn / bdf_window_frame
(WIN_ROW_NUMBER, WIN_RANK, WIN_DENSE_RANK, WIN_PERCENT_RANK, WIN_CUME_DIST, WIN_LAG, WIN_LEAD, WIN_SUM, WIN_COUNT, WIN_MIN, WIN_MAX,
 WIN_AVG, WIN_FIRST_VALUE, WIN_LAST_VALUE, WIN_NTH_VALUE) = range(15)
WINDOW_FNS = {"row_number": WIN_ROW_NUMBER, "rank": WIN_RANK, "dense_rank": WIN_DENSE_RANK, "percent_rank": WIN_PERCENT_RANK,
              "cume_dist": WIN_CUME_DIST, "lag": WIN_LAG, "lead": WIN_LEAD, "sum": WIN_SUM, "count": WIN_COUNT, "min": WIN_MIN,
              "max": WIN_MAX, "avg": WIN_AVG, "first_value": WIN_FIRST_VALUE, "last_value": WIN_LAST_VALUE, "nth_value": WIN_NTH_VALUE}
FRAME_ROWS, FRAME_RANGE, FRAME_PARTITION, FRAME_ROWS_BETWEEN, FRAME_RANGE_BETWEEN = range(5)
BOUNDED_FRAMES = {"rows": FRAME_ROWS_BETWEEN, "range": FRAME_RANGE_BETWEEN}   # ("rows" | "range", start, end) frames
WINDOW_FRAMES = {"rows": FRAME_ROWS, "range": FRAME_RANGE, "partition": FRAME_PARTITION}
# list columns (bdf_list_*)
LIST_BASE = 32
LIST_CONTAINS, LIST_POSITION = range(2)
LIST_MAX, LIST_MIN, LIST_SIZE = range(3)
LIST_REMOVE, LIST_SORT, LIST_DISTINCT, LIST_REPEAT = range(4)
LIST_EXCEPT, LIST_INTERSECT, LIST_UNION = range(3)
# dates and timestamps (bdf_temporal_*)
TEMPORAL_NONE, DATE32, DATE64, TIMESTAMP, TIME32, TIME64 = range(6)
SECOND, MILLISECOND, MICROSECOND, NANOSECOND = range(4)
(T_YEAR, T_QUARTER, T_MONTH, T_DAY_OF_MONTH, T_DAY_OF_YEAR, T_DAY_OF_WEEK, T_HOUR, T_MINUTE, T_SECOND, T_TO_DATE, T_DATE_ADD, T_DATE_SUB,
 T_ADD_MONTHS, T_LAST_DAY, T_NEXT_DAY, T_DATE_TRUNC, T_UNIX_TIMESTAMP, T_TO_TIMESTAMP) = range(18)
TEMPORAL_FNS = {"year": T_YEAR, "quarter": T_QUARTER, "month": T_MONTH, "day_of_month": T_DAY_OF_MONTH, "day_of_year": T_DAY_OF_YEAR,
                "day_of_week": T_DAY_OF_WEEK, "hour": T_HOUR, "minute": T_MINUTE, "second": T_SECOND, "to_date": T_TO_DATE,
                "date_add": T_DATE_ADD, "date_sub": T_DATE_SUB, "add_months": T_ADD_MONTHS, "last_day": T_LAST_DAY, "next_day": T_NEXT_DAY,
                "date_trunc": T_DATE_TRUNC, "unix_timestamp": T_UNIX_TIMESTAMP, "to_timestamp": T_TO_TIMESTAMP}
T_DATE_DIFF, T_MONTHS_BETWEEN = range(2)
TRUNC_UNITS = {"year": 0, "quarter": 1, "month": 2, "week": 3, "day": 4, "hour": 5, "minute": 6, "second": 7}
TIME_UNITS = {"s": SECOND, "ms": MILLISECOND, "us": MICROSECOND, "ns": NANOSECOND}


class View(C.Structure):
    _fields_ = [("values", C.c_void_p), ("validity", C.c_void_p), ("len", C.c_int64), ("offset", C.c_int64),
                ("null_count", C.c_int64)]


class Out(C.Structure):
    _fields_ = [("values", C.c_void_p), ("validity", C.c_void_p), ("len", C.c_int64), ("null_count", C.c_int64),
                ("has_validity", C.c_int32)]


class Agg4(C.Structure):
    _fields_ = [("sum", C.c_uint64), ("min", C.c_uint64), ("max", C.c_uint64), ("count", C.c_int64),
                ("rows", C.c_int64), ("any_valid", C.c_int32), ("would_panic", C.c_int32), ("n_chunks", C.c_int64)]


class MomentRec(C.Structure):
    _fields_ = [("count", C.c_int64), ("mean", C.c_double), ("m2", C.c_double), ("m3", C.c_double), ("m4", C.c_double)]


class DistinctRec(C.Structure):
    _fields_ = [("count", C.c_int64), ("sum", C.c_uint64)]


class ExprNode(C.Structure):
    _fields_ = [("op", C.c_int32), ("a", C.c_int32), ("b", C.c_int32)]


class Arg(C.Structure):
    """bdf_arg: a column (column != NULL) or a scalar's T::Native bits; valid == 0 is a NULL literal."""
    _fields_ = [("column", C.c_void_p), ("bits", C.c_uint64), ("valid", C.c_int32)]


class SortKeyC(C.Structure):
    _fields_ = [("column", C.c_void_p), ("descending", C.c_int32)]


class GroupOut(C.Structure):
    _fields_ = [("sum", C.c_void_p), ("count", C.c_void_p), ("min", C.c_void_p), ("max", C.c_void_p)]


class GroupAggC(C.Structure):
    _fields_ = [("column", C.c_void_p), ("function", C.c_int32)]


class WindowCall(C.Structure):
    _fields_ = [("function", C.c_int32), ("frame", C.c_int32), ("column", C.c_void_p), ("offset", C.c_int64), ("default_bits", C.c_uint64),
                ("has_default", C.c_int32), ("ignore_nulls", C.c_int32), ("start", C.c_int64), ("end", C.c_int64), ("start_f", C.c_double),
                ("end_f", C.c_double)]


class AsofSpec(C.Structure):
    _fields_ = [("direction", C.c_int32), ("allow_exact_matches", C.c_int32), ("has_tolerance", C.c_int32), ("tolerance", C.c_int64),
                ("tolerance_f", C.c_double)]


class TemporalTypeC(C.Structure):
    _fields_ = [("kind", C.c_int32), ("unit", C.c_int32), ("tz", C.c_char_p)]


class ListView(C.Structure):
    _fields_ = [("offsets", C.c_void_p), ("validity", C.c_void_p), ("len", C.c_int64), ("offset", C.c_int64), ("null_count", C.c_int64),
                ("values", View)]


class ListOut(C.Structure):
    _fields_ = [("offsets", C.c_void_p), ("validity", C.c_void_p), ("values", C.c_void_p), ("value_validity", C.c_void_p),
                ("null_count", C.c_int64), ("value_null_count", C.c_int64), ("has_validity", C.c_int32), ("has_value_validity", C.c_int32)]


class JsonOptions(C.Structure):
    _fields_ = [("max_records", C.c_int64), ("batch_size", C.c_int64)]


class ParquetOptions(C.Structure):
    _fields_ = [("batch_size", C.c_int64)]


class ParquetWriteOptions(C.Structure):
    _fields_ = [("compression", C.c_int32), ("dictionary", C.c_int32), ("row_group_rows", C.c_int64)]


class CsvOptions(C.Structure):
    _fields_ = [("has_header", C.c_int32), ("delimiter", C.c_uint8), ("max_records", C.c_int64), ("batch_size", C.c_int64)]


class CsvWriteOptions(C.Structure):
    _fields_ = [("has_header", C.c_int32), ("delimiter", C.c_uint8)]


class JsonWriteOptions(C.Structure):
    _fields_ = [("explicit_nulls", C.c_int32)]


class LaunchRecord(C.Structure):
    _fields_ = [("kernel", C.c_int32), ("dtype", C.c_int32), ("rows", C.c_int64), ("bytes", C.c_int64),
                ("ms", C.c_float)]


class ArrowError(Exception):
    """arrow::error::ArrowError as surfaced by the reference API."""


class ComputeError(ArrowError):
    pass


class DivideByZero(ArrowError):
    def __init__(self, msg="Divide by zero error"):
        super().__init__(msg)


class ParseError(ArrowError):
    """ArrowError::ParseError: a CSV value does not parse as its column's type."""


class UnsupportedType(ArrowError):
    """A trait bound the reference enforces at compile time (T::Native: Float / Signed / Ord ...)."""


class ReferencePanic(RuntimeError):
    """The reference panics on this input (e.g. max() .unwrap() on an all-null chunk, aggregate.rs:19)."""


_lib: Optional[C.CDLL] = None


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'`. "
            "rust-dataframe_b200 has no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    P = C.POINTER
    vp, i32, i64, u64 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64
    sig = {
        "bdf_abi_version": ([], C.c_int),
        "bdf_last_error": ([], C.c_char_p),
        "bdf_init": ([C.c_int, P(vp)], C.c_int),
        "bdf_init_multi": ([C.c_int, P(C.c_int), P(vp)], C.c_int),
        "bdf_fleet_size": ([vp], C.c_int),
        "bdf_destroy": ([vp], None),
        "bdf_synchronize": ([vp], C.c_int),
        "bdf_device_info": ([vp, P(i32), P(i32), P(i32), P(i64)], C.c_int),
        "bdf_comm_unique_id": ([P(C.c_uint8)], C.c_int),
        "bdf_comm_attach": ([vp, P(C.c_uint8), C.c_int, C.c_int], C.c_int),
        "bdf_comm_detach": ([vp], C.c_int),
        "bdf_comm_info": ([vp, P(i32), P(i32), P(i32), P(i64)], C.c_int),
        "bdf_comm_collective": ([vp, C.c_int], C.c_int),
        "bdf_comm_barrier": ([vp], C.c_int),
        "bdf_comm_set_combine": ([vp, C.c_int], C.c_int),
        "bdf_comm_get_combine": ([vp], C.c_int),
        "bdf_comm_all_reduce_f64": ([vp, C.c_int, i64, P(C.c_double)], C.c_int),
        "bdf_aggregate_all_many_dev": ([vp, i32, P(vp), P(Agg4)], C.c_int),
        "bdf_aggregate_all_many_dev_async": ([vp, i32, P(vp), P(vp)], C.c_int),
        "bdf_future_count": ([vp], C.c_int),
        "bdf_host_alloc": ([vp, C.c_size_t, P(vp)], C.c_int),
        "bdf_host_free": ([vp, vp], C.c_int),
        "bdf_host_register": ([vp, vp, C.c_size_t], C.c_int),
        "bdf_host_unregister": ([vp, vp], C.c_int),
        "bdf_binary": ([vp, C.c_int, C.c_int, i64, P(View), i64, P(View), P(Out)], C.c_int),
        "bdf_unary": ([vp, C.c_int, C.c_int, i64, P(View), P(Out)], C.c_int),
        "bdf_cast": ([vp, C.c_int, C.c_int, i64, P(View), P(Out)], C.c_int),
        "bdf_aggregate": ([vp, C.c_int, C.c_int, i64, P(View), vp, P(i32)], C.c_int),
        "bdf_aggregate_all": ([vp, C.c_int, i64, P(View), P(Agg4)], C.c_int),
        "bdf_avg": ([vp, C.c_int, i64, P(View), P(C.c_double), P(i32)], C.c_int),
        "bdf_upload": ([vp, C.c_int, i64, P(View), C.c_int, P(vp)], C.c_int),
        "bdf_upload_many": ([vp, i64, P(i32), P(i64), P(P(View)), C.c_int, P(vp)], C.c_int),
        "bdf_col_wait": ([vp, vp], C.c_int),
        "bdf_col_describe": ([vp, P(i32), P(i64), P(i64)], C.c_int),
        "bdf_col_chunk_info": ([vp, vp, i64, P(i64), P(i64), P(i32)], C.c_int),
        "bdf_binary_dev": ([vp, C.c_int, vp, vp, P(vp)], C.c_int),
        "bdf_unary_dev": ([vp, C.c_int, vp, P(vp)], C.c_int),
        "bdf_cast_dev": ([vp, C.c_int, vp, P(vp)], C.c_int),
        "bdf_aggregate_dev": ([vp, C.c_int, vp, vp, P(i32)], C.c_int),
        "bdf_aggregate_all_dev": ([vp, vp, P(Agg4)], C.c_int),
        "bdf_avg_dev": ([vp, vp, P(C.c_double), P(i32)], C.c_int),
        "bdf_moments": ([vp, C.c_int, i64, P(View), P(MomentRec)], C.c_int),
        "bdf_moments_dev": ([vp, vp, P(MomentRec)], C.c_int),
        "bdf_moments_stat": ([P(MomentRec), C.c_int, P(C.c_double), P(i32)], C.c_int),
        "bdf_moments_merge": ([P(MomentRec), P(MomentRec), P(MomentRec)], C.c_int),
        "bdf_distinct": ([vp, C.c_int, i64, P(View), P(DistinctRec)], C.c_int),
        "bdf_distinct_dev": ([vp, vp, P(DistinctRec)], C.c_int),
        "bdf_percentile": ([vp, C.c_int, i64, P(View), i32, P(C.c_double), P(C.c_double), P(i32)], C.c_int),
        "bdf_percentile_dev": ([vp, vp, i32, P(C.c_double), P(C.c_double), P(i32)], C.c_int),
        "bdf_mode": ([vp, C.c_int, i64, P(View), P(u64), P(i64), P(i32)], C.c_int),
        "bdf_mode_dev": ([vp, vp, P(u64), P(i64), P(i32)], C.c_int),
        "bdf_uniques_dev": ([vp, vp, P(vp), P(vp)], C.c_int),
        "bdf_hist_dev": ([vp, vp, i32, P(C.c_double), P(C.c_double), P(i64)], C.c_int),
        "bdf_hist_density": ([i32, P(C.c_double), P(i64), P(C.c_double)], C.c_int),
        "bdf_expr_check": ([i32, P(i32), i32, P(ExprNode), P(i32), P(i32)], C.c_int),
        "bdf_eval_expr_dev": ([vp, i32, P(vp), i32, P(ExprNode), P(vp)], C.c_int),
        "bdf_eval_expr_agg_dev": ([vp, i32, P(vp), i32, P(ExprNode), P(vp), P(Agg4)], C.c_int),
        "bdf_eval_expr_agg_dev_async": ([vp, i32, P(vp), i32, P(ExprNode), P(vp), P(vp)], C.c_int),
        "bdf_sort_indices_dev": ([vp, i32, P(SortKeyC), P(vp)], C.c_int),
        "bdf_top_k_indices_dev": ([vp, i32, P(SortKeyC), i64, P(vp)], C.c_int),
        "bdf_take_dev": ([vp, vp, vp, P(vp)], C.c_int),
        "bdf_group_aggregate_dev": ([vp, vp, i32, P(vp), P(vp), P(GroupOut), P(i64)], C.c_int),
        "bdf_group_by_dev": ([vp, i32, P(vp), i32, P(GroupAggC), P(vp), P(vp), P(i64)], C.c_int),
        "bdf_group_by_lists_dev": ([vp, i32, P(vp), i32, P(GroupAggC), P(vp), P(vp), P(vp), P(i64)], C.c_int),
        "bdf_join_indices_dev": ([vp, i32, i32, P(vp), P(vp), P(vp), P(vp), P(i64)], C.c_int),
        "bdf_join_asof_dev": ([vp, vp, vp, i32, P(vp), P(vp), P(AsofSpec), P(vp)], C.c_int),
        "bdf_duplicated_dev": ([vp, i32, P(vp), i32, P(vp)], C.c_int),
        "bdf_set_op_dev": ([vp, i32, i32, P(vp), P(vp), P(vp)], C.c_int),
        "bdf_concat_dev": ([vp, i32, P(vp), P(vp)], C.c_int),
        "bdf_list_concat_dev": ([vp, i32, P(vp), P(vp)], C.c_int),
        "bdf_bool_widen_dev": ([vp, vp, P(vp)], C.c_int),
        "bdf_window_dev": ([vp, i32, P(vp), i32, P(SortKeyC), i32, P(WindowCall), P(vp)], C.c_int),
        "bdf_compare_dev": ([vp, C.c_int, vp, vp, C.c_double, P(vp)], C.c_int),
        "bdf_boolean_dev": ([vp, C.c_int, vp, vp, P(vp)], C.c_int),
        "bdf_filter_dev": ([vp, vp, vp, P(vp)], C.c_int),
        "bdf_rowwise_dev": ([vp, C.c_int, i32, P(Arg), P(vp)], C.c_int),
        "bdf_case_when_dev": ([vp, i32, P(vp), P(Arg), P(vp)], C.c_int),
        "bdf_null_test_dev": ([vp, C.c_int, vp, P(vp)], C.c_int),
        "bdf_download": ([vp, vp, P(Out)], C.c_int),
        "bdf_download_begin": ([vp, vp, P(Out)], C.c_int),
        "bdf_download_end": ([vp, vp, P(Out)], C.c_int),
        "bdf_binary_agg_dev": ([vp, C.c_int, vp, vp, P(vp), P(Agg4)], C.c_int),
        "bdf_binary_agg_dev_async": ([vp, C.c_int, vp, vp, P(vp), P(vp)], C.c_int),
        "bdf_aggregate_all_dev_async": ([vp, vp, P(vp)], C.c_int),
        "bdf_future_wait": ([vp, vp, P(Agg4)], C.c_int),
        "bdf_col_free": ([vp, vp], None),
        "bdf_profile_enable": ([vp, C.c_int], C.c_int),
        "bdf_profile_read": ([vp, P(LaunchRecord), i64, P(i64)], C.c_int),
        "bdf_launch_count": ([vp], i64),
        "bdf_timer_start": ([vp], C.c_int),
        "bdf_timer_stop": ([vp, P(C.c_float)], C.c_int),
        "bdf_flush_l2": ([vp, C.c_size_t], C.c_int),
        "bdf_ipc_open": ([C.c_char_p, P(vp)], C.c_int),
        "bdf_ipc_close": ([vp], None),
        "bdf_ipc_describe": ([vp, P(i32), P(i64), P(i64)], C.c_int),
        "bdf_ipc_column": ([vp, i32, P(C.c_char_p), P(i32), P(i32)], C.c_int),
        "bdf_ipc_batch_rows": ([vp, i64, P(i64)], C.c_int),
        "bdf_ipc_view": ([vp, i64, i32, P(View)], C.c_int),
        "bdf_ipc_read": ([vp, vp, i32, P(i32), C.c_int, P(vp)], C.c_int),
        "bdf_ipc_read_batches": ([vp, vp, i32, P(i32), i64, P(i64), C.c_int, P(vp)], C.c_int),
        "bdf_ipc_write_host": ([C.c_char_p, i32, P(C.c_char_p), P(i32), i64, P(P(View))], C.c_int),
        "bdf_ipc_write": ([vp, C.c_char_p, i32, P(C.c_char_p), P(vp)], C.c_int),
        "bdf_csv_open": ([vp, C.c_char_p, P(CsvOptions), i32, P(i32), P(vp)], C.c_int),
        "bdf_csv_describe": ([vp, P(i32), P(i64), P(i64)], C.c_int),
        "bdf_csv_column": ([vp, i32, P(C.c_char_p), P(i32), P(i32)], C.c_int),
        "bdf_csv_read": ([vp, vp, i32, P(i32), P(vp)], C.c_int),
        "bdf_csv_stats": ([vp, P(i64), P(i64), P(C.c_double)], C.c_int),
        "bdf_csv_close": ([vp, vp], None),
        "bdf_csv_write": ([vp, C.c_char_p, i32, P(C.c_char_p), P(vp), P(CsvWriteOptions)], C.c_int),
        "bdf_json_open": ([vp, C.c_char_p, P(JsonOptions), i32, P(C.c_char_p), P(i32), P(vp)], C.c_int),
        "bdf_json_describe": ([vp, P(i32), P(i64), P(i64)], C.c_int),
        "bdf_json_column": ([vp, i32, P(C.c_char_p), P(i32), P(i32)], C.c_int),
        "bdf_json_read": ([vp, vp, i32, P(i32), P(vp)], C.c_int),
        "bdf_json_read_list": ([vp, vp, i32, P(vp)], C.c_int),
        "bdf_json_stats": ([vp, P(i64), P(i64), P(C.c_double)], C.c_int),
        "bdf_json_close": ([vp, vp], None),
        "bdf_parquet_open": ([C.c_char_p, P(ParquetOptions), P(vp)], C.c_int),
        "bdf_parquet_describe": ([vp, P(i32), P(i64), P(i64)], C.c_int),
        "bdf_parquet_column": ([vp, i32, P(C.c_char_p), P(i32), P(i32)], C.c_int),
        "bdf_parquet_temporal_column": ([vp, i32, P(TemporalTypeC)], C.c_int),
        "bdf_parquet_check": ([vp, i32], C.c_int),
        "bdf_parquet_read": ([vp, vp, i32, P(i32), P(vp)], C.c_int),
        "bdf_parquet_stats": ([vp, P(i64), P(i64), P(C.c_double)], C.c_int),
        "bdf_parquet_close": ([vp], None),
        "bdf_parquet_write": ([vp, C.c_char_p, i32, P(C.c_char_p), P(vp), P(TemporalTypeC), P(ParquetWriteOptions)], C.c_int),
        "bdf_generate": ([vp, C.c_int, C.c_int, C.c_double, C.c_double, u64, u64, i64, P(i64), i64, C.c_uint32, P(vp)],
                         C.c_int),
        "bdf_list_upload": ([vp, C.c_int, i64, P(ListView), C.c_int, P(vp)], C.c_int),
        "bdf_list_describe": ([vp, P(i32), P(i64), P(i64)], C.c_int),
        "bdf_list_chunk_info": ([vp, vp, i64, P(i64), P(i64), P(i64)], C.c_int),
        "bdf_list_download": ([vp, vp, P(ListOut)], C.c_int),
        "bdf_list_values": ([vp], vp),
        "bdf_list_free": ([vp, vp], None),
        "bdf_list_find_dev": ([vp, C.c_int, vp, u64, P(vp)], C.c_int),
        "bdf_list_reduce_dev": ([vp, C.c_int, vp, P(vp)], C.c_int),
        "bdf_list_transform_dev": ([vp, C.c_int, vp, u64, i64, P(vp)], C.c_int),
        "bdf_list_set_dev": ([vp, C.c_int, vp, vp, P(vp)], C.c_int),
        "bdf_list_explode_dev": ([vp, vp, P(vp), P(vp)], C.c_int),
        "bdf_list_take_dev": ([vp, vp, vp, P(vp)], C.c_int),
        "bdf_list_filter_dev": ([vp, vp, vp, P(vp)], C.c_int),
        "bdf_ipc_list_column": ([vp, i32, P(i32)], C.c_int),
        "bdf_ipc_read_list": ([vp, vp, i32, C.c_int, P(vp)], C.c_int),
        "bdf_temporal": ([vp, C.c_int, P(TemporalTypeC), i64, i64, P(View), P(Out)], C.c_int),
        "bdf_temporal_dev": ([vp, C.c_int, P(TemporalTypeC), i64, vp, P(vp)], C.c_int),
        "bdf_temporal_binary_dev": ([vp, C.c_int, P(TemporalTypeC), vp, P(TemporalTypeC), vp, P(vp)], C.c_int),
        "bdf_temporal_result": ([C.c_int, P(TemporalTypeC), i64, P(i32), P(TemporalTypeC)], C.c_int),
        "bdf_ipc_temporal_column": ([vp, i32, P(TemporalTypeC)], C.c_int),
        "bdf_ipc_read_temporal": ([vp, vp, i32, C.c_int, P(vp)], C.c_int),
        "bdf_ipc_write_typed": ([vp, C.c_char_p, i32, P(C.c_char_p), P(vp), P(TemporalTypeC)], C.c_int),
        "bdf_ipc_write_lists": ([vp, C.c_char_p, i32, P(C.c_char_p), P(vp), P(TemporalTypeC), P(vp)], C.c_int),
        "bdf_json_write": ([vp, C.c_char_p, i32, P(C.c_char_p), P(vp), P(TemporalTypeC), P(vp), P(JsonWriteOptions)], C.c_int),
    }
    for name, (args, res) in sig.items():
        fn = getattr(L, name)  # AttributeError if the library does not export a declared symbol
        fn.argtypes = args
        fn.restype = res
    if L.bdf_abi_version() != 3:
        raise RuntimeError("libb200df.so ABI version mismatch")
    _lib = L
    return L


EXPORTED_SYMBOLS = [
    "bdf_abi_version", "bdf_last_error", "bdf_init", "bdf_init_multi", "bdf_fleet_size", "bdf_destroy", "bdf_synchronize", "bdf_device_info",
    "bdf_comm_unique_id", "bdf_comm_attach", "bdf_comm_detach", "bdf_comm_info", "bdf_comm_collective", "bdf_comm_barrier", "bdf_comm_set_combine", "bdf_comm_get_combine",
    "bdf_comm_all_reduce_f64", "bdf_aggregate_all_many_dev", "bdf_aggregate_all_many_dev_async", "bdf_future_count",
    "bdf_host_alloc", "bdf_host_free", "bdf_host_register", "bdf_host_unregister", "bdf_binary", "bdf_unary", "bdf_cast",
    "bdf_aggregate", "bdf_aggregate_all", "bdf_avg", "bdf_upload", "bdf_upload_many", "bdf_col_wait", "bdf_col_describe",
    "bdf_col_chunk_info", "bdf_binary_dev", "bdf_unary_dev", "bdf_cast_dev", "bdf_aggregate_dev",
    "bdf_aggregate_all_dev", "bdf_avg_dev", "bdf_expr_check", "bdf_eval_expr_dev", "bdf_eval_expr_agg_dev", "bdf_eval_expr_agg_dev_async", "bdf_sort_indices_dev", "bdf_top_k_indices_dev", "bdf_take_dev", "bdf_group_aggregate_dev", "bdf_group_by_dev", "bdf_group_by_lists_dev", "bdf_join_indices_dev", "bdf_join_asof_dev", "bdf_duplicated_dev", "bdf_set_op_dev", "bdf_concat_dev", "bdf_list_concat_dev", "bdf_bool_widen_dev", "bdf_window_dev", "bdf_compare_dev", "bdf_boolean_dev", "bdf_filter_dev", "bdf_rowwise_dev", "bdf_case_when_dev", "bdf_null_test_dev", "bdf_download", "bdf_download_begin", "bdf_download_end",
    "bdf_binary_agg_dev", "bdf_binary_agg_dev_async", "bdf_aggregate_all_dev_async", "bdf_future_wait", "bdf_col_free", "bdf_profile_enable", "bdf_profile_read",
    "bdf_launch_count", "bdf_timer_start", "bdf_timer_stop", "bdf_flush_l2", "bdf_generate",
    "bdf_ipc_open", "bdf_ipc_close", "bdf_ipc_describe", "bdf_ipc_column", "bdf_ipc_batch_rows", "bdf_ipc_view", "bdf_ipc_read", "bdf_ipc_read_batches",
    "bdf_ipc_write_host", "bdf_ipc_write",
    "bdf_csv_open", "bdf_csv_describe", "bdf_csv_column", "bdf_csv_read", "bdf_csv_stats", "bdf_csv_close", "bdf_csv_write",
    "bdf_json_open", "bdf_json_describe", "bdf_json_column", "bdf_json_read", "bdf_json_read_list", "bdf_json_stats", "bdf_json_close", "bdf_json_write",
    "bdf_moments", "bdf_moments_dev", "bdf_moments_stat", "bdf_moments_merge", "bdf_distinct", "bdf_distinct_dev",
    "bdf_list_upload", "bdf_list_describe", "bdf_list_chunk_info", "bdf_list_download", "bdf_list_values", "bdf_list_free",
    "bdf_list_find_dev", "bdf_list_reduce_dev", "bdf_list_transform_dev", "bdf_list_set_dev", "bdf_list_explode_dev",
    "bdf_list_take_dev", "bdf_list_filter_dev",
    "bdf_ipc_list_column", "bdf_ipc_read_list",
    "bdf_temporal", "bdf_temporal_dev", "bdf_temporal_binary_dev", "bdf_temporal_result", "bdf_ipc_temporal_column", "bdf_ipc_read_temporal",
    "bdf_ipc_write_typed", "bdf_ipc_write_lists",
    "bdf_parquet_open", "bdf_parquet_describe", "bdf_parquet_column", "bdf_parquet_temporal_column", "bdf_parquet_check", "bdf_parquet_read",
    "bdf_parquet_stats", "bdf_parquet_close", "bdf_parquet_write",
    "bdf_percentile", "bdf_percentile_dev", "bdf_mode", "bdf_mode_dev", "bdf_uniques_dev", "bdf_hist_dev", "bdf_hist_density",
]


def raise_for_status(st: int) -> None:
    if st == OK:
        return
    msg = (lib().bdf_last_error() or b"").decode("utf-8", "replace")
    if st == LENGTH_MISMATCH:
        raise ComputeError("Cannot perform math operation on arrays of different length")
    if st == DIVIDE_BY_ZERO:
        raise DivideByZero()
    if st == UNSUPPORTED:
        raise UnsupportedType(msg)
    if st == WOULD_PANIC:
        raise ReferencePanic(msg)
    if st == OOM:
        raise MemoryError(msg)
    if st == PARSE:
        raise ParseError(msg)
    raise ComputeError(f"[bdf status {st}] {msg}")


def make_views(chunks: Sequence[PrimitiveArray]):
    arr = (View * max(len(chunks), 1))()
    for i, c in enumerate(chunks):
        arr[i].values = c.values.ctypes.data if c.values.size else None
        arr[i].validity = c.validity.ctypes.data if c.validity is not None else None
        arr[i].len = c.length
        arr[i].offset = c.offset
        arr[i].null_count = c.null_count
    return arr


class PinnedBuffer:
    """cudaHostAlloc'ed bytes exposed as numpy arrays (freed with the object)."""

    def __init__(self, ctx: "Context", nbytes: int):
        self._ctx = ctx
        self.nbytes = int(nbytes)
        p = C.c_void_p()
        raise_for_status(lib().bdf_host_alloc(ctx.handle, max(self.nbytes, 1), C.byref(p)))
        self.ptr = p.value
        self._raw = (C.c_uint8 * max(self.nbytes, 1)).from_address(self.ptr)

    def array(self, dtype, count: int, byte_offset: int = 0) -> np.ndarray:
        a = np.frombuffer(self._raw, dtype=dtype, count=count, offset=byte_offset)
        return a

    def close(self):
        if self.ptr and self._ctx.handle:
            lib().bdf_host_free(self._ctx.handle, C.c_void_p(self.ptr))
        self.ptr = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Context:
    """One bdf_ctx = one GPU.  One process drives one GPU (torchrun gives each rank its LOCAL_RANK)."""

    def __init__(self, device: Optional[int] = None):
        if device is None:
            device = int(os.environ.get("LOCAL_RANK", "0"))
        h = C.c_void_p()
        raise_for_status(lib().bdf_init(int(device), C.byref(h)))
        self.handle = h
        self.device = int(device)

    @classmethod
    def multi(cls, n_gpus: int = 0, devices: Optional[Sequence[int]] = None) -> "Context":
        """ONE context over several GPUs of the box (bdf_init_multi; 0 = all visible): the library shards every call by
        row range, each GPU works over its own PCIe link, aggregates are combined by the grouped ncclAllReduce."""
        self = cls.__new__(cls)
        h = C.c_void_p()
        devs = (C.c_int * len(devices))(*devices) if devices else None
        raise_for_status(lib().bdf_init_multi(int(n_gpus if not devices else len(devices)), devs, C.byref(h)))
        self.handle = h
        self.device = int(devices[0]) if devices else 0
        return self

    @property
    def n_gpus(self) -> int:
        return int(lib().bdf_fleet_size(self.handle))

    def close(self):
        if getattr(self, "handle", None):
            lib().bdf_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- misc --
    def synchronize(self):
        raise_for_status(lib().bdf_synchronize(self.handle))

    def device_info(self):
        sm, ma, mi, hbm = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int64()
        raise_for_status(lib().bdf_device_info(self.handle, C.byref(sm), C.byref(ma), C.byref(mi), C.byref(hbm)))
        return {"sm_count": sm.value, "cc": (ma.value, mi.value), "hbm_bytes": hbm.value}

    def pinned(self, nbytes: int) -> PinnedBuffer:
        return PinnedBuffer(self, nbytes)

    # -- multi-GPU: this context as a rank of a communicator (include/b200df.h "multi-GPU") --
    @staticmethod
    def comm_unique_id() -> bytes:
        buf = (C.c_uint8 * 128)()
        raise_for_status(lib().bdf_comm_unique_id(buf))
        return bytes(buf)

    def comm_attach(self, unique_id: bytes, rank: int, world: int):
        """ncclCommInitRank: afterwards every aggregate entry is collective and returns the aggregate of the whole
        (sharded) column on every rank."""
        buf = (C.c_uint8 * 128)(*unique_id)
        raise_for_status(lib().bdf_comm_attach(self.handle, buf, int(rank), int(world)))

    def comm_detach(self):
        raise_for_status(lib().bdf_comm_detach(self.handle))

    def comm_info(self) -> dict:
        r, w, v, n = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int64()
        raise_for_status(lib().bdf_comm_info(self.handle, C.byref(r), C.byref(w), C.byref(v), C.byref(n)))
        return {"rank": r.value, "world": w.value, "nccl_version": v.value, "collectives": n.value}

    def comm_collective(self, on: bool):
        raise_for_status(lib().bdf_comm_collective(self.handle, 1 if on else 0))

    def comm_barrier(self):
        raise_for_status(lib().bdf_comm_barrier(self.handle))

    def comm_set_combine(self, peer_memory: bool):
        """True: NVLink peer-memory mailboxes (one kernel of the library); False: the grouped ncclAllReduce."""
        raise_for_status(lib().bdf_comm_set_combine(self.handle, 1 if peer_memory else 0))

    def comm_get_combine(self) -> str:
        return "peer-memory" if lib().bdf_comm_get_combine(self.handle) else "nccl"

    def comm_all_reduce(self, values, op: int = SUM):
        """Blocking all-reduce of a few float64 values (timing max-over-ranks and the like)."""
        arr = np.ascontiguousarray(np.atleast_1d(np.asarray(values, dtype=np.float64))).copy()
        raise_for_status(lib().bdf_comm_all_reduce_f64(self.handle, op, arr.shape[0], arr.ctypes.data_as(C.POINTER(C.c_double))))
        return arr

    def pinned_array(self, dtype: int, values: np.ndarray, mask: Optional[np.ndarray] = None) -> PrimitiveArray:
        """Copy a numpy array (and optional bool mask, True = valid) into pinned host memory."""
        n = int(values.shape[0])
        w = width_of(dtype)
        vbytes = (n * w + 63) // 64 * 64
        bbytes = ((n + 7) // 8 + 63) // 64 * 64 if mask is not None else 0
        buf = self.pinned(vbytes + bbytes)
        v = buf.array(NP_DTYPES[dtype], n)
        v[:] = values
        validity, nulls = None, 0
        if mask is not None:
            validity = buf.array(np.uint8, (n + 7) // 8, vbytes)
            validity[:] = np.packbits(np.asarray(mask, dtype=bool), bitorder="little")
            nulls = int(n - np.count_nonzero(mask))
        return PrimitiveArray(dtype, v, validity, 0, n, nulls, keepalive=buf)

    def profile_enable(self, on: bool = True):
        raise_for_status(lib().bdf_profile_enable(self.handle, 1 if on else 0))

    def profile_read(self, cap: int = 65536) -> List[dict]:
        buf = (LaunchRecord * cap)()
        n = C.c_int64(0)
        raise_for_status(lib().bdf_profile_read(self.handle, buf, cap, C.byref(n)))
        return [{"kernel": LAUNCH_KERNEL_NAMES[buf[i].kernel], "dtype": buf[i].dtype, "rows": buf[i].rows,
                 "bytes": buf[i].bytes, "ms": buf[i].ms} for i in range(n.value)]

    def launch_count(self) -> int:
        return int(lib().bdf_launch_count(self.handle))

    def timer_start(self):
        raise_for_status(lib().bdf_timer_start(self.handle))

    def timer_stop(self) -> float:
        ms = C.c_float(0)
        raise_for_status(lib().bdf_timer_stop(self.handle, C.byref(ms)))
        return float(ms.value)

    def flush_l2(self, nbytes: int = 256 << 20):
        raise_for_status(lib().bdf_flush_l2(self.handle, nbytes))


_default_ctx: Optional[Context] = None


def default_context() -> Context:
    """Process-wide lazy singleton (what the Rust shim does with a OnceCell)."""
    global _default_ctx
    if _default_ctx is None:
        _default_ctx = Context()
    return _default_ctx


def alloc_outputs(dtype: int, lens: Sequence[int], ctx: Optional[Context] = None, pinned: bool = False):
    """Caller-side output buffers (the Rust shim uses MutableBuffer::new): returns (Out[], [(values, bitmap)])."""
    outs = (Out * max(len(lens), 1))()
    bufs = []
    if dtype == BOOL:  # bit-packed values
        for i, n in enumerate(lens):
            v = np.zeros((n + 7) // 8, dtype=np.uint8)
            b = np.zeros((n + 7) // 8, dtype=np.uint8)
            outs[i].values = v.ctypes.data if v.size else None
            outs[i].validity = b.ctypes.data if b.size else None
            outs[i].len = n
            bufs.append((v, b, None))
        return outs, bufs
    for i, n in enumerate(lens):
        if pinned:
            w = width_of(dtype)
            vbytes = (n * w + 63) // 64 * 64
            pb = ctx.pinned(vbytes + ((n + 7) // 8 + 63) // 64 * 64)
            v = pb.array(NP_DTYPES[dtype], n)
            b = pb.array(np.uint8, (n + 7) // 8, vbytes)
            keep = pb
        else:
            v = np.empty(n, dtype=NP_DTYPES[dtype])
            b = np.zeros((n + 7) // 8, dtype=np.uint8)
            keep = None
        outs[i].values = v.ctypes.data if n else None
        outs[i].validity = b.ctypes.data if b.size else None
        outs[i].len = n
        bufs.append((v, b, keep))
    return outs, bufs


def collect_outputs(dtype: int, outs, bufs) -> List[PrimitiveArray]:
    res = []
    if dtype == BOOL:
        from .arrays import BooleanArray

        for i, (v, b, keep) in enumerate(bufs):
            has_v = bool(outs[i].has_validity)
            res.append(BooleanArray(v, b if has_v else None, 0, int(outs[i].len), int(outs[i].null_count) if has_v else 0))
        return res
    for i, (v, b, keep) in enumerate(bufs):
        has_v = bool(outs[i].has_validity)
        res.append(PrimitiveArray(dtype, v, b if has_v else None, 0, int(outs[i].len),
                                  int(outs[i].null_count) if has_v else 0, keepalive=keep))
    return res
