"""rust-dataframe_b200: the Hopper (sm_90a) execution path for rust-dataframe's per-RecordBatch compute
(elementwise add/sub/mul/div, trig, numeric cast, sum/min/max/count with null-bitmap propagation).

The product is ``libb200df.so`` -- hand-written CUDA kernels behind the C ABI in ``include/b200df.h``.
This package is the thin host-side mirror of the reference's operator interface over that ABI
(``ScalarFunctions``, ``AggregateFunctions``, ``cast``) plus the device-resident ``Column`` handle.
Import as ``rust_dataframe_b200`` (alias module at the repository root).
"""
from . import _native as native
from ._native import (ArrowError, ComputeError, Context, DivideByZero, ParseError, ReferencePanic, UnsupportedType,
                      default_context)
from .arrays import (BooleanArray, DTYPE_NAMES, ListArray, F32, F64, I8, I16, I32, I64, NP_DTYPES, U8, U16, U32, U64, PrimitiveArray, TemporalType,
                     dtype_of, width_of)
from .ipc import IpcFile, write_ipc, write_ipc_host
from .csv_reader import CsvFile, write_csv
from .json_reader import JsonFile, write_json
from .parquet_reader import ParquetFile, write_parquet
from . import frame
from .frame import DeviceFrame, plan_aggregate, plan_fusion, plan_join, plan_set_op, plan_window
from .functions import (AggFuture, AggregateFunctions, ArrayFunctions, Column, ListColumn, ScalarFunctions, CaseWhen, cast, coalesce, concat, duplicated, eval_expr, eval_expr_agg, group_aggregate, group_by, join_asof_indices, join_indices,
                        greatest, hist_density, least, moments_merge, moments_stat, nanvl, sort_columns, set_op_mask, sort_indices, temporal_result, top_k_indices, when, window)

__all__ = [
    "native", "ArrowError", "ComputeError", "Context", "DivideByZero", "ParseError", "ReferencePanic", "UnsupportedType",
    "default_context", "PrimitiveArray", "BooleanArray", "ListArray", "ScalarFunctions", "AggregateFunctions", "ArrayFunctions", "Column", "ListColumn", "AggFuture", "cast", "eval_expr", "eval_expr_agg", "group_aggregate", "group_by", "join_indices", "join_asof_indices", "sort_indices", "sort_columns", "top_k_indices", "IpcFile", "CsvFile", "JsonFile", "ParquetFile", "write_parquet", "write_csv", "write_json", "write_ipc", "write_ipc_host", "frame", "DeviceFrame", "plan_aggregate", "plan_fusion", "plan_join", "plan_set_op", "plan_window", "concat", "duplicated", "set_op_mask", "window", "moments_stat", "moments_merge", "hist_density",
    "TemporalType", "temporal_result", "coalesce", "greatest", "least", "nanvl", "when", "CaseWhen",
    "I8", "I16", "I32", "I64", "U8", "U16", "U32", "U64", "F32", "F64", "NP_DTYPES", "DTYPE_NAMES", "dtype_of", "width_of",
]
