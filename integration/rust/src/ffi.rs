//! FFI surface of libb200df.so (mirrors include/b200df.h).  UNCOMPILED in this repository's image -- see ../README.md.
use std::ffi::CStr;
use std::os::raw::{c_char, c_int, c_void};

use arrow::array::{Array, PrimitiveArray};
use arrow::datatypes::{ArrowPrimitiveType, DataType};
use arrow::error::ArrowError;

#[repr(C)]
pub struct BdfView {
    pub values: *const c_void,   // base of the values buffer, NOT offset-adjusted
    pub validity: *const u8,     // null when the array has no null buffer
    pub len: i64,
    pub offset: i64,             // elements; applies to values and validity bits
    pub null_count: i64,         // -1 = unknown
}

#[repr(C)]
pub struct BdfOut {
    pub values: *mut c_void,
    pub validity: *mut u8,
    pub len: i64,                // in: capacity (= result length); out: length
    pub null_count: i64,
    pub has_validity: i32,
}

pub enum BdfCtx {}
pub enum BdfCol {}   // a column resident in HBM (one chunk per RecordBatch)
pub enum BdfIpc {}   // a mapped Arrow IPC file
pub enum BdfParquet {}   // the mapped files of a Parquet read, footers and page headers parsed
pub enum BdfCsv {}
pub const BDF_PARSE: i32 = 9;   // -> ArrowError::ParseError(last_error())
pub const BDF_UTF8: i32 = 11;   // CSV schema entry: a string column the device skips
// include/b200df.h "null handling and conditional selection": column == null is a scalar (T::Native bits, Boolean 0 / 1);
// valid == 0 is a NULL literal.
#[repr(C)]
#[derive(Clone, Copy)]
pub struct BdfArg { pub column: *const BdfCol, pub bits: u64, pub valid: i32 }
pub const BDF_ROW_COALESCE: c_int = 0;
pub const BDF_ROW_GREATEST: c_int = 1;
pub const BDF_ROW_LEAST: c_int = 2;
pub const BDF_ROW_NANVL: c_int = 3;
pub const BDF_IS_NULL: c_int = 0;
pub const BDF_IS_NOT_NULL: c_int = 1;
pub const BDF_IS_NAN: c_int = 2;

#[repr(C)]
pub struct BdfCsvOptions { pub has_header: i32, pub delimiter: u8, pub max_records: i64 /* <0: all */, pub batch_size: i64 }
#[repr(C)]
#[derive(Clone, Copy)]
pub struct BdfParquetOptions { pub batch_size: i64 }
#[repr(C)]
#[derive(Clone, Copy)]
pub struct BdfCsvWriteOptions { pub has_header: i32, pub delimiter: u8 }
#[repr(C)]
#[derive(Clone, Copy)]
pub struct BdfJsonWriteOptions { pub explicit_nulls: i32 }
#[repr(C)]
#[derive(Clone, Copy)]
pub struct BdfParquetWriteOptions { pub compression: i32, pub dictionary: i32, pub row_group_rows: i64 }

#[repr(C)]
pub struct BdfListView { pub offsets: *const i32, pub validity: *const u8, pub len: i64, pub offset: i64, pub null_count: i64, pub values: BdfView }
#[repr(C)]
pub struct BdfListOut {
    pub offsets: *mut i32, pub validity: *mut u8, pub values: *mut c_void, pub value_validity: *mut u8,
    pub null_count: i64, pub value_null_count: i64, pub has_validity: i32, pub has_value_validity: i32,
}
pub enum BdfList {}
pub const BDF_LIST_BASE: i32 = 32;   // bdf_ipc_list_column: BDF_LIST_BASE + T
pub const BDF_LIST_CONTAINS: i32 = 0;
pub const BDF_LIST_POSITION: i32 = 1;
pub const BDF_LIST_MAX: i32 = 0;
pub const BDF_LIST_MIN: i32 = 1;
pub const BDF_LIST_SIZE: i32 = 2;
pub const BDF_LIST_REMOVE: i32 = 0;
pub const BDF_LIST_SORT: i32 = 1;
pub const BDF_LIST_DISTINCT: i32 = 2;
pub const BDF_LIST_REPEAT: i32 = 3;
pub const BDF_LIST_EXCEPT: i32 = 0;
pub const BDF_LIST_INTERSECT: i32 = 1;
pub const BDF_LIST_UNION: i32 = 2;
#[repr(C)]
pub struct BdfExprNode { pub op: i32, pub a: i32, pub b: i32 }   // op: bdf_binop, or BDF_EXPR_UNARY + bdf_unop
pub const BDF_EXPR_UNARY: i32 = 100;
/// bdf_group_out: per value column; `min` / `max` are NULL for Float columns (T::Native: Ord).
#[repr(C)]
#[derive(Clone, Copy)]
pub struct BdfGroupOut {
    pub sum: *mut BdfCol,
    pub count: *mut BdfCol,
    pub min: *mut BdfCol,
    pub max: *mut BdfCol,
}

/// bdf_group_agg: one (value column, function) pair of a flattened `Vec<Aggregation>`; `function` is a `bdf_group_fn`.
#[repr(C)]
#[derive(Clone, Copy)]
pub struct BdfGroupAgg { pub column: *const BdfCol, pub function: i32 }
/// bdf_group_fn, in AggregateFunction order.
pub const BDF_GROUP_SUM: i32 = 0;
pub const BDF_GROUP_MAX: i32 = 1;
pub const BDF_GROUP_MIN: i32 = 2;
pub const BDF_GROUP_AVG: i32 = 3;
pub const BDF_GROUP_COUNT: i32 = 4;
pub const BDF_GROUP_COUNT_DISTINCT: i32 = 5;
pub const BDF_GROUP_FIRST: i32 = 6;
// (BDF_GROUP_LAST = 7 follows; then the statistical functions, continuing AggregateFunction's order, and the population forms)
pub const BDF_GROUP_KURTOSIS: i32 = 8;
pub const BDF_GROUP_SKEWNESS: i32 = 9;
pub const BDF_GROUP_STDDEV: i32 = 10;
pub const BDF_GROUP_SUM_DISTINCT: i32 = 11;
pub const BDF_GROUP_VARIANCE: i32 = 12;
pub const BDF_GROUP_STDDEV_POP: i32 = 13;
pub const BDF_GROUP_VAR_POP: i32 = 14;
pub const BDF_GROUP_MEDIAN: i32 = 32;   // the distributions start a block of their own
pub const BDF_GROUP_MODE: i32 = 33;
pub const BDF_GROUP_COLLECT_LIST: i32 = 48;   // the list builders: bdf_group_by_lists_dev only
pub const BDF_GROUP_COLLECT_SET: i32 = 49;
/// bdf_moment_rec: count, mean and the central sums m2, m3, m4 of the valid values (read `as f64`).
#[repr(C)]
#[derive(Clone, Copy, Default)]
pub struct BdfMomentRec { pub count: i64, pub mean: f64, pub m2: f64, pub m3: f64, pub m4: f64 }
/// bdf_distinct_rec: the number of distinct valid values and their sum (T::Native bits in the low bytes).
#[repr(C)]
#[derive(Clone, Copy, Default)]
pub struct BdfDistinctRec { pub count: i64, pub sum: u64 }
/// bdf_stat
pub const BDF_STAT_VARIANCE: i32 = 0;
pub const BDF_STAT_VAR_POP: i32 = 1;
pub const BDF_STAT_STDDEV: i32 = 2;
pub const BDF_STAT_STDDEV_POP: i32 = 3;
pub const BDF_STAT_SKEWNESS: i32 = 4;
pub const BDF_STAT_KURTOSIS: i32 = 5;
pub const BDF_GROUP_LAST: i32 = 7;

#[repr(C)]
pub struct BdfSortKey { pub column: *const BdfCol, pub descending: i32 }
/// bdf_window_call (include/b200df.h): one window function over the shared WindowSpec.  `column` is null for the five ranking
/// functions; `offset` / `default_bits` / `has_default` are LAG / LEAD's (`offset` is also NTH_VALUE's n), `frame` (bdf_window_frame) the
/// aggregates' and value functions'.  `start` / `end` are ROWS_BETWEEN's and an integer RANGE_BETWEEN's offsets (i64::MIN / i64::MAX =
/// UNBOUNDED), `start_f` / `end_f` a float RANGE_BETWEEN's (-inf / +inf); `ignore_nulls` is the value functions'.
#[repr(C)]
#[derive(Clone, Copy)]
pub struct BdfWindowCall {
    pub function: i32, pub frame: i32, pub column: *const BdfCol, pub offset: i64, pub default_bits: u64, pub has_default: i32,
    pub ignore_nulls: i32, pub start: i64, pub end: i64, pub start_f: f64, pub end_f: f64,
}
/// bdf_asof_spec: the rules of one as-of join (include/b200df.h "as-of join").  `tolerance` bounds an integer or temporal key's distance in
/// its own units, `tolerance_f` a Float32 / Float64 key's (+inf allowed); both only when `has_tolerance` is 1.
#[repr(C)]
#[derive(Clone, Copy)]
pub struct BdfAsofSpec { pub direction: i32, pub allow_exact_matches: i32, pub has_tolerance: i32, pub tolerance: i64, pub tolerance_f: f64 }
/// bdf_asof_direction.
pub const BDF_ASOF_BACKWARD: i32 = 0;
pub const BDF_ASOF_FORWARD: i32 = 1;
pub const BDF_ASOF_NEAREST: i32 = 2;
// bdf_keep / bdf_setop
pub const BDF_KEEP_FIRST: i32 = 0;
pub const BDF_KEEP_LAST: i32 = 1;
pub const BDF_KEEP_NONE: i32 = 2;
pub const BDF_SETOP_INTERSECT: i32 = 0;
pub const BDF_SETOP_INTERSECT_ALL: i32 = 1;
pub const BDF_SETOP_EXCEPT: i32 = 2;
pub const BDF_SETOP_EXCEPT_ALL: i32 = 3;
/// bdf_join_type: JoinType's four, then the existence joins.
pub const BDF_JOIN_LEFT_SEMI: i32 = 4;
pub const BDF_JOIN_LEFT_ANTI: i32 = 5;
/// bdf_window_fn, in WindowFunctions order, then the aggregates.
pub const BDF_WIN_ROW_NUMBER: i32 = 0;
pub const BDF_WIN_RANK: i32 = 1;
pub const BDF_WIN_DENSE_RANK: i32 = 2;
pub const BDF_WIN_PERCENT_RANK: i32 = 3;
pub const BDF_WIN_CUME_DIST: i32 = 4;
pub const BDF_WIN_LAG: i32 = 5;
pub const BDF_WIN_LEAD: i32 = 6;
pub const BDF_WIN_SUM: i32 = 7;
pub const BDF_WIN_COUNT: i32 = 8;
pub const BDF_WIN_MIN: i32 = 9;
pub const BDF_WIN_MAX: i32 = 10;
pub const BDF_WIN_AVG: i32 = 11;
pub const BDF_WIN_FIRST_VALUE: i32 = 12;
pub const BDF_WIN_LAST_VALUE: i32 = 13;
pub const BDF_WIN_NTH_VALUE: i32 = 14;
/// bdf_window_frame: ROWS = partition start .. current row, RANGE = .. the current row's last peer, PARTITION = the whole partition;
/// ROWS_BETWEEN / RANGE_BETWEEN = WindowSpec's rows_between / range_between with signed offsets.
pub const BDF_FRAME_ROWS: i32 = 0;
pub const BDF_FRAME_RANGE: i32 = 1;
pub const BDF_FRAME_PARTITION: i32 = 2;
pub const BDF_FRAME_ROWS_BETWEEN: i32 = 3;
pub const BDF_FRAME_RANGE_BETWEEN: i32 = 4;
pub const BDF_ASYNC: c_int = 1;

/// All four aggregates of one pass (include/b200df.h `bdf_agg4`, ABI version 2: `n_chunks` added).
#[repr(C)]
pub struct BdfAgg4 { pub sum: u64, pub min: u64, pub max: u64, pub count: i64, pub rows: i64, pub any_valid: i32, pub would_panic: i32, pub n_chunks: i64 }
pub enum BdfFuture {}

pub const BDF_OK: c_int = 0;
pub const BDF_LENGTH_MISMATCH: c_int = 1;
pub const BDF_DIVIDE_BY_ZERO: c_int = 2;
pub const BDF_WOULD_PANIC: c_int = 7;

extern "C" {
    pub fn bdf_upload(ctx: *mut BdfCtx, dtype: c_int, n_chunks: i64, input: *const BdfView, flags: c_int, out: *mut *mut BdfCol) -> c_int;
    pub fn bdf_rowwise_dev(ctx: *mut BdfCtx, func: c_int, n_args: i32, args: *const BdfArg, out: *mut *mut BdfCol) -> c_int;
    pub fn bdf_case_when_dev(ctx: *mut BdfCtx, n_branches: i32, conditions: *const *const BdfCol, values: *const BdfArg /* n_branches + 1 */,
                             out: *mut *mut BdfCol) -> c_int;
    pub fn bdf_null_test_dev(ctx: *mut BdfCtx, func: c_int, input: *const BdfCol, out: *mut *mut BdfCol) -> c_int;
    pub fn bdf_init(device: c_int, out: *mut *mut BdfCtx) -> c_int;
    /// ONE context over `n_gpus` GPUs of the box (0 = all visible): the library shards every call by row range, each GPU
    /// moves its pieces over its own PCIe link, aggregates are combined over NVLink (grouped ncclAllReduce / peer-memory
    /// mailboxes).  What a single Rust process binds; every entry below accepts it.
    pub fn bdf_init_multi(n_gpus: c_int, devices: *const c_int, out: *mut *mut BdfCtx) -> c_int;
    pub fn bdf_fleet_size(ctx: *mut BdfCtx) -> c_int;
    /// Process per GPU (MPI-style launchers): rank 0 makes the id, ships the 128 bytes, every rank attaches its one-GPU context.
    pub fn bdf_comm_unique_id(id: *mut u8) -> c_int;
    pub fn bdf_comm_attach(ctx: *mut BdfCtx, id: *const u8, rank: c_int, world: c_int) -> c_int;
    pub fn bdf_aggregate_all(ctx: *mut BdfCtx, dtype: c_int, n: i64, input: *const BdfView, out: *mut BdfAgg4) -> c_int;
    pub fn bdf_aggregate_all_many_dev(ctx: *mut BdfCtx, n_cols: i32, cols: *const *const BdfCol, out: *mut BdfAgg4) -> c_int;
    pub fn bdf_binary_agg_dev_async(ctx: *mut BdfCtx, op: c_int, left: *const BdfCol, right: *const BdfCol, out: *mut *mut BdfCol,
                                    fut: *mut *mut BdfFuture) -> c_int;
    pub fn bdf_future_wait(ctx: *mut BdfCtx, fut: *mut BdfFuture, out: *mut BdfAgg4) -> c_int;
    pub fn bdf_last_error() -> *const c_char;
    pub fn bdf_host_register(ctx: *mut BdfCtx, p: *mut c_void, bytes: usize) -> c_int;
    pub fn bdf_host_unregister(ctx: *mut BdfCtx, p: *mut c_void) -> c_int;
    pub fn bdf_binary(ctx: *mut BdfCtx, op: c_int, dtype: c_int, n_left: i64, left: *const BdfView, n_right: i64,
                      right: *const BdfView, out: *mut BdfOut) -> c_int;
    pub fn bdf_unary(ctx: *mut BdfCtx, op: c_int, dtype: c_int, n: i64, input: *const BdfView, out: *mut BdfOut) -> c_int;
    pub fn bdf_cast(ctx: *mut BdfCtx, from: c_int, to: c_int, n: i64, input: *const BdfView, out: *mut BdfOut) -> c_int;
    pub fn bdf_aggregate(ctx: *mut BdfCtx, op: c_int, dtype: c_int, n: i64, input: *const BdfView, out_scalar: *mut c_void,
                         is_some: *mut i32) -> c_int;
    pub fn bdf_avg(ctx: *mut BdfCtx, dtype: c_int, n: i64, input: *const BdfView, out: *mut f64, is_some: *mut i32) -> c_int;
    // statistical aggregates: a context computes the moment record; a pure function derives a statistic from it
    pub fn bdf_moments(ctx: *mut BdfCtx, dtype: c_int, n: i64, input: *const BdfView, out: *mut BdfMomentRec) -> c_int;
    pub fn bdf_moments_stat(m: *const BdfMomentRec, stat: c_int, out: *mut f64, is_some: *mut i32) -> c_int;
    pub fn bdf_moments_merge(a: *const BdfMomentRec, b: *const BdfMomentRec, out: *mut BdfMomentRec) -> c_int;
    pub fn bdf_distinct(ctx: *mut BdfCtx, dtype: c_int, n: i64, input: *const BdfView, out: *mut BdfDistinctRec) -> c_int;
    // distributions: Spark's exact percentile and mode (host in), uniques and numpy's histogram (device in), numpy's density
    pub fn bdf_percentile(ctx: *mut BdfCtx, dtype: c_int, n: i64, input: *const BdfView, n_p: i32, p: *const f64, out: *mut f64,
                          is_some: *mut i32) -> c_int;
    pub fn bdf_mode(ctx: *mut BdfCtx, dtype: c_int, n: i64, input: *const BdfView, bits: *mut u64, freq: *mut i64, is_some: *mut i32) -> c_int;
    pub fn bdf_uniques_dev(ctx: *mut BdfCtx, input: *const BdfCol, values: *mut *mut BdfCol, counts: *mut *mut BdfCol) -> c_int;
    pub fn bdf_hist_dev(ctx: *mut BdfCtx, input: *const BdfCol, nbins: i32, range: *const f64, edges: *mut f64, counts: *mut i64) -> c_int;
    pub fn bdf_hist_density(nbins: i32, edges: *const f64, counts: *const i64, out: *mut f64) -> c_int;
    // device-resident columns (the lazy evaluator keeps a frame's numeric columns in HBM between Calculations)
    pub fn bdf_upload_many(ctx: *mut BdfCtx, n_cols: i64, dtypes: *const i32, n_chunks: *const i64, input: *const *const BdfView, flags: c_int,
                           out: *mut *mut BdfCol) -> c_int;
    pub fn bdf_binary_dev(ctx: *mut BdfCtx, op: c_int, left: *const BdfCol, right: *const BdfCol, out: *mut *mut BdfCol) -> c_int;
    pub fn bdf_unary_dev(ctx: *mut BdfCtx, op: c_int, input: *const BdfCol, out: *mut *mut BdfCol) -> c_int;
    pub fn bdf_cast_dev(ctx: *mut BdfCtx, to: c_int, input: *const BdfCol, out: *mut *mut BdfCol) -> c_int;
    pub fn bdf_eval_expr_dev(ctx: *mut BdfCtx, n_inputs: i32, inputs: *const *const BdfCol, n_nodes: i32, nodes: *const BdfExprNode,
                             out: *mut *mut BdfCol) -> c_int;
    pub fn bdf_download(ctx: *mut BdfCtx, col: *const BdfCol, out: *mut BdfOut) -> c_int;
    pub fn bdf_col_free(ctx: *mut BdfCtx, col: *mut BdfCol);
    // DataFrame::sort
    pub fn bdf_sort_indices_dev(ctx: *mut BdfCtx, n_keys: i32, keys: *const BdfSortKey, indices: *mut *mut BdfCol) -> c_int;
    pub fn bdf_top_k_indices_dev(ctx: *mut BdfCtx, n_keys: i32, keys: *const BdfSortKey, k: i64, indices: *mut *mut BdfCol) -> c_int;
    pub fn bdf_take_dev(ctx: *mut BdfCtx, values: *const BdfCol, indices: *const BdfCol, out: *mut *mut BdfCol) -> c_int;
    // group-by aggregate (Transformation::GroupAggregate, src/evaluation.rs:73; planned shape src/expression.rs:114-221)
    pub fn bdf_group_aggregate_dev(ctx: *mut BdfCtx, key: *const BdfCol, n_values: i32, values: *const *const BdfCol, out_keys: *mut *mut BdfCol,
                                   out: *mut BdfGroupOut, n_groups: *mut i64) -> c_int;
    // group-by over 1..16 key columns with a flat list of (column, function) pairs; every returned column is the caller's to free
    pub fn bdf_group_by_dev(ctx: *mut BdfCtx, n_keys: i32, keys: *const *const BdfCol, n_aggs: i32, aggs: *const BdfGroupAgg,
                            out_keys: *mut *mut BdfCol, out: *mut *mut BdfCol, n_groups: *mut i64) -> c_int;
    // the same with collect_list / collect_set: a collect aggregation writes out_lists[j] (one chunk) and sets out[j] = NULL
    pub fn bdf_group_by_lists_dev(ctx: *mut BdfCtx, n_keys: i32, keys: *const *const BdfCol, n_aggs: i32, aggs: *const BdfGroupAgg,
                                  out_keys: *mut *mut BdfCol, out: *mut *mut BdfCol, out_lists: *mut *mut BdfList, n_groups: *mut i64) -> c_int;
    // equi-join (calc_equijoin_indices): join_type in JoinType order (LeftJoin, RightJoin, InnerJoin, FullJoin); two UInt32 index
    // columns, NULL = no partner, to take every column of each side with.  BDF_JOIN_LEFT_SEMI / _ANTI: only left_indices (the left
    // rows with / without a partner, ascending); right_indices may be null and is set to null
    pub fn bdf_join_indices_dev(ctx: *mut BdfCtx, join_type: i32, n_keys: i32, left_keys: *const *const BdfCol, right_keys: *const *const BdfCol,
                                left_indices: *mut *mut BdfCol, right_indices: *mut *mut BdfCol, n_rows: *mut i64) -> c_int;
    // as-of join (pandas' merge_asof): one UInt32 column, a right row number per left row in left order, NULL = no partner
    pub fn bdf_join_asof_dev(ctx: *mut BdfCtx, left_on: *const BdfCol, right_on: *const BdfCol, n_by: i32, left_by: *const *const BdfCol,
                             right_by: *const *const BdfCol, spec: *const BdfAsofSpec, right_indices: *mut *mut BdfCol) -> c_int;
    // distinct rows and set operations: a Boolean mask over the (left) rows, chunked like the keys, no nulls (include/b200df.h)
    pub fn bdf_duplicated_dev(ctx: *mut BdfCtx, n_keys: i32, keys: *const *const BdfCol, keep: i32, mask: *mut *mut BdfCol) -> c_int;
    pub fn bdf_set_op_dev(ctx: *mut BdfCtx, op: i32, n_keys: i32, left: *const *const BdfCol, right: *const *const BdfCol,
                          mask: *mut *mut BdfCol) -> c_int;
    // the chunks of cols[0], then those of cols[1], ... copied on the device; one dtype
    pub fn bdf_concat_dev(ctx: *mut BdfCtx, n: i32, cols: *const *const BdfCol, out: *mut *mut BdfCol) -> c_int;
    pub fn bdf_list_concat_dev(ctx: *mut BdfCtx, n: i32, lists: *const *const BdfList, out: *mut *mut BdfList) -> c_int;
    // a Boolean column as UInt8 0 / 1 (nulls kept), the form in which a Boolean payload goes through bdf_filter_dev
    pub fn bdf_bool_widen_dev(ctx: *mut BdfCtx, input: *const BdfCol, out: *mut *mut BdfCol) -> c_int;
    // window functions over one WindowSpec (src/window.rs:8-22; WindowFunctions, src/functions/window.rs:1-11): n_calls one-chunk columns
    // in the caller's row order, every one the caller's to free
    pub fn bdf_window_dev(ctx: *mut BdfCtx, n_partition: i32, partition_by: *const *const BdfCol, n_order: i32, order_by: *const BdfSortKey,
                          n_calls: i32, calls: *const BdfWindowCall, out: *mut *mut BdfCol) -> c_int;
    // CSV files straight to the device (DataFrame::from_csv): rules, departures and memory in include/b200df.h
    pub fn bdf_csv_open(ctx: *mut BdfCtx, path: *const c_char, options: *const BdfCsvOptions, n_schema: i32, schema_dtypes: *const i32,
                        out: *mut *mut BdfCsv) -> c_int;
    pub fn bdf_csv_describe(file: *const BdfCsv, n_columns: *mut i32, n_batches: *mut i64, n_rows: *mut i64) -> c_int;
    pub fn bdf_csv_column(file: *const BdfCsv, col: i32, name: *mut *const c_char, dtype: *mut i32, nullable: *mut i32) -> c_int;
    pub fn bdf_csv_read(ctx: *mut BdfCtx, file: *const BdfCsv, n_cols: i32, cols: *const i32, out: *mut *mut BdfCol) -> c_int;
    pub fn bdf_csv_stats(file: *const BdfCsv, n_fields: *mut i64, exact_fields: *mut i64, upload_ms: *mut f64) -> c_int;
    pub fn bdf_csv_close(ctx: *mut BdfCtx, file: *mut BdfCsv);
    // CSV files straight from the device (DataFrame::to_csv): chunk b of every column = RecordBatch b; options NULL: a header and ','
    pub fn bdf_csv_write(ctx: *mut BdfCtx, path: *const c_char, n_cols: i32, names: *const *const c_char, cols: *const *const BdfCol,
                         options: *const BdfCsvWriteOptions) -> c_int;
    // line-delimited JSON straight from the device (DataFrame::to_json): column j is lists[j] when that is non-null (cols[j] then
    // null); types / lists may be null; options NULL: explicit_nulls = 0
    pub fn bdf_json_write(ctx: *mut BdfCtx, path: *const c_char, n_cols: i32, names: *const *const c_char, cols: *const *const BdfCol,
                          types: *const BdfTemporalType, lists: *const *const BdfList, options: *const BdfJsonWriteOptions) -> c_int;
    // Arrow IPC files (DataFrame::from_arrow / to_arrow)
    pub fn bdf_ipc_open(path: *const c_char, out: *mut *mut BdfIpc) -> c_int;
    pub fn bdf_ipc_close(file: *mut BdfIpc);
    pub fn bdf_ipc_describe(file: *const BdfIpc, n_columns: *mut i32, n_batches: *mut i64, n_rows: *mut i64) -> c_int;
    pub fn bdf_ipc_column(file: *const BdfIpc, col: i32, name: *mut *const c_char, dtype: *mut i32, nullable: *mut i32) -> c_int;
    pub fn bdf_ipc_read(ctx: *mut BdfCtx, file: *const BdfIpc, n_cols: i32, cols: *const i32, flags: c_int, out: *mut *mut BdfCol) -> c_int;
    pub fn bdf_ipc_read_batches(ctx: *mut BdfCtx, file: *const BdfIpc, n_cols: i32, cols: *const i32, n_batches: i64, batches: *const i64,
                                flags: c_int, out: *mut *mut BdfCol) -> c_int;
    // List<T> columns and ArrayFunctions (src/functions/array.rs): rules, departures and limits in include/b200df.h
    pub fn bdf_list_upload(ctx: *mut BdfCtx, child_dtype: c_int, n_chunks: i64, lists: *const BdfListView, flags: c_int, out: *mut *mut BdfList) -> c_int;
    pub fn bdf_list_describe(list: *const BdfList, child_dtype: *mut i32, n_chunks: *mut i64, total_len: *mut i64) -> c_int;
    pub fn bdf_list_chunk_info(ctx: *mut BdfCtx, list: *const BdfList, chunk: i64, len: *mut i64, null_count: *mut i64, n_elements: *mut i64) -> c_int;
    pub fn bdf_list_download(ctx: *mut BdfCtx, list: *const BdfList, out: *mut BdfListOut) -> c_int;
    pub fn bdf_list_values(list: *const BdfList) -> *const BdfCol;
    pub fn bdf_list_free(ctx: *mut BdfCtx, list: *mut BdfList);
    pub fn bdf_list_find_dev(ctx: *mut BdfCtx, func: c_int, list: *const BdfList, value_bits: u64, out: *mut *mut BdfCol) -> c_int;
    pub fn bdf_list_reduce_dev(ctx: *mut BdfCtx, func: c_int, list: *const BdfList, out: *mut *mut BdfCol) -> c_int;
    pub fn bdf_list_transform_dev(ctx: *mut BdfCtx, func: c_int, list: *const BdfList, value_bits: u64, count: i64, out: *mut *mut BdfList) -> c_int;
    pub fn bdf_list_set_dev(ctx: *mut BdfCtx, func: c_int, a: *const BdfList, b: *const BdfList, out: *mut *mut BdfList) -> c_int;
    pub fn bdf_list_explode_dev(ctx: *mut BdfCtx, list: *const BdfList, rows: *mut *mut BdfCol, values: *mut *mut BdfCol) -> c_int;
    // whole lists between rows: take gives one chunk, filter keeps the chunks (RecordBatch-aligned with bdf_filter_dev)
    pub fn bdf_list_take_dev(ctx: *mut BdfCtx, list: *const BdfList, indices: *const BdfCol, out: *mut *mut BdfList) -> c_int;
    pub fn bdf_list_filter_dev(ctx: *mut BdfCtx, list: *const BdfList, mask: *const BdfCol, out: *mut *mut BdfList) -> c_int;
    pub fn bdf_ipc_list_column(file: *const BdfIpc, col: i32, dtype: *mut i32) -> c_int;
    pub fn bdf_ipc_read_list(ctx: *mut BdfCtx, file: *const BdfIpc, col: i32, flags: c_int, out: *mut *mut BdfList) -> c_int;
    pub fn bdf_ipc_write(ctx: *mut BdfCtx, path: *const c_char, n_cols: i32, names: *const *const c_char, cols: *const *const BdfCol) -> c_int;
    // dates and timestamps (include/b200df.h "dates and timestamps")
    pub fn bdf_temporal(ctx: *mut BdfCtx, func: c_int, ty: *const BdfTemporalType, arg: i64, n: i64, input: *const BdfView, out: *mut BdfOut) -> c_int;
    pub fn bdf_temporal_dev(ctx: *mut BdfCtx, func: c_int, ty: *const BdfTemporalType, arg: i64, input: *const BdfCol, out: *mut *mut BdfCol) -> c_int;
    pub fn bdf_temporal_binary_dev(ctx: *mut BdfCtx, func: c_int, ta: *const BdfTemporalType, a: *const BdfCol, tb: *const BdfTemporalType,
                                   b: *const BdfCol, out: *mut *mut BdfCol) -> c_int;
    pub fn bdf_temporal_result(func: c_int, ty: *const BdfTemporalType, arg: i64, out_dtype: *mut i32, out_type: *mut BdfTemporalType) -> c_int;
    pub fn bdf_ipc_temporal_column(file: *const BdfIpc, col: i32, out: *mut BdfTemporalType) -> c_int;
    pub fn bdf_ipc_read_temporal(ctx: *mut BdfCtx, file: *const BdfIpc, col: i32, flags: c_int, out: *mut *mut BdfCol) -> c_int;
    pub fn bdf_ipc_write_typed(ctx: *mut BdfCtx, path: *const c_char, n_cols: i32, names: *const *const c_char, cols: *const *const BdfCol,
                               types: *const BdfTemporalType) -> c_int;
    // column j is lists[j] (List<item: T>) when that is non-null, cols[j] otherwise
    pub fn bdf_ipc_write_lists(ctx: *mut BdfCtx, path: *const c_char, n_cols: i32, names: *const *const c_char, cols: *const *const BdfCol,
                               types: *const BdfTemporalType, lists: *const *const BdfList) -> c_int;
    // Parquet files straight to the device (include/b200df.h "Parquet files straight to the device")
    pub fn bdf_parquet_open(path: *const c_char, options: *const BdfParquetOptions, out: *mut *mut BdfParquet) -> c_int;
    pub fn bdf_parquet_describe(file: *const BdfParquet, n_columns: *mut i32, n_batches: *mut i64, n_rows: *mut i64) -> c_int;
    pub fn bdf_parquet_column(file: *const BdfParquet, col: i32, name: *mut *const c_char, dtype: *mut i32, nullable: *mut i32) -> c_int;
    pub fn bdf_parquet_temporal_column(file: *const BdfParquet, col: i32, out: *mut BdfTemporalType) -> c_int;
    pub fn bdf_parquet_check(file: *const BdfParquet, col: i32) -> c_int;
    pub fn bdf_parquet_read(ctx: *mut BdfCtx, file: *const BdfParquet, n_cols: i32, cols: *const i32, out: *mut *mut BdfCol) -> c_int;
    pub fn bdf_parquet_stats(file: *const BdfParquet, n_pages: *mut i64, uploaded_bytes: *mut i64, upload_ms: *mut f64) -> c_int;
    pub fn bdf_parquet_close(file: *mut BdfParquet);
    // Parquet files straight from the device (DataFrame::to_parquet): types NULL or one per column (kind 0: none); options NULL: the
    // defaults (uncompressed, dictionary on, one row group per chunk)
    pub fn bdf_parquet_write(ctx: *mut BdfCtx, path: *const c_char, n_cols: i32, names: *const *const c_char, cols: *const *const BdfCol,
                             types: *const BdfTemporalType, options: *const BdfParquetWriteOptions) -> c_int;
}

/// bdf_temporal_type: kind (0 none, 1 Date32, 2 Date64, 3 Timestamp, 4 Time32, 5 Time64), unit (arrow TimeUnit order), tz (Timestamp).
#[repr(C)]
pub struct BdfTemporalType { pub kind: i32, pub unit: i32, pub tz: *const c_char }

/// The bdf_temporal_type of an arrow DataType (None for a non-temporal type).  The tz string must outlive the call: the caller keeps
/// the CString.
pub fn temporal_type(t: &DataType, tz_keep: &mut Option<std::ffi::CString>) -> Option<BdfTemporalType> {
    use arrow::datatypes::{DateUnit, TimeUnit};
    let unit = |u: &TimeUnit| match u { TimeUnit::Second => 0, TimeUnit::Millisecond => 1, TimeUnit::Microsecond => 2, TimeUnit::Nanosecond => 3 };
    match t {
        DataType::Date32(DateUnit::Day) => Some(BdfTemporalType { kind: 1, unit: 0, tz: std::ptr::null() }),
        DataType::Date64(DateUnit::Millisecond) => Some(BdfTemporalType { kind: 2, unit: 1, tz: std::ptr::null() }),
        DataType::Timestamp(u, tz) => {
            *tz_keep = tz.as_ref().map(|s| std::ffi::CString::new(s.as_str()).unwrap());
            Some(BdfTemporalType { kind: 3, unit: unit(u), tz: tz_keep.as_ref().map_or(std::ptr::null(), |c| c.as_ptr()) })
        }
        DataType::Time32(u) => Some(BdfTemporalType { kind: 4, unit: unit(u), tz: std::ptr::null() }),
        DataType::Time64(u) => Some(BdfTemporalType { kind: 5, unit: unit(u), tz: std::ptr::null() }),
        _ => None,
    }
}

/// Process-wide context.  A plain process gets ONE context over every GPU of the box (`bdf_init_multi(0, ..)`: the library
/// shards each call over the GPUs -- the role rayon's par_iter plays in the reference, src/functions/scalar.rs:28-31).  Under a
/// process-per-GPU launcher (RANK / WORLD_SIZE / LOCAL_RANK set) each process takes its LOCAL_RANK's GPU and the launcher's
/// side channel carries the communicator id: see `attach` below.  Set BDF_ONE_GPU=1 to pin a plain process to GPU 0.
pub fn ctx() -> *mut BdfCtx {
    use std::sync::Once;
    static INIT: Once = Once::new();
    static mut CTX: *mut BdfCtx = std::ptr::null_mut();
    unsafe {
        INIT.call_once(|| {
            let mut c = std::ptr::null_mut();
            let launcher = std::env::var("WORLD_SIZE").ok().and_then(|s| s.parse::<i32>().ok()).map_or(false, |w| w > 1);
            let st = if launcher || std::env::var("BDF_ONE_GPU").is_ok() {
                let dev = std::env::var("LOCAL_RANK").ok().and_then(|s| s.parse().ok()).unwrap_or(0);
                bdf_init(dev, &mut c)
            } else {
                bdf_init_multi(0, std::ptr::null(), &mut c)
            };
            assert_eq!(st, BDF_OK, "libb200df initialisation failed: {}", last_error());
            CTX = c;
        });
        CTX
    }
}

/// A one-GPU context for the entries a multi-GPU context does not offer (sort / take / filter move rows between chunks; the IPC
/// readers map one file): GPU LOCAL_RANK (0 in a plain process).  The same object as `ctx()` under a process-per-GPU launcher.
pub fn ctx_one_gpu() -> *mut BdfCtx {
    use std::sync::Once;
    static INIT: Once = Once::new();
    static mut CTX: *mut BdfCtx = std::ptr::null_mut();
    unsafe {
        INIT.call_once(|| {
            let all = ctx();
            if bdf_fleet_size(all) <= 1 { CTX = all; return; }
            let mut c = std::ptr::null_mut();
            let st = bdf_init(0, &mut c);
            assert_eq!(st, BDF_OK, "bdf_init failed: {}", last_error());
            CTX = c;
        });
        CTX
    }
}

/// Process per GPU: make this process's context a rank of the job's communicator.  `id` = the 128 bytes rank 0 obtained from
/// `bdf_comm_unique_id` and the launcher distributed (an MPI broadcast, a file, a TCP store ...).  Afterwards every aggregate
/// entry returns the aggregate of the whole sharded column on every rank.
pub fn attach(id: &[u8; 128], rank: i32, world: i32) -> Result<(), ArrowError> {
    let st = unsafe { bdf_comm_attach(ctx(), id.as_ptr(), rank, world) };
    if st == BDF_OK { Ok(()) } else { Err(to_arrow_error(st)) }
}

pub fn last_error() -> String {
    unsafe { CStr::from_ptr(bdf_last_error()) }.to_string_lossy().into_owned()
}

/// bdf_dtype: Arrow DataType order Int8..UInt64, Float32, Float64.
pub fn dtype_id(t: &DataType) -> c_int {
    match t {
        DataType::Int8 => 0, DataType::Int16 => 1, DataType::Int32 => 2, DataType::Int64 => 3,
        DataType::UInt8 => 4, DataType::UInt16 => 5, DataType::UInt32 => 6, DataType::UInt64 => 7,
        DataType::Float32 => 8, DataType::Float64 => 9,
        other => panic!("{:?} is not a primitive numeric type", other),
    }
}

pub fn view<T: ArrowPrimitiveType>(a: &PrimitiveArray<T>) -> BdfView {
    let d = a.data();
    BdfView {
        values: d.buffers()[0].raw_data() as *const c_void,
        validity: d.null_buffer().map_or(std::ptr::null(), |b| b.raw_data()),
        len: a.len() as i64,
        offset: a.offset() as i64,
        null_count: a.null_count() as i64,
    }
}

pub fn to_arrow_error(st: c_int) -> ArrowError {
    match st {
        BDF_LENGTH_MISMATCH => ArrowError::ComputeError("Cannot perform math operation on arrays of different length".to_string()),
        BDF_DIVIDE_BY_ZERO => ArrowError::DivideByZero,
        _ => ArrowError::ComputeError(last_error()),
    }
}
