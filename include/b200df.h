/*
 * b200df.h -- C ABI of libb200df.so: the Hopper (sm_90a) execution path for rust-dataframe's
 * per-RecordBatch compute.  Plain pointers and sizes only; no C++/torch/arrow types cross this boundary.
 *
 * Reference = nevi-me/rust-dataframe @ a8310afd (paths relative to the reference root).  The reference
 * has no FFI today; the seam is the set of Rust functions below, whose BODIES become one call each
 * (INTEGRATION.md shows the Rust binding).  One call carries ALL chunks of the column(s)
 * (Vec<&PrimitiveArray<T>>, one entry per RecordBatch -- src/table.rs:114-123), so batching, streams and
 * device memory are owned by the library.
 *
 *   bdf_binary      replaces the bodies of ScalarFunctions::{add,subtract,multiply,par_multiply,divide}
 *                   (src/functions/scalar.rs:16-103 -> arrow::compute::{add,subtract,multiply,divide}) and
 *                   atan2/hypot/log (scalar.rs:148,274,291 -> math_op scalar.rs:499-523)
 *   bdf_unary       replaces ScalarFunctions::{abs,sin,cos,tan,acos,...} (scalar.rs:106-457 -> scalar_op
 *                   scalar.rs:525-540)
 *   bdf_cast        replaces the arrow::compute::cast call of Function::Cast (src/evaluation.rs:296-315)
 *   bdf_aggregate   replaces AggregateFunctions::{sum,min,max,count} (src/functions/aggregate.rs:12-93)
 *   bdf_avg         replaces AggregateFunctions::avg (aggregate.rs:32-65)
 *   bdf_*_dev       the same operators on device-resident columns, so a chain of Calculations
 *                   (src/evaluation.rs:66-96 evaluates one after another) uploads once and downloads once.
 *
 * Threads: a context may be called from several threads; calls on one context are serialised (a one-GPU context by a lock around each
 * entry, a multi-GPU context around each fan-out to its GPUs), so the reference's callers need no locking of their own -- but
 * bdf_destroy must not race with another call, and a column or future handle belongs to the thread that is using it.
 *
 * Error convention: every entry returns a bdf_status; BDF_OK == 0.  bdf_last_error() gives a
 * thread-local message.  No exception or abort crosses the ABI.  Mapping to the reference's errors:
 *   BDF_LENGTH_MISMATCH -> ArrowError::ComputeError("Cannot perform math operation on arrays of different length")
 *                          (text as src/functions/scalar.rs:508-511)
 *   BDF_DIVIDE_BY_ZERO  -> ArrowError::DivideByZero
 *   BDF_UNSUPPORTED     -> a trait bound the reference enforces at compile time (e.g. sin on integers,
 *                          max on floats: T::Native: Float / Ord)
 *   BDF_WOULD_PANIC     -> the reference panics here (max/min .unwrap() on an all-null or empty chunk,
 *                          aggregate.rs:19,29); the binding turns it back into a panic
 *   BDF_PARSE           -> ArrowError::ParseError(bdf_last_error()) (the CSV reader)
 *   BDF_CUDA / BDF_OOM / BDF_INVALID -> ArrowError::ComputeError(bdf_last_error())
 * There is NO CPU fallback: without a usable CUDA device bdf_init fails with BDF_CUDA.
 *
 * Ownership: host buffers (inputs and outputs) belong to the caller; the library never frees them and,
 * except for BDF_ASYNC uploads, never touches them after the call returns.  Device memory, streams and
 * events belong to bdf_ctx / bdf_col handles.  A bdf_ctx serialises concurrent callers with a mutex.
 */
#ifndef B200DF_H
#define B200DF_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default) /* the library is built with -fvisibility=hidden; these are its exports */
#endif

#define BDF_ABI_VERSION 3

/* Arrow primitive types, in arrow::datatypes::DataType order. */
typedef enum {
    BDF_I8 = 0, BDF_I16, BDF_I32, BDF_I64, BDF_U8, BDF_U16, BDF_U32, BDF_U64, BDF_F32, BDF_F64, BDF_NTYPES
} bdf_dtype;

typedef enum { BDF_ADD = 0, BDF_SUB, BDF_MUL, BDF_DIV, BDF_ATAN2, BDF_HYPOT, BDF_LOG, BDF_NBINARY } bdf_binop;

typedef enum {
    BDF_ABS = 0, BDF_SIN, BDF_COS, BDF_TAN,
    BDF_ACOS, BDF_ASIN, BDF_ATAN, BDF_CBRT, BDF_CEIL, BDF_COSH, BDF_DEGREES, BDF_EXP, BDF_EXPM1,
    BDF_FLOOR, BDF_LOG10, BDF_LOG2, BDF_RADIANS, BDF_ROUND, BDF_SINH, BDF_SQRT, BDF_TANH, BDF_NUNARY
} bdf_unop;

typedef enum { BDF_SUM = 0, BDF_MIN, BDF_MAX, BDF_COUNT, BDF_NAGG } bdf_aggop;

/* SURVEY 8(f) N2 (the step after the hot path): boolean columns are Arrow BooleanArrays -- `values` is a bit-packed
 * LSB-first bitmap whose `offset` counts bits -- identified by dtype BDF_BOOL in bdf_upload / bdf_col_describe. */
#define BDF_BOOL 10
typedef enum { BDF_GT = 0, BDF_GE, BDF_EQ, BDF_NE, BDF_LT, BDF_LE } bdf_cmpop;
typedef enum { BDF_AND = 0, BDF_OR, BDF_NOT } bdf_boolop;

typedef enum {
    BDF_OK = 0, BDF_LENGTH_MISMATCH = 1, BDF_DIVIDE_BY_ZERO = 2, BDF_UNSUPPORTED = 3, BDF_CUDA = 4,
    BDF_NCCL = 5 /* the communicator (bdf_comm_*) or a collective failed */, BDF_OOM = 6, BDF_WOULD_PANIC = 7, BDF_INVALID = 8,
    BDF_PARSE = 9 /* a CSV value does not parse as its column's type: ArrowError::ParseError(bdf_last_error()) */
} bdf_status;

/* One chunk = one PrimitiveArray<T> in Arrow memory layout (ArrayData: buffers[0], null bitmap, len, offset). */
typedef struct {
    const void*    values;     /* base of the values buffer, NOT offset-adjusted                         */
    const uint8_t* validity;   /* LSB-first bitmap, 1 = valid; NULL when the array has no null buffer     */
    int64_t        len;        /* logical length in elements                                              */
    int64_t        offset;     /* element offset, applies to values and to validity bits (sliced arrays)  */
    int64_t        null_count; /* cached ArrayData::null_count, or -1 if unknown                          */
} bdf_view;

/* Output chunk.  values >= len*width bytes, validity >= ceil(len/8) bytes, both caller-allocated
 * (arrow MutableBuffer).  validity is written at bit offset 0 with zero padding bits.  validity may be
 * NULL only if the result carries no bitmap (has_validity == 0 on return), else BDF_INVALID. */
typedef struct {
    void*    values;
    uint8_t* validity;
    int64_t  len;          /* IN: capacity in elements (must equal the result length); OUT: length */
    int64_t  null_count;   /* OUT */
    int32_t  has_validity; /* OUT: 0 => every slot valid and no bitmap was written */
} bdf_out;

/* All four aggregates from one pass.  Each value slot holds T::Native in its low bytes (little endian). */
typedef struct {
    uint64_t sum, min, max;  /* bit patterns of T::Native, zero-padded to 8 bytes                      */
    int64_t  count;          /* non-null slots                                                         */
    int64_t  rows;           /* total slots                                                            */
    int32_t  any_valid;      /* 0 => min/max are None                                                  */
    int32_t  would_panic;    /* 1 => some chunk is empty/all-null: reference max/min .unwrap() panics  */
    int64_t  n_chunks;       /* chunks aggregated (0 => Iterator::max over an empty Vec: None)         */
} bdf_agg4;

typedef struct bdf_ctx bdf_ctx;
typedef struct bdf_col bdf_col;
typedef struct bdf_future bdf_future; /* an aggregate whose kernels are enqueued but not yet waited for */

/* ---- lifecycle ------------------------------------------------------------------------------ */
int          bdf_abi_version(void);
const char*  bdf_last_error(void);
int          bdf_init(int device, bdf_ctx** out);   /* one context per GPU (one process per GPU) */
/* ONE context over n_gpus GPUs of the box (0 = all visible; devices == NULL: 0..n-1): what a single Rust process binds.
 * Every entry below accepts it: the rows of a call are cut into one contiguous range per GPU (the axis the reference's
 * rayon par_iter parallelises, src/functions/scalar.rs:28-31,99-102 -- cuts inside a chunk fall on 64-row boundaries,
 * so a piece is a zero-copy Arrow slice), every GPU moves and computes its pieces over its own PCIe link, and aggregates
 * are combined by the grouped ncclAllReduce (ncclCommInitAll).  Results, chunk structure, null counts and errors are
 * those of the one-GPU context.  Not offered on a multi-GPU context: sort / take / filter (rows change chunks) and the
 * IPC readers (BDF_UNSUPPORTED). */
int          bdf_init_multi(int n_gpus, const int* devices, bdf_ctx** out);
int          bdf_fleet_size(bdf_ctx* ctx);           /* GPUs behind the context (1 for bdf_init) */
void         bdf_destroy(bdf_ctx* ctx);
int          bdf_synchronize(bdf_ctx* ctx);
int          bdf_device_info(bdf_ctx* ctx, int32_t* sm_count, int32_t* cc_major, int32_t* cc_minor, int64_t* hbm_bytes);

/* ---- multi-GPU (SURVEY 8(e)): one context per GPU, the contexts of a job form a communicator ---------------------
 * The Vec<RecordBatch> is sharded over the GPUs by chunk (parallel over the same axis as the reference's rayon
 * par_iter, src/functions/scalar.rs:28-31,99-102): elementwise operators and casts need no exchange at all.  The
 * cross-chunk fold of an aggregate (src/functions/aggregate.rs:12-31,70-93) becomes [this GPU's chunks] -> ONE grouped
 * ncclAllReduce over NVLink (sum/count/rows: ncclSum on the wrapping 64-bit patterns; min/max: ncclMin/ncclMax on
 * order-preserving keys; float sums: all-gathered and folded in rank order), enqueued by the library on the stream
 * that produced the partials -- no host round trip.  After bdf_comm_attach every aggregate entry (bdf_aggregate*,
 * bdf_avg*, bdf_binary_agg_dev*, bdf_eval_expr_agg_dev*) is COLLECTIVE: all ranks make the same calls in the same
 * order and every rank receives the aggregate of the whole column; DivideByZero is agreed on by all ranks.
 * bdf_comm_collective(ctx, 0) switches back to per-rank results.  NCCL is bound at run time (libnccl.so.2).
 *   process per GPU:  rank 0 calls bdf_comm_unique_id, ships the 128 bytes to the others (any side channel), every
 *                     rank calls bdf_comm_attach(ctx, id, rank, world)  [ncclCommInitRank];
 *   one process:      bdf_init_multi (below) owns all GPUs of the box  [ncclCommInitAll]. */
#define BDF_COMM_ID_BYTES 128
int  bdf_comm_unique_id(uint8_t* id /* BDF_COMM_ID_BYTES */);
int  bdf_comm_attach(bdf_ctx* ctx, const uint8_t* id, int rank, int world);
int  bdf_comm_detach(bdf_ctx* ctx);
int  bdf_comm_info(bdf_ctx* ctx, int32_t* rank, int32_t* world, int32_t* nccl_version, int64_t* collectives_enqueued);
int  bdf_comm_collective(bdf_ctx* ctx, int on);
/* How the partial aggregates travel: 0 = the grouped ncclAllReduce, 1 = NVLink peer-memory mailboxes (one small kernel of
 * the library stores every rank's record into every peer and folds in rank order; needs peer access between all GPUs).
 * Default: 1 where available, unless the environment says BDF_COMBINE=nccl.  Results are identical (integers: order
 * independent; float sums: rank-order fold in both).  Collective: every rank switches at the same point. */
int  bdf_comm_set_combine(bdf_ctx* ctx, int mode);
int  bdf_comm_get_combine(bdf_ctx* ctx);
int  bdf_comm_barrier(bdf_ctx* ctx);    /* drains this context's streams, then returns once every rank has arrived */
int  bdf_comm_all_reduce_f64(bdf_ctx* ctx, int op /* BDF_SUM | BDF_MIN | BDF_MAX */, int64_t n, double* inout); /* blocking */

/* Pinned host memory ("Arrow buffers are pinned and copied to device once per batch"). */
int          bdf_host_alloc(bdf_ctx* ctx, size_t bytes, void** out);
int          bdf_host_free(bdf_ctx* ctx, void* p);
int          bdf_host_register(bdf_ctx* ctx, void* p, size_t bytes);
int          bdf_host_unregister(bdf_ctx* ctx, void* p);

/* ---- host in / host out: drop-in bodies for the reference functions --------------------------- */
/* zip() semantics: n = min(n_left, n_right) chunks are processed (scalar.rs:28-31). */
int bdf_binary(bdf_ctx* ctx, int op, int dtype, int64_t n_left, const bdf_view* left, int64_t n_right,
               const bdf_view* right, bdf_out* out);
int bdf_unary(bdf_ctx* ctx, int op, int dtype, int64_t n_chunks, const bdf_view* in, bdf_out* out);
int bdf_cast(bdf_ctx* ctx, int from, int to, int64_t n_chunks, const bdf_view* in, bdf_out* out);
/* out_scalar: T::Native for SUM/MIN/MAX, int64_t for COUNT.  *is_some == 0 <=> Rust None. */
int bdf_aggregate(bdf_ctx* ctx, int op, int dtype, int64_t n_chunks, const bdf_view* in, void* out_scalar,
                  int32_t* is_some);
int bdf_aggregate_all(bdf_ctx* ctx, int dtype, int64_t n_chunks, const bdf_view* in, bdf_agg4* out);
int bdf_avg(bdf_ctx* ctx, int dtype, int64_t n_chunks, const bdf_view* in, double* out, int32_t* is_some);

/* ---- device-resident columns -------------------------------------------------------------------- */
#define BDF_ASYNC 1 /* bdf_upload returns before the copies finish: host buffers must stay valid and
                       unmodified until bdf_col_wait / bdf_synchronize / a download of a dependent column */
int  bdf_upload(bdf_ctx* ctx, int dtype, int64_t n_chunks, const bdf_view* in, int flags, bdf_col** out);
/* Several columns in one call, copies issued chunk-major (a0,b0,a1,b1,...) so that an operator over them
 * can start on chunk i as soon as ITS inputs have landed while later chunks are still crossing PCIe. */
int  bdf_upload_many(bdf_ctx* ctx, int64_t n_cols, const int32_t* dtypes, const int64_t* n_chunks,
                     const bdf_view* const* in, int flags, bdf_col** out /* n_cols entries */);
int  bdf_col_wait(bdf_ctx* ctx, const bdf_col* col);
int  bdf_col_describe(const bdf_col* col, int32_t* dtype, int64_t* n_chunks, int64_t* total_len);
int  bdf_col_chunk_info(bdf_ctx* ctx, const bdf_col* col, int64_t chunk, int64_t* len, int64_t* null_count,
                        int32_t* has_validity);
int  bdf_binary_dev(bdf_ctx* ctx, int op, const bdf_col* left, const bdf_col* right, bdf_col** out);
int  bdf_unary_dev(bdf_ctx* ctx, int op, const bdf_col* in, bdf_col** out);
int  bdf_cast_dev(bdf_ctx* ctx, int to, const bdf_col* in, bdf_col** out);
int  bdf_aggregate_dev(bdf_ctx* ctx, int op, const bdf_col* in, void* out_scalar, int32_t* is_some);
int  bdf_aggregate_all_dev(bdf_ctx* ctx, const bdf_col* in, bdf_agg4* out);
int  bdf_avg_dev(bdf_ctx* ctx, const bdf_col* in, double* out, int32_t* is_some);
int  bdf_download(bdf_ctx* ctx, const bdf_col* col, bdf_out* out /* n_chunks entries */);
/* ---- N2: BooleanFilter comparisons / boolean kernels / filter on device columns ------------------------------
 * bdf_compare_dev  BooleanFilter::{Gt,Ge,Eq,Ne,Lt,Le} (src/expression.rs:820-852): both sides are cast to Float64, then
 *                  compared (IEEE, computed under nulls); validity = AND.  right == NULL compares with `scalar`
 *                  (BooleanInput::Scalar broadcast, :783-802).  Result: a BDF_BOOL column.
 * bdf_boolean_dev  arrow compute::{and,or,not} on boolean columns (values op values, validity AND); b ignored for NOT.
 * bdf_filter_dev   ChunkedArray::filter (src/table.rs:97-107): arrow compute::filter per chunk pair; a slot is kept
 *                  iff the mask is valid and true there.  Result chunk lengths are data dependent (bdf_col_chunk_info). */
int  bdf_compare_dev(bdf_ctx* ctx, int op, const bdf_col* left, const bdf_col* right, double scalar, bdf_col** out);
int  bdf_boolean_dev(bdf_ctx* ctx, int op, const bdf_col* a, const bdf_col* b, bdf_col** out);
int  bdf_filter_dev(bdf_ctx* ctx, const bdf_col* values, const bdf_col* mask, bdf_col** out);
/* ---- null handling and conditional selection (Spark's coalesce / greatest / least / nanvl / isnull / isnan / CASE WHEN) --------
 * The functions the reference names in src/functions/scalar.rs with empty bodies (coalesce, greatest, least, nanv1), with
 * Spark's definitions, and the null tests and the conditional that make them usable.
 *   coalesce(a1..an)        1..64 arguments: per row, the first argument valid there; NULL where every argument is NULL.  NaN
 *                           is a value, not a null.  fill_null(x, v) is coalesce(x, v); nvl / ifnull are two-argument coalesce.
 *   greatest / least(a1..an) 2..64 arguments: nulls are skipped, NULL only where every argument is NULL.  Values are ordered as
 *                           DataFrame::sort orders them (every NaN equal and greater than +inf, -0.0 == 0.0); among equal values
 *                           the earliest argument wins, so greatest(-0.0, 0.0) returns the bits of -0.0.
 *   nanvl(a, b)             Float32 / Float64: a where a is valid and not NaN, b where a is NaN (even a NULL b), NULL where a is.
 *   case_when               1..64 branches: a row takes the value of the first branch whose condition is valid and true there
 *                           (a NULL condition counts as false, as in SQL), else values[n_branches]; a NULL literal there is the
 *                           missing ELSE.
 *   is_null / is_not_null / is_nan  a Boolean column with no bitmap; is_nan of a NULL slot, of an integer or of a Boolean column
 *                           is false.
 * Every value of a result is copied bit for bit from the argument that supplied it (NaN payloads and the sign of zero survive):
 * no arithmetic, so results are identical under any chunking and on any number of GPUs.
 * Types: the value columns of a call share one dtype (else BDF_INVALID; a temporal column is its storage type here) and at least
 * one value is a column, which gives the result type.  Boolean values are allowed in coalesce and case_when, not in greatest,
 * least or nanvl (BDF_UNSUPPORTED); nanvl of an integer type is BDF_UNSUPPORTED.  A condition must be a Boolean column
 * (BDF_INVALID).  A scalar holds T::Native bits (Boolean: 0 or 1).
 * Chunks: zipped as the element-wise operators zip them -- n = the smallest chunk count among the column arguments, conditions
 * included; chunk i of every column must have the same length (BDF_LENGTH_MISMATCH).  Chunk i of the result is RecordBatch i;
 * it has a bitmap when some value argument can be NULL in that chunk (a bitmap there, or a NULL scalar in the call), and null
 * counts are exact.  Chunk groups are those of the other element-wise operators: work on a chunk starts once that chunk of every
 * column argument has landed.  Launch records: BDF_K_BINARY for value results, BDF_K_COMPARE for the null tests.
 * Limit: a call's per-chunk descriptor takes 48 + 32 x (conditions + values) bytes of the context's 32 MiB descriptor ring, so a
 * call of c chunks needs c x that many bytes: about 8,000 chunks with 64 branches, about 16,000 with 64 coalesce arguments, about
 * 300,000 with two.  A larger call returns BDF_OOM; split it by chunks. */
typedef struct { const bdf_col* column; uint64_t bits; int32_t valid; } bdf_arg;   /* column == NULL: a scalar, T::Native bits
                                                                                      (Boolean 0/1); valid == 0: a NULL literal */
typedef enum { BDF_ROW_COALESCE = 0, BDF_ROW_GREATEST, BDF_ROW_LEAST, BDF_ROW_NANVL } bdf_row_fn;
typedef enum { BDF_IS_NULL = 0, BDF_IS_NOT_NULL, BDF_IS_NAN } bdf_null_test;
int  bdf_rowwise_dev(bdf_ctx* ctx, int fn, int32_t n_args, const bdf_arg* args, bdf_col** out);
int  bdf_case_when_dev(bdf_ctx* ctx, int32_t n_branches, const bdf_col* const* conditions,
                       const bdf_arg* values /* n_branches + 1, last = else */, bdf_col** out);
int  bdf_null_test_dev(bdf_ctx* ctx, int fn, const bdf_col* in, bdf_col** out);
/* ---- N3: consecutive Calculations fused into one pass -----------------------------------------------------------
 * Evaluate::evaluate (src/evaluation.rs:66-96) materialises every Calculation; when the intermediates are not kept, the
 * chain can be evaluated per element in ONE kernel: inputs are read once, only the final column is written
 * (config 2: 40 B/row instead of 88).  The program is straight-line: slots 0..n_inputs-1 are the input columns,
 * node k writes slot n_inputs+k and may read any earlier slot; the last node is the result (Float64).  An input column
 * of another numeric type is read through `as f64` -- a Function::Cast to Float64 (never fails, validity unchanged)
 * folded into the load.  Every node
 * is the same operator the unfused call would run, so arithmetic chains are bit-identical; DivideByZero is raised iff
 * a slot valid for that divide node has a zero divisor.  At most 6 inputs and 12 nodes. */
#define BDF_EXPR_UNARY 100 /* node.op = bdf_binop for binary nodes, BDF_EXPR_UNARY + bdf_unop for unary nodes (operand a) */
typedef struct { int32_t op, a, b; } bdf_expr_node;
int  bdf_eval_expr_dev(bdf_ctx* ctx, int32_t n_inputs, const bdf_col* const* inputs, int32_t n_nodes, const bdf_expr_node* nodes,
                       bdf_col** out);
/* Would bdf_eval_expr_dev accept this program?  Needs no context and no GPU: validates the nodes and runs the host compiler,
 * so a planner can decide what to fuse before it touches data.  input_dtypes may be NULL (all Float64).  Returns the status
 * the evaluation would return for the program itself (BDF_OK, BDF_INVALID, BDF_UNSUPPORTED); on success reports the
 * accumulator program's instruction count and how many of the two temporaries it uses. */
int  bdf_expr_check(int32_t n_inputs, const int32_t* input_dtypes, int32_t n_nodes, const bdf_expr_node* nodes, int32_t* n_instructions,
                    int32_t* n_temporaries);
/* ... with a trailing aggregate (AggregateFunctions::sum / count of the chain's last column, src/functions/aggregate.rs:22-31,
 * 70-93) folded into the same pass, like bdf_binary_agg_dev.  `out` may be NULL: the column is then never written (the
 * chain is only aggregated: sum(sin(((a+b)*c)/d)) reads 32 B/row and writes nothing).  Float64 result: agg->sum and
 * agg->count are set, min/max are not (T::Native: Ord).  The _async form returns a future for bdf_future_wait. */
int  bdf_eval_expr_agg_dev(bdf_ctx* ctx, int32_t n_inputs, const bdf_col* const* inputs, int32_t n_nodes, const bdf_expr_node* nodes,
                           bdf_col** out, bdf_agg4* agg);
int  bdf_eval_expr_agg_dev_async(bdf_ctx* ctx, int32_t n_inputs, const bdf_col* const* inputs, int32_t n_nodes,
                                 const bdf_expr_node* nodes, bdf_col** out, bdf_future** fut);
/* Split download: _begin enqueues the device->host copies (they start as soon as each chunk group is
 * ready), _end waits for them and fills len / null_count / has_validity.  Same `out` array for both. */
int  bdf_download_begin(bdf_ctx* ctx, const bdf_col* col, bdf_out* out);
int  bdf_download_end(bdf_ctx* ctx, const bdf_col* col, bdf_out* out);
/* Fused operator + aggregate (SURVEY K5 / 8(f) N3): out = left (op) right AND sum/min/max/count of `out`,
 * computed while `out` is being written -- one pass, 3 x width bytes/row instead of 4 x.  op in
 * {ADD,SUB,MUL,DIV}.  The column is materialised exactly as bdf_binary_dev would.  agg->would_panic is
 * not evaluated here (always 0); use bdf_aggregate_dev for the reference's unwrap() behaviour. */
int  bdf_binary_agg_dev(bdf_ctx* ctx, int op, const bdf_col* left, const bdf_col* right, bdf_col** out, bdf_agg4* agg);
/* Asynchronous aggregates: the call enqueues the kernels and returns a future; bdf_future_wait blocks until
 * the result has reached the host, converts it and CONSUMES the future (out may be NULL to discard). */
int  bdf_binary_agg_dev_async(bdf_ctx* ctx, int op, const bdf_col* left, const bdf_col* right, bdf_col** out, bdf_future** fut);
int  bdf_aggregate_all_dev_async(bdf_ctx* ctx, const bdf_col* in, bdf_future** fut);
/* sum/min/max/count of up to 64 columns in one call (BASELINE config 3: 8 x Int64): one reduction per column, ONE host
 * wait and -- on a rank of a communicator -- ONE grouped collective for all of them.  out / the future carry n_cols
 * records in column order; the blocking form also evaluates would_panic. */
int  bdf_aggregate_all_many_dev(bdf_ctx* ctx, int32_t n_cols, const bdf_col* const* cols, bdf_agg4* out /* n_cols */);
int  bdf_aggregate_all_many_dev_async(bdf_ctx* ctx, int32_t n_cols, const bdf_col* const* cols, bdf_future** fut);
int  bdf_future_count(const bdf_future* fut);   /* records bdf_future_wait will write */
int  bdf_future_wait(bdf_ctx* ctx, bdf_future* fut, bdf_agg4* out /* bdf_future_count(fut) records */);
void bdf_col_free(bdf_ctx* ctx, bdf_col* col);

/* ---- DataFrame::sort (src/dataframe.rs:194-222): lexsort_to_indices + take ------------------------------------------
 * bdf_sort_indices_dev  arrow compute::lexsort_to_indices over the criteria columns (numeric, equal lengths, any chunking;
 *                       row numbers count through the chunks): a STABLE sort; per criterion ascending or descending,
 *                       nulls always last (the reference passes nulls_first: false), NaN greater than every number,
 *                       -0.0 == 0.0.  Result: one UInt32 chunk of row numbers.  BDF_INVALID for zero criteria
 *                       ("Sort criteria cannot be empty").
 * bdf_take_dev          Column::take (src/table.rs:218-241) -> arrow compute::take: out[i] = values[indices[i]], one
 *                       chunk (the reference's repartitioning loop always produces a single chunk); a null index or a
 *                       null value gives a null slot; an index past the end is an error (BDF_INVALID).  Any numeric
 *                       or boolean values column; indices: a UInt32 column. */
typedef struct { const bdf_col* column; int32_t descending; } bdf_sort_key;
int  bdf_sort_indices_dev(bdf_ctx* ctx, int32_t n_keys, const bdf_sort_key* keys, bdf_col** indices);
int  bdf_take_dev(bdf_ctx* ctx, const bdf_col* values, const bdf_col* indices, bdf_col** out);

/* ---- top-k: DataFrame::sort followed by limit (SQL's ORDER BY ... LIMIT k, pandas' nsmallest / nlargest) -------------------
 * bdf_top_k_indices_dev  The first min(k, n) row numbers of bdf_sort_indices_dev(ctx, n_keys, keys), bit for bit, for every input:
 *                        the same criteria, stability, directions, nulls last, NaN greatest and -0.0 == 0.0.  Result: one UInt32
 *                        chunk without nulls.  The sort's errors, statuses and messages in the sort's order (a multi-GPU context,
 *                        null arguments, "Sort criteria cannot be empty", non-numeric criteria, different lengths, more than
 *                        2^32-1 rows); then k < 0 -> BDF_INVALID.  k == 0 gives an empty column; k >= n the whole sort.
 * Path.  When k > 5n / 8 the call runs the full sort and keeps its first k entries.  Otherwise it chooses the k rows without sorting
 *   all of them: one round per criterion finds the threshold key of the rows still to choose with the radix select of the exact
 *   percentiles, marks the rows before it as chosen and the rows equal to it as the next round's tie set; the first ties in row order
 *   fill the rest.  Only the k chosen rows are then gathered and sorted.  The crossover was measured on an H100 (DESIGN §8).
 * Memory (k <= 5n / 8).  Two bitmaps over n rows and a UInt32 iota (4.25 B/row), the select's candidate scratch (at most the
 *   criterion's key width per valid row, usually far less), and for a tie set of m rows its row ids and one gathered criterion
 *   (at most 16 B per tie row); then the k-row gathers and sort.  The full sort takes 24 B/row of scratch.
 * Launch records: BDF_K_SELECT (threshold passes, marks and the tie prefix), BDF_K_FILTER (compactions), BDF_K_TAKE (gathers),
 *   BDF_K_SORT (the sort of the k chosen rows, or of all rows above the crossover). */
int  bdf_top_k_indices_dev(bdf_ctx* ctx, int32_t n_keys, const bdf_sort_key* keys, int64_t k, bdf_col** indices);

/* ---- group-by aggregate (the tail of SURVEY 8(f) N4: `Transformation::GroupAggregate`, a panic! in the reference,
 * src/evaluation.rs:73; its intended shape is src/expression.rs:114-221) ---------------------------------------------------
 * Rows are grouped by ONE numeric key column; every value column is folded per group with the aggregates of
 * AggregateFunctions (sum: wrapping for integers, double accumulation for floats; count of valid slots; min / max for integers).
 * Groups come out in ascending key order, the null key (one group) last -- the order of DataFrame::sort; NaN keys form one
 * group after every number, -0.0 and 0.0 are one group.  Results: one chunk per column, n_groups rows; sum (dtype of the value
 * column, never null: an all-null group sums to 0 like AggregateFunctions::sum), count (Int64), min / max (NULL for a group
 * without a valid value; not produced for float columns -- T::Native: Ord -- the pointers are NULL then). */
typedef struct { bdf_col *sum, *count, *min, *max; } bdf_group_out;
int  bdf_group_aggregate_dev(bdf_ctx* ctx, const bdf_col* key, int32_t n_values, const bdf_col* const* values, bdf_col** out_keys,
                             bdf_group_out* out /* n_values */, int64_t* n_groups);

/* ---- group-by over several key columns (`GroupAggregate(Vec<String>, Vec<Aggregation>)`; the planned schema is
 * Dataset::try_aggregate, src/expression.rs:114-221; the functions are AggregateFunction, :696-710) ---------------------------
 * Groups.  Rows are grouped by the tuple of 1..16 numeric key columns.  Per key column: nulls form one value, all NaNs are one
 *   value, -0.0 == 0.0.
 * Group order.  The order DataFrame::sort gives with every criterion ascending: lexicographic over the keys, and within each
 *   key the null after every value (NaN after every number).  With one key this is the order of bdf_group_aggregate_dev.
 * Output keys.  n_keys columns, each one chunk of n_groups rows, null where that key is null.
 * Aggregations.  0..64 (value column, function) pairs -- what Vec<Aggregation> flattens to; every result is one chunk of
 *   n_groups rows and a new column the caller frees:
 *   SUM             dtype of x; integers wrap, floats accumulate in double with a fixed fold order.  Never NULL.
 *   COUNT           Int64: the number of valid slots.
 *   MIN / MAX       dtype of x; NULL for a group without a valid value.  Floats are ordered by IEEE totalOrder after every
 *                   NaN is made the positive quiet NaN: -0.0 < +0.0, NaN above +inf (where the sort puts NaN).  MAX is NaN if
 *                   the group holds a NaN, MIN is NaN only if every valid value is NaN.
 *   AVG             Float64: the sum of the valid values, accumulated in double in the group's fixed fold order, over the count;
 *                   NULL when the count is 0 (the None of AggregateFunctions::avg).  Int64 / UInt64 columns are refused
 *                   (BDF_UNSUPPORTED "avg needs f64: From<T::Native>", as bdf_avg).
 *   FIRST / LAST    dtype of x: the value at the first / last row of the group in the caller's row order (chunk order, then
 *                   row; the stable sort keeps it inside a group); NULL when that row's value is null (positional, like
 *                   pandas first(skipna=False): nulls are not skipped).
 *   COUNT_DISTINCT  Int64: the number of distinct valid values in the group, equality as for keys; nulls are not counted.
 *                   Costs one more stable sort of all rows per COUNT_DISTINCT aggregation.
 * Deterministic: the same inputs give the same bits, hot keys included (no atomics on values).
 * Departures from the planned schema, on purpose: counts come back as Int64 (the frame layer casts them to the planned UInt32,
 *   as for bdf_group_aggregate_dev); avg stays Float64 where try_aggregate types it as x (a mean truncated to an integer is
 *   not a mean, and AggregateFunctions::avg returns f64).
 * Errors: n_keys outside 1..16, n_aggs outside 0..64, a null pointer -> BDF_INVALID; a non-numeric key or value column, an
 *   unknown function, avg of Int64 / UInt64 -> BDF_UNSUPPORTED; columns of different lengths -> BDF_LENGTH_MISMATCH; a
 *   multi-GPU context (rows change chunks, as for sort / take / filter) -> BDF_UNSUPPORTED; more than 2^32-1 rows -> the
 *   sort's BDF_UNSUPPORTED.  On failure nothing is returned and nothing leaks. */
/* The statistical functions (section "statistical aggregates" below) per group:
 *   KURTOSIS / SKEWNESS / STDDEV / VARIANCE / STDDEV_POP / VAR_POP   Float64: the statistic of the group's moment record, NULL where
 *                   it is None.  Any numeric x (Int64 / UInt64 included).  The record is folded per group by the fold paths and the
 *                   fixed order of SUM (a one-value record merged per valid value; moments.cuh), then one kernel derives the statistic.
 *   SUM_DISTINCT    dtype of x: the sum of the group's distinct valid values (equality as COUNT_DISTINCT), which come out of the same
 *                   second sort in ascending order and are folded with SUM's fold (integers wrap, floats in double from +0.0, rounded
 *                   once).  Never NULL: a group without a valid value sums to 0.  A NaN among them makes the sum NaN. */
typedef enum { BDF_GROUP_SUM = 0, BDF_GROUP_MAX, BDF_GROUP_MIN, BDF_GROUP_AVG, BDF_GROUP_COUNT, BDF_GROUP_COUNT_DISTINCT, BDF_GROUP_FIRST,
               BDF_GROUP_LAST, BDF_GROUP_KURTOSIS, BDF_GROUP_SKEWNESS, BDF_GROUP_STDDEV, BDF_GROUP_SUM_DISTINCT, BDF_GROUP_VARIANCE,
               BDF_GROUP_STDDEV_POP, BDF_GROUP_VAR_POP,
               BDF_GROUP_MEDIAN = 32, BDF_GROUP_MODE } bdf_group_fn;   /* AggregateFunction order and the population forms; 32..: the distributions */
/* The distribution functions (section "distributions" below) per group, after the second sort of COUNT_DISTINCT.  They are not members of
 * AggregateFunction, so they start a block of their own at 32 and 15..31 stay unknown function ids (BDF_UNSUPPORTED):
 *   MEDIAN  Float64: the percentile at p = 0.5 of the group's valid values, by the whole-column rule; NULL without a valid value.
 *   MODE    dtype of x: the group's most frequent valid value by the whole-column rule; NULL without a valid value. */
typedef struct { const bdf_col* column; int32_t function; } bdf_group_agg;
int  bdf_group_by_dev(bdf_ctx* ctx, int32_t n_keys, const bdf_col* const* keys, int32_t n_aggs, const bdf_group_agg* aggs,
                      bdf_col** out_keys /* n_keys */, bdf_col** out /* n_aggs */, int64_t* n_groups);
/* Lists per group (ArrayFunction::CollectList / CollectSet, src/expression.rs; Spark's collect_list / collect_set, made deterministic).
 * bdf_group_by_lists_dev is bdf_group_by_dev that also takes the two list builders, all in one call over ONE sort of the keys.  A
 * collect aggregation writes out_lists[j] and sets out[j] = NULL; every other aggregation writes out[j] and sets out_lists[j] = NULL.
 * bdf_group_by_dev keeps refusing ids 48 and 49 (BDF_UNSUPPORTED): its outputs cannot hold a list.  Keys, value columns, group order
 * and errors are those of bdf_group_by_dev.  Every list result has ONE chunk of n_groups lists, no NULL list and no null element:
 *   COLLECT_LIST  The valid values of the group in row order (chunk order, then row).  Null values are skipped; a group without a
 *                 valid value gives a valid EMPTY list.
 *   COLLECT_SET   The distinct valid values of the group, ascending in DataFrame::sort's order (NaN greatest).  Equality is that of
 *                 COUNT_DISTINCT: all NaNs are one value, -0.0 == 0.0; the bits kept are those of the value's first occurrence in
 *                 row order.  Empty and null rules as COLLECT_LIST.  Costs the second sort of COUNT_DISTINCT, once per value column
 *                 however many COLLECT_SET aggregations name it.
 * More than 2^31 - 1 elements in one result -> BDF_UNSUPPORTED (Int32 offsets).  On failure nothing is returned and nothing leaks. */
typedef enum { BDF_GROUP_COLLECT_LIST = 48, BDF_GROUP_COLLECT_SET } bdf_group_list_fn;   /* function ids of bdf_group_agg: a block of their own */
typedef struct bdf_list bdf_list;
int  bdf_group_by_lists_dev(bdf_ctx* ctx, int32_t n_keys, const bdf_col* const* keys, int32_t n_aggs, const bdf_group_agg* aggs,
                            bdf_col** out_keys /* n_keys */, bdf_col** out /* n_aggs */, bdf_list** out_lists /* n_aggs */, int64_t* n_groups);

/* ---- equi-join (Transformation::Join -> DataFrame::join, src/dataframe.rs:626-719; the body of calc_equijoin_indices,
 * src/functions/join.rs:19-137) ------------------------------------------------------------------------------------------------
 * Criterion k is the pair (left_keys[k], right_keys[k]), 1..16 of them, numeric.  The result is two UInt32 columns of n_rows rows,
 * one chunk each: row numbers that count through the chunks of each side, NULL = no partner.  They feed bdf_take_dev directly, the
 * way DataFrame::join feeds Column::take.
 * Match.  A left row and a right row match when, for every criterion, both slots are valid and their values are equal.  Equality is
 *   the key equality of sort and group-by: all NaNs are equal, -0.0 == 0.0.  A row with a null in any criterion matches nothing.
 * Order (fixed, so the result is deterministic):
 *   INNER, LEFT  left rows in row order; each left row's matches in ascending right row order.  LEFT: a left row without a match
 *                appears once, in its place, with a NULL right index (null-key rows count as having no match).
 *   RIGHT        exactly LEFT with the sides swapped, and the two output columns swapped back: right rows in row order.
 *   FULL         the LEFT output, then every right row no left row matched, in right row order, with a NULL left index.
 * Departures from the reference, on purpose:
 *   1. pair order: as above, instead of HashMap iteration order;
 *   2. null keys: the reference hashes a null-key row under its truncated key bytes, so null rows can match each other, and also
 *      appends the row again as unmatched (a LEFT join can list it twice); here a null-key row never matches and appears once;
 *   3. FULL: the reference's FullJoin arm (join.rs:109-133) emits only the matched pairs and the null-key rows, dropping every
 *      unmatched row whose key is valid; here FULL is the SQL full outer join;
 *   4. float keys: the reference compares raw bytes (-0.0 != 0.0); here floats follow the key equality above (Postgres's too);
 *   5. zero criteria: in the reference every row then matches every row (a cross join); here it is refused.
 * Errors (nothing is returned and nothing leaks): n_keys outside 1..16 ("Join criteria cannot be empty" for 0) or a null pointer
 *   -> BDF_INVALID; an unknown join type or a non-numeric key -> BDF_UNSUPPORTED; a criterion whose two columns have different
 *   dtypes -> BDF_UNSUPPORTED "Join columns must have compatible types" (the text of try_join); key columns of one side with
 *   different lengths -> BDF_LENGTH_MISMATCH; a side of more than 2^32-1 rows -> the sort's BDF_UNSUPPORTED; a multi-GPU context
 *   -> BDF_UNSUPPORTED (as sort / take / filter / group-by); an output that does not fit in device memory -> BDF_OOM.
 * Existence joins (Spark's left_semi / left_anti; not in the reference, whose JoinType has the first four):
 *   LEFT_SEMI    every left row that has at least one match, once, however many partners it has;
 *   LEFT_ANTI    every other left row, rows with a null in any criterion included (a null key matches nothing: Spark's left_anti
 *                for an equi-join, not SQL's NOT IN).
 *   *left_indices is one UInt32 chunk without nulls: left row numbers in ascending order, *n_rows of them.  No right indices are
 *   made: right_indices may be NULL, and if it is not, *right_indices is set to NULL.  Match rules and errors are those above. */
typedef enum { BDF_JOIN_LEFT = 0, BDF_JOIN_RIGHT, BDF_JOIN_INNER, BDF_JOIN_FULL, BDF_JOIN_LEFT_SEMI, BDF_JOIN_LEFT_ANTI } bdf_join_type;   /* JoinType order, then the existence joins */
int  bdf_join_indices_dev(bdf_ctx* ctx, int32_t join_type, int32_t n_keys, const bdf_col* const* left_keys, const bdf_col* const* right_keys,
                          bdf_col** left_indices, bdf_col** right_indices, int64_t* n_rows);

/* ---- as-of join (pandas' merge_asof, polars' join_asof, DuckDB's ASOF JOIN; not in the reference) ----------------------------------
 * For every left row, one right row: the last one at or before its `on` key (BACKWARD), the first one at or after it (FORWARD), or the
 * nearer of those two (NEAREST), among the right rows whose 0..16 `by` keys equal the left row's.
 * Output.  *right_indices: one UInt32 chunk of as many rows as the left side; row i belongs to left row i (left order is kept, so the
 *   left columns need no take) and holds a right row number counting through the chunks, NULL when the row has no partner.  Take the
 *   right columns with bdf_take_dev / bdf_list_take_dev.
 * Candidates of left row i: the right rows j whose every `by` pair is valid on both sides and equal under the join's key equality (all
 *   NaNs equal, -0.0 == 0.0), and whose right_on[j] is valid and not NaN.  A left row whose `on` is null or NaN, or one of whose `by`
 *   keys is null, gets NULL.
 * Choice.  Keys compare in the sort's order, -0.0 == 0.0.  With l the left key and r the right keys:
 *   BACKWARD  among the candidates with r <= l (r < l without exact matches) the greatest r; of equal r the LAST in right row order;
 *   FORWARD   among the candidates with r >= l (r > l) the least r; of equal r the FIRST in right row order;
 *   NEAREST   b = the BACKWARD pick, f = the FORWARD pick: the one that exists, else b when l - r_b <= r_f - l (ties go backward), else f.
 * Tolerance (has_tolerance != 0): the pick becomes NULL when its distance is greater than the tolerance.  Integer and temporal keys:
 *   `tolerance`, in the key's own units; the distance is exact (INT64_MAX against INT64_MIN is 2^64 - 1).  Float32 / Float64 keys:
 *   `tolerance_f` (may be +inf); the distance is (double)l - (double)r or the reverse, rounded once, Float32 widened exactly; equal keys,
 *   infinities included, are at distance 0.
 * Departures from pandas, on purpose: neither side needs to be sorted; left order is kept; null and NaN keys simply match nothing
 *   (pandas refuses them).
 * Errors (nothing is returned and nothing leaks): n_by outside 0..16, a null pointer, a negative or NaN tolerance -> BDF_INVALID; an
 *   unknown direction, a non-numeric or Boolean key -> BDF_UNSUPPORTED; an `on` or `by` pair of different dtypes -> BDF_UNSUPPORTED
 *   "Join columns must have compatible types"; key columns of one side with different lengths -> BDF_LENGTH_MISMATCH; more than
 *   2^32-1 right rows -> the sort's BDF_UNSUPPORTED; a multi-GPU context -> BDF_UNSUPPORTED.
 * The right side is sorted once by (by..., on), stably; every left row then binary-searches its `by` run and, inside it, its `on` key,
 *   reading the left chunks in place.  The result does not depend on timing (no atomics on results). */
typedef enum { BDF_ASOF_BACKWARD = 0, BDF_ASOF_FORWARD, BDF_ASOF_NEAREST } bdf_asof_direction;
typedef struct {
    int32_t direction;            /* bdf_asof_direction */
    int32_t allow_exact_matches;  /* 1: <= / >= ; 0: < / > */
    int32_t has_tolerance;
    int64_t tolerance;            /* integer and temporal on-keys, in the key's own units, >= 0 */
    double  tolerance_f;          /* Float32 / Float64 on-keys, >= 0, may be +inf */
} bdf_asof_spec;
int  bdf_join_asof_dev(bdf_ctx* ctx, const bdf_col* left_on, const bdf_col* right_on, int32_t n_by, const bdf_col* const* left_by,
                       const bdf_col* const* right_by, const bdf_asof_spec* spec, bdf_col** right_indices);

/* ---- distinct rows and set operations (pandas' duplicated / drop_duplicates / concat; Spark's distinct, dropDuplicates, union,
 * intersect, intersectAll, subtract, exceptAll; not in the reference) --------------------------------------------------------------
 * Every operation is a Boolean mask over the (left) rows, to be applied with bdf_filter_dev / bdf_list_filter_dev: the result keeps
 * the caller's row order and needs no second sort.
 * Equality.  Two rows are equal when every key is equal under group-by's equality: nulls equal each other, all NaNs are one value,
 *   and -0.0 == 0.0.
 * Keys.  1..16 key columns per side, each one of the ten numeric types or Boolean.  Boolean keys are accepted by these entries only:
 *   inside them they are widened to one byte per row (bdf_bool_widen_dev); bdf_sort_indices_dev and bdf_group_by_dev still refuse them.
 * bdf_duplicated_dev  *mask: one Boolean slot per row, no nulls, chunked like the keys; true for the rows pandas' duplicated(keep=...)
 *   marks: KEEP_FIRST every row of a run of equal rows except its first in row order; KEEP_LAST every row except its last; KEEP_NONE
 *   every row of a run longer than one.
 * bdf_set_op_dev  *mask: one Boolean slot per LEFT row, no nulls, chunked like left[0]; true = kept.  In a run of equal rows with cl
 *   left and cr right rows, the run keeps its first q left rows in row order:
 *     INTERSECT       q = cl > 0 && cr > 0 ? 1 : 0
 *     INTERSECT_ALL   q = min(cl, cr)
 *     EXCEPT          q = cr == 0 ? 1 : 0          (Spark's subtract: distinct)
 *     EXCEPT_ALL      q = max(cl - cr, 0)
 *   Row counts and row order follow Spark; which copies are kept (the earliest) is this library's definition, so the result is
 *   deterministic.  Kept rows keep their own bits: when the first occurrence is -0.0, the result holds -0.0.
 * bdf_concat_dev / bdf_list_concat_dev  the chunks of cols[0], then those of cols[1], and so on, copied device to device; bitmaps
 *   start at bit 0 of every result chunk.  All inputs must have one dtype (child dtype for lists), else BDF_UNSUPPORTED.
 * bdf_bool_widen_dev  a Boolean column as UInt8 0 / 1, chunked like it, nulls kept: a Boolean payload column goes through
 *   bdf_filter_dev this way, and bdf_compare_dev(NE, 0) turns it back.
 * Errors (nothing is returned and nothing leaks): n_keys outside 1..16, n < 1, a null pointer, an unknown keep or op -> BDF_INVALID; a
 *   non-numeric key -> BDF_UNSUPPORTED; a key position whose left and right dtypes differ -> BDF_UNSUPPORTED "Union can only be
 *   performed on tables with compatible column types"; key columns of one side with different lengths -> BDF_LENGTH_MISMATCH; more
 *   than 2^32-1 rows in the sort (left + right for the set operations) -> the sort's BDF_UNSUPPORTED; a multi-GPU context ->
 *   BDF_UNSUPPORTED, as for sort / group-by / join.
 * The keys are sorted stably once (a set operation sorts the left rows, then the right rows, as one column), so a run's left rows
 *   come first and its left count is the distance from the run start to its first right row.  Launch records: BDF_K_GROUP. */
typedef enum { BDF_KEEP_FIRST = 0, BDF_KEEP_LAST, BDF_KEEP_NONE } bdf_keep;
typedef enum { BDF_SETOP_INTERSECT = 0, BDF_SETOP_INTERSECT_ALL, BDF_SETOP_EXCEPT, BDF_SETOP_EXCEPT_ALL } bdf_setop;
int  bdf_duplicated_dev(bdf_ctx* ctx, int32_t n_keys, const bdf_col* const* keys, int32_t keep, bdf_col** mask);
int  bdf_set_op_dev(bdf_ctx* ctx, int32_t op, int32_t n_keys, const bdf_col* const* left, const bdf_col* const* right, bdf_col** mask);
int  bdf_concat_dev(bdf_ctx* ctx, int32_t n, const bdf_col* const* cols, bdf_col** out);
int  bdf_list_concat_dev(bdf_ctx* ctx, int32_t n, const bdf_list* const* lists, bdf_list** out);
int  bdf_bool_widen_dev(bdf_ctx* ctx, const bdf_col* in, bdf_col** out);

/* ---- window functions (WindowFunctions, src/functions/window.rs:1-11; WindowSpec, src/window.rs:8-22: stubs in the reference) ----
 * One call computes n_calls window columns that share one specification, so the rows are sorted once.
 * Rows and order.  Partitions are the runs of equal tuples of the 0..16 numeric partition_by columns; within a partition rows are
 *   ordered by the 0..16 numeric order_by columns, each ascending or descending.  Both use the key rules of sort, group-by and join:
 *   nulls are one value and come last in both directions (as DataFrame::sort puts them), all NaNs are one value greater than every
 *   number, -0.0 == 0.0.  Peers are rows of a partition with equal order tuples.  Ties are broken by the caller's row order (chunk
 *   order, then row), which the stable sort keeps, so ROW_NUMBER, LAG / LEAD and the ROWS frame are deterministic where SQL leaves
 *   them unspecified.
 * Output.  One chunk per call, in the caller's row order: row r of every output belongs to input row r (a window adds columns to a
 *   frame, it does not reorder it).  Every output is a new column the caller frees.
 * Ranking functions (column == NULL; never NULL):
 *   ROW_NUMBER    UInt32: the 1-based position in the partition.
 *   RANK          UInt32: 1 + the number of rows of the partition before the first peer.
 *   DENSE_RANK    UInt32: 1 + the number of distinct peer groups of the partition before this one.
 *   PERCENT_RANK  Float64: (double)(rank - 1) / (double)(partition rows - 1); 0 for a one-row partition.
 *   CUME_DIST     Float64: (double)(rows of the partition up to and including the last peer) / (double)(partition rows).
 *   Both Float64 functions are one IEEE division, so their results are bit-exact.
 * LAG / LEAD (column x of any numeric type, offset k >= 0): x at the row k positions before / after this row in the partition, in the
 *   dtype of x.  A row outside the partition gives the default (default_bits: T::Native of x in the low bytes, as bdf_agg4) when
 *   has_default, else NULL; a row inside whose x is null gives NULL (RESPECT NULLS).  k = 0 is x itself.
 * Aggregates of x over a frame: ROWS = the first row of the partition through the current row; RANGE = through the current row's last
 *   peer (SQL's default frame with an ORDER BY); PARTITION = the whole partition (SQL's default without one; also writes a group total
 *   back onto every row).  Types and null rules are those of bdf_group_by_dev:
 *   SUM    dtype of x; integers wrap, floats accumulate in double and are rounded once.  Never NULL: a frame without a valid value sums
 *          to 0, like AggregateFunctions::sum (SQL would give NULL).
 *   COUNT  Int64: the valid slots of the frame.
 *   MIN / MAX  dtype of x; NULL without a valid value; floats by the totalOrder rule of bdf_group_by_dev.
 *   AVG    Float64: the double sum over the count; NULL when the count is 0; Int64 / UInt64 refused.
 * Degenerate specifications: without order columns every row of a partition is a peer (rank 1; ROWS follows row order); without
 *   partition columns the whole column is one partition; with neither, nothing is sorted or gathered for ROWS: the aggregates are
 *   row-order running aggregates over the caller's chunks read in place.
 * Deterministic: the same inputs give the same bits, float sums included (a segmented scan over a fixed tile decomposition; no atomics
 *   on values).
 * Errors (nothing is returned and nothing leaks): n_partition or n_order outside 0..16, n_calls outside 0..64, a null pointer, a
 *   negative offset, a ranking call with a column, a LAG / LEAD / aggregate call without one, or a call without any column at all (no
 *   keys and only ranking functions: no rows to number) -> BDF_INVALID; an unknown function or frame, a non-numeric column, AVG of
 *   Int64 / UInt64 ("avg needs f64: From<T::Native>"), more than 2^32-1 rows (the sort's message), a multi-GPU context ->
 *   BDF_UNSUPPORTED; columns of different lengths -> BDF_LENGTH_MISMATCH. */
/* Bounded frames (WindowSpec's rows_between / range_between).  A zero-initialised call's new fields change nothing above.
 * Frame resolution.  Every frame is a range of sorted positions [s, e] inside the current row's partition [ps, pe]; s > e is empty.
 *   ROWS_BETWEEN   s = max(ps, i + start), e = min(pe, i + end) in saturating arithmetic; an UNBOUNDED start is ps, an UNBOUNDED end pe.
 *   RANGE_BETWEEN  exactly one order column.  With v the current row's key, an ascending key gives the rows whose key k is valid, not
 *                  NaN and v + start <= k <= v + end; a descending key v - end <= k <= v - start (PRECEDING always points towards the
 *                  start of the sorted order).  As positions: s is the first row of the partition's valid non-NaN keys that meets the
 *                  start bound (the row after them when none does), e the last that meets the end bound (the row before them when
 *                  none does).  Integer (and temporal) keys use start / end and compare exactly, with no wrap: a bound outside the
 *                  type's range takes in every row on that side, and an unsigned key accepts a negative start.  Float keys use
 *                  start_f / end_f and compare with (double)v + start_f rounded once; -0.0 == 0.0 and +-inf keys follow IEEE
 *                  arithmetic.  When the current key is null or NaN, an offset bound is the first (start) or last (end) row of the
 *                  row's own peer run.  An UNBOUNDED bound is always the partition's edge, so UNBOUNDED FOLLOWING includes the null
 *                  and NaN keys where they sort.
 *   Offsets follow Spark's rowsBetween / rangeBetween: negative = PRECEDING, 0 = CURRENT ROW, positive = FOLLOWING; INT64_MIN /
 *   INT64_MAX (-inf / +inf for start_f / end_f) = UNBOUNDED.
 *   Equivalent specifications run the existing frame and give its bits: ROWS_BETWEEN(UNBOUNDED, 0) = ROWS, ROWS_BETWEEN(UNBOUNDED,
 *   UNBOUNDED) = PARTITION, RANGE_BETWEEN(UNBOUNDED, 0) = RANGE, RANGE_BETWEEN(UNBOUNDED, UNBOUNDED) = PARTITION.
 * Aggregates over a bounded frame keep the types and null rules above: an empty frame gives SUM 0, COUNT 0 and NULL for MIN, MAX and
 *   AVG.  COUNT, integer SUM (wrapping) and MIN / MAX (totalOrder for floats) are exact.  Float SUM and every AVG stay within
 *   16 * log2(max(k, 2)) * 2^-53 * sum(|x|) over the frame's k rows, plus the final f32 rounding, and are the same bits on every run
 *   and under any chunking: each frame is combined from a radix-32 hierarchy of block prefixes and suffixes, every term a sum over part
 *   of the frame, in an order fixed by (s, e); the cost per row does not grow with the frame's width.  A float prefix-sum difference
 *   does not meet this bar, and neither does a sliding add / subtract: their error grows with the magnitudes of the partition, not of
 *   the frame.  (Integer sums could use prefix differences: wrapping arithmetic makes them exact.)
 * FIRST_VALUE / LAST_VALUE / NTH_VALUE (column x of any numeric type; the output has x's dtype; any frame, the three above included).
 *   RESPECT NULLS (ignore_nulls = 0): x at s, at e, or at s + n - 1 when that is at most e (n = offset); NULL when that row's x is null
 *   or the frame is empty.  IGNORE NULLS: the first, last or n-th valid x in [s, e]; NULL when the frame holds fewer valid values.
 * Errors of bounded frames (BDF_INVALID; nothing is returned and nothing leaks): start > end; a start of UNBOUNDED FOLLOWING or an end
 *   of UNBOUNDED PRECEDING; a NaN float offset; RANGE_BETWEEN without exactly one order column; NTH_VALUE with n < 1; ignore_nulls on a
 *   function other than the three value functions. */
typedef enum { BDF_WIN_ROW_NUMBER = 0, BDF_WIN_RANK, BDF_WIN_DENSE_RANK, BDF_WIN_PERCENT_RANK, BDF_WIN_CUME_DIST,
               BDF_WIN_LAG, BDF_WIN_LEAD, BDF_WIN_SUM, BDF_WIN_COUNT, BDF_WIN_MIN, BDF_WIN_MAX, BDF_WIN_AVG,
               BDF_WIN_FIRST_VALUE, BDF_WIN_LAST_VALUE, BDF_WIN_NTH_VALUE } bdf_window_fn;
typedef enum { BDF_FRAME_ROWS = 0, BDF_FRAME_RANGE, BDF_FRAME_PARTITION, BDF_FRAME_ROWS_BETWEEN, BDF_FRAME_RANGE_BETWEEN } bdf_window_frame;
typedef struct {
    int32_t function;        /* bdf_window_fn */
    int32_t frame;           /* bdf_window_frame; aggregates and value functions */
    const bdf_col* column;   /* LAG / LEAD / aggregates / value functions; NULL for the five ranking functions */
    int64_t offset;          /* LAG / LEAD, >= 0; NTH_VALUE's n, >= 1 */
    uint64_t default_bits;   /* LAG / LEAD: T::Native of `column` in the low bytes (as bdf_agg4) */
    int32_t has_default;
    int32_t ignore_nulls;    /* FIRST_VALUE / LAST_VALUE / NTH_VALUE: IGNORE NULLS */
    int64_t start, end;      /* ROWS_BETWEEN, and RANGE_BETWEEN over an integer or temporal order key: signed offsets */
    double start_f, end_f;   /* RANGE_BETWEEN over a Float32 / Float64 order key; -inf / +inf = UNBOUNDED */
} bdf_window_call;
int  bdf_window_dev(bdf_ctx* ctx, int32_t n_partition, const bdf_col* const* partition_by, int32_t n_order, const bdf_sort_key* order_by,
                    int32_t n_calls, const bdf_window_call* calls, bdf_col** out /* n_calls */);

/* ---- statistical aggregates (AggregateFunctions::{variance, stddev, skewness, kurtosis, count_distinct, sum_distinct}: empty stubs in
 * the reference, src/functions/aggregate.rs:81,94-102, "TODO population and sample stddevs / variances"; the names follow Spark, and so
 * do the definitions) -----------------------------------------------------------------------------------------------------------------
 * Input.  A column of any of the ten numeric types; every valid value is read `as f64` (Int64 / UInt64 beyond 2^53 round to nearest,
 *   Float32 is exact); nulls are skipped.  Unlike avg, Int64 / UInt64 are accepted: avg's refusal mirrors its declared bound
 *   f64: From<T::Native>, the stubs declare none, and the CSV reader infers Int64 for every integer column.
 * The moment record of the valid values x1..xn: count = n, mean, and the central sums m2 = sum (x - mean)^2, m3 = sum (x - mean)^3,
 *   m4 = sum (x - mean)^4 -- computed in one pass, as accurately as two passes would (never as sum x^2 - n mean^2).  If every valid
 *   value is equal, mean is exactly that value and m2 = m3 = m4 = 0 exactly.  If any valid value is NaN or +-inf, mean, m2, m3 and m4
 *   are NaN.  Overflow of an intermediate follows IEEE arithmetic (inf / NaN) and is not an error.
 * The statistics, each from the record with exactly this operation order (n = (double)count, no FMA contraction, IEEE sqrt):
 *   VAR_POP = m2 / n                 VARIANCE = m2 / (n - 1)        (sample; Spark's variance)
 *   STDDEV_POP = sqrt(VAR_POP)       STDDEV = sqrt(VARIANCE)        (sample; Spark's stddev)
 *   SKEWNESS = (sqrt(n) * m3) / (m2 * sqrt(m2))                     KURTOSIS = (n * m4) / (m2 * m2) - 3   (excess)
 *   None (is_some = 0; NULL per group): every statistic when count = 0; the sample forms also when count = 1; SKEWNESS and KURTOSIS
 *   also when m2 = 0 (Spark 3 with null on divide by zero).
 * Multi-GPU: every GPU computes the record of its rows; the records are combined with bdf_moments_merge in rank order (on a
 *   communicator they are all-gathered first), so every rank returns the same bits, and a fleet or communicator of one GPU returns
 *   the one-GPU bits.
 * count_distinct / sum_distinct use the key equality of sort, group-by and join (all NaNs are one value, -0.0 == 0.0); nulls are not
 *   counted.  count is Int64; sum has the dtype of x (T::Native bits in the low bytes, zero-padded, as bdf_agg4): integers wrap, floats
 *   are the distinct values accumulated in double in ascending value order from +0.0 (group-by's SUM fold) and rounded once.  Never
 *   None: no valid values sum to 0, like AggregateFunctions::sum.  A NaN among the values makes the sum NaN.  The values are sorted
 *   (the group-by's second sort with the whole column as one group), so both need every row on one GPU: on either kind of multi-GPU
 *   context they are BDF_UNSUPPORTED.
 * Deterministic: the same inputs with the same chunking give the same bits (no atomics on values; fold orders depend only on shapes).
 * Errors (nothing is written, nothing leaks): a null pointer or an unknown bdf_stat -> BDF_INVALID; a non-numeric or Boolean column ->
 *   BDF_UNSUPPORTED. */
typedef struct { int64_t count; double mean, m2, m3, m4; } bdf_moment_rec;
typedef struct { int64_t count; uint64_t sum; /* T::Native bits, as bdf_agg4 */ } bdf_distinct_rec;
typedef enum { BDF_STAT_VARIANCE = 0, BDF_STAT_VAR_POP, BDF_STAT_STDDEV, BDF_STAT_STDDEV_POP, BDF_STAT_SKEWNESS, BDF_STAT_KURTOSIS } bdf_stat;
int  bdf_moments(bdf_ctx* ctx, int dtype, int64_t n_chunks, const bdf_view* in, bdf_moment_rec* out);   /* host in */
int  bdf_moments_dev(bdf_ctx* ctx, const bdf_col* in, bdf_moment_rec* out);
/* No context, no GPU: the formulas above, and the pairwise merge (Chan / Pebay, moments.cuh) the library itself uses across ranks. */
int  bdf_moments_stat(const bdf_moment_rec* m, int stat, double* out, int32_t* is_some);
int  bdf_moments_merge(const bdf_moment_rec* a, const bdf_moment_rec* b, bdf_moment_rec* out);
int  bdf_distinct(bdf_ctx* ctx, int dtype, int64_t n_chunks, const bdf_view* in, bdf_distinct_rec* out);   /* host in */
int  bdf_distinct_dev(bdf_ctx* ctx, const bdf_col* in, bdf_distinct_rec* out);

/* ---- distributions (Column::hist and Column::uniques, src/table.rs:244-345; Spark's percentile, median and mode for the
 * "mode, median" of the reference's README) -------------------------------------------------------------------------------------
 * Input.  A column of any of the ten numeric types; nulls are skipped.  Keys are the sort's (all NaNs are one value, greater than every
 *   number; -0.0 == 0.0).
 * Percentile (Spark's exact percentile): n = the valid values, pos = (double)(n - 1) * p, lo = floor(pos), hi = ceil(pos); a and b are
 *   the lo-th and hi-th valid values in key order, read `as f64` (Int64 / UInt64 beyond 2^53 round to nearest).  The result is a when
 *   lo == hi or a == b, else (hi - pos) * a + (pos - lo) * b -- exactly these IEEE operations, no FMA.  A selected -0.0 is +0.0, and
 *   every NaN result (a selected NaN, or -inf and +inf interpolated) is the positive quiet NaN: the result is a function of the keys,
 *   whichever rows held them.  median is p = 0.5.  is_some[i] = 0 (out[i] = 0) when the column has no valid value.
 *   Whole columns are selected, not sorted: an MSD radix select over the keys (a digit histogram of the column read in place, then
 *   only the keys of the chosen buckets, compacted into a scratch of at most the valid values).
 * Mode: the valid value with the most rows; ties go to the smallest in key order (Spark 4's mode(col, deterministic => true)).  bits
 *   is the value of the class's first row in the caller's row order (chunk order, then row), T::Native in the low bytes as bdf_agg4
 *   (so a class of -0.0 and 0.0 returns whichever came first, as sum_distinct's representative); freq is the class's row count.
 *   is_some = 0 (bits = freq = 0) without a valid value.
 * Uniques: the distinct valid values in ascending key order, each class represented as mode represents it, as one chunk without
 *   nulls; counts[i] (Int64) is the number of rows of class i.  Departures from Column::uniques: (1) the order is ascending, not
 *   HashSet order; (2) nulls are skipped (the reference reads the bytes of null slots); (3) NaN is one value (the reference panics in
 *   noisy_float::r64); (4) all ten numeric types, not only Int64 / Float64; (5) Utf8 is not supported (no string columns on the device).
 * Histogram: numpy.histogram's uniform bins, which are the definition (histo_fp's bucket rule is a departure not followed).  Every
 *   value is read `as f64`.  Range: the explicit {lo, hi}, else [min, max] of the valid non-NaN values (a -0.0 bound is +0.0), else
 *   [0, 1] when there is none; lo == hi becomes [lo - 0.5, hi + 0.5].  edges[i] = (double)i * ((hi - lo) / nbins) + lo, two
 *   roundings (np.linspace; when the step rounds to 0: ((double)i / nbins) * (hi - lo) + lo), edges[nbins] = hi.  A value x with
 *   lo <= x <= hi goes to bin i = min((int)((x - lo) / (hi - lo) * nbins), nbins - 1), then numpy's one-step correction: i - 1 when
 *   x < edges[i], else i + 1 when x >= edges[i + 1] and i != nbins - 1.  NaN and values outside an explicit range are not counted.
 *   Departure: numpy refuses a NaN in an automatic range; here NaN is skipped.  Up to 2048 bins are counted per CTA in shared memory,
 *   more with global atomics; either way the counts are exact.
 * bdf_hist_density (no context, no GPU): numpy's density=True, out[i] = ((double)counts[i] / (edges[i + 1] - edges[i])) /
 *   (double)sum(counts) -- NaN everywhere when no value was counted, as numpy.  Column::hist accepts density and ignores it.
 * Deterministic: every result is exact (selected keys, integer counts, one interpolation), so the same rows give the same bits on
 *   every call and under any chunking; atomics only add integers.
 * Errors (nothing is written, nothing leaks): a null pointer, n_p outside 1..1024, a p outside [0, 1] or NaN, nbins outside 1..2^24
 *   -> BDF_INVALID; an explicit range with lo > hi -> BDF_INVALID "max must be larger than min in range parameter.", one that is not
 *   finite -> BDF_INVALID "supplied range of [lo, hi] is not finite"; an automatic range with an infinity -> BDF_INVALID "autodetected
 *   range of [lo, hi] is not finite"; a non-numeric or Boolean column -> BDF_UNSUPPORTED; more than 2^32-1 rows -> the sort's
 *   BDF_UNSUPPORTED; a multi-GPU context of either kind -> BDF_UNSUPPORTED (every row of the column must be on one GPU); a scratch
 *   that does not fit -> BDF_OOM.
 * Launch records: BDF_K_SELECT for the select passes, BDF_K_HIST for the range and count passes. */
int  bdf_percentile(bdf_ctx* ctx, int dtype, int64_t n_chunks, const bdf_view* in, int32_t n_p, const double* p, double* out,
                    int32_t* is_some);   /* host in */
int  bdf_percentile_dev(bdf_ctx* ctx, const bdf_col* in, int32_t n_p, const double* p, double* out, int32_t* is_some);
int  bdf_mode(bdf_ctx* ctx, int dtype, int64_t n_chunks, const bdf_view* in, uint64_t* bits, int64_t* freq, int32_t* is_some);   /* host in */
int  bdf_mode_dev(bdf_ctx* ctx, const bdf_col* in, uint64_t* bits, int64_t* freq, int32_t* is_some);
int  bdf_uniques_dev(bdf_ctx* ctx, const bdf_col* in, bdf_col** values, bdf_col** counts /* may be NULL */);
int  bdf_hist_dev(bdf_ctx* ctx, const bdf_col* in, int32_t nbins, const double* range /* NULL or {lo, hi} */, double* edges /* nbins + 1 */,
                  int64_t* counts /* nbins */);
int  bdf_hist_density(int32_t nbins, const double* edges, const int64_t* counts, double* out);

/* ---- N4: Arrow IPC files either side of the path ---------------------------------------------------------------
 * DataFrame::from_arrow (src/dataframe.rs:391-407: arrow::ipc::reader::FileReader, every RecordBatch -> one chunk per
 * column) and DataFrame::to_arrow (:515-525: arrow::ipc::writer::FileWriter).  The file is mapped and its footer, schema
 * and RecordBatch metadata are decoded by the library itself (Arrow IPC file format, metadata V4/V5, uncompressed,
 * little endian); body buffers are used in place.  Columns of the ten numeric types and Boolean can be read; any other
 * column (strings, lists, structs, dictionaries, temporal types ...) is skipped and reported with dtype -1.
 *   bdf_ipc_open / _close / _describe / _column / _batch_rows / _view need no context (and no GPU);
 *   bdf_ipc_view      a zero-copy bdf_view of one column of one RecordBatch, pointing into the mapping;
 *   bdf_ipc_read      the chosen columns straight to the device, one chunk per RecordBatch (flags: BDF_ASYNC; keep the
 *                     file open until bdf_col_wait / bdf_synchronize then);
 *   bdf_ipc_write_host  write host arrays ([column][batch] views, any offset) as an IPC file (V5, 64-byte aligned bodies);
 *   bdf_ipc_write     device columns (equal chunk structure: chunk b of every column = RecordBatch b) -> IPC file. */
typedef struct bdf_ipc bdf_ipc;
int  bdf_ipc_open(const char* path, bdf_ipc** out);
void bdf_ipc_close(bdf_ipc* file);
int  bdf_ipc_describe(const bdf_ipc* file, int32_t* n_columns, int64_t* n_batches, int64_t* n_rows);
int  bdf_ipc_column(const bdf_ipc* file, int32_t col, const char** name, int32_t* dtype, int32_t* nullable);
int  bdf_ipc_batch_rows(const bdf_ipc* file, int64_t batch, int64_t* rows);
int  bdf_ipc_view(const bdf_ipc* file, int64_t batch, int32_t col, bdf_view* out);
int  bdf_ipc_read(bdf_ctx* ctx, const bdf_ipc* file, int32_t n_cols, const int32_t* cols, int flags, bdf_col** out /* n_cols */);
/* A subset of the RecordBatches, in the given order (multi-GPU: rank r of N reads batches r, r+N, ... -- SURVEY 8(e)). */
int  bdf_ipc_read_batches(bdf_ctx* ctx, const bdf_ipc* file, int32_t n_cols, const int32_t* cols, int64_t n_batches,
                          const int64_t* batches, int flags, bdf_col** out /* n_cols */);
int  bdf_ipc_write_host(const char* path, int32_t n_cols, const char* const* names, const int32_t* dtypes, int64_t n_batches,
                        const bdf_view* const* cols /* [n_cols][n_batches] */);
int  bdf_ipc_write(bdf_ctx* ctx, const char* path, int32_t n_cols, const char* const* names, const bdf_col* const* cols);

/* ---- CSV files straight to the device (DataFrame::from_csv, src/dataframe.rs:349-389; LazyFrame::read(Csv), src/evaluation.rs:328) ----
 * The reference reads with arrow-rs's csv::Reader (ReaderBuilder::infer_schema(max_records).has_header(..).with_batch_size(1024)) over
 * the csv / csv-core crates.  Those crates are not restated from source: the rules below are RECALLED, parity unpinned, except the
 * uk_cities reads the reference tests pin (3 columns, 37 rows, the lat/lng values).
 * Records (csv-core, default configuration): a DFA over bytes with states StartRecord, StartField, InField, InQuoted, QuoteInQuoted.
 *   '"' opens a quoted field only at the start of a field (elsewhere in an unquoted field it is a literal byte); inside quotes ""
 *   is one '"' and a lone '"' closes the quotes; bytes after the close up to the next delimiter / terminator are appended
 *   literally ("ab"cd -> abcd); the delimiter, '\r' and '\n' are literal inside quotes.  A record ends at '\r', '\n' or "\r\n";
 *   runs of terminators are skipped (blank lines make no record).  End of file ends the last record; an unterminated quote at
 *   end of file simply ends the field (csv-core's end-of-input from InQuoted ends the field and the record).  A leading UTF-8
 *   BOM (EF BB BF) is skipped (the csv crate strips it).  Every record must have as many fields as the first one (the reader is
 *   not flexible), else BDF_INVALID "CSV error: record R (line: L, byte: B): found record with N fields, but the previous record
 *   has M fields" (R counts records from 0, the header included; L is 1 + the '\n' bytes before the record; B its byte offset).
 *   With has_header the first record gives the names, else they are column_1, column_2, ...
 * Inference (infer_file_schema) over the first max_records data records (all when max_records < 0): an empty field (unquoted or
 *   "") is a null and adds no type; otherwise, in order: the unquoted value starts with '"' -> Utf8; (?i)^(true)$|^(false)$ ->
 *   Boolean; ^-?(\d+\.\d+)$ -> Float64; ^-?(\d+)$ -> Int64; else Utf8.  Per column: one type -> it; {Int64, Float64} -> Float64;
 *   anything else, a column without any type included -> Utf8.  nullable = an empty field was seen there.  So 1e5, .5, +1 and inf
 *   infer as Utf8.  Departure: \d is ASCII 0-9 here; Rust's regex \d also matches other Unicode digits.
 * Values: an empty field is NULL; otherwise Rust's FromStr of the column type on the unquoted value.  Integers [+-]?[0-9]+, unsigned
 *   types refuse '-' (even -0), overflow is an error.  Floats: [+-]? then digits with an optional '.' and optional [eE][+-]?digits
 *   (1. and .5 parse, . and 1e do not), or inf / infinity / nan in any case; CORRECTLY ROUNDED to the column type (Float32 straight
 *   from the decimal, never through Float64); -nan is NaN with the sign bit.  Boolean: to_lowercase() == "true" / "false".
 *   A failure: BDF_PARSE "Error while parsing value {s} for column {c} at line {l}", s the unquoted value, c the column's index in
 *   the file, l the data record's index from 0 plus 1 with a header (records, not physical lines).  The reported field is the
 *   first the reference would meet: by RecordBatch, then by column in the requested order, then by row.
 * Types: the ten numeric types and Boolean are read; Utf8 (and anything else) is not on the device path: bdf_csv_column reports it
 *   with dtype -1 and bdf_csv_read refuses it (read such columns on the CPU, e.g. arrow's reader with a projection of just them).
 *   An explicit schema gives one dtype per column: 0..9, BDF_BOOL, or BDF_UTF8 / -1 (skipped); any other value -> BDF_UNSUPPORTED.
 * Output: one chunk of batch_size rows per RecordBatch (the last one shorter), null counts set, no validity bitmap in a chunk
 *   without nulls.
 * Departures from the reference, on purpose: (1) from_csv truncates the frame at the first batch that fails to parse (Err(e) =>
 *   has_next = false); here the read fails with BDF_PARSE.  (2) unequal field counts: inside the inferred records the reference
 *   panics (build(..).unwrap()), after them it truncates; here both give BDF_INVALID.  (3) a file without data records (a header
 *   only, or empty) makes the reference panic at batches[0]: BDF_WOULD_PANIC.  (4) ASCII digits, above.
 * Memory: bdf_csv_open keeps the file's bytes and the field index (8 B per field) in HBM until bdf_csv_close and needs about 0.25 B
 *   per file byte more while tokenizing; a read needs its outputs and, when it reads a float column, a list for the float fields
 *   the fast path cannot round, allocated up front: max(65536, float fields / 64) entries of 40 B (at least 2.6 MB, about 0.63 B
 *   per float field).  What does not fit gives BDF_OOM; a failed call leaks nothing.  A multi-GPU context -> BDF_UNSUPPORTED.
 *   Float fields whose rounding the device cannot decide (more than 19 significant digits where the truncation is ambiguous, or an
 *   ambiguous 128-bit product) are rounded exactly on the host (strtod / strtof in the C locale) and written back; bdf_csv_stats
 *   counts them.  More of them than max(65536, float fields / 64) in one read -> BDF_UNSUPPORTED. */
#define BDF_UTF8 11   /* schema entry only: a string column (not read on the device) */
typedef struct { int32_t has_header; uint8_t delimiter; int64_t max_records /* <0: all */; int64_t batch_size; } bdf_csv_options;
typedef struct bdf_csv bdf_csv;
int  bdf_csv_open(bdf_ctx* ctx, const char* path, const bdf_csv_options* options, int32_t n_schema, const int32_t* schema_dtypes /* NULL: infer */,
                  bdf_csv** out);
int  bdf_csv_describe(const bdf_csv* file, int32_t* n_columns, int64_t* n_batches, int64_t* n_rows);
int  bdf_csv_column(const bdf_csv* file, int32_t col, const char** name, int32_t* dtype /* -1 off the path */, int32_t* nullable);
int  bdf_csv_read(bdf_ctx* ctx, const bdf_csv* file, int32_t n_cols, const int32_t* cols, bdf_col** out /* n_cols */);   /* projection */
/* fields in the file; float fields the last read rounded on the host; host time of the file's upload in bdf_csv_open */
int  bdf_csv_stats(const bdf_csv* file, int64_t* n_fields, int64_t* exact_fields, double* upload_ms);
void bdf_csv_close(bdf_ctx* ctx, bdf_csv* file);   /* the context that opened it */

/* ---- CSV files straight from the device (DataFrame::to_csv, src/dataframe.rs:527-543; Evaluate::write(Csv(path, options)),
 * src/evaluation.rs:343) ------------------------------------------------------------------------------------------------------------
 * The reference writes with arrow-rs's csv::Writer over the csv crate.  Neither is restated from source: the rules below are RECALLED,
 * parity unpinned (the reference's own tests only check that the write succeeds).
 * Layout.  A header record with the column names unless has_header = 0, then one record per row in row order (chunk order, then
 *   row); fields separated by the delimiter; every record ends with "\n" (the csv crate's default terminator), the last one too.  A
 *   frame without rows is the header alone (an empty file without one).
 * NULL.  An empty field.  A record of exactly one field that is empty (a one-column frame, a NULL row) is written "" as the csv crate
 *   does -- and as the round trip needs: the reader skips blank lines.
 * Values (Rust's ToString / Display of the native value):
 *   integers (the 8 types)  plain decimal, '-' for negatives (-9223372036854775808, 18446744073709551615);
 *   Boolean                 true / false;
 *   Float32 / Float64       the SHORTEST digit string that reads back to the same value in that type (Float32 as an f32, never via
 *                           f64), the one closest to the exact value when several do; written positionally, never with an exponent:
 *                           1 (not 1.0), 0.1, 100000000000000000000 for 1e20, 0.0000001 for 1e-7, 340282350000000000000000000000000000000
 *                           for f32::MAX; the longest field is 327 bytes (the negative smallest f64 subnormal).  NaN whatever its sign
 *                           or payload, inf, -inf.  -0.0 is written -0: a decision (Rust before 1.53 printed 0), so that the value
 *                           survives a round trip.  Later arrow versions format floats with lexical_core instead (1.0, exponent
 *                           forms); which form the reference's pinned branch used is not known.
 * Header names are quoted as the csv crate's QuoteStyle::Necessary does: a name containing the delimiter, '"', '\r' or '\n' (or the
 *   only, empty, name) is put in quotes with every '"' doubled.  Values never need quotes: the delimiter may not occur in them.
 * Options.  options == NULL: a header and ','.  The reference's plan carries CsvWriteOptions { has_headers, delimiter }
 *   (src/expression.rs:380-384) but Evaluate::write ignores them; here they are honoured (a departure).  Allowed delimiters are bytes
 *   that cannot occur in a formatted value: not NUL, a digit, '-', '.', '"', '\r', '\n' or a letter of NaN / inf / true / false
 *   (N a i n f t r u e l s); any other -> BDF_INVALID.
 * Types.  The ten numeric types and Boolean.  A frame with a Utf8 column is written on the CPU (arrow's writer), as for reading.
 * Reading it back.  With Display an all-integral Float64 column (1, 2) is inferred as Int64 by the reader (the reference behaves the
 *   same); exact round trips need an explicit schema.  With one, every value reads back bit for bit (NaN as a NaN: Display drops its
 *   sign and payload).
 * Input.  As bdf_ipc_write: chunk b of every column has the same length; any other chunk structure -> BDF_LENGTH_MISMATCH.  Any number
 *   of columns.
 * Memory.  The rows go in blocks whose text surely fits a device buffer: two 64 MiB text buffers, the byte offsets of up to 2^21 rows
 *   (16 MiB) and 32 B per (chunk, column) of the column table in HBM; the context's pinned staging slots (6 x 8 MiB, shared with
 *   uploads) carry the text to the file, written with pwrite by the staging threads.  Neither grows with the file.
 * Errors (nothing leaks): a null pointer, n_cols <= 0 or a refused delimiter -> BDF_INVALID; a path that cannot be created or written
 *   -> BDF_INVALID with the OS error text (the file is then incomplete); a multi-GPU context -> BDF_UNSUPPORTED (as the reader). */
typedef struct { int32_t has_header; uint8_t delimiter; } bdf_csv_write_options;
int  bdf_csv_write(bdf_ctx* ctx, const char* path, int32_t n_cols, const char* const* names, const bdf_col* const* cols,
                   const bdf_csv_write_options* options /* NULL: a header and ',' */);

/* ---- list columns and ArrayFunctions (src/functions/array.rs; size / explode: ScalarFunctions stubs, scalar.rs:237,414) ----------
 * Layout.  Arrow List<T> with 32-bit offsets, T one of the ten numeric types, one chunk per RecordBatch.  A bdf_list holds per chunk the
 *   list validity, len + 1 Int32 offsets rebased to start at 0, and the elements as an ordinary bdf_col whose chunk i holds exactly the
 *   elements [offsets[0], offsets[len]) of list chunk i (bdf_list_values lends it out: every column operator works on the elements).
 *   LargeList, nested lists, FixedSizeList and Boolean / Utf8 children are not on the device path (BDF_UNSUPPORTED).
 * bdf_list_view.  The list's offset applies to offsets and validity; `values` is the child array, whose own offset and validity apply
 *   (offsets index the child from values.offset).  Only the elements the lists reference cross PCIe.  A null list whose offsets span
 *   elements is uploaded as it is; every function below ignores those elements.
 * Limits.  Elements per chunk below 2^31 (Int32 offsets), elements per call below 2^32 (the sort's UInt32 row numbers): beyond either,
 *   BDF_UNSUPPORTED.  A list-returning function gives ONE chunk (as take and sort do), so its elements must also stay below 2^31.
 *   A multi-GPU context -> BDF_UNSUPPORTED for every list entry (as sort / take).
 * Rules shared by every function:
 *   Equality is the key equality of sort, group-by, join and count_distinct: integers exact, all NaNs one value, -0.0 == 0.0 (a
 *     deliberate departure from the reference's PartialEq, for NaN only).
 *   The search value is T::Native bits in the low bytes of a uint64_t (as bdf_window_call.default_bits).
 *   A null list gives a valid EMPTY list in every list-returning function (the reference's ListBuilder::append(true) on a.is_null(i)).
 *   Deterministic: the same bits on every run, no atomics on values.
 * Per function ("pinned" = one of the reference's six array tests covers it; "unpinned" = follows Spark 2.4 where the reference is
 *   silent or its body is private and broken):
 *   CONTAINS (array.rs:15)   Boolean, chunks of the input.  Null list -> NULL; otherwise true iff a VALID element equals v (a null slot
 *                            never matches, so a valid list never gives NULL).  Pinned.
 *   POSITION (:233)          Int32, chunks of the input, never NULL: the 1-based index of the first valid element equal to v (null slots
 *                            count as positions), 0 without one; a null list -> 0 (as the reference appends).  Pinned.
 *   MAX / MIN (:182, :206)   T, chunks of the input.  Null elements are skipped; a list whose elements are all null -> NULL; a null list
 *                            -> NULL; a valid EMPTY list -> BDF_WOULD_PANIC (.max().unwrap()).  Floats (an extension) use group-by's
 *                            float rule: IEEE totalOrder keys, -0.0 < +0.0, NaN greatest, returned as the positive quiet NaN.
 *   SIZE (scalar.rs:414)     Int32, chunks of the input: the slot count; a null list -> -1 (Spark 2.4).
 *   REMOVE (:262)            Elements equal to v removed, order kept; null elements are kept as null.  Pinned (offsets, value count).
 *   SORT (:328)              Ascending in DataFrame::sort's order (NaN greatest, -0.0 == 0.0, ties in input order), nulls last.  Pinned.
 *   DISTINCT (:39)           The first occurrence of each value in input order; at most one null, at the first null's place.  Unpinned.
 *   REPEAT (:294)            The list concatenated `count` times; 0 -> empty; count < 0 -> BDF_INVALID (the reference casts it to usize);
 *                            nulls repeat as nulls.  Unpinned.
 *   EXCEPT / INTERSECT / UNION (:66, :110, :356)  Distinct results in the order of first appearance: except = in a, not in b;
 *                            intersect = in a and in b; union = a then b.  Null elements are one value.  A null a -> a valid empty list;
 *                            a null b counts as empty.  Different list counts per chunk -> BDF_LENGTH_MISMATCH ("Expected array a and b
 *                            to have the same length").  Unpinned.
 *   EXPLODE (scalar.rs:237)  Two one-chunk columns: UInt32 parent row numbers (counted through the chunks) and the T values, one row
 *                            per element of every valid list, in order; null and empty lists give no row (Spark); null elements give
 *                            null values.  Other columns follow with bdf_take_dev(col, rows).
 * Errors (nothing is returned and nothing leaks): a null pointer or an unknown function -> BDF_INVALID; a non-numeric child, the limits
 *   above, a multi-GPU context -> BDF_UNSUPPORTED; children of different dtypes in a set function -> BDF_UNSUPPORTED. */
#define BDF_LIST_BASE 32   /* bdf_ipc_list_column reports a List<T> column as BDF_LIST_BASE + T */
typedef struct {
    const int32_t* offsets;   /* base of the offsets buffer, NOT offset-adjusted: entries offset .. offset + len are read    */
    const uint8_t* validity;  /* list validity, LSB-first, 1 = valid; NULL when every list is valid                          */
    int64_t        len;       /* lists                                                                                      */
    int64_t        offset;    /* list offset (sliced ListArray)                                                             */
    int64_t        null_count;
    bdf_view       values;    /* the child array                                                                            */
} bdf_list_view;
/* One downloaded list chunk.  offsets >= len + 1 Int32, validity >= ceil(len / 8) bytes (may be NULL if the chunk has no null list),
 * values >= elements x width bytes, value_validity >= ceil(elements / 8) bytes (may be NULL if no element is null); sizes come from
 * bdf_list_chunk_info.  Bitmaps are written at bit 0. */
typedef struct {
    int32_t* offsets;
    uint8_t* validity;
    void*    values;
    uint8_t* value_validity;
    int64_t  null_count, value_null_count;   /* OUT */
    int32_t  has_validity, has_value_validity; /* OUT */
} bdf_list_out;
typedef enum { BDF_LIST_CONTAINS = 0, BDF_LIST_POSITION } bdf_list_find_fn;
typedef enum { BDF_LIST_MAX = 0, BDF_LIST_MIN, BDF_LIST_SIZE } bdf_list_reduce_fn;
typedef enum { BDF_LIST_REMOVE = 0, BDF_LIST_SORT, BDF_LIST_DISTINCT, BDF_LIST_REPEAT } bdf_list_transform_fn;
typedef enum { BDF_LIST_EXCEPT = 0, BDF_LIST_INTERSECT, BDF_LIST_UNION } bdf_list_set_fn;
int  bdf_list_upload(bdf_ctx* ctx, int child_dtype, int64_t n_chunks, const bdf_list_view* in, int flags, bdf_list** out);
int  bdf_list_describe(const bdf_list* list, int32_t* child_dtype, int64_t* n_chunks, int64_t* total_len);
int  bdf_list_chunk_info(bdf_ctx* ctx, const bdf_list* list, int64_t chunk, int64_t* len, int64_t* null_count, int64_t* n_elements);
int  bdf_list_download(bdf_ctx* ctx, const bdf_list* list, bdf_list_out* out /* n_chunks */);
const bdf_col* bdf_list_values(const bdf_list* list);   /* owned by the list */
void bdf_list_free(bdf_ctx* ctx, bdf_list* list);
int  bdf_list_find_dev(bdf_ctx* ctx, int fn, const bdf_list* list, uint64_t value_bits, bdf_col** out);
int  bdf_list_reduce_dev(bdf_ctx* ctx, int fn, const bdf_list* list, bdf_col** out);
int  bdf_list_transform_dev(bdf_ctx* ctx, int fn, const bdf_list* list, uint64_t value_bits /* REMOVE */, int64_t count /* REPEAT */,
                            bdf_list** out);
int  bdf_list_set_dev(bdf_ctx* ctx, int fn, const bdf_list* a, const bdf_list* b, bdf_list** out);
int  bdf_list_explode_dev(bdf_ctx* ctx, const bdf_list* list, bdf_col** rows, bdf_col** values);
/* Whole lists moved between rows: the list columns of a frame through take (DataFrame::sort, join, limit) and filter.
 *   bdf_list_take_dev    out[i] = list[indices[i]] (Column::take), indices a UInt32 column whose row numbers count through the list's
 *                        chunks.  ONE chunk.  A null index gives a null list, a null list stays null, null elements stay null with
 *                        their bits.  Offsets start at 0 and only the elements of valid lists are copied.  An index past the end ->
 *                        BDF_INVALID.
 *   bdf_list_filter_dev  The lists where the Boolean mask is valid and true (ChunkedArray::filter).  The chunks of the input are kept:
 *                        chunk i holds the kept lists of chunk i, so list columns stay RecordBatch-aligned with the numeric columns
 *                        bdf_filter_dev filters.  Mask chunk lengths that differ from the list's -> BDF_LENGTH_MISMATCH.
 *   Both: exact null counts (bdf_list_chunk_info); more than 2^31 - 1 result elements in one chunk -> BDF_UNSUPPORTED (Int32 offsets);
 *   a multi-GPU context -> BDF_UNSUPPORTED.  On failure nothing is returned and nothing leaks. */
int  bdf_list_take_dev(bdf_ctx* ctx, const bdf_list* list, const bdf_col* indices /* UInt32 */, bdf_list** out);
int  bdf_list_filter_dev(bdf_ctx* ctx, const bdf_list* list, const bdf_col* mask /* Boolean */, bdf_list** out);
/* List<T> columns of an IPC file.  bdf_ipc_column keeps reporting them with dtype -1 (outside the column path: bdf_ipc_read and
 * bdf_ipc_view refuse them, and readers that take every column of dtype >= 0 are unaffected); bdf_ipc_list_column gives
 * BDF_LIST_BASE + T for a List of one numeric T and -1 for every other column (LargeList, nested lists, List<bool> ...);
 * bdf_ipc_read_list uploads one, one chunk per RecordBatch, offsets and child buffers taken from the mapping (no context needed for
 * the first, none of the three needs a GPU except the read). */
int  bdf_ipc_list_column(const bdf_ipc* file, int32_t col, int32_t* dtype);
int  bdf_ipc_read_list(bdf_ctx* ctx, const bdf_ipc* file, int32_t col, int flags, bdf_list** out);

/* ---- line-delimited JSON files straight to the device (DataFrame::from_json, src/dataframe.rs; LazyFrame::read(Json),
 * src/evaluation.rs:329) ----------------------------------------------------------------------------------------------------------
 * The reference reads with arrow-rs's json::Reader (infer_json_schema over max_records, then batches of batch_size, default 1024)
 * over serde_json.  Neither is restated from source: every rule marked RECALLED below is recalled, parity unpinned (the reference
 * has no JSON test); the others are this library's decisions, listed under Departures.
 * Records.  A record is one line: '\n' ends it, and a '\r' before the '\n' is whitespace (JSON's whitespace is ' ', '\t', '\r',
 *   '\n').  Lines made only of whitespace are skipped.  A leading UTF-8 BOM is skipped.  End of file ends the last record.  Every
 *   record is one JSON object (RFC 8259; RECALLED: serde_json's grammar); anything else is BDF_INVALID "JSON error at line L, byte
 *   B: what": a record that is not an object, malformed JSON, a number outside JSON's grammar (NaN, Infinity, +1, 01, 1., .5), an
 *   unterminated string, an invalid escape, a raw control byte in a string, unbalanced brackets, trailing bytes after the object,
 *   or nesting deeper than 128 levels (RECALLED: serde_json's recursion limit).  L counts lines from 1; B is the byte offset of the
 *   error in the file (the BOM counted).  A raw '\n' cannot occur in a valid string, so records are split without string state.
 * Keys.  Compared after their escapes are decoded ("\u0061" is the key a; a lone surrogate escape decodes to U+FFFD).  Columns come
 *   in the order each key is first seen in the file.  A key repeated in one record: the last value wins (RECALLED: serde_json's
 *   Map).  At most 65536 distinct raw keys per file, else BDF_UNSUPPORTED; two different keys with the same 64-bit hash are detected
 *   (every key is compared byte for byte) and give BDF_UNSUPPORTED.
 * Inference (no schema) over the first max_records records (all of them when max_records < 0); the columns are the keys seen
 *   there.  Each value is put in one class: null adds no type and makes the column nullable; true / false Boolean; an integer
 *   literal (no fraction, no exponent) in i64 range Int64; any other number Float64; a string Utf8; an object a struct; an array a
 *   List of its non-null elements' coerced class.  Per key (RECALLED: arrow's coercion): one type -> it; {Int64, Float64} ->
 *   Float64; List<Int64> with List<Float64> -> List<Float64>; a numeric scalar with a numeric list -> a List of the coerced element
 *   type (arrow's "scalar and list -> list"); anything involving Utf8, a struct, Boolean mixed with another type, nested lists, a
 *   list with a non-numeric element, or only lists that never had a typed element (or only nulls) -> off the device path:
 *   bdf_json_column reports dtype -1, as bdf_csv_column does for Utf8.  A key missing from an inferred record makes its column
 *   nullable.
 * Explicit schema.  (name, dtype) pairs: dtype 0..9, BDF_BOOL, BDF_LIST_BASE + T for a numeric T, or BDF_UTF8 / -1 to skip the
 *   column (reported with dtype -1); any other -> BDF_UNSUPPORTED, a repeated name -> BDF_INVALID.  Keys not in the schema are
 *   ignored; every schema column is nullable.
 * Values.  An absent key or null gives NULL.  Integer columns take integer literals in range for the column type (unsigned types
 *   refuse a '-' sign, even -0).  Float columns take any JSON number, CORRECTLY ROUNDED to the column type (Float32 straight from the
 *   decimal, never through Float64: the CSV reader's Eisel-Lemire path and its exact host fallback).  Boolean columns take true /
 *   false.  A List<T> column takes an array: each element converted like a scalar of T, a null (or non-converting) element a null
 *   element; a bare number is a one-element list; [] a valid empty list.  Anything that does not convert is NULL: a float or an
 *   out-of-range integer into an integer column, a string, a Boolean into a number column, a number into a Boolean column, an
 *   object, an array into a scalar column.  (RECALLED: arrow's reader leaves a non-conforming value null.  pyarrow's reader
 *   instead ERRORS on such a value once the column's type is fixed: departure 4.)
 * Output.  One chunk of batch_size rows per RecordBatch (the last one shorter), null counts set, no validity bitmap in a chunk
 *   without nulls.  bdf_json_read reads numeric and Boolean columns (a projection); bdf_json_read_list reads one List<T> column as a
 *   bdf_list, one chunk per RecordBatch with offsets from 0 in every chunk (no list bitmap in a chunk without null lists, no element
 *   bitmap in a chunk without null elements).
 * Departures from the reference, on purpose: (1) from_json stops at the first Err batch and keeps what it has; here the open (or
 *   the read) fails.  (2) an empty file, or one of blank lines only, makes the reference panic at batches[0]: BDF_WOULD_PANIC.
 *   (3) field order is first-seen; the recalled arrow reader of that era kept the inferred fields in a HashMap, so its order was
 *   unstable.  (4) a value that does not convert is NULL here, where pyarrow errors.  (5) bytes are not checked for valid UTF-8
 *   (serde_json reads from a str, so invalid UTF-8 is an error there).  (6) a '\r' alone does not end a record.
 * Memory.  bdf_json_open keeps the file's bytes, 32 B per object member and 4 B per (record, column) in HBM until bdf_json_close and
 *   needs 16 B per line and 8 B per '\n' more while it indexes; the file itself must fit as for CSV, else BDF_OOM before anything
 *   is uploaded; anything else that does not fit gives BDF_OOM.  A read needs its outputs and, for float columns, a list of at most
 *   max(65536, floats / 64) entries of 40 B for the values the device cannot round (rounded on the host with strtod / strtof in the
 *   C locale; bdf_json_stats counts them; more -> BDF_UNSUPPORTED).  A failed call leaks nothing.  A multi-GPU context ->
 *   BDF_UNSUPPORTED. */
typedef struct { int64_t max_records /* <0: all */; int64_t batch_size; } bdf_json_options;
typedef struct bdf_json bdf_json;
int  bdf_json_open(bdf_ctx* ctx, const char* path, const bdf_json_options* options, int32_t n_schema, const char* const* schema_names,
                   const int32_t* schema_dtypes /* both NULL: infer */, bdf_json** out);
int  bdf_json_describe(const bdf_json* file, int32_t* n_columns, int64_t* n_batches, int64_t* n_rows);
int  bdf_json_column(const bdf_json* file, int32_t col, const char** name, int32_t* dtype /* -1 off the path */, int32_t* nullable);
int  bdf_json_read(bdf_ctx* ctx, const bdf_json* file, int32_t n_cols, const int32_t* cols, bdf_col** out /* n_cols */);   /* projection */
int  bdf_json_read_list(bdf_ctx* ctx, const bdf_json* file, int32_t col, bdf_list** out);
/* object members in the file; float values the last read rounded on the host; host time of the file's upload in bdf_json_open */
int  bdf_json_stats(const bdf_json* file, int64_t* n_members, int64_t* exact_fields, double* upload_ms);
void bdf_json_close(bdf_ctx* ctx, bdf_json* file);   /* the context that opened it */

/* ---- dates and timestamps (ScalarFunctions::hour, src/functions/scalar.rs:267-273 -> arrow compute::hour; the Spark date functions
 * that are empty stubs in the same file: add_months, date_add, date_sub, date_trunc, date_diff, day_of_month, day_of_week, day_of_year,
 * last_day, minute, month, months_between, next_day, quarter, second, to_date, unix_timestamp, year ...) ----------------------------------
 * Types.  A temporal column is an ORDINARY bdf_col of its physical dtype; a bdf_temporal_type travels beside it (no new bdf_dtype), so
 *   sort, group-by, join, window, take, filter and min / max work on temporal columns unchanged:
 *     Date32     BDF_I32  days since 1970-01-01 (unit ignored)      Date64     BDF_I64  milliseconds (unit BDF_MILLISECOND)
 *     Timestamp  BDF_I64  in its unit (any), tz optional             Time32     BDF_I32  time of day, s or ms
 *     Time64     BDF_I64  time of day, us or ns
 *   Any other (kind, unit), or a column whose physical dtype does not match its type -> BDF_INVALID.  "Date kinds" below = Date32,
 *   Date64 and Timestamp; "time kinds" = Time32 and Time64.
 * Calendar.  Proleptic Gregorian, no leap seconds.  A value v of a date kind is split by FLOOR division into days = floor(v / units_per_day)
 *   and a time of day 0 <= tod < units_per_day (so -1 us is 1969-12-31T23:59:59.999999).  Definition, not parity: old arrow versions
 *   truncated toward zero here (recalled).  Civil fields come from days by Hinnant's civil_from_days (PAPERS.md).
 * Range.  The dates of chrono's NaiveDate, years -262144 ..= 262143 (days -96465658 ..= 95026601), where arrow's value_as_datetime gives
 *   None.  A date outside it gives NULL: the date a function reads (the local date for the civil functions, the UTC date for
 *   UNIX_TIMESTAMP and TO_TIMESTAMP) and a computed result date alike.  A result that does not fit its output type is NULL too (a
 *   Timestamp(s) in year 3000 converted to ns; date_trunc(year) of a ns value in 1677 whose year start is below i64::MIN).  A Time32 /
 *   Time64 value outside [0, one day) gives NULL for HOUR / MINUTE / SECOND.  Otherwise a result slot is valid iff its input slot is (the
 *   two-column functions: iff both are).  Every result carries a validity bitmap (its null count may be 0).
 * Time zones.  Values are UTC instants.  The functions that read civil fields apply a Timestamp's tz when it is NULL, "UTC", "Z" or
 *   "+00:00" (no shift) or a fixed offset "+HH:MM" / "-HH:MM" (HH 00..23, MM 00..59): local time = instant + offset, and DATE_TRUNC turns
 *   the truncated local time back into an instant (local - offset).  Any other tz string -- a named zone such as "Europe/Paris" --
 *   gives BDF_UNSUPPORTED there: there is no tz database on the device, and UTC fields would be silently wrong.  UNIX_TIMESTAMP and
 *   TO_TIMESTAMP keep instants and accept any tz.  (Departure: the arrow of the reference's era ignored tz.)
 * Functions (bdf_temporal_fn; "arg" is the int64_t argument, ignored where the table has none):
 *   YEAR, QUARTER (1..4), MONTH (1..12), DAY_OF_MONTH, DAY_OF_YEAR (1..366)   date kinds -> Int32: the civil fields.
 *   DAY_OF_WEEK      date kinds -> Int32, Spark's numbering: 1 = Sunday .. 7 = Saturday.
 *   HOUR, MINUTE, SECOND   date and time kinds -> Int32 of the (local) time of day; Date32 gives 0 (arrow's hour goes through midnight);
 *                    SECOND has no fraction.
 *   TO_DATE          date kinds -> Date32: the civil date.
 *   DATE_ADD / DATE_SUB   date kinds, arg = days in Int32 range -> Date32: to_date(x) + arg / - arg.
 *   ADD_MONTHS       date kinds, arg = months in Int32 range -> Date32, SPARK 2.4's rule: the target month is (year, month) + arg; if the
 *                    start day is the last day of its month, or lies past the end of the target month, the result is the target month's
 *                    last day, else the same day.  So 2019-02-28 + 1 = 2019-03-31 and 2016-08-31 + 1 = 2016-09-30.  Spark 3 dropped the
 *                    first half of this rule (2019-02-28 + 1 = 2019-03-28 there).
 *   LAST_DAY         date kinds -> Date32: the last day of the month.
 *   NEXT_DAY         date kinds, arg = day of week 1..7 (Spark numbering) -> Date32: the first date strictly after to_date(x) with that
 *                    weekday.  arg outside 1..7 -> BDF_INVALID (a constant here, not Spark's per-row string that gives NULL).
 *   DATE_TRUNC       date kinds, arg = bdf_trunc_unit -> the input's type (Timestamp: unit and tz kept): floor in local time to the start
 *                    of the year / quarter / month / week (Monday) / day / hour / minute / second.  Date32 with a unit below DAY returns
 *                    x.  Time kinds -> BDF_UNSUPPORTED.
 *   UNIX_TIMESTAMP   date kinds -> Int64: floor seconds since the epoch (Date32: days x 86400).
 *   TO_TIMESTAMP     date kinds, arg = target bdf_time_unit -> Timestamp(arg, tz of a Timestamp input, else NULL): the same instant,
 *                    floor-divided when the target unit is coarser.
 *   A time kind with any function but HOUR / MINUTE / SECOND -> BDF_UNSUPPORTED.
 * Two-column functions (bdf_temporal_binary_fn): a and b may be different date kinds; each side's tz rules apply.
 *   DATE_DIFF(end = a, start = b)  -> Int32: days(to_date(a)) - days(to_date(b)), Spark's datediff.
 *   MONTHS_BETWEEN(t1 = a, t2 = b) -> Float64, Spark 2.4 with roundOff = true, in exactly this IEEE double sequence (no FMA):
 *                    monthDiff = (double)((y1 * 12 + m1) - (y2 * 12 + m2)); if d1 == d2 or both are the last day of their month: monthDiff;
 *                    else secDiff = (double)((d1 - d2) * 86400 + (s1 - s2)) with s the whole seconds of the local time of day (0 for
 *                    Date32), diff = monthDiff + secDiff / 2678400.0, t = diff * 1e8, k = floor(t), k += 1 if t - k >= 0.5 (Java 8's
 *                    Math.round, ties toward +inf), result k / 1e8.  ('1997-02-28 10:30:00', '1996-10-30') = 3.94959677.
 * Results are deterministic and bit-exact: integer arithmetic, plus the one double sequence above.
 * Comparison.  bdf_compare_dev goes through Float64: exact for Date32 / Time32 values (and for to_date / unix_timestamp results within
 *   +-2^53), not for Date64 / Timestamp / Time64 instants.  The Python layer therefore refuses compare on a column tagged with a 64-bit
 *   temporal type (a departure from refusing every tagged column: a date-range filter on to_date() needs it).
 * Parity unpinned: the reference pins none of this (no test of hour; the stubs have no body).  arrow's and chrono's behaviour and Spark
 *   2.4's rules and documentation examples are RECALLED.
 * Chunks.  bdf_temporal / bdf_temporal_dev keep the input's chunks (as bdf_unary); bdf_temporal_binary_dev zips chunks as bdf_binary_dev
 *   (BDF_LENGTH_MISMATCH on unequal chunk lengths).  All three accept a multi-GPU context and return the one-GPU bits.
 * Errors (nothing is returned and nothing leaks): a null pointer, an unknown function, an invalid type, a wrong physical dtype or a bad arg
 *   -> BDF_INVALID; a function the kind does not have or a named tz -> BDF_UNSUPPORTED. */
typedef enum { BDF_TEMPORAL_NONE = 0, BDF_DATE32, BDF_DATE64, BDF_TIMESTAMP, BDF_TIME32, BDF_TIME64 } bdf_temporal_kind;
typedef enum { BDF_SECOND = 0, BDF_MILLISECOND, BDF_MICROSECOND, BDF_NANOSECOND } bdf_time_unit;   /* arrow TimeUnit order */
typedef struct { int32_t kind; int32_t unit; const char* tz; /* Timestamp only; NULL = none */ } bdf_temporal_type;
typedef enum {
    BDF_TEMPORAL_YEAR = 0, BDF_TEMPORAL_QUARTER, BDF_TEMPORAL_MONTH, BDF_TEMPORAL_DAY_OF_MONTH, BDF_TEMPORAL_DAY_OF_YEAR, BDF_TEMPORAL_DAY_OF_WEEK,
    BDF_TEMPORAL_HOUR, BDF_TEMPORAL_MINUTE, BDF_TEMPORAL_SECOND, BDF_TEMPORAL_TO_DATE, BDF_TEMPORAL_DATE_ADD, BDF_TEMPORAL_DATE_SUB,
    BDF_TEMPORAL_ADD_MONTHS, BDF_TEMPORAL_LAST_DAY, BDF_TEMPORAL_NEXT_DAY, BDF_TEMPORAL_DATE_TRUNC, BDF_TEMPORAL_UNIX_TIMESTAMP,
    BDF_TEMPORAL_TO_TIMESTAMP, BDF_NTEMPORAL
} bdf_temporal_fn;
typedef enum { BDF_TEMPORAL_DATE_DIFF = 0, BDF_TEMPORAL_MONTHS_BETWEEN } bdf_temporal_binary_fn;
typedef enum { BDF_TRUNC_YEAR = 0, BDF_TRUNC_QUARTER, BDF_TRUNC_MONTH, BDF_TRUNC_WEEK, BDF_TRUNC_DAY, BDF_TRUNC_HOUR, BDF_TRUNC_MINUTE,
               BDF_TRUNC_SECOND } bdf_trunc_unit;
/* host in / host out: the drop-in body of ScalarFunctions::hour<T>(Vec<&PrimitiveArray<T>>) -> Vec<Int32Array> and of the stubs.  `out`
 * holds the result's dtype (bdf_temporal_result). */
int  bdf_temporal(bdf_ctx* ctx, int fn, const bdf_temporal_type* type, int64_t arg, int64_t n_chunks, const bdf_view* in, bdf_out* out);
int  bdf_temporal_dev(bdf_ctx* ctx, int fn, const bdf_temporal_type* type, int64_t arg, const bdf_col* in, bdf_col** out);
int  bdf_temporal_binary_dev(bdf_ctx* ctx, int fn, const bdf_temporal_type* ta, const bdf_col* a, const bdf_temporal_type* tb, const bdf_col* b,
                             bdf_col** out);
/* No context, no GPU: validates (fn, type, arg) exactly as the entries do and reports the result's dtype and temporal type (kind 0 for a
 * plain Int32 / Int64 result; out_type->tz points at type->tz). */
int  bdf_temporal_result(int fn, const bdf_temporal_type* type, int64_t arg, int32_t* out_dtype, bdf_temporal_type* out_type);
/* Temporal columns of an IPC file.  bdf_ipc_column keeps reporting Date / Time / Timestamp columns with dtype -1 (as List columns);
 * bdf_ipc_temporal_column gives the type (kind 0 for any other column, or for a Date / Time field whose unit and width do not form a
 * valid type); tz points into the open file.  bdf_ipc_read_temporal uploads one such column, one chunk per RecordBatch, its buffers
 * checked at read time.  bdf_ipc_write_typed is bdf_ipc_write with a type per column (kind 0: as the column's dtype; types == NULL:
 * all kind 0); it writes the Date / Time / Timestamp field types, tz included.  Duration, Interval and Decimal stay outside the path. */
int  bdf_ipc_temporal_column(const bdf_ipc* file, int32_t col, bdf_temporal_type* out);
int  bdf_ipc_read_temporal(bdf_ctx* ctx, const bdf_ipc* file, int32_t col, int flags, bdf_col** out);
int  bdf_ipc_write_typed(bdf_ctx* ctx, const char* path, int32_t n_cols, const char* const* names, const bdf_col* const* cols,
                         const bdf_temporal_type* types /* n_cols entries, or NULL */);
/* bdf_ipc_write_typed with list columns: column j is lists[j] when that is non-NULL (then cols[j] must be NULL and types[j].kind 0),
 * otherwise cols[j] as in bdf_ipc_write_typed.  A list is written as List<item: T>, field and child both nullable, the child named
 * "item" as pyarrow names it; its FieldNodes are the list's and then the child's, its buffers the list validity, the Int32 offsets
 * (from 0), the child validity and the child values, each on a 64-byte file offset.  List chunk b is RecordBatch b: any other chunk
 * structure -> BDF_LENGTH_MISMATCH.  bdf_ipc_read_list reads such a column back. */
int  bdf_ipc_write_lists(bdf_ctx* ctx, const char* path, int32_t n_cols, const char* const* names, const bdf_col* const* cols,
                         const bdf_temporal_type* types /* or NULL */, const bdf_list* const* lists /* n_cols entries, or NULL */);

/* ---- Parquet files straight to the device (DataFrame::from_parquet, src/dataframe.rs) ----------------------------------------------
 * The reference reads a file, or every file of a directory, with parquet's ParquetFileArrowReader in batches of 1024 rows.  Rules
 * marked RECALLED are recalled from arrow-rs of that era, parity unpinned; the others are this library's decisions.
 * Files.  "PAR1" at both ends and a Thrift compact-protocol FileMetaData footer, parsed on the host: every read is bounds-checked,
 *   nesting is limited to 32 levels and unknown field ids are skipped (so footers with page indexes, bloom filters, size or geo
 *   statistics parse).  An encrypted file ("PARE") or a ColumnChunk.file_path pointing into another file -> BDF_UNSUPPORTED.
 * Pages.  DATA_PAGE (V1), DATA_PAGE_V2 (is_compressed = false included) and at most one DICTIONARY_PAGE, first in its chunk;
 *   INDEX_PAGE is skipped.  Page CRCs are NOT checked.
 * Codecs.  UNCOMPRESSED and SNAPPY.  Any other (GZIP, BROTLI, LZ4, LZ4_RAW, ZSTD, LZO) -> BDF_UNSUPPORTED naming the codec when that
 *   column is read (or checked); the file still opens and the other columns still read.
 * Encodings.  Values: PLAIN; PLAIN_DICTIONARY / RLE_DICTIONARY ids over a PLAIN dictionary page; RLE for Boolean; BYTE_STREAM_SPLIT for
 *   the fixed-width types.  A chunk may switch from dictionary to PLAIN pages part-way (what a writer does when the dictionary
 *   outgrows its limit).  Definition levels: the RLE / bit-packed hybrid.  DELTA_*, the deprecated BIT_PACKED levels, and any
 *   other encoding -> BDF_UNSUPPORTED for that column, naming the encoding.
 * Types.  Only top-level primitive columns, required or optional (maximum definition level 0 or 1).  A group, a repeated field or any
 *   other type is one column of dtype -1, stepped over (as the CSV reader steps over Utf8).  Logical types win over converted types:
 *     BOOLEAN -> Boolean;  FLOAT -> Float32;  DOUBLE -> Float64
 *     INT32, none / INT(8|16|32, signed) / INT_8, INT_16, INT_32    -> Int32 / Int8, Int16, Int32
 *     INT32, INT(8|16|32, unsigned) / UINT_8, UINT_16, UINT_32      -> UInt8, UInt16, UInt32
 *     INT64, none / INT(64, signed) / INT_64; INT(64, unsigned) / UINT_64 -> Int64; UInt64
 *     INT32 DATE -> Date32;  INT32 TIME(MILLIS) / TIME_MILLIS -> Time32(ms);  INT64 TIME(MICROS | NANOS) / TIME_MICROS -> Time64(us | ns)
 *     INT64 TIMESTAMP(unit, isAdjustedToUTC) -> Timestamp(unit, "UTC" if adjusted, else no tz); TIMESTAMP_MILLIS / _MICROS (converted
 *       only, which the format defines as adjusted to UTC) -> Timestamp(ms | us, "UTC")
 *     INT96, DECIMAL, FLOAT16, BYTE_ARRAY, FIXED_LEN_BYTE_ARRAY, anything else -> dtype -1
 *   Temporal columns report their physical dtype (BDF_I32 / BDF_I64) from bdf_parquet_column; bdf_parquet_temporal_column gives the tag.
 *   Narrow integers: an INT(8|16) value stored in INT32 that does not fit its type is TRUNCATED to its low bits.
 *   Timestamp tz: when the footer holds an ARROW:schema entry (an Arrow IPC schema message, base64) whose top-level field at the same
 *   position has the same name and is a Timestamp of the same unit, the tz is that field's (as pyarrow restores a "+01:00" or
 *   "Europe/Paris" column).  A malformed entry is ignored.  The unit is always Parquet's: departure (1), pyarrow restores a
 *   Timestamp(s) column from Arrow's metadata; here it reads as Timestamp(ms), and a Date64 column (stored as DATE) as Date32.
 *   Because the units then differ, such a Timestamp(s, tz) column also loses a named tz: it reads as Timestamp(ms, "UTC") (the
 *   Parquet type's isAdjustedToUTC), where pyarrow restores Timestamp(s, tz).
 * Output.  One chunk of batch_size rows (default 1024) per RecordBatch: the batches run across the row groups of one file, and each
 *   file starts a new chunk (RECALLED; parity unpinned).  Null counts are set; a chunk without nulls has no validity bitmap; a required
 *   column is not nullable.  A null slot holds 0.
 * Directories.  The regular files of the directory in byte order of their names (departure (2): the reference takes read_dir's
 *   unspecified order); names starting with '.' or '_' (_SUCCESS) are skipped (departure (3): the reference fails on them); files
 *   with zero row groups are skipped.  The first file left gives the schema; every other file must have the same column names, dtypes
 *   and temporal types (tz included), else BDF_INVALID naming the file and column; nullable is the OR over the files.  No file left
 *   -> BDF_WOULD_PANIC (the reference's schema.unwrap()).
 * Errors.  Found on the host: BDF_INVALID "Parquet error in FILE[, row group G][, column C][, page P]: what" -- bad magic, a footer or
 *   column chunk outside the file, a page header or page running past its chunk, data-page num_values not adding up to the row
 *   group's rows, more than one dictionary page, dictionary ids without a dictionary.  A bad footer fails bdf_parquet_open; a bad
 *   chunk fails bdf_parquet_check and a read of its column.  Found on the device (a per-page error word, read back once at the end
 *   of the read): the same status and message shape -- a corrupt snappy stream, a decompressed size that differs from the page
 *   header, a dictionary index outside the dictionary, a level, index or value stream that ends early.
 * Memory.  A read uploads the projected column chunks only, still compressed (bdf_parquet_stats counts their bytes), and needs
 *   the decompressed size of its snappy pages, run tables of 8 B per entry (per level or index stream, at most min(values, stream
 *   bytes) + 1 entries), and its outputs; what does not fit gives
 *   BDF_OOM before anything is uploaded.  A failed call leaks nothing.  The open needs no context and no GPU; a read on a multi-GPU
 *   context -> BDF_UNSUPPORTED. */
typedef struct { int64_t batch_size; } bdf_parquet_options;
typedef struct bdf_parquet bdf_parquet;
int  bdf_parquet_open(const char* path /* a file or a directory */, const bdf_parquet_options* options /* NULL: defaults */, bdf_parquet** out);
int  bdf_parquet_describe(const bdf_parquet* file, int32_t* n_columns, int64_t* n_batches, int64_t* n_rows);
int  bdf_parquet_column(const bdf_parquet* file, int32_t col, const char** name, int32_t* dtype /* physical; -1 off the path */, int32_t* nullable);
int  bdf_parquet_temporal_column(const bdf_parquet* file, int32_t col, bdf_temporal_type* out);   /* kind 0: not temporal */
/* No GPU: the status a read of col would give for every cause the host can detect (off the path, codec, encoding, a bad chunk). */
int  bdf_parquet_check(const bdf_parquet* file, int32_t col);
int  bdf_parquet_read(bdf_ctx* ctx, const bdf_parquet* file, int32_t n_cols, const int32_t* cols, bdf_col** out /* n_cols */);   /* projection */
/* of the last read: data and dictionary pages decoded, compressed bytes uploaded, host time of the upload */
int  bdf_parquet_stats(const bdf_parquet* file, int64_t* n_pages, int64_t* uploaded_bytes, double* upload_ms);
void bdf_parquet_close(bdf_parquet* file);

/* ---- Parquet files straight from the device (DataFrame::to_parquet, src/dataframe.rs:545-560) ----------------------------------------
 * The reference writes with parquet's ArrowWriter, one write(batch) per RecordBatch.  Rules marked RECALLED are recalled from parquet-rs
 * of that era (WriterProperties defaults, the early ArrowWriter), parity unpinned; the others are this library's decisions.
 * Defaults (options == NULL, RECALLED).  UNCOMPRESSED, dictionary on, statistics on, writer version 1.0 (DATA_PAGE V1 pages), one row
 *   group per RecordBatch, which here is one per chunk; an empty chunk is skipped.  Snappy and row_group_rows are options, as
 *   bdf_csv_write_options are: row_group_rows = N > 0 cuts row groups of N rows across the chunks.
 * Schema.  Every column is OPTIONAL (maximum definition level 1), as bdf_ipc_write marks every field nullable.  Types are the inverse of
 *   the reader's table:
 *     Int8 / Int16 / Int32 -> INT32 INT(8|16|32, signed);  UInt8 / UInt16 / UInt32 -> INT32 INT(8|16|32, unsigned), widened on the device
 *     Int64 / UInt64 -> INT64 INT(64, signed / unsigned);  Float32 -> FLOAT;  Float64 -> DOUBLE;  Boolean -> BOOLEAN
 *     Date32 -> INT32 DATE;  Date64 -> INT32 DATE, floor(ms / 86 400 000)
 *     Time32(s | ms) -> INT32 TIME(MILLIS), seconds x 1000;  Time64(us | ns) -> INT64 TIME(MICROS | NANOS)
 *     Timestamp(s) -> INT64 TIMESTAMP(MILLIS), x 1000;  Timestamp(ms | us | ns, tz) -> INT64 TIMESTAMP(unit, isAdjustedToUTC = tz != NULL)
 *   The converted types are written too where the format has them (INT_8 .. UINT_64, DATE, TIME_MILLIS, TIME_MICROS, and
 *   TIMESTAMP_MILLIS / _MICROS for a Timestamp with a tz: the format defines those as adjusted to UTC).  An ARROW:schema key-value
 *   entry holds the base64 of the IPC Schema message bdf_ipc_write_typed writes (every Arrow type, tz included).  pyarrow reads such a
 *   file exactly as it reads its own file of the same table: the time zone, fixed or named, comes back from the entry, while Date64,
 *   Time32(s) and Timestamp(s) come back in Parquet's units (Date32 days, milliseconds), as for pyarrow's own files.
 * Pages.  2^17 rows per data page, the last page of a row group fewer; a page never crosses a row group.  Definition levels: a 4-byte
 *   length, then the RLE / bit-packed hybrid in bit width 1 -- one RLE run for a page without nulls or with only nulls, else one
 *   bit-packed run copied from the validity bits.  Values: PLAIN (Boolean bit-packed) or dictionary ids.  Page CRCs are not written.
 * Dictionary (not for Boolean).  A column chunk's dictionary is its distinct values by raw bit pattern (so -0.0 and 0.0, and NaNs with
 *   different payloads, are separate entries and round-trip bit for bit), in ascending order of the bits read as unsigned integers: a
 *   decision, parquet-rs uses first-seen order.  Date64 values of one day are separate entries with the same stored date.  RECALLED
 *   v1.0 encodings: the dictionary page is PLAIN_DICTIONARY and the data pages PLAIN_DICTIONARY ids: one byte of bit width,
 *   max(1, ceil(log2 entries)), then one bit-packed run per page.  A chunk whose dictionary would exceed 1 MiB (entries x physical width,
 *   parquet-rs's default limit) is written PLAIN as a whole, without a dictionary page: a departure, parquet-rs falls back part-way
 *   through a chunk.  So is a chunk without a valid value.
 * Snappy.  Each page body (levels and values; a dictionary page's values) is one snappy stream, built from independently compressed
 *   64 KiB fragments, as the format allows.  Every page of a SNAPPY chunk is compressed, even when that makes it larger.
 * Statistics.  Per column chunk: null_count, min_value, max_value (the deprecated min / max are not written), and column_orders =
 *   TYPE_DEFINED_ORDER for every column.  Signed or unsigned order as the logical type says, false < true, over the stored physical
 *   values (after the x 1000 and Date64 conversions).  Floats skip NaN; a zero minimum is written -0.0 and a zero maximum +0.0.  A chunk
 *   without a valid non-NaN value has no min / max.
 * File.  "PAR1", per row group and column the dictionary page and the data pages, the Thrift compact-protocol FileMetaData (version 1,
 *   root schema element and leaves, row groups with total_byte_size and num_rows, created_by "b200df parquet writer", the ARROW:schema
 *   entry and the column orders), its length, "PAR1".  A frame without rows is a file with zero row groups (RECALLED: what an
 *   ArrowWriter closed without a write leaves); pyarrow reads it as an empty table, and bdf_parquet_open gives BDF_WOULD_PANIC for it,
 *   as the reference's from_parquet would (schema.unwrap()).  The same frame and options give the same bytes, call after call.
 * Input.  As bdf_csv_write: chunk b of every column has the same length, else BDF_LENGTH_MISMATCH.  The ten numeric types and Boolean;
 *   types[j] (NULL: none) tags Int32 / Int64 columns as Date, Time or Timestamp (kind 0: none).  A tag is checked as
 *   bdf_ipc_write_typed checks it (bdf_temporal_result's validation of kind and unit, then the physical dtype): a bad tag, or a column
 *   that cannot hold it (a Boolean column included) -> BDF_INVALID.  Any other column type -> BDF_UNSUPPORTED.  At most 2^32 - 1 rows
 *   and at most 2^20 column chunks (row groups x columns) per file, else BDF_INVALID.
 * Memory.  The pages go in blocks of consecutive pages, in file order, through two fixed 64 MiB device buffers (and an 80 MiB fragment
 *   buffer for snappy); the context's pinned staging slots (shared with uploads) carry headers and bodies to the file, written with
 *   pwrite by the staging threads.  Neither grows with the file.  What does, beside the frame itself:
 *     - the page and tile tables: about 40 B per 2048 rows and column, on the device and the host;
 *     - while the dictionary of one column is found (one column at a time): one sort of that column and its sorted copies
 *       (sorted_runs, as group-by) and the row-group ids, about 50 B per row for an 8-byte column, plus 4 B of id per row;
 *     - kept until the write ends, for each chunk written with a dictionary: 4 B of id per row of the chunk and its entries (at most
 *       1 MiB).  A column whose chunks all fall back to PLAIN keeps nothing.
 * Errors (nothing leaks): a null pointer, n_cols <= 0, compression not 0 / 1, dictionary not 0 / 1 or row_group_rows < 0 ->
 *   BDF_INVALID; a multi-GPU context -> BDF_UNSUPPORTED; BDF_OOM before the file is created.  Every refusal above happens before the
 *   file is created, so an existing file at the path is left as it was.  The file is written in place, as the CSV writer writes (no
 *   temporary file and rename: writing to /dev/null stays possible); a path that cannot be created or written -> BDF_INVALID with the
 *   OS text, and a failed call leaves a file without its trailing magic, which every reader rejects.
 * Launch records (BDF_K_PARQUET_WRITE): dtype BDF_U32 for the dictionary steps, -1 for the encode of a block (count, layout, encode),
 *   BDF_U8 for its snappy fragments and compaction. */
typedef struct {
    int32_t compression;      /* 0 UNCOMPRESSED, 1 SNAPPY */
    int32_t dictionary;       /* 0 off, 1 on */
    int64_t row_group_rows;   /* 0: one row group per chunk; N > 0: N rows per row group, cut across chunks */
} bdf_parquet_write_options;
int  bdf_parquet_write(bdf_ctx* ctx, const char* path, int32_t n_cols, const char* const* names, const bdf_col* const* cols,
                       const bdf_temporal_type* types /* n_cols entries or NULL, as bdf_ipc_write_typed */,
                       const bdf_parquet_write_options* options /* NULL: the defaults above */);

/* ---- line-delimited JSON files straight from the device (DataFrame::to_json) -------------------------------------------------------
 * The reference has no JSON writer (its README leaves "JSON: Write" unchecked).  The rules follow arrow-rs's json::LineDelimitedWriter
 * over serde_json, the reference's own dependencies; they are RECALLED, parity unpinned.  Departures are marked as such.
 * Records.  One JSON object per row in row order (chunk order, then row), each followed by "\n", the last one too; compact as serde_json
 *   writes it (no spaces).  A frame without rows writes an empty file, which bdf_json_open refuses with BDF_WOULD_PANIC (the reference
 *   panics on an empty file): such a file does not read back.
 * Members.  In column order, "name":value.  Names are escaped as serde_json escapes a string: \" \\ \b \f \n \r \t, other bytes below
 *   0x20 as \u00xx (lowercase hex), every other byte as it is.
 * NULL.  A NULL member is left out (arrow-rs's default, Spark's ignoreNullFields), so an all-NULL row is {}.  explicit_nulls = 1
 *   writes "name":null instead (pandas' habit).  A null element inside a list is always null.
 * Values:
 *   integers (the 8 types)  plain decimal (-9223372036854775808, 18446744073709551615); Boolean true / false.
 *   Float32 / Float64       the SHORTEST digits that read back to the same value in the column's own type, the closest of them when
 *                           several do (the CSV writer's digits).  Float32 is formatted as an f32, never widened: a departure, as
 *                           serde_json's Value widens f32 to f64.  Layout: ryu's (RECALLED: the ryu crate's format64 / format32).  With
 *                           kk the decimal exponent of the first digit plus one (10^(kk-1) <= |v| < 10^kk): integral values as digits
 *                           and ".0" while kk <= 16 (Float32 13); the point inside the digits for 0 < kk <= 16 (13); 0.000ddd for
 *                           -5 < kk <= 0 (Float32 -6 < kk); otherwise d.ddde and the exponent, '-' for a negative one, no '+', no
 *                           padding.  1.0, -0.0, 0.001, 1e16, 1e-7, 5e-324, 3.4028235e38 (f32::MAX).  So an all-integral Float64 column
 *                           reads back as Float64 under inference (unlike the CSV writer's 1).
 *                           NaN, inf and -inf are not JSON numbers: they are written as null (serde_json does the same), so the member
 *                           is left out unless explicit_nulls.  THEY DO NOT SURVIVE A ROUND TRIP: they come back NULL.
 *   temporal (types[j])     JSON strings, as bdf_parquet_write takes the types.  Date32 / Date64: "YYYY-MM-DD", the floor day.
 *                           Timestamp: "YYYY-MM-DDTHH:MM:SS" and a fraction of a fixed number of digits for its unit (none for s, 3 for
 *                           ms, 6 for us, 9 for ns), split by floor division as the temporal functions split (-1 us is
 *                           "1969-12-31T23:59:59.999999").  Time zones follow the temporal functions' rules: no tz, no suffix; "UTC",
 *                           "Z" or "+00:00": UTC fields and the suffix Z; a fixed offset +-HH:MM: the local fields (instant + offset)
 *                           and that offset as the suffix (RFC 3339); a named zone -> BDF_UNSUPPORTED.  Time32 / Time64: "HH:MM:SS"
 *                           with the same fraction rule.  Years as chrono's %Y: 4 digits for 0000..9999, '+' and the digits above 9999
 *                           (+10000), '-' and at least 4 digits below 0 (-0001).  A date outside chrono's range (years -262144 ..=
 *                           262143) or a time of day outside [0, one day) -> BDF_INVALID naming the column and the value, found from
 *                           the column's min and max before the file is opened: nothing becomes NULL silently.
 *   List<T> (lists[j])      [e,e,...] with each element formatted as a scalar of T, [] for an empty list; a null list is a NULL member.
 * Columns.  Column j is lists[j] when lists is given and lists[j] is non-NULL (then cols[j] must be NULL and types[j].kind 0, as in
 *   bdf_ipc_write_lists), otherwise cols[j]: one of the ten numeric types or Boolean, tagged with types[j] when types is given and
 *   types[j].kind != 0 (the physical dtype must match the kind).  Chunk b of every column (the lists' chunk b) has the same number of
 *   rows, else BDF_LENGTH_MISMATCH; sliced chunks and bit offsets are taken as they are.  Any number of columns.
 * Reading it back.  bdf_json_open with an explicit schema reads numeric, Boolean and List<T> columns back bit for bit (NaN and +-inf as
 *   NULL); temporal strings are not read back as temporal columns.
 * Memory.  The rows go in windows of at most 2^21 rows and 2^23 list elements, and each window's text in blocks cut at row boundaries
 *   where it fills a 64 MiB text buffer.  In HBM: two 64 MiB text buffers, 16 MiB of row offsets, 64 MiB of element offsets (with
 *   list columns), 16 MiB per list column for the list positions, 48 B per (chunk, column) plus 64 B per column of tables and a
 *   block table of 64 KiB plus 32 KiB per list column (in HBM and pinned); the context's pinned staging slots (6 x 8 MiB, shared with
 *   uploads) carry the text to the file, written with pwrite by the staging threads.  None of it grows with the file.  Only the longest single row can add more: a row with
 *   more than 2^23 elements needs 8 B per element of it, and a row whose text is longer than 64 MiB a buffer of its own size (one
 *   List<Float64> of 10^7 elements: about 80 MB and 250 MB).
 * Errors (nothing leaks; a refused call writes no file): a null pointer, n_cols <= 0, both or neither of cols[j] and lists[j], a
 *   temporal type on a list column, an invalid temporal type or a value outside its range -> BDF_INVALID; a named tz or an
 *   unsupported dtype -> BDF_UNSUPPORTED; a path that cannot be created or written -> BDF_INVALID with the OS error text (the file is
 *   then incomplete); a multi-GPU context -> BDF_UNSUPPORTED.
 * Launch records (BDF_K_JSON_WRITE): dtype BDF_U64 for the measure passes (element and row lengths), BDF_U32 for their scans, BDF_U8
 *   for the emit passes (rows and elements), -1 for the one-thread planning steps (window ends, block cuts). */
typedef struct { int32_t explicit_nulls; } bdf_json_write_options;
int  bdf_json_write(bdf_ctx* ctx, const char* path, int32_t n_cols, const char* const* names, const bdf_col* const* cols,
                    const bdf_temporal_type* types /* n_cols or NULL */, const bdf_list* const* lists /* n_cols or NULL */,
                    const bdf_json_write_options* options /* NULL: explicit_nulls = 0 */);

/* ---- measurement support ------------------------------------------------------------------------ */
/* Per-launch CUDA-event timing on the library's compute stream (the stream the kernels run on). */
typedef struct {
    int32_t kernel;   /* bdf_kernel_id, or an id that follows it (BDF_K_JSON_WRITE) */
    int32_t dtype;    /* output dtype   */
    int64_t rows;     /* elements processed by the launch */
    int64_t bytes;    /* algorithmic bytes of the launch (SURVEY 8(d) per-row figure x rows) */
    float   ms;       /* device time between the bracketing events */
} bdf_launch_record;
typedef enum { BDF_K_BINARY = 0, BDF_K_UNARY, BDF_K_CAST, BDF_K_REDUCE, BDF_K_GENERATE, BDF_K_AVG, BDF_K_COMPARE, BDF_K_FILTER, BDF_K_EXPR, BDF_K_SORT, BDF_K_TAKE, BDF_K_GROUP, BDF_K_JOIN, BDF_K_CSV, BDF_K_WINDOW, BDF_K_MOMENTS, BDF_K_CSV_WRITE, BDF_K_LIST, BDF_K_TEMPORAL, BDF_K_JSON, BDF_K_PARQUET, BDF_K_PARQUET_WRITE, BDF_K_SELECT, BDF_K_HIST } bdf_kernel_id;
/* Kernel ids that follow the enum.  bdf_kernel_id stays as published, ending at BDF_K_HIST: callers size their tables of kernel
 * names by its members, so a later id is a constant here instead.  bdf_launch_record.kernel may hold one of them. */
enum { BDF_K_JSON_WRITE = BDF_K_HIST + 1 };
int     bdf_profile_enable(bdf_ctx* ctx, int on);
int     bdf_profile_read(bdf_ctx* ctx, bdf_launch_record* buf, int64_t cap, int64_t* n); /* syncs; drains */
int64_t bdf_launch_count(bdf_ctx* ctx);           /* kernels launched since bdf_init */
/* Stream-ordered stopwatch on the compute stream: start/stop record events; stop syncs and reports ms. */
int     bdf_timer_start(bdf_ctx* ctx);
int     bdf_timer_stop(bdf_ctx* ctx, float* ms);
/* Writes `bytes` of device memory (an L2 flush when bytes > L2 size). */
int     bdf_flush_l2(bdf_ctx* ctx, size_t bytes);

/* Counter-based synthetic columns generated on the device (bench / large-config tests; SURVEY 8(d)).
 * Reproduces oracle/oracle.c:orc_generate bit-for-bit.  kind 0: real uniform [lo,hi), 1: real +-[1,2),
 * 2: integer full range, 3: integer uniform [-2^40,2^40).  null_mod 0: no bitmap. */
int bdf_generate(bdf_ctx* ctx, int dtype, int kind, double lo, double hi, uint64_t seed, uint64_t col_id,
                 int64_t n_chunks, const int64_t* chunk_lens, int64_t row0, uint32_t null_mod, bdf_col** out);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* B200DF_H */
